"""Row-slab decomposition plan (SURVEY §8e) — the host-side arithmetic of the multi-GPU path.

Mirrors csrc/fluid.cu (create_common; block_depth, the depth of a solve; JacobiPlan, the launch split that
run_jacobi and solve_host_banded iterate over; draw_ghost_rows and the bands of a slab frame) so that the schedule
can be checked on CPU (tests/test_slab_schedule_gloo.py, tests/test_band_schedule_cpu.py,
tests/test_slab_draw_plan_cpu.py) and so that launchers know which rows a rank owns.
One process per GPU; rank g of G owns sim rows [g*H//G, (g+1)*H//G) and the matching dye rows.
Messages (NCCL send/recv inside the library, both neighbours in one group) happen ONLY on:
  * Jacobi, communication-avoiding ("deep") form: ONE group per solve with iters+1 rows of pressure
    and iters rows of divergence; launch i then produces owned rows +- (sweeps still to come + 1).
    Fallback when the ghost zone is thinner than iters+1: as many rows of divergence as the first
    (deepest) launch has sweeps, once, then K rows of pressure before each launch of depth K (K+1
    before the last, which also produces one row beyond each slab edge so that gradientSubtract
    needs no message);
  * advection: G rows of the projected velocity, then Gd rows of dye;
  * a frame (render, canvas, capture): draw_ghost_rows of dye, then with BLOOM / SUNRAYS one all-gather each of
    the bands draw_plan gives (every rank ends with the whole prefiltered bloom FBO / sunrays mask).
curl / vorticity / divergence run on ghost rows the previous step computed redundantly
(velocity is advected on owned rows +-3: curl needs +-2, vorticity +-1, divergence +-0).
"""
from __future__ import annotations

from dataclasses import dataclass

KMAX = 13
DEFAULT_BLOCK = 10
DEFAULT_HALO = 64
VELOCITY_GHOST = 3


def rows(extent: int, rank: int, world: int) -> tuple[int, int]:
    return extent * rank // world, extent * (rank + 1) // world


def jacobi_launches(iters: int, block: int = DEFAULT_BLOCK) -> list[int]:
    """Balanced split of `iters` sweeps into ceil(iters/block) launches, deeper ones first (fluid.cu JacobiPlan)."""
    if iters <= 0:
        return []
    block = max(1, min(block, KMAX))
    n = (iters + block - 1) // block
    base, extra = divmod(iters, n)
    return [base + (1 if k < extra else 0) for k in range(n)]


def host_bands(sim_h: int, iters: int, bands: int = 16, block: int = 0) -> list[dict]:
    """Plan of `fluid_pressure_solve_host` on one GPU (fluid.cu solve_host_banded): the grid is cut into row
    bands; band b is solved as soon as upload chunk b has arrived and is downloaded while later chunks upload.
    Returns one dict per band: owned rows [lo, hi), upload chunk [up_lo, up_hi) (what the band needs beyond the
    earlier chunks: rows up to hi + iters), and per launch (K, out_lo, out_hi) — launch k produces the band's
    rows +- the sweeps still to come.  block: JACOBI_BLOCK, 0 = DEFAULT_BLOCK (fluid.cu block_depth of a band).
    Empty list: the one-piece path (grid too short for two bands)."""
    nb = min(bands, 16, sim_h // max(256, 4 * iters)) if iters > 0 else 0
    block = block if block > 0 else DEFAULT_BLOCK
    if nb < 2:
        return []
    band = (sim_h + nb - 1) // nb
    out = []
    for b in range(nb):
        lo = min(b * band, sim_h); hi = min(lo + band, sim_h)
        if hi <= lo:
            break
        up_lo = 0 if b == 0 else min(lo + iters, sim_h)
        up_hi = sim_h if hi == sim_h else min(hi + iters, sim_h)
        launches, remaining = [], iters
        for K in jacobi_launches(iters, block):
            remaining -= K
            launches.append((K, max(lo - remaining, 0), min(hi + remaining, sim_h)))
        out.append(dict(lo=lo, hi=hi, up_lo=up_lo, up_hi=up_hi, launches=launches))
    return out


@dataclass
class SlabPlan:
    sim_h: int
    dye_h: int
    rank: int
    world: int
    halo: int = DEFAULT_HALO
    iterations: int = 20

    def __post_init__(self):
        self.row0, self.row1 = rows(self.sim_h, self.rank, self.world)
        self.drow0, self.drow1 = rows(self.dye_h, self.rank, self.world)
        self.G = 0
        if self.world > 1:
            per_sim = max(1, -(-self.dye_h // self.sim_h))
            # clipped with the SHORTEST slab (floor(H/world)) so that all ranks agree on the halo height
            self.G = min(max(self.halo, self.iterations + 2), self.sim_h // self.world, (self.dye_h // self.world) // per_sim)
        self.Gd = self.G * max(1, -(-self.dye_h // self.sim_h))
        if self.world > 1 and self.G < 14:
            raise ValueError(f"slab of {self.row1 - self.row0} rows is too short for a 14-row halo")

    def block(self, requested: int = 0) -> int:
        """Depth of the solve's launches (fluid.cu block_depth): `requested` (JACOBI_BLOCK) if > 0, else KMAX on
        one GPU and DEFAULT_BLOCK on a slab; at most KMAX, and on a slab below the ghost rows."""
        kb = requested if requested > 0 else (DEFAULT_BLOCK if self.world > 1 else KMAX)
        kb = min(kb, KMAX)
        return min(kb, self.G - 1) if self.world > 1 else kb

    def jacobi_messages(self, iters: int, requested_block: int = 0):
        """[(field, rows)] in issue order for one pressure solve."""
        ks = jacobi_launches(iters, self.block(requested_block))
        if not ks or self.world == 1:
            return []
        if self.deep(iters):
            return [("pressure+divergence", iters + 1)]
        msgs = [("divergence", max(ks))]
        for i, k in enumerate(ks):
            msgs.append(("pressure", k + (1 if i == len(ks) - 1 else 0)))
        return msgs

    def deep(self, iters: int) -> bool:
        return self.world > 1 and iters + 1 <= self.G and iters + 1 <= self.row1 - self.row0

    def launch_extents(self, iters: int, requested_block: int = 0):
        """[(K, ext)]: launch of depth K produces owned rows +- ext (clipped to the domain)."""
        ks = jacobi_launches(iters, self.block(requested_block))
        out, rem = [], iters
        for i, k in enumerate(ks):
            rem -= k
            if self.world == 1:
                out.append((k, 0))
            elif self.deep(iters):
                out.append((k, rem + 1))
            else:
                out.append((k, 1 if i == len(ks) - 1 else 0))
        return out

    def max_backtrace_rows(self) -> int:
        """Largest dt*|v| (in sim rows) the advection halo covers: G - ghost compute - bilinear tap."""
        return self.G - VELOCITY_GHOST - 2


def draw_ghost_rows(dye_h: int, height: int, bloom_h: int = 0, sunrays: bool = False) -> int:
    """Dye ghost rows a slab frame samples beyond the rows a rank owns (fluid.cu draw_ghost_rows), the same on every
    rank.  Every band starts at floor(n * rank / world) of its own grid, so a band of a `height`-row target may begin
    up to one target row before the dye rows it covers.  The display and shading taps (+-1 target row) then reach
    less than 1.5 * dye_h / height + 1.5 dye rows beyond the owned ones, the bloom prefilter's band of a bloom_h-row
    FBO less than dye_h / (2 * bloom_h) + 1.5, and the sunrays mask (at dye texel centres, its +y tap weighted 0)
    one.  bloom_h = 0: no prefilter (BLOOM off, or a pyramid of fewer than 2 levels)."""
    need = -(-3 * dye_h // (2 * height)) + 2
    if bloom_h > 0:
        need = max(need, -(-dye_h // (2 * bloom_h)) + 2)
    if sunrays:
        need = max(need, 1)
    return need


def draw_plan(dye_h: int, height: int, rank: int, world: int, bloom_h: int = 0, sunrays: bool = False) -> dict:
    """What rank `rank` of `world` does for one frame of a `height`-row target: `band`, the target rows it draws
    (fluid_render_band); `bloom_rows`, the rows of the bloom_h-row FBO it prefilters (None without a prefilter);
    `mask_rows`, the dye rows it draws the sunrays mask on (its own; None without SUNRAYS); `ghost`, the dye ghost
    rows it refreshes first; `gathers`, the all-gathers that follow."""
    return dict(band=rows(height, rank, world),
                bloom_rows=rows(bloom_h, rank, world) if bloom_h > 0 else None,
                mask_rows=rows(dye_h, rank, world) if sunrays else None,
                ghost=draw_ghost_rows(dye_h, height, bloom_h, sunrays),
                gathers=int(bloom_h > 0) + int(sunrays))


def gather_bytes(dye_w: int, dye_h: int, bloom_w: int = 0, bloom_h: int = 0, sunrays: bool = False) -> int:
    """Bytes of the buffers one frame's gathers assemble: the prefiltered bloom FBO (RGBA fp32) and the sunrays
    mask's alpha (fp32).  Each rank receives all of them but its own band, so a frame moves (world - 1) times this
    in all."""
    return 16 * bloom_w * bloom_h + (4 * dye_w * dye_h if sunrays else 0)
