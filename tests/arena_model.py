"""The field arena of a single-GPU handle, restated from `field_layout` in fluid.cu, and what each entry
point may write in it.

Every field of a handle lives in one allocation: velocity x2, dye x2, pressure x2, divergence, curl, each
slot starting on a 2 MiB boundary, then 1 KiB of peer-memory flag words.  A field's extent is W * H * bytes
per cell; the rest of its slot is padding that no kernel may touch.  Where an extent is a multiple of
2 MiB there is no padding, and a store one row too far lands in the next slot.

`may_change` lists the byte ranges a call may modify given the read slot of each pair before the call;
every other byte of [0, bytes) must come out of the call unchanged.  `changes_outside` and `describe`
name the bytes that moved anyway: slot and row / column, padding of a slot, or the flag words."""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np

ALIGN = 2 << 20
FLAG_BYTES = 1024
PAIRS = ("velocity", "dye", "pressure")


@dataclass(frozen=True)
class Layout:
    W: int
    H: int
    Wd: int
    Hd: int
    half: bool
    v: tuple
    dye: tuple
    p: tuple
    div: int
    curl: int
    flags: int
    bytes: int

    def cell(self, field):
        """Bytes per cell: float2 / float4 / float, or their fp16 forms in half storage."""
        return {"velocity": 8, "dye": 16}.get(field, 4) // (2 if self.half else 1)

    def width(self, field):
        return self.Wd if field == "dye" else self.W

    def extent(self, field):
        return self.width(field) * (self.Hd if field == "dye" else self.H) * self.cell(field)

    def slot(self, field, k=0):
        """Offset of slot k of a pair, or of divergence / curl."""
        return {"velocity": self.v, "dye": self.dye, "pressure": self.p}[field][k] if field in PAIRS \
            else getattr(self, {"divergence": "div", "curl": "curl"}[field])

    def slots(self):
        """(name, field, offset) of every slot in arena order."""
        out = [(f"{f}[{k}]", f, self.slot(f, k)) for f in PAIRS for k in (0, 1)]
        return sorted(out + [(f, f, self.slot(f)) for f in ("divergence", "curl")], key=lambda s: s[2])


def _round(n):
    return (n + ALIGN - 1) // ALIGN * ALIGN


def layout(W, H, Wd, Hd, half=False) -> Layout:
    """field_layout(h, W*H, Wd*Hd) of fluid.cu for a single-GPU handle."""
    s = 2 if half else 1
    n, nd = W * H, Wd * Hd
    o = 0
    offs = []
    for bytes_ in (n * 8 // s,) * 2 + (nd * 16 // s,) * 2 + (n * 4 // s,) * 4:
        offs.append(o)
        o += _round(bytes_)
    return Layout(W, H, Wd, Hd, half, tuple(offs[0:2]), tuple(offs[2:4]), tuple(offs[4:6]), offs[6], offs[7],
                  o, o + FLAG_BYTES)


# What each call may modify (extents only, never padding).  `.read` / `.write` are the slots of a pair as
# they were before the call.  fluid_write(f) is "write" with the field named.
MAY_CHANGE = {
    "read": (),
    "render": (),
    "render_sunrays": ("dye.write",),                     # the sunrays mask is drawn into dye.write (S:1300)
    "curl": ("curl",),
    "divergence": ("divergence",),
    "vorticity": ("velocity.write",),
    "gradient_subtract": ("velocity.write",),
    "advect_velocity": ("velocity.write",),
    "advect_dye": ("dye.write",),
    "curl_vorticity_divergence": ("velocity.write", "curl", "divergence"),
    "clear_pressure": ("pressure.write",),
    "jacobi": ("pressure.read", "pressure.write"),
    "pressure_solve": ("pressure.read", "pressure.write"),
    "pressure_solve_host": ("pressure.read", "pressure.write", "divergence"),
    "splats": ("velocity.write", "dye.write"),             # launches after the first run in place on .write
    "step": ("velocity.read", "velocity.write", "dye.write", "pressure.read", "pressure.write", "divergence", "curl"),
}


def extent_range(L: Layout, target: str, par: dict):
    """[lo, hi) of `field` (divergence / curl) or `field.read` / `field.write` with pair parities `par`."""
    field, _, side = target.partition(".")
    if field in PAIRS:
        k = par[field] ^ (side == "write")
        lo = L.slot(field, k)
    else:
        lo = L.slot(field)
    return lo, lo + L.extent(field)


def may_change(call: str, L: Layout, par: dict, field: str | None = None):
    """The byte ranges `call` may modify, given the slot (0 / 1) each pair's .read is in before it."""
    if call == "write":
        targets = (field + ".read",) if field in PAIRS else (field,)
    else:
        targets = MAY_CHANGE[call]
    return [extent_range(L, t, par) for t in targets]


def describe(L: Layout, off: int) -> str:
    """Where byte `off` of the arena is: a slot's row / column / byte in the cell, a slot's padding, or the
    flag words."""
    if off >= L.flags:
        return f"flag words +{off - L.flags}" if off < L.bytes else f"past the arena +{off - L.bytes}"
    for name, field, lo in reversed(L.slots()):
        if off >= lo:
            rel = off - lo
            if rel >= L.extent(field):
                return f"padding of {name} +{rel - L.extent(field)}"
            row_bytes = L.width(field) * L.cell(field)
            return f"{name} row {rel // row_bytes} column {rel % row_bytes // L.cell(field)} byte {rel % L.cell(field)}"
    raise AssertionError(off)


def outside(offsets, ranges):
    """The offsets (ascending integer array) that lie in none of `ranges`."""
    offsets = np.asarray(offsets, np.int64)
    keep = np.ones(offsets.shape, bool)
    for lo, hi in ranges:
        keep &= (offsets < lo) | (offsets >= hi)
    return offsets[keep]


def report(L: Layout, offsets, limit: int = 8):
    """`describe` of the first `limit` offsets."""
    return [f"{int(o)}: {describe(L, int(o))}" for o in np.asarray(offsets)[:limit]]


def changes_outside(before: np.ndarray, after: np.ndarray, ranges, L: Layout, limit: int = 8):
    """(number of bytes of [0, L.bytes) that changed outside `ranges`, report of the first ones)."""
    moved = outside(np.flatnonzero(before[:L.bytes] != after[:L.bytes]), ranges)
    return len(moved), report(L, moved, limit)


def put(arena: np.ndarray, offset: int, field_values: np.ndarray, half: bool = False):
    """Stores a field's values at `offset` of a uint8 arena image, in the storage format."""
    b = np.ascontiguousarray(field_values, np.float16 if half else np.float32).view(np.uint8).reshape(-1)
    arena[offset:offset + b.size] = b


def fresh(L: Layout) -> np.ndarray:
    """The image of a new arena (make_arena): zero everywhere, dye alpha 1 in both dye slots."""
    a = np.zeros(L.bytes, np.uint8)
    one = np.zeros((L.Hd, L.Wd, 4), np.float32)
    one[..., 3] = 1
    for k in (0, 1):
        put(a, L.dye[k], one, L.half)
    return a
