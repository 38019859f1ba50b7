// jacobi.cuh — the pressure loop of step() (script.js S:1259-1266, pressureShader S:868-890).
//
//   p'[i,j] = ((((p[c(i-1),j] + p[c(i+1),j]) + p[i,c(j-1)]) + p[i,c(j+1)]) - div[i,j]) * 0.25
//
// Three kernels, all bit-identical per cell to the reference's one-blit-per-sweep loop:
//   jacobi_scalar_kernel  any W,H; one cell per thread (tiny / odd-sized grids).
//   jacobi_sweep_kernel   W%4==0; one float4 per thread, shuffles for x-neighbours; ONE sweep
//                         per launch == the literal S:1262 loop (12 B/update of HBM traffic).
//   jacobi_tb_kernel<K>   K sweeps per launch (temporal blocking) as a register-streaming stencil:
//     * a warp owns a 128-column window (lane l holds columns 4l..4l+3 as one float4) and streams
//       upward over a chunk of rows; no __syncthreads anywhere, warps are independent;
//     * time level t (t = 0..K-1) lives in a rotating 3-row register window; when level 0 loads
//       row r, level t produces row r-t, so the K sweeps form a software pipeline in y;
//     * x-neighbours across lanes come from __shfl_up/down.  Lane 0 has no left neighbour and lane 31
//       no right one: at level 1 they take the level-0 column just outside the window (x0-1, x0+128)
//       from the staged p box, which is 4 columns wider than the window on each side, so level 1 is
//       right on all 128 columns; from level 2 on their shuffles return garbage that creeps inward
//       one column per level.  Level K is wrong in its outer K-1 columns: HX = roundup(K-1,4) halo
//       columns on each side of the window are recomputed by the neighbouring window (overlapped
//       tiling);
//     * CLAMP_TO_EDGE in x is an even reflection p[-1-m] = p[m]; because L+R is the first add of
//       the expression (commutative) the reflected columns evolve bit-identically, so mirroring
//       the LOADS implements the boundary for all K levels.  In y the expression is not
//       symmetric in B/T, so rows 0 and H-1 select "below := centre" / "above := centre"
//       explicitly (EDGE instantiation, only on the few steps that touch those rows);
//     * div[r] is needed by level t when it produces row r, i.e. K times at K different steps:
//       each lane keeps its float4 of the last K+3 rows in a register ring (see tb_block);
//     * p / div rows are staged ahead into a per-warp shared-memory ring, so the few resident
//       warps still keep enough bytes in flight for HBM: one lane issues 2-D tensor-map TMA boxes
//       (cp.async.bulk.tensor, SASS UTMALDG) of the window's rows with mbarrier complete_tx.
//   The optional SCALE template fuses the clear pass (S:1253-1257, p <- PRESSURE*p) into the
//   level-0 load of the first launch: one fp32 multiply, same rounding as the separate blit.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace fk {

// ---- the member table of a batch handle --------------------------------------------------------------
// Each member's step scalars and dt in device memory: MP_KEYS rows of B floats, row k holding every member's
// value of scalar k (MP_RADIUS: correctRadius(SPLAT_RADIUS / 100) as splats use it).  The host changes it only
// by stream-ordered copies, so a step graph never bakes a value in.  A kernel whose grid has one layer per member
// reads member blockIdx.z's value (B == gridDim.z).
enum MemberParam { MP_DT, MP_CURL, MP_PRESSURE, MP_VELOCITY_DISSIPATION, MP_DENSITY_DISSIPATION, MP_RADIUS, MP_KEYS };
__device__ __forceinline__ float member_param(const float* __restrict__ tab, MemberParam k) {
    return __ldg(tab + (size_t)k * gridDim.z + blockIdx.z);
}

struct JacobiArgs {
    const float* pin;    // local row 0 of the source pressure buffer
    const float* div;    // local row 0 of divergence
    float* pout;         // local row 0 of the destination pressure buffer
    int W, H;            // GLOBAL grid size (clamp rules refer to it)
    int row_off;         // global row index of local row 0 (0 on a single GPU)
    int out_lo, out_hi;  // global rows [out_lo, out_hi) to produce
    int rows_per_chunk;  // tb kernel: output rows per warp stream
    float scale;         // SCALE: value of config.PRESSURE
    int* err;            // device error word (3 = a bounded mbarrier wait gave up)
    const unsigned char* tiny_map;   // tb kernel: where divergence defeats the fma contraction (may be null)
    unsigned long long* exact_streams;   // tb kernel: warps that ran the un-contracted tail (may be null)
};

// the two tensor maps a temporally blocked launch reads through: p describes the buffer passed as
// JacobiArgs::pin, d the one passed as div, both from their local row 0.  64-byte aligned
// CUtensorMap images, passed by value as a __grid_constant__ kernel parameter
struct __align__(64) TmapPair {
    unsigned char p[128];
    unsigned char d[128];
};

// ------------------------------------------------------------------------------------------------
// S: storage policy (passes.cuh).  The pointers of JacobiArgs address S::T1 elements: fp16 ones in
// half storage, where do_scale is false (the clear pass is a launch of its own there).
template <class S>
__global__ void __launch_bounds__(256) jacobi_scalar_kernel(JacobiArgs a, bool do_scale) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int j = a.out_lo + blockIdx.y * blockDim.y + threadIdx.y;
    if (i >= a.W || j >= a.out_hi) return;
    const int il = max(i - 1, 0), ir = min(i + 1, a.W - 1);
    const int jb = max(j - 1, 0) - a.row_off, jt = min(j + 1, a.H - 1) - a.row_off;
    const int jl = j - a.row_off;
    const auto* pin = reinterpret_cast<const typename S::T1*>(a.pin);
    const auto* div = reinterpret_cast<const typename S::T1*>(a.div);
    const float s = do_scale ? a.scale : 1.0f;
    float L = S::ld(pin, (size_t)jl * a.W + il), R = S::ld(pin, (size_t)jl * a.W + ir);
    float B = S::ld(pin, (size_t)jb * a.W + i), T = S::ld(pin, (size_t)jt * a.W + i);
    if (do_scale) { L = s * L; R = s * R; B = s * B; T = s * T; }
    S::st(reinterpret_cast<typename S::T1*>(a.pout), (size_t)jl * a.W + i,
          ((((L + R) + B) + T) - S::ld(div, (size_t)jl * a.W + i)) * 0.25f);
}

// ------------------------------------------------------------------------------------------------
// One sweep, one float4 per thread.  blockDim = (32 * WARPS_X, ROWS): a warp spans 128 columns.
template <bool SCALE>
__global__ void __launch_bounds__(256) jacobi_sweep_kernel(JacobiArgs a) {
    const int W4 = a.W >> 2;
    const int g = blockIdx.x * blockDim.x + threadIdx.x;  // float4 column group
    const int j = a.out_lo + blockIdx.y * blockDim.y + threadIdx.y;
    const bool live = (g < W4) && (j < a.out_hi);
    const int gc = min(g, W4 - 1), jc = min(j, a.out_hi - 1);
    const int jl = jc - a.row_off;
    const int jb = max(jc - 1, 0) - a.row_off, jt = min(jc + 1, a.H - 1) - a.row_off;
    const float4* P = reinterpret_cast<const float4*>(a.pin);
    float4 c = __ldg(P + (size_t)jl * W4 + gc);
    float4 b = __ldg(P + (size_t)jb * W4 + gc);
    float4 t = __ldg(P + (size_t)jt * W4 + gc);
    const float4 d = __ldg(reinterpret_cast<const float4*>(a.div) + (size_t)jl * W4 + gc);
    if (SCALE) {
        const float s = a.scale;
        c.x = s * c.x; c.y = s * c.y; c.z = s * c.z; c.w = s * c.w;
        b.x = s * b.x; b.y = s * b.y; b.z = s * b.z; b.w = s * b.w;
        t.x = s * t.x; t.y = s * t.y; t.z = s * t.z; t.w = s * t.w;
    }
    float l = __shfl_up_sync(0xffffffffu, c.w, 1);
    float r = __shfl_down_sync(0xffffffffu, c.x, 1);
    const int lane = threadIdx.x & 31;
    if (lane == 0) {   // warp edge: fetch the neighbour (or clamp at the wall)
        float e = (gc > 0) ? __ldg(a.pin + (size_t)jl * a.W + 4 * gc - 1) : 0.0f;
        l = (gc > 0) ? (SCALE ? a.scale * e : e) : c.x;
    }
    if (lane == 31 || gc == W4 - 1) {
        float e = (gc < W4 - 1) ? __ldg(a.pin + (size_t)jl * a.W + 4 * gc + 4) : 0.0f;
        r = (gc < W4 - 1) ? (SCALE ? a.scale * e : e) : c.w;
    }
    float4 o;
    o.x = ((((l + c.y) + b.x) + t.x) - d.x) * 0.25f;
    o.y = ((((c.x + c.z) + b.y) + t.y) - d.y) * 0.25f;
    o.z = ((((c.y + c.w) + b.z) + t.z) - d.z) * 0.25f;
    o.w = ((((c.z + r) + b.w) + t.w) - d.w) * 0.25f;
    if (live) reinterpret_cast<float4*>(a.pout)[(size_t)jl * W4 + gc] = o;
}

// ------------------------------------------------------------------------------------------------
// Temporally blocked kernel, generation 7.
//
// Arithmetic.  Out of registers the kernel is bound by fp32 LANE-OPERATIONS per update (scalar
// FADD / FMUL / FFMA, 32 lanes per cycle per SM sub-partition).  The reference expression costs 5:
// ((((L+R)+B)+T)-d)*0.25.  The last two contract into ONE fma with a pre-scaled divergence,
//        fma(S, 0.25, -0.25*d)  ==  (S - d) * 0.25      bit for bit,
// whenever d == 0 or |d| >= 2^-123, and rn(S-d) is finite:  -0.25*d is then exact;
// for |S-d| >= 2^-124 scaling by 2^-2 commutes with the rounding of S-d (normal results); for
// |S-d| < 2^-124 <= |d|/2 Sterbenz makes S-d exact, so both sides round the same real number once.
// Two ends of the exponent range break it.
//   * A divergence value with 0 < |d| < 2^-123 (subnormal-range far fields of a Gaussian splat do
//     produce them) can double-round differently, so the producers of `divergence` keep a coarse map —
//     one byte per 128-column x 32-row cell — of where such values occur, and a warp whose footprint
//     touches a flagged cell runs the EXACT instantiation (subtract, then multiply) from the start.
//   * Finite S and d whose difference rounds to +-inf (|S-d| >= 2^128 - 2^103): the reference gives
//     inf, the fma the finite S/4 - d/4.  This needs max(|S|, |d|) >= 2^127 - 2^102, which no sweep of
//     a launch reaches while every level-0 input — PRESSURE*p as loaded, and d — is below BIG_IN = 2^122
//     (each sweep grows |p| by at most |d|/4: after 12 sweeps |p| < 2^125, so |S| <= 2^127 - 2^103;
//     proof in tests/test_fma_contraction_cpu.py).  A contracted stream tracks the largest level-0
//     magnitude it loads (fmaxf: NaN drops out, it meets both tails alike; inf counts) and, if that
//     reached BIG_IN, runs again through the EXACT instantiation, overwriting the rows it stored.
//     The edge columns that lanes 0 and 31 read for level 1 are level-0 inputs like any other (they
//     reach valid outputs whenever K-1 is a multiple of 4), so they are folded into the same maximum.
// 4 lane-ops per update instead of 5 everywhere else, plus 8 FMNMX per row on the ALU pipe.
//
// Staging.  p / div rows reach a warp through a shared-memory ring filled by 2-D tensor-map TMA
// (cp.async.bulk.tensor.2d, SASS UTMALDG): one elected lane arms an mbarrier and fetches a
// 136-column x 3-row box of p and of div at x0-4 per pipeline block: the window plus one float4 on
// each side.  Rows stay 16-byte aligned for every lane's LDS.128, and the edge columns x0-1 and x0+128
// of p lie inside.  div goes through the same box although its outer columns are never read: at
// HX = 12 (depths 10-13) rows from x0-4 start on a 32-byte sector of global memory and rows from x0 do
// not, and where the box starts moved a launch by 3-5 % (DESIGN 5.10).  Columns outside the grid and
// rows outside the mapped buffer are zero-filled by the hardware (never used by a valid output).
constexpr int TB_BOX = 136;                          // columns of a staged box: the window and 4 on each side
template <int K>
struct TB {
    static constexpr int HX = (K + 2) / 4 * 4;       // x halo (columns) on each side of a window: roundup(K-1, 4)
    static constexpr int VALID = 128 - 2 * HX;       // columns a window produces
    static constexpr int RD = K + 3;                 // div register-ring slots
    static constexpr int U = 3;                      // pipeline steps per unrolled block
    // NS stages, each a 3-row box of div followed by a 3-row box of p (row = 544 B), each box padded to a
    // multiple of 128 B, the alignment TMA needs of its destination; then NS mbarriers
    // Three stages: the boxes of a block are requested at the end of the block two before it.  A fourth
    // stage, more bytes in flight per warp, made the solve slower (DESIGN 5.12).
    static constexpr int NS = 3;
    static constexpr int ROW4 = TB_BOX / 4;          // float4 per staged row
    static constexpr int P4 = (U * ROW4 + 7) / 8 * 8;                   // float4 offset of the p box in a stage
    static constexpr int TX = 2 * U * ROW4 * (int)sizeof(float4);       // bytes one stage's two boxes bring
    static constexpr int STAGE4 = 2 * P4;                               // float4 per stage
    static constexpr int SMEM = NS * STAGE4 * (int)sizeof(float4) + NS * 8;
};

// coarse map of "divergence has a value with 0 < |d| < 2^-123 here": one byte per cell
constexpr int TINY_CW = 128, TINY_CH = 32;
constexpr float TINY_DIV = 9.4039548e-38f;           // 2^-123
__host__ __device__ inline int tiny_map_w(int W) { return (W + TINY_CW - 1) / TINY_CW; }
__host__ __device__ inline int tiny_map_h(int H) { return (H + TINY_CH - 1) / TINY_CH; }
__device__ __forceinline__ bool is_tiny_div(float d) { return d != 0.0f && fabsf(d) < TINY_DIV; }
// level-0 inputs of a contracted stream at or above this magnitude send it through the EXACT tail
constexpr float BIG_IN = 5.3169119831396635e36f;     // 2^122

// ---- TMA (2-D tensor map) + mbarrier ----------------------------------------------------------------
// Waits are bounded: a mis-armed barrier costs an error word, never a hung kernel.
__device__ __forceinline__ unsigned smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(void* bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_expect_tx(void* bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const void* tmap, int x, int y, void* bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
                 ::"r"(smem_u32(smem_dst)), "l"(tmap), "r"(x), "r"(y), "r"(smem_u32(bar)) : "memory");
}
// the box of member m of a batch handle's (W, H, B) tensor map, one member deep: rows past the member's
// first or last read as zero, exactly like rows past a single handle's 2-D map
__device__ __forceinline__ void tma_load_3d(void* smem_dst, const void* tmap, int x, int y, int m, void* bar) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                 ::"r"(smem_u32(smem_dst)), "l"(tmap), "r"(x), "r"(y), "r"(m), "r"(smem_u32(bar)) : "memory");
}
// BATCH: blockIdx.z is the member
template <bool BATCH>
__device__ __forceinline__ void tma_load_box(void* smem_dst, const void* tmap, int x, int y, void* bar) {
    if constexpr (BATCH) tma_load_3d(smem_dst, tmap, x, y, (int)blockIdx.z, bar);
    else tma_load_2d(smem_dst, tmap, x, y, bar);
}
__device__ __forceinline__ void mbar_inval(void* bar) {
    asm volatile("mbarrier.inval.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(void* bar, unsigned parity) {
    unsigned ok;
    asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
    return ok != 0;
}
__device__ __forceinline__ void mbar_wait(void* bar, unsigned parity, int* err) {
    if (mbar_try_wait(bar, parity)) return;              // the common case: the box landed long ago
#pragma unroll 1
    for (int tries = 0; tries < (1 << 16); ++tries)      // each try_wait already blocks for a HW time slice
        if (mbar_try_wait(bar, parity)) return;
    if (err) *err = 3;
}

__device__ __forceinline__ float4 lds128(const float4* p) {
    float4 v;
    const unsigned a = (unsigned)__cvta_generic_to_shared(p);
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(a) : "memory");
    return v;
}

__device__ __forceinline__ float lds32(const float* p) {
    float v;
    const unsigned a = (unsigned)__cvta_generic_to_shared(p);
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(a) : "memory");
    return v;
}

__device__ __forceinline__ void sts32(const float* p, float v) {
    const unsigned a = (unsigned)__cvta_generic_to_shared(p);
    asm volatile("st.shared.f32 [%0], %1;" ::"r"(a), "f"(v) : "memory");
}

__device__ __forceinline__ float4 rev4(float4 v, bool rev) {
    return rev ? make_float4(v.w, v.z, v.y, v.x) : v;
}

// one Jacobi update of a float4 of row `c`, with rows below/above and the neighbours l / r across lanes.
//   EXACT:  o = ((((L + R) + below) + above) - d) * 0.25          (d = divergence)
//   else :  o = fma(((L + R) + below) + above, 0.25, d)           (d = -0.25 * divergence)
// Every operation is an explicit IEEE round-to-nearest intrinsic, so the result does not depend on
// the build's --fmad setting: the fma is the only contraction, and it is the one proven exact above.
template <bool EXACT>
__device__ __forceinline__ float4 jacobi4(const float l, const float r, const float4 below, const float4 c,
                                          const float4 above, const float4 d) {
    float4 o;
    o.x = __fadd_rn(__fadd_rn(__fadd_rn(l, c.y), below.x), above.x);
    o.y = __fadd_rn(__fadd_rn(__fadd_rn(c.x, c.z), below.y), above.y);
    o.z = __fadd_rn(__fadd_rn(__fadd_rn(c.y, c.w), below.z), above.z);
    o.w = __fadd_rn(__fadd_rn(__fadd_rn(c.z, r), below.w), above.w);
    if (EXACT) {
        o.x = __fmul_rn(__fsub_rn(o.x, d.x), 0.25f);
        o.y = __fmul_rn(__fsub_rn(o.y, d.y), 0.25f);
        o.z = __fmul_rn(__fsub_rn(o.z, d.z), 0.25f);
        o.w = __fmul_rn(__fsub_rn(o.w, d.w), 0.25f);
    } else {
        o.x = __fmaf_rn(o.x, 0.25f, d.x);
        o.y = __fmaf_rn(o.y, 0.25f, d.y);
        o.z = __fmaf_rn(o.z, 0.25f, d.z);
        o.w = __fmaf_rn(o.w, 0.25f, d.w);
    }
    return o;
}

// Per-warp stream state that survives across unrolled blocks.
struct TBStream {
    float4* op;          // where level K's row of THIS step goes (advances one row per step)
    int rout;            // global row index op points at  (= ys + s - K)
    // alignas: rout alone in its 8 bytes, the layout this kernel has been measured with.  Packing stg
    // next to rout renumbers the PTX registers, and ptxas then schedules the whole kernel differently.
    alignas(8) int stg;  // stage consumed by this block (0..NS-1)
    unsigned phase;      // mbarrier parity of that stage
    int yfill;           // local row coordinate of the next box to fetch
};

struct TBTma {           // warp-uniform TMA bookkeeping
    const void* tm_p;    // tensor map of the source pressure buffer
    const void* tm_d;    // tensor map of divergence
    unsigned long long* bars;   // NS mbarriers
    float4* slots;       // stage q at slots + q * STAGE4
    int x0;              // first (possibly negative) column of the window
    int lane;
    int* err;
};

// One unrolled block of 3 pipeline steps.
//   * p windows: 3 register slots per level, rotating with period 3 == the unroll, so they are
//     addressed with compile-time constants and never moved;
//   * div: level t needs div[r] when it produces row r, i.e. at K different steps.  The last K+3
//     rows live in the register ring dr[]: the row staged at phase ph sits in dr[K+ph], level t
//     reads dr[K+ph-t], and the ring is shifted down by 3 at the end of the block (MOVs issue on
//     the ALU pipe, beside the fp32 pipe that bounds the kernel);
//   * EDGE instantiates the wall selects in y, REV the mirrored-lane reversal in x, EXACT the
//     un-contracted tail; all are chosen by warp-uniform branches OUTSIDE the steady-state loop;
//   * level 1 is the only level whose edge lanes have a real neighbour outside the window: the row it
//     centres on was staged one step earlier and is still in shared memory (this block's stage, or row 2
//     of the previous block's, which is refilled only at the end of this block), so lanes 0 and 31
//     read that row's column x0-1 / x0+128 through `ering` instead of keeping it in a register;
//   * a contracted block folds the magnitudes of its level-0 inputs into `big` (BIG_IN above).
template <int K, bool SCALE, bool EDGE, bool REV, bool EXACT, bool BATCH>
__device__ __forceinline__ void tb_block(float4 (&w)[K][3], float4 (&dr)[TB<K>::RD], TBStream& st, float& big,
                                         const float4* __restrict__ ring, const float* __restrict__ ering,
                                         const TBTma& tm, const int W4,
                                         const int y0, const int y1, const int H,
                                         const bool rev, const bool lane_out, const float scale) {
    using T = TB<K>;
    mbar_wait(tm.bars + st.stg, st.phase, tm.err);
    const float4* srow = ring + st.stg * T::STAGE4;
    const float* erow = ering + st.stg * (4 * T::STAGE4);
    const float* erow_prev = ering + ((unsigned)(st.stg + T::NS - 1) % T::NS) * (4 * T::STAGE4) + 2 * TB_BOX;
    // The K levels x 3 steps of a block form a dependency lattice: node (ph, t) needs node
    // (ph, t-1) of the same step (the fresh row above) and rows of level t-1 from the two previous
    // steps.  Source order is step by step; ptxas interleaves the chains itself.
#pragma unroll
    for (int ph = 0; ph < 3; ++ph) {
#pragma unroll
        for (int t = 0; t <= K; ++t) {
            if (t == 0) {
                // ---- level 0: the oldest staged row ---------------------------------------------------
                float4 in = lds128(srow + ph * T::ROW4);
                float4 dv = lds128(srow - T::P4 + ph * T::ROW4);    // the div box starts P4 float4 below the p box
                if (REV) { in = rev4(in, rev); dv = rev4(dv, rev); }
                if (SCALE) {
                    in.x = scale * in.x; in.y = scale * in.y; in.z = scale * in.z; in.w = scale * in.w;
                }
                if (!EXACT) {                     // d' = -0.25 * d, exact outside the flagged cells
                    big = fmaxf(big, fmaxf(fmaxf(fmaxf(fabsf(in.x), fabsf(in.y)), fmaxf(fabsf(in.z), fabsf(in.w))),
                                           fmaxf(fmaxf(fabsf(dv.x), fabsf(dv.y)), fmaxf(fabsf(dv.z), fabsf(dv.w)))));
                    dv.x = __fmul_rn(dv.x, -0.25f); dv.y = __fmul_rn(dv.y, -0.25f);
                    dv.z = __fmul_rn(dv.z, -0.25f); dv.w = __fmul_rn(dv.w, -0.25f);
                }
                w[0][(ph + 2) % 3] = in;
                dr[K + ph] = dv;
            } else {
                // ---- level t of step ph ---------------------------------------------------------------
                const float4 c = w[t - 1][(ph + 1) % 3];
                float4 below = w[t - 1][(ph + 0) % 3];
                float4 above = w[t - 1][(ph + 2) % 3];
                if (EDGE) {                       // warp-uniform conditions
                    const int r = st.rout + ph + (K - t);   // row produced by level t at this step
                    if (r == 0) below = c;        // CLAMP_TO_EDGE: p[i,-1] = p[i,0]
                    if (r == H - 1) above = c;    //                p[i,H]  = p[i,H-1]
                }
                const float4 d = dr[K + ph - t];  // div row staged t steps ago
                float l = __shfl_up_sync(0xffffffffu, c.w, 1);
                float r = __shfl_down_sync(0xffffffffu, c.x, 1);
                if (t == 1) {                     // c is level 0: the edge lanes' neighbours are input data
                    float e = lds32(ph == 0 ? erow_prev : erow + (ph - 1) * TB_BOX);
                    if (SCALE) e = scale * e;
                    if (!EXACT) big = fmaxf(big, fabsf(e));
                    l = (tm.lane == 0) ? e : l;
                    r = (tm.lane == 31) ? e : r;
                }
                const float4 o = jacobi4<EXACT>(l, r, below, c, above, d);
                if (t < K) {
                    w[t][(ph + 2) % 3] = o;
                } else if (lane_out && (unsigned)(st.rout + ph - y0) < (unsigned)(y1 - y0)) {
                    st.op[ph * W4] = o;
                }
            }
        }
    }
    st.rout += 3;
    st.op += 3 * W4;
#pragma unroll
    for (int j = 0; j < K; ++j) dr[j] = dr[j + 3];
    // Refill the stage consumed ONE BLOCK AGO with the box NS-1 blocks ahead: every value read
    // from it has been used by now, so all lanes' reads of it have completed.
    __syncwarp();
    if (tm.lane == 0) {
        const int q = (st.stg == 0) ? T::NS - 1 : st.stg - 1;
        float4* dst = tm.slots + q * T::STAGE4;
        mbar_expect_tx(tm.bars + q, (unsigned)T::TX);
        tma_load_box<BATCH>(dst, tm.tm_d, tm.x0 - 4, st.yfill, tm.bars + q);
        tma_load_box<BATCH>(dst + T::P4, tm.tm_p, tm.x0 - 4, st.yfill, tm.bars + q);
    }
    st.yfill += 3;
    if (st.stg + 1 == T::NS) { st.stg = 0; st.phase ^= 1u; } else { ++st.stg; }
}

// returns this lane's largest level-0 magnitude (0 for an EXACT stream)
template <int K, bool SCALE, bool REV, bool EXACT, bool BATCH>
__device__ __forceinline__ float tb_stream(const JacobiArgs& a, const void* tm_p, const void* tm_d,
                                          float4* __restrict__ smem4, const int lane, const int x0,
                                          const int lc, const int gx, const bool rev,
                                          const bool lane_out, const int y0, const int y1,
                                          const int ys) {
    using T = TB<K>;
    const int W = a.W, H = a.H, W4 = W >> 2;
    const int nsteps = y1 - ys + K;                   // level K emits row ys+s-K at step s

    const ptrdiff_t base = -(ptrdiff_t)a.row_off * W4;
    float4* Og = reinterpret_cast<float4*>(a.pout) + base + (lane_out ? (gx >> 2) : 0);

    // rotating windows: w[t][(ph+0)%3] = row r-1, [(ph+1)%3] = row r, [(ph+2)%3] = fresh row r+1
    float4 w[K][3];
#pragma unroll
    for (int t = 0; t < K; ++t)
#pragma unroll
        for (int q = 0; q < 3; ++q) w[t][q] = make_float4(0.f, 0.f, 0.f, 0.f);
    float4 dr[T::RD];
#pragma unroll
    for (int q = 0; q < T::RD; ++q) dr[q] = make_float4(0.f, 0.f, 0.f, 0.f);

    TBStream st{};
    TBTma tm{};
    // every lane reads its (mirrored / clamped) column group out of the window's 128 columns of the
    // staged boxes.  In the last window the mirror image of the outermost lanes lies left of the window
    // (x0 > lc); those lanes feed no output (beyond lane_out and the shuffle cone), so they read the
    // window's first column instead of shared memory below it.  `ring`: this lane's float4 in p row 0
    // of stage 0 (the boxes start at column x0 - 4).
    const float4* ring = smem4 + T::P4 + ((min(max(lc, x0), x0 + 124) - (x0 - 4)) >> 2);
    // `ering`: in the same row, the column lane 0 / lane 31 takes as its outer neighbour at level 1:
    // x0 - 1 / x0 + 128, mirrored about the walls like lc, and clamped into the box where the image
    // lies outside it (the last window again: no output depends on it).  The other lanes read a column
    // of their own group, which changes nothing about `big`.
    int ec = min(max(lc, x0), x0 + 124);
    if (lane == 0 || lane == 31) {
        ec = (lane == 0) ? x0 - 1 : x0 + 128;
        if (ec < 0) ec = -1 - ec;                              // p[-1-m] = p[m]
        else if (ec >= W) ec = 2 * W - 1 - ec;                 // p[W+m]  = p[W-1-m]
        ec = min(max(min(max(ec, 0), W - 1), x0 - 4), x0 + TB_BOX - 5);
    }
    const float* ering = reinterpret_cast<const float*>(smem4 + T::P4) + (ec - (x0 - 4));
    // the first step's level 1 (a dead warm-up node) reads the row "staged one step earlier" from a stage
    // no box has reached yet: it must not bring whatever shared memory held into `big`
    sts32(ering + (T::NS - 1) * (4 * T::STAGE4) + 2 * TB_BOX, 0.0f);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // ordered before the TMA write that refills that stage
    tm.tm_p = tm_p; tm.tm_d = tm_d;
    tm.bars = reinterpret_cast<unsigned long long*>(smem4 + T::NS * T::STAGE4);
    tm.slots = smem4;
    tm.x0 = x0; tm.err = a.err;
    tm.lane = (int)threadIdx.x;                       // == lane (one warp per CTA): nothing to keep live in the out-of-line streams
    st.stg = 0; st.phase = 0;
    st.yfill = ys - a.row_off;
    if (lane == 0) {
#pragma unroll
        for (int q = 0; q < T::NS; ++q) mbar_init(tm.bars + q, 1);
        mbar_fence_init();
    }
    __syncwarp();
    // boxes of blocks 0 .. NS-2 into stages 0 .. NS-2; stage NS-1 is filled at the end of block 0
#pragma unroll
    for (int q = 0; q < T::NS - 1; ++q) {
        if (lane == 0) {
            float4* dst = tm.slots + q * T::STAGE4;
            mbar_expect_tx(tm.bars + q, (unsigned)T::TX);
            tma_load_box<BATCH>(dst, tm_d, x0 - 4, st.yfill, tm.bars + q);
            tma_load_box<BATCH>(dst + T::P4, tm_p, x0 - 4, st.yfill, tm.bars + q);
        }
        st.yfill += 3;
    }
    st.rout = ys - K;
    st.op = Og + (ptrdiff_t)st.rout * W4;             // only dereferenced for rows in [y0, y1)

    // A block touches a wall row when its rows [ys+s0-K, ys+s0+2] reach row 0 or row H-1: the
    // first blocks of a bottom chunk and the last ones of a top chunk.  Wall and steady-state
    // blocks run in SEPARATE loops (not one loop with a branch) so that the steady-state loop
    // has its own register assignment and its window rotation closes without moves.
    int s0 = 0;
    float big = 0.0f;
#pragma unroll 1
    while (s0 < nsteps) {                             // at most: wall blocks, steady blocks, wall blocks
#pragma unroll 1
        for (; s0 < nsteps && ((ys + s0 - K <= 0) || (ys + s0 + 2 >= H - 1)); s0 += 3)
            tb_block<K, SCALE, true, REV, EXACT, BATCH>(w, dr, st, big, ring, ering, tm, W4, y0, y1, H, rev, lane_out, a.scale);
#pragma unroll 1
        for (; s0 < nsteps && !((ys + s0 - K <= 0) || (ys + s0 + 2 >= H - 1)); s0 += 3)
            tb_block<K, SCALE, false, REV, EXACT, BATCH>(w, dr, st, big, ring, ering, tm, W4, y0, y1, H, rev, lane_out, a.scale);
    }
    // drain the over-fetched tail before the CTA (and its shared memory) goes away
#pragma unroll
    for (int q = 0; q < T::NS - 1; ++q) {
        mbar_wait(tm.bars + st.stg, st.phase, tm.err);
        if (st.stg + 1 == T::NS) { st.stg = 0; st.phase ^= 1u; } else { ++st.stg; }
    }
    return big;
}

template <int K, bool SCALE, bool BATCH>
__device__ __noinline__ void tb_stream_exact(const JacobiArgs& a, const void* tm_p, const void* tm_d,
                                             float4* __restrict__ smem4, const int lane, const int x0,
                                             const int lc, const int gx, const bool rev, const bool lane_out,
                                             const int y0, const int y1, const int ys, const bool any_rev) {
    if (lane == 0 && a.exact_streams) atomicAdd(a.exact_streams, 1ull);
    if (any_rev) tb_stream<K, SCALE, true, true, BATCH>(a, tm_p, tm_d, smem4, lane, x0, lc, gx, rev, lane_out, y0, y1, ys);
    else tb_stream<K, SCALE, false, true, BATCH>(a, tm_p, tm_d, smem4, lane, x0, lc, gx, rev, lane_out, y0, y1, ys);
}

// One warp per CTA: every quantity that steers control flow derives from blockIdx and kernel
// arguments only, so the compiler can prove the warp converged at each shuffle (no WARPSYNC /
// BSSY scaffolding) and keeps loop state in uniform registers.
#ifndef FLUID_TB_MINBLOCKS
#define FLUID_TB_MINBLOCKS 1     // tuning builds: resident CTAs per SM the register allocation must allow
#endif
#ifdef FLUID_TB_MAXNREG            // tuning builds: cap registers directly (192 -> 10 one-warp CTAs per SM)
#define FLUID_TB_BOUNDS __maxnreg__(FLUID_TB_MAXNREG)
#else
#define FLUID_TB_BOUNDS __launch_bounds__(32, FLUID_TB_MINBLOCKS)
#endif
// BATCH: a batch handle's launch, blockIdx.z the member.  The maps are 3-D (W, H, B); pout and the tiny map
// move to the member's array and map region, and SCALE takes the member's PRESSURE from member_table (a.scale is
// not read).  Only that instantiation reads member_table.
template <int K, bool SCALE, bool BATCH = false>
__global__ void FLUID_TB_BOUNDS jacobi_tb_kernel(JacobiArgs a, const __grid_constant__ TmapPair maps,
                                                 const float* __restrict__ member_table) {
    using T = TB<K>;
    if constexpr (BATCH) {
        a.pout += (size_t)blockIdx.z * a.W * a.H;
        if (a.tiny_map) a.tiny_map += (size_t)blockIdx.z * tiny_map_w(a.W) * tiny_map_h(a.H);
        if constexpr (SCALE) a.scale = member_param(member_table, MP_PRESSURE);
    }
    extern __shared__ __align__(128) float4 smem4[];
    // Programmatic dependent launch: back-to-back blocked launches of one solve are chained with
    // cudaLaunchAttributeProgrammaticStreamSerialization, so the NEXT launch's CTAs are already
    // resident (index math done, parked at griddepcontrol.wait) while this grid drains — the
    // single-wave tail and the launch gap overlap instead of adding up.  Both instructions are
    // no-ops for a launch without the attribute.
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    const int lane = threadIdx.x;
    const int nxw = (a.W + T::VALID - 1) / T::VALID;
    const int wid = blockIdx.x;
    const int wx = wid % nxw;
    const int cy = wid / nxw;

    // ---- x geometry of this lane: mirrored / clamped float4 column group ------------------------
    const int W = a.W, H = a.H;
    const int gx = wx * T::VALID - T::HX + 4 * lane;  // first global column of this lane
    int lc = gx;
    bool rev = false;
    if (gx < 0) { lc = -gx - 4; rev = true; }                 // p[-1-m] = p[m]
    else if (gx >= W) { lc = 2 * W - 4 - gx; rev = true; }    // p[W+m]  = p[W-1-m]
    lc = min(max(lc, 0), W - 4);
    const bool any_rev = (wx == 0) || ((wx + 1) * T::VALID + T::HX > W);   // warp-uniform
    const bool lane_out = (lane >= T::HX / 4) && (lane < 32 - T::HX / 4) && (gx >= 0) && (gx < W);
    const int x0 = wx * T::VALID - T::HX;

    // ---- y geometry of this warp's stream ----------------------------------------------------------
    const int y0 = a.out_lo + cy * a.rows_per_chunk;
    const int y1 = min(y0 + a.rows_per_chunk, a.out_hi);
    const int ys = max(y0 - K, 0);                    // first input row
    const int ye = min(y1 - 1 + K, H - 1);            // last input row

    asm volatile("griddepcontrol.wait;" ::: "memory");      // everything below reads what the previous launch wrote

    // ---- does the divergence this stream reads hold a value that defeats the fma contraction? ----
    bool exact = false;
    if (a.tiny_map) {
        const int mw = tiny_map_w(W);
        const int cx0 = max(x0, 0) / TINY_CW, cx1 = min(x0 + 127, W - 1) / TINY_CW;
        const int cy0 = ys / TINY_CH, cy1 = ye / TINY_CH;
        const int ncx = cx1 - cx0 + 1, n = ncx * (cy1 - cy0 + 1);
        unsigned f = 0;
        for (int k = lane; k < n; k += 32) f |= a.tiny_map[(cy0 + k / ncx) * mw + cx0 + k % ncx];
        exact = __any_sync(0xffffffffu, f != 0);
    }
    const void* tp = &maps.p;
    const void* td = &maps.d;
    // The common case first, so that it is laid out first: code placement matters to this kernel (it
    // runs one or two warps per scheduler, straight out of the instruction caches).  The un-contracted
    // instantiations are kept out of line for the same reason.  Every contracted stream, mirrored
    // window or not, runs ONE instantiation (REV: 8 selects per step, the identity where rev is false):
    // an SM whose resident warps ran two separate steady-state loops would keep two loop bodies in its
    // instruction cache, and a loop body twice as large measured 11 % slower (DESIGN §5.8).
    if (!exact) {
        const float big = tb_stream<K, SCALE, true, false, BATCH>(a, tp, td, smem4, lane, x0, lc, gx, rev, lane_out, y0, y1, ys);
        // an input that could make S - d overflow within this launch: solve the stream again with the exact
        // tail.  It stores the same rows, nobody else reads pout before the grid ends (pin != pout), and its
        // stages were drained, so the barriers are retired and made afresh
        exact = __any_sync(0xffffffffu, big >= BIG_IN);
        if (exact && lane == 0) {
            unsigned long long* bars = reinterpret_cast<unsigned long long*>(smem4 + T::NS * T::STAGE4);
            for (int q = 0; q < T::NS; ++q) mbar_inval(bars + q);
        }
        __syncwarp();
        if (!exact) return;
    }
    tb_stream_exact<K, SCALE, BATCH>(a, tp, td, smem4, lane, x0, lc, gx, rev, lane_out, y0, y1, ys, any_rev);
}

// ---- producers of the tiny-divergence map ----------------------------------------------------------
// Host-written divergence (fluid_write, fluid_pressure_solve_host) and ghost rows received from a
// neighbour are scanned by this kernel; the kernels that COMPUTE divergence flag cells themselves.
// The map must have been zeroed for the rows being scanned (cudaMemsetAsync by the caller).
__global__ void __launch_bounds__(256) tiny_scan_kernel(const float* __restrict__ div, unsigned char* __restrict__ map,
                                                        int W, int row_off, int j_lo, int j_hi) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int j = j_lo + blockIdx.y;
    if (i >= W || j >= j_hi) return;
    if (is_tiny_div(__ldg(div + (size_t)(j - row_off) * W + i)))
        map[(j / TINY_CH) * tiny_map_w(W) + i / TINY_CW] = 1;
}

}  // namespace fk
