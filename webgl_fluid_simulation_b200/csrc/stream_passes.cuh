// stream_passes.cuh — the 5-point-stencil passes of step() other than the Jacobi loop, as
// ROW-STREAMING warp kernels (generation 2 of curl / vorticity / divergence and gradientSubtract).
//
// Shape shared by the kernels in this file (the same idea as jacobi_tb_kernel, one sweep deep):
//   * a warp owns a window of 128 columns — lane l holds columns 4l..4l+3 as float4 (scalar fields)
//     or two float4 (velocity, interleaved xy) — and streams UP a chunk of rows, keeping the rows a
//     stencil still needs in registers: every field row is read from HBM once per chunk (+ halo
//     rows), with 16-byte coalesced loads and stores;
//   * x-neighbours across lanes come from __shfl_up/down; there is no shared memory and no
//     __syncthreads: warps are independent (4 per CTA only to amortise CTA launch);
//   * CLAMP_TO_EDGE (S:1051-1052) / the explicit walls of divergenceShader (S:804-807) are selects
//     on the lanes / rows that touch a wall, in GLOBAL coordinates (`Grid`), so the kernels serve a
//     full grid and a row slab alike;
//   * arithmetic is the GLSL expression order, op for op (library built with --fmad=false, IEEE
//     div / sqrt): results are bit-identical to the one-blit-per-pass kernels of passes.cuh, which
//     stay as the fallback for widths that are not a multiple of 4 and as the `FLUID_FLAG_UNFUSED`
//     test surface.
#pragma once
#include "passes.cuh"

namespace fk {

struct StreamArgs {
    Grid g;               // global size, row_off of the local buffers, rows [j_lo, j_hi) to produce
    int rows_per_chunk;   // output rows per warp stream
    int nxw;              // windows per row
};

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

// ---- gradientSubtractShader S:892-913 -----------------------------------------------------------
//   v.x -= p[c(i+1),j] - p[c(i-1),j];   v.y -= p[i,c(j+1)] - p[i,c(j-1)]
// 20 B per cell (read p 4 + v 8, write v 8).  Windows do not overlap: the two lanes at the ends of a
// warp fetch their one missing neighbour with a scalar load (L1/L2 hit: the next warp streams it).
constexpr int GS_WARPS = 4;
constexpr int GS_U = 4;                                          // rows per software-pipeline group
// BATCH: blockIdx.z is the member of a batch handle, whose fields are dense (B, H, W) arrays (one GPU)
template <bool BATCH = false>
__global__ void __launch_bounds__(32 * GS_WARPS) gradient_stream_kernel(const float* __restrict__ p,
                                                                       const float2* __restrict__ v,
                                                                       float2* __restrict__ vout, StreamArgs a) {
    if constexpr (BATCH) {
        const size_t mo = (size_t)blockIdx.z * a.g.W * a.g.H;
        p += mo; v += mo; vout += mo;
    }
    const int lane = threadIdx.x & 31;
    const int wid = blockIdx.x * GS_WARPS + (threadIdx.x >> 5);
    const int wx = wid % a.nxw, cy = wid / a.nxw;
    const int W = a.g.W, H = a.g.H;
    const int y0 = a.g.j_lo + cy * a.rows_per_chunk;
    const int y1 = min(y0 + a.rows_per_chunk, a.g.j_hi);
    if (y0 >= y1) return;                                   // warp-uniform
    const int c0 = wx * 128 + 4 * lane;
    const bool live = c0 < W;
    const int cc = live ? c0 : W - 4;                       // dead lanes of the last window re-read its last group
    const bool wall_l = (c0 == 0), wall_r = (c0 + 4 == W);
    const bool edge_l = (lane == 0) && !wall_l, edge_r = (lane == 31) && !wall_r && live;

    const float* prow = p + (ptrdiff_t)(0 - a.g.row_off) * W + cc;      // + j*W : row j, this lane's group
    auto P = [&](int j) { return ldg4(prow + (ptrdiff_t)j * W); };
    float4 below = P(max(y0 - 1, 0)), cur = P(y0);
    // GS_U rows per iteration, every load of the group issued before the first use: 3 x GS_U
    // 16-byte loads in flight per lane is what keeps HBM busy with this little arithmetic
#pragma unroll 1
    for (int j0 = y0; j0 < y1; j0 += GS_U) {
        float4 ab[GS_U], va[GS_U], vb[GS_U];
        float el[GS_U], er[GS_U];
#pragma unroll
        for (int u = 0; u < GS_U; ++u) {
            const int j = min(j0 + u, y1 - 1);              // the tail of a chunk re-reads its last row (not stored)
            ab[u] = P(min(j + 1, H - 1));
            const float4* vr = reinterpret_cast<const float4*>(v + (ptrdiff_t)(j - a.g.row_off) * W + cc);
            va[u] = __ldg(vr); vb[u] = __ldg(vr + 1);
            el[u] = edge_l ? __ldg(prow + (ptrdiff_t)j * W - 1) : 0.f;
            er[u] = edge_r ? __ldg(prow + (ptrdiff_t)j * W + 4) : 0.f;
        }
#pragma unroll
        for (int u = 0; u < GS_U; ++u) {
            const int j = j0 + u;
            const float4 above = ab[u];
            float l = __shfl_up_sync(0xffffffffu, cur.w, 1);
            float r = __shfl_down_sync(0xffffffffu, cur.x, 1);
            if (edge_l) l = el[u];
            if (edge_r) r = er[u];
            if (wall_l) l = cur.x;                          // CLAMP_TO_EDGE: p[-1,j] = p[0,j]
            if (wall_r) r = cur.w;
            float4 oa, ob;
            oa.x = va[u].x - (cur.y - l);        oa.y = va[u].y - (above.x - below.x);
            oa.z = va[u].z - (cur.z - cur.x);    oa.w = va[u].w - (above.y - below.y);
            ob.x = vb[u].x - (cur.w - cur.y);    ob.y = vb[u].y - (above.z - below.z);
            ob.z = vb[u].z - (r - cur.z);        ob.w = vb[u].w - (above.w - below.w);
            if (live && j < y1) {
                float4* o = reinterpret_cast<float4*>(vout + (ptrdiff_t)(j - a.g.row_off) * W + cc);
                o[0] = oa; o[1] = ob;
            }
            below = cur; cur = above;
        }
    }
}

// ---- curl -> vorticity -> divergence in one streaming pass (S:1234-1251) -------------------------
//   curl  C[j] = 0.5*(((vy[c(i+1)] - vy[c(i-1)]) - vx[c(j+1)]) + vx[c(j-1)])          (S:814-833)
//   new v N[j] = vorticity_apply(V[j]; C at c(i-1), c(i+1), c(j+1), c(j-1), centre)      (S:835-866)
//   div   D[j] = 0.5*(((Nx[i+1] - Nx[i-1]) + Ny[j+1]) - Ny[j-1]),  walls: -centre       (S:786-812)
// 24 B per cell (read v 8; write v 8 + divergence 4 + curl 4) instead of 44 B for the three blits.
// Software pipeline in y: the step that takes V[s] produces C[s-1], N[s-2] and D[s-3]; the three
// rows of V, C and N a step still needs rotate through register slots with period 3 == the unroll,
// so nothing is ever moved.  Velocity rows reach the warp through a per-warp shared-memory ring
// filled by cp.async (16 B per lane, RING rows in flight): the global-load latency is paid in the
// ring, not in registers.  Windows overlap by one lane (4 columns) on each side: lanes 1..30 of a
// warp produce output, 120 columns.
constexpr int CVD2_WARPS = 4;
constexpr int CVD2_VALID = 120;
#ifndef FLUID_CVD_MINBLOCKS            // tuning builds
#define FLUID_CVD_MINBLOCKS 4
#endif
#ifndef FLUID_CVD_RING
#define FLUID_CVD_RING 6
#endif
constexpr int CVD2_MINBLOCKS = FLUID_CVD_MINBLOCKS;              // register budget: 4 CTAs = 16 streams per SM at 118 registers (FLUID_CVD_MINBLOCKS: tuning builds)
constexpr int CVD2_RING = FLUID_CVD_RING;                        // rows in flight per warp (1 KB each)
constexpr int CVD2_SMEM = CVD2_WARPS * CVD2_RING * 64 * (int)sizeof(float4);

// cp.async (LDGSTS): global -> shared without passing through registers.  Each lane copies, and
// later reads back, ONLY its own 16 bytes of a row, so the per-thread completion wait
// (cp.async.wait_group) is all the synchronisation the ring needs.
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gmem_src) {
    const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(d), "l"(gmem_src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

struct Vel4 { float x[4], y[4]; };          // 4 consecutive cells of a velocity row

__device__ __forceinline__ Vel4 unpack_vel(const float4 a, const float4 b) {
    Vel4 r;
    r.x[0] = a.x; r.y[0] = a.y; r.x[1] = a.z; r.y[1] = a.w;
    r.x[2] = b.x; r.y[2] = b.y; r.x[3] = b.z; r.y[3] = b.w;
    return r;
}

struct CvdStream {
    const float4* src;    // next velocity row to stage (this lane's two float4)
    int jload;            // LOGICAL row index src stands for (clamped to [0, H-1] when dereferenced)
    int slot;             // ring slot consumed by the next step
    float4* o_curl;       // where curl row s-1 of the current step goes, ditto below (advance one row per step)
    float4* o_vel;
    float4* o_div;
};

// one pipeline step: takes V[s] from the ring, produces C[s-1], N[s-2], D[s-3]
template <int PH>
__device__ __forceinline__ void cvd_step(Vel4 (&V)[3], float (&C)[3][4], Vel4 (&N)[3], CvdStream& st,
                                         float4* __restrict__ ring, const int s, const int y0, const int y1,
                                         const int H, const int W4, const bool out_lane, const bool wall_l,
                                         const bool wall_r, const float curl_k, const float dt,
                                         unsigned char* __restrict__ tiny_cell) {
    // slot indices: X[(PH+2)%3] is the row produced / taken at this step, (PH+1)%3 one step older,
    // (PH+0)%3 two steps older
    constexpr int NEW = (PH + 2) % 3, MID = (PH + 1) % 3, OLD = (PH + 0) % 3;
    // ---- take V[s]; refill the ring slot with the row RING steps ahead -------------------------------
    cp_async_wait<CVD2_RING - 1>();
    float4* cell = ring + st.slot * 64;
    V[NEW] = unpack_vel(lds128(cell), lds128(cell + 32));
    cp_async16(cell, st.src); cp_async16(cell + 32, st.src + 1);
    cp_async_commit();
    if (st.jload >= 0 && st.jload < H - 1) st.src += 2 * W4;     // CLAMP_TO_EDGE of the velocity fetch in y
    ++st.jload;
    st.slot = (st.slot + 1 == CVD2_RING) ? 0 : st.slot + 1;

    // ---- curl row s-1 from V[s-2] (OLD), V[s-1] (MID), V[s] (NEW) --------------------------------------
    {
        float l = __shfl_up_sync(0xffffffffu, V[MID].y[3], 1);
        float r = __shfl_down_sync(0xffffffffu, V[MID].y[0], 1);
        if (wall_l) l = V[MID].y[0];                        // vy[c(-1)] = vy[0]
        if (wall_r) r = V[MID].y[3];
        const float L[4] = {l, V[MID].y[0], V[MID].y[1], V[MID].y[2]};
        const float R[4] = {V[MID].y[1], V[MID].y[2], V[MID].y[3], r};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float vort = ((R[k] - L[k]) - V[NEW].x[k]) + V[OLD].x[k];
            C[NEW][k] = 0.5f * vort;                        // slot NEW of C now holds curl row s-1
        }
        if (out_lane && (unsigned)(s - 1 - y0) < (unsigned)(y1 - y0))
            *st.o_curl = make_float4(C[NEW][0], C[NEW][1], C[NEW][2], C[NEW][3]);
    }
    // ---- new velocity row jn = s-2 from curl rows s-3 (OLD), s-2 (MID), s-1 (NEW) and V[s-2] (OLD) -------
    {
        const int jn = s - 2;
        float l = __shfl_up_sync(0xffffffffu, C[MID][3], 1);
        float r = __shfl_down_sync(0xffffffffu, C[MID][0], 1);
        if (wall_l) l = C[MID][0];                          // curl[c(-1)] = curl[0]
        if (wall_r) r = C[MID][3];
        const float L[4] = {l, C[MID][0], C[MID][1], C[MID][2]};
        const float R[4] = {C[MID][1], C[MID][2], C[MID][3], r};
        const bool bot = (jn <= 0), top = (jn >= H - 1);    // curl[c(j-1)] / curl[c(j+1)] at the walls
        VortPre pre[4];
        bool ok = true;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float T = top ? C[MID][k] : C[NEW][k];
            const float B = bot ? C[MID][k] : C[OLD][k];
            pre[k] = vort_pre(L[k], R[k], T, B);
            ok &= pre[k].ok;
        }
        if (__all_sync(0xffffffffu, ok)) {                  // warp-uniform: the branch-free quotients are exact here
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float2 nv = vort_post(make_float2(V[OLD].x[k], V[OLD].y[k]), pre[k], C[MID][k], curl_k, dt);
                N[NEW].x[k] = nv.x; N[NEW].y[k] = nv.y;     // slot NEW of N now holds new-velocity row s-2
            }
        } else {
#pragma unroll
            for (int k = 0; k < 4; ++k) {                   // rare (subnormal / non-finite operands): nvcc's guarded sqrt / divisions
                const float T = top ? C[MID][k] : C[NEW][k];
                const float B = bot ? C[MID][k] : C[OLD][k];
                const float2 nv = vorticity_apply(make_float2(V[OLD].x[k], V[OLD].y[k]), L[k], R[k], T, B, C[MID][k], curl_k, dt);
                N[NEW].x[k] = nv.x; N[NEW].y[k] = nv.y;
            }
        }
        if (out_lane && (unsigned)(jn - y0) < (unsigned)(y1 - y0)) {
            st.o_vel[0] = make_float4(N[NEW].x[0], N[NEW].y[0], N[NEW].x[1], N[NEW].y[1]);
            st.o_vel[1] = make_float4(N[NEW].x[2], N[NEW].y[2], N[NEW].x[3], N[NEW].y[3]);
        }
    }
    // ---- divergence row jd = s-3 from new-velocity rows s-4 (OLD), s-3 (MID), s-2 (NEW) ----------------
    {
        const int jd = s - 3;
        float l = __shfl_up_sync(0xffffffffu, N[MID].x[3], 1);
        float r = __shfl_down_sync(0xffffffffu, N[MID].x[0], 1);
        if (wall_l) l = -N[MID].x[0];                       // vL.x < 0  ->  L = -C.x   (S:804)
        if (wall_r) r = -N[MID].x[3];                       // vR.x > 1  ->  R = -C.x   (S:805)
        const float L[4] = {l, N[MID].x[0], N[MID].x[1], N[MID].x[2]};
        const float R[4] = {N[MID].x[1], N[MID].x[2], N[MID].x[3], r};
        const bool bot = (jd == 0), top = (jd == H - 1);
        float d[4];
        bool tiny = false;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float T = top ? -N[MID].y[k] : N[NEW].y[k];   // vT.y > 1  ->  T = -C.y   (S:806)
            const float B = bot ? -N[MID].y[k] : N[OLD].y[k];   // vB.y < 0  ->  B = -C.y   (S:807)
            d[k] = 0.5f * (((R[k] - L[k]) + T) - B);
            tiny |= is_tiny_div(d[k]);
        }
        if (out_lane && (unsigned)(jd - y0) < (unsigned)(y1 - y0)) {
            *st.o_div = make_float4(d[0], d[1], d[2], d[3]);
            if (tiny && tiny_cell) tiny_cell[(jd / TINY_CH) * tiny_map_w(4 * W4)] = 1;
        }
    }
    st.o_curl += W4; st.o_vel += 2 * W4; st.o_div += W4;
}

// BATCH: blockIdx.z is the member of a batch handle; each member flags its own region of the tiny map, and
// dtp is the member table (jacobi.cuh), from which the member takes its dt and CURL (curl_k is not read)
template <bool BATCH = false>
__global__ void __launch_bounds__(32 * CVD2_WARPS, CVD2_MINBLOCKS) cvd_stream_kernel(const float2* __restrict__ v,
                                                                    float* __restrict__ curl,
                                                                    float2* __restrict__ vout,
                                                                    float* __restrict__ div, StreamArgs a,
                                                                    float curl_k, const float* __restrict__ dtp,
                                                                    unsigned char* __restrict__ tiny_map) {
    if constexpr (BATCH) {
        const size_t mo = (size_t)blockIdx.z * a.g.W * a.g.H;
        v += mo; curl += mo; vout += mo; div += mo;
        if (tiny_map) tiny_map += (size_t)blockIdx.z * tiny_map_w(a.g.W) * tiny_map_h(a.g.H);
    }
    extern __shared__ __align__(16) float4 cvd_smem[];
    const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
    const int wid = blockIdx.x * CVD2_WARPS + wib;
    const int wx = wid % a.nxw, cy = wid / a.nxw;
    const int W = a.g.W, H = a.g.H, W4 = W >> 2;
    const int y0 = a.g.j_lo + cy * a.rows_per_chunk;
    const int y1 = min(y0 + a.rows_per_chunk, a.g.j_hi);
    if (y0 >= y1) return;                                   // warp-uniform
    const float dt = BATCH ? member_param(dtp, MP_DT) : __ldg(dtp);
    if constexpr (BATCH) curl_k = member_param(dtp, MP_CURL);

    const int c0 = wx * CVD2_VALID - 4 + 4 * lane;          // first column of this lane (may be off-grid)
    const bool out_lane = (lane >= 1) && (lane <= 30) && (c0 >= 0) && (c0 < W);
    const bool wall_l = (c0 == 0), wall_r = (c0 + 4 == W);
    // off-grid lanes (left of column 0 / right of column W-1 in the edge windows) load some valid
    // address and compute garbage that nobody reads: wall lanes take their clamped neighbour from
    // their own registers
    const int cc = min(max(c0, 0), W - 4);
    float4* ring = cvd_smem + wib * (CVD2_RING * 64) + lane;       // row q: ring[q*64] and ring[q*64+32]

    // D[y0] needs N[y0-1], which needs C[y0-2], which needs V[y0-3]: step s = y0-3 is the first, the
    // last one takes V[y1+2].  Outputs of the first steps fall outside [y0, y1) and are not stored.
    const int s_first = y0 - 3, s_last = y1 + 2;
    CvdStream st;
    st.jload = s_first;
    st.src = reinterpret_cast<const float4*>(v + ((ptrdiff_t)(min(max(s_first, 0), H - 1) - a.g.row_off) * W + cc));
    st.slot = 0;
#pragma unroll
    for (int q = 0; q < CVD2_RING; ++q) {
        cp_async16(ring + q * 64, st.src); cp_async16(ring + q * 64 + 32, st.src + 1);
        cp_async_commit();
        if (st.jload >= 0 && st.jload < H - 1) st.src += 2 * W4;
        ++st.jload;
    }
    const int oc = out_lane ? c0 : 0;
    st.o_curl = reinterpret_cast<float4*>(curl + ((ptrdiff_t)(s_first - 1 - a.g.row_off) * W + oc));
    st.o_vel = reinterpret_cast<float4*>(vout + ((ptrdiff_t)(s_first - 2 - a.g.row_off) * W + oc));
    st.o_div = reinterpret_cast<float4*>(div + ((ptrdiff_t)(s_first - 3 - a.g.row_off) * W + oc));
    unsigned char* tiny_cell = tiny_map ? tiny_map + (oc / TINY_CW) : nullptr;

    Vel4 V[3], N[3];
    float C[3][4];
#pragma unroll
    for (int q = 0; q < 3; ++q)
#pragma unroll
        for (int k = 0; k < 4; ++k) { V[q].x[k] = V[q].y[k] = N[q].x[k] = N[q].y[k] = 0.f; C[q][k] = 0.f; }

#pragma unroll 1
    for (int s = s_first; s <= s_last; s += 3) {
        cvd_step<0>(V, C, N, st, ring, s, y0, y1, H, W4, out_lane, wall_l, wall_r, curl_k, dt, tiny_cell);
        cvd_step<1>(V, C, N, st, ring, s + 1, y0, y1, H, W4, out_lane, wall_l, wall_r, curl_k, dt, tiny_cell);
        cvd_step<2>(V, C, N, st, ring, s + 2, y0, y1, H, W4, out_lane, wall_l, wall_r, curl_k, dt, tiny_cell);
    }
    cp_async_wait<0>();
}

}  // namespace fk
