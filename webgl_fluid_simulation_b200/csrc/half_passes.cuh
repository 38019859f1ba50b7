// half_passes.cuh — the HALF-FLOAT STORAGE mode (FLUID_FLAG_HALF_STORAGE): what the reference
// really stores.  script.js keeps every field in half-float textures (ext.halfFloatTexType, S:138-147;
// RGBA16F dye, RG16F velocity, R16F pressure / divergence / curl, S:986-1006): each blit computes in
// fp32 and the result is rounded to fp16 when it is written.  The fp32-storage kernels of this
// library are what BASELINE.json's metric asks for; this mode reproduces the reference's own
// storage format bit for bit — same arithmetic (the shared device functions of passes.cuh), fp16
// round-to-nearest-even on every pass write, one launch per reference blit — and halves the
// algorithmic bytes (Jacobi: 6 B per update), which gives the second roofline point of bench.py.
//
// Deliberately simple: one thread per cell (4 cells for the Jacobi sweep), single GPU.  The
// temporally blocked / streaming machinery stays fp32-only: a temporally blocked half kernel would
// have to round every level to fp16 anyway (the reference rounds after EVERY sweep).
#pragma once
#include <cuda_fp16.h>

#include "passes.cuh"

namespace fk {
namespace hs {

typedef __half h1;
typedef __half2 h2;
struct __align__(8) h4 { __half2 a, b; };

__device__ __forceinline__ float ld(const h1* p, int i) { return __half2float(__ldg(p + i)); }
__device__ __forceinline__ float2 ld(const h2* p, int i) { return __half22float2(__ldg(p + i)); }
__device__ __forceinline__ float4 ld(const h4* p, int i) {
    const uint2 raw = __ldg(reinterpret_cast<const uint2*>(p) + i);
    const float2 a = __half22float2(*reinterpret_cast<const h2*>(&raw.x)), b = __half22float2(*reinterpret_cast<const h2*>(&raw.y));
    return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ void st(h1* p, int i, float v) { p[i] = __float2half_rn(v); }
__device__ __forceinline__ void st(h2* p, int i, float2 v) { p[i] = __floats2half2_rn(v.x, v.y); }
__device__ __forceinline__ void st(h4* p, int i, float4 v) {
    h4 o; o.a = __floats2half2_rn(v.x, v.y); o.b = __floats2half2_rn(v.z, v.w);
    p[i] = o;
}

#define HS_CELL()                                                                      \
    const int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y * blockDim.y + threadIdx.y; \
    if (i >= W || j >= H) return;                                                      \
    const int il = max(i - 1, 0), ir = min(i + 1, W - 1), jb = max(j - 1, 0), jt = min(j + 1, H - 1)

__global__ void __launch_bounds__(256) curl_kernel(const h2* __restrict__ v, h1* __restrict__ curl, int W, int H) {
    HS_CELL();
    const float L = ld(v, j * W + il).y, R = ld(v, j * W + ir).y, T = ld(v, jt * W + i).x, B = ld(v, jb * W + i).x;
    const float vort = ((R - L) - T) + B;
    st(curl, j * W + i, 0.5f * vort);
}
__global__ void __launch_bounds__(256) vorticity_kernel(const h2* __restrict__ v, const h1* __restrict__ curl,
                                                        h2* __restrict__ vout, int W, int H, float curl_k,
                                                        const float* __restrict__ dtp) {
    HS_CELL();
    st(vout, j * W + i, vorticity_apply(ld(v, j * W + i), ld(curl, j * W + il), ld(curl, j * W + ir), ld(curl, jt * W + i),
                                        ld(curl, jb * W + i), ld(curl, j * W + i), curl_k, __ldg(dtp)));
}
__global__ void __launch_bounds__(256) divergence_kernel(const h2* __restrict__ v, h1* __restrict__ div, int W, int H) {
    HS_CELL();
    float L = ld(v, j * W + il).x, R = ld(v, j * W + ir).x, T = ld(v, jt * W + i).y, B = ld(v, jb * W + i).y;
    const float2 C = ld(v, j * W + i);
    if (i == 0) L = -C.x;
    if (i == W - 1) R = -C.x;
    if (j == H - 1) T = -C.y;
    if (j == 0) B = -C.y;
    st(div, j * W + i, 0.5f * (((R - L) + T) - B));
}
__global__ void __launch_bounds__(256) scale_kernel(const h1* __restrict__ in, h1* __restrict__ out, int n, float value) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n) st(out, k, value * ld(in, k));
}
// one Jacobi sweep (S:868-890), one cell per thread: 6 B per update (read p 2 + div 2, write p 2)
__global__ void __launch_bounds__(256) jacobi_kernel(const h1* __restrict__ p, const h1* __restrict__ div,
                                                     h1* __restrict__ pout, int W, int H) {
    HS_CELL();
    const float L = ld(p, j * W + il), R = ld(p, j * W + ir), B = ld(p, jb * W + i), T = ld(p, jt * W + i);
    st(pout, j * W + i, ((((L + R) + B) + T) - ld(div, j * W + i)) * 0.25f);
}
// the same sweep, 8 cells (16 bytes) per thread, shuffles for the x-neighbours: width % 8 == 0
__global__ void __launch_bounds__(256) jacobi8_kernel(const h1* __restrict__ p, const h1* __restrict__ div,
                                                      h1* __restrict__ pout, int W, int H) {
    const int W8 = W >> 3;
    const int g = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y * blockDim.y + threadIdx.y;
    const bool live = g < W8 && j < H;
    const int gc = min(g, W8 - 1), jc = min(j, H - 1);
    const int jb = max(jc - 1, 0), jt = min(jc + 1, H - 1);
    auto row8 = [&](const h1* base, int r, float (&o)[8]) {
        const uint4 raw = __ldg(reinterpret_cast<const uint4*>(base + (size_t)r * W) + gc);
        const unsigned w[4] = {raw.x, raw.y, raw.z, raw.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) { const float2 f = __half22float2(*reinterpret_cast<const h2*>(&w[k])); o[2 * k] = f.x; o[2 * k + 1] = f.y; }
    };
    float c[8], b[8], t[8], d[8];
    row8(p, jc, c); row8(p, jb, b); row8(p, jt, t); row8(div, jc, d);
    float l = __shfl_up_sync(0xffffffffu, c[7], 1), r = __shfl_down_sync(0xffffffffu, c[0], 1);
    const int lane = threadIdx.x & 31;
    if (lane == 0) l = gc > 0 ? ld(p, jc * W + 8 * gc - 1) : c[0];
    if (lane == 31 || gc == W8 - 1) r = gc < W8 - 1 ? ld(p, jc * W + 8 * gc + 8) : c[7];
    float o[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) {
        const float L = k == 0 ? l : c[k - 1], R = k == 7 ? r : c[k + 1];
        o[k] = ((((L + R) + b[k]) + t[k]) - d[k]) * 0.25f;
    }
    if (live) {
        uint4 raw;
        unsigned* w = &raw.x;
#pragma unroll
        for (int k = 0; k < 4; ++k) { const h2 q = __floats2half2_rn(o[2 * k], o[2 * k + 1]); w[k] = *reinterpret_cast<const unsigned*>(&q); }
        reinterpret_cast<uint4*>(pout + (size_t)jc * W)[gc] = raw;
    }
}
__global__ void __launch_bounds__(256) gradient_kernel(const h1* __restrict__ p, const h2* __restrict__ v,
                                                       h2* __restrict__ vout, int W, int H) {
    HS_CELL();
    float2 vel = ld(v, j * W + i);
    vel.x = vel.x - (ld(p, j * W + ir) - ld(p, j * W + il));
    vel.y = vel.y - (ld(p, jt * W + i) - ld(p, jb * W + i));
    st(vout, j * W + i, vel);
}

// bilerp of S:758-770 on half textures (texels widen exactly; arithmetic in fp32 like the shader)
template <typename T, typename F>
__device__ __forceinline__ F bilerp_h(const T* __restrict__ tex, int W, const Taps& t);
template <>
__device__ __forceinline__ float2 bilerp_h<h2, float2>(const h2* __restrict__ tex, int W, const Taps& t) {
    const float2 a = ld(tex, t.j0 * W + t.i0), b = ld(tex, t.j0 * W + t.i1), c = ld(tex, t.j1 * W + t.i0), d = ld(tex, t.j1 * W + t.i1);
    float2 r;
    r.x = mixf(mixf(a.x, b.x, t.fx), mixf(c.x, d.x, t.fx), t.fy);
    r.y = mixf(mixf(a.y, b.y, t.fx), mixf(c.y, d.y, t.fx), t.fy);
    return r;
}
template <>
__device__ __forceinline__ float4 bilerp_h<h4, float4>(const h4* __restrict__ tex, int W, const Taps& t) {
    const float4 a = ld(tex, t.j0 * W + t.i0), b = ld(tex, t.j0 * W + t.i1), c = ld(tex, t.j1 * W + t.i0), d = ld(tex, t.j1 * W + t.i1);
    float4 r;
    r.x = mixf(mixf(a.x, b.x, t.fx), mixf(c.x, d.x, t.fx), t.fy);
    r.y = mixf(mixf(a.y, b.y, t.fx), mixf(c.y, d.y, t.fx), t.fy);
    r.z = mixf(mixf(a.z, b.z, t.fx), mixf(c.z, d.z, t.fx), t.fy);
    r.w = mixf(mixf(a.w, b.w, t.fx), mixf(c.w, d.w, t.fx), t.fy);
    return r;
}

// advectionShader S:746-784 (MANUAL_FILTERING form, like the fp32 kernels): velocity sampled at the
// target cell's uv on the sim grid, back-trace with the SIM texel size, source on its own grid
template <typename T, typename F>
__global__ void __launch_bounds__(256) advect_kernel(const h2* __restrict__ vel, int Wv, int Hv, const T* __restrict__ src,
                                                     T* __restrict__ out, int W, int H, const float* __restrict__ dtp,
                                                     float dissipation, float tsx, float tsy, float dsx, float dsy) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y * blockDim.y + threadIdx.y;
    if (i >= W || j >= H) return;
    const float dt = __ldg(dtp);       // tsx.. = fp32 of the JS doubles 1/W (S:1061-1062), computed on the host
    const float uvx = ((float)i + 0.5f) / (float)W, uvy = ((float)j + 0.5f) / (float)H;
    const float2 vv = bilerp_h<h2, float2>(vel, Wv, bilerp_taps(uvx, uvy, tsx, tsy, Wv, Hv));
    const float cx = uvx - (dt * vv.x) * tsx, cy = uvy - (dt * vv.y) * tsy;
    const F r = bilerp_h<T, F>(src, W, bilerp_taps(cx, cy, dsx, dsy, W, H));
    const float decay = 1.0f + dissipation * dt;
    F o = r;
    float* oc = reinterpret_cast<float*>(&o);
#pragma unroll
    for (int k = 0; k < (int)(sizeof(F) / sizeof(float)); ++k) oc[k] = oc[k] / decay;
    st(out, j * W + i, o);
}

// storage policy of splats_kernel (passes.cuh): round() is the st() + ld() pair above, the RN-even
// store of one splat() call and the exact widening read of the next.  Plain loads: launches after a
// block's first run in place.
struct SplatHalf {
    typedef h2 V;
    typedef h4 D;
    template <int C> static __device__ __forceinline__ void load(const void* p, size_t o, float* v) {
        if (C == 2) {
            const float2 t = __half22float2(static_cast<const h2*>(p)[o]); v[0] = t.x; v[1] = t.y;
        } else {
            const h4 t = static_cast<const h4*>(p)[o];
            const float2 a = __half22float2(t.a), b = __half22float2(t.b);
            v[0] = a.x; v[1] = a.y; v[2] = b.x; v[3] = b.y;
        }
    }
    template <int C> static __device__ __forceinline__ void store(void* p, size_t o, const float* v) {
        if (C == 2) static_cast<h2*>(p)[o] = __floats2half2_rn(v[0], v[1]);
        else { h4 t; t.a = __floats2half2_rn(v[0], v[1]); t.b = __floats2half2_rn(v[2], v[3]); static_cast<h4*>(p)[o] = t; }
    }
    template <int C> static __device__ __forceinline__ void round(float* v) {
#pragma unroll
        for (int q = 0; q < C; q += 2) {
            const float2 t = __half22float2(__floats2half2_rn(v[q], v[q + 1]));
            v[q] = t.x; v[q + 1] = t.y;
        }
    }
};

// host <-> device conversions of fluid_read / fluid_write (the ABI speaks fp32)
__global__ void __launch_bounds__(256) widen_kernel(const h1* __restrict__ in, float* __restrict__ out, size_t n) {
    const size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n) out[k] = __half2float(in[k]);
}
__global__ void __launch_bounds__(256) narrow_kernel(const float* __restrict__ in, h1* __restrict__ out, size_t n) {
    const size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n) out[k] = __float2half_rn(in[k]);
}
__global__ void __launch_bounds__(256) fill_alpha_kernel(h4* __restrict__ d, size_t n) {
    const size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n) st(d, (int)k, make_float4(0.f, 0.f, 0.f, 1.f));
}

}  // namespace hs
}  // namespace fk
