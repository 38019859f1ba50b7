// half_passes.cuh — the HALF-FLOAT STORAGE mode (FLUID_FLAG_HALF_STORAGE): what the reference
// really stores.  script.js keeps every field in half-float textures (ext.halfFloatTexType, S:138-147;
// RGBA16F dye, RG16F velocity, R16F pressure / divergence / curl, S:986-1006): each blit computes in
// fp32 and the result is rounded to fp16 when it is written.  The fp32-storage kernels of this
// library are what BASELINE.json's metric asks for; this mode reproduces the reference's own
// storage format bit for bit — same arithmetic, fp16 round-to-nearest-even on every pass write, one
// launch per reference blit — and halves the algorithmic bytes (Jacobi: 6 B per update), which gives
// the second roofline point of bench.py.
//
// The passes are the one-cell kernels of passes.cuh / jacobi.cuh instantiated with StoreHalf below,
// single GPU.  The temporally blocked / streaming machinery stays fp32-only: a temporally blocked
// half kernel would have to round every level to fp16 anyway (the reference rounds after EVERY sweep).
#pragma once
#include <cuda_fp16.h>

#include "passes.cuh"

namespace fk {
namespace hs {

typedef __half h1;
typedef __half2 h2;
struct __align__(8) h4 { __half2 a, b; };

// storage policy (passes.cuh StoreF32): texels widen exactly to fp32, stores round to nearest even
struct StoreHalf {
    typedef h1 T1;
    typedef h2 T2;
    typedef h4 T4;
    static __device__ __forceinline__ float ldg(const h1* p, size_t i) { return __half2float(__ldg(p + i)); }
    static __device__ __forceinline__ float2 ldg(const h2* p, size_t i) { return __half22float2(__ldg(p + i)); }
    static __device__ __forceinline__ float4 ldg(const h4* p, size_t i) {
        const uint2 raw = __ldg(reinterpret_cast<const uint2*>(p) + i);
        const float2 a = __half22float2(*reinterpret_cast<const h2*>(&raw.x)), b = __half22float2(*reinterpret_cast<const h2*>(&raw.y));
        return make_float4(a.x, a.y, b.x, b.y);
    }
    static __device__ __forceinline__ float ld(const h1* p, size_t i) { return __half2float(p[i]); }
    static __device__ __forceinline__ float2 ld(const h2* p, size_t i) { return __half22float2(p[i]); }
    static __device__ __forceinline__ float4 ld(const h4* p, size_t i) {
        const h4 t = p[i];
        const float2 a = __half22float2(t.a), b = __half22float2(t.b);
        return make_float4(a.x, a.y, b.x, b.y);
    }
    static __device__ __forceinline__ void st(h1* p, size_t i, float v) { p[i] = __float2half_rn(v); }
    static __device__ __forceinline__ void st(h2* p, size_t i, float2 v) { p[i] = __floats2half2_rn(v.x, v.y); }
    static __device__ __forceinline__ void st(h4* p, size_t i, float4 v) {
        h4 o; o.a = __floats2half2_rn(v.x, v.y); o.b = __floats2half2_rn(v.z, v.w);
        p[i] = o;
    }
    template <int C> static __device__ __forceinline__ void round(float* v) {
#pragma unroll
        for (int q = 0; q < C; q += 2) {
            const float2 t = __half22float2(__floats2half2_rn(v[q], v[q + 1]));
            v[q] = t.x; v[q + 1] = t.y;
        }
    }
};

// one Jacobi sweep (S:868-890), 8 cells (16 bytes) per thread, shuffles for the x-neighbours: width % 8 == 0
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
    if (lane == 0) l = gc > 0 ? StoreHalf::ldg(p, jc * W + 8 * gc - 1) : c[0];
    if (lane == 31 || gc == W8 - 1) r = gc < W8 - 1 ? StoreHalf::ldg(p, jc * W + 8 * gc + 8) : c[7];
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

// host <-> device conversions of fluid_read / fluid_write (the ABI speaks fp32)
__global__ void __launch_bounds__(256) widen_kernel(const h1* __restrict__ in, float* __restrict__ out, size_t n) {
    const size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n) out[k] = __half2float(in[k]);
}
__global__ void __launch_bounds__(256) narrow_kernel(const float* __restrict__ in, h1* __restrict__ out, size_t n) {
    const size_t k = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n) out[k] = __float2half_rn(in[k]);
}

}  // namespace hs
}  // namespace fk
