// postfx.cuh — the display-side post-FX of render() (SURVEY §8f rank 1, second half): bloom
// (applyBloom S:1350-1394; shaders S:614-674) and sunrays (applySunrays + blur S:1396-1419; shaders
// S:461-494, S:676-724) and the display shader for every keyword set with BLOOM or SUNRAYS (S:549-612).
//
// Every kernel is one reference blit: one thread per target texel, sources fetched through the
// GL_LINEAR formula of passes.cuh (linear_fetch4).  Arithmetic order follows the GLSL; with the
// library's --fmad=false / IEEE div+sqrt build everything is bit-identical to the CPU oracle except
// the display's pow() (linearToGamma), which is tolerance-checked like splat's exp().
#pragma once
#include <cuda_runtime.h>

#include "passes.cuh"

namespace fk {

__device__ __forceinline__ float linear_fetch1(const float* __restrict__ tex, int W, int H, float uvx, float uvy) {
    const float u = uvx * (float)W - 0.5f, v = uvy * (float)H - 0.5f;
    const float fi = floorf(u), fj = floorf(v);
    const float a = u - fi, b = v - fj;
    const int i0 = texel_index(fi, W), i1 = texel_index(fi + 1.0f, W);
    const int j0 = texel_index(fj, H), j1 = texel_index(fj + 1.0f, H);
    const float w00 = (1.0f - a) * (1.0f - b), w10 = a * (1.0f - b), w01 = (1.0f - a) * b, w11 = a * b;
    return ((w00 * __ldg(&tex[(size_t)j0 * W + i0]) + w10 * __ldg(&tex[(size_t)j0 * W + i1])) +
            w01 * __ldg(&tex[(size_t)j1 * W + i0])) + w11 * __ldg(&tex[(size_t)j1 * W + i1]);
}

// REPEAT-wrapped LINEAR fetch of the first channel of an RGB (3 floats / texel) texture: the
// dithering texture (createTextureAsync S:1128-1158: LINEAR, REPEAT).
__device__ __forceinline__ float linear_fetch_rgb_r_repeat(const float* __restrict__ tex, int W, int H, float uvx, float uvy) {
    const float u = uvx * (float)W - 0.5f, v = uvy * (float)H - 0.5f;
    const float fi = floorf(u), fj = floorf(v);
    const float a = u - fi, b = v - fj;
    long long i0 = (long long)fi % W, j0 = (long long)fj % H;
    if (i0 < 0) i0 += W;
    if (j0 < 0) j0 += H;
    const long long i1 = (i0 + 1) % W, j1 = (j0 + 1) % H;
    const float w00 = (1.0f - a) * (1.0f - b), w10 = a * (1.0f - b), w01 = (1.0f - a) * b, w11 = a * b;
    return ((w00 * __ldg(&tex[((size_t)j0 * W + i0) * 3]) + w10 * __ldg(&tex[((size_t)j0 * W + i1) * 3])) +
            w01 * __ldg(&tex[((size_t)j1 * W + i0) * 3])) + w11 * __ldg(&tex[((size_t)j1 * W + i1) * 3]);
}

// bloomPrefilterShader S:614-631
__global__ void __launch_bounds__(256) bloom_prefilter_kernel(const float4* __restrict__ dye, int Wd, int Hd,
                                                              float4* __restrict__ out, int w, int h, float curve0,
                                                              float curve1, float curve2, float threshold) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y * blockDim.y + threadIdx.y;
    if (i >= w || j >= h) return;
    const float uvx = ((float)i + 0.5f) / (float)w, uvy = ((float)j + 0.5f) / (float)h;
    const float4 c = linear_fetch4(dye, Wd, Hd, uvx, uvy);
    const float br = fmaxf(c.x, fmaxf(c.y, c.z));
    float rq = fminf(fmaxf(br - curve0, 0.0f), curve1);
    rq = (curve2 * rq) * rq;
    const float f = fmaxf(rq, br - threshold) / fmaxf(br, 0.0001f);
    out[(size_t)j * w + i] = make_float4(c.x * f, c.y * f, c.z * f, 0.0f);
}

// bloomBlurShader S:633-651 / bloomFinalShader S:653-674; add = blendFunc(ONE, ONE) (S:1374-1375)
__global__ void __launch_bounds__(256) box4_kernel(const float4* __restrict__ src, int ws, int hs,
                                                   float4* __restrict__ dst, int w, int h, float scale, int add) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y * blockDim.y + threadIdx.y;
    if (i >= w || j >= h) return;
    const float tsx = (float)(1.0 / (double)ws), tsy = (float)(1.0 / (double)hs);
    const float uvx = ((float)i + 0.5f) / (float)w, uvy = ((float)j + 0.5f) / (float)h;
    const float4 L = linear_fetch4(src, ws, hs, uvx - tsx, uvy), R = linear_fetch4(src, ws, hs, uvx + tsx, uvy);
    const float4 T = linear_fetch4(src, ws, hs, uvx, uvy + tsy), B = linear_fetch4(src, ws, hs, uvx, uvy - tsy);
    float4 s;
    s.x = ((((0.0f + L.x) + R.x) + T.x) + B.x) * 0.25f * scale;
    s.y = ((((0.0f + L.y) + R.y) + T.y) + B.y) * 0.25f * scale;
    s.z = ((((0.0f + L.z) + R.z) + T.z) + B.z) * 0.25f * scale;
    s.w = ((((0.0f + L.w) + R.w) + T.w) + B.w) * 0.25f * scale;
    float4* o = dst + (size_t)j * w + i;
    if (add) { const float4 d = *o; s.x = s.x + d.x; s.y = s.y + d.y; s.z = s.z + d.z; s.w = s.w + d.w; }
    *o = s;
}

// sunraysMaskShader S:676-691 (target = dye.write, like the reference: S:1300)
__global__ void __launch_bounds__(256) sunrays_mask_kernel(const float4* __restrict__ dye, float4* __restrict__ mask,
                                                           int Wd, int Hd) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y * blockDim.y + threadIdx.y;
    if (i >= Wd || j >= Hd) return;
    const float uvx = ((float)i + 0.5f) / (float)Wd, uvy = ((float)j + 0.5f) / (float)Hd;
    float4 c = linear_fetch4(dye, Wd, Hd, uvx, uvy);
    const float br = fmaxf(c.x, fmaxf(c.y, c.z));
    c.w = 1.0f - fminf(fmaxf(br * 20.0f, 0.0f), 0.8f);
    mask[(size_t)j * Wd + i] = c;
}

// sunraysShader S:693-724
__global__ void __launch_bounds__(256) sunrays_kernel(const float4* __restrict__ mask, int Wm, int Hm,
                                                      float* __restrict__ out, int w, int h, float weight) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y * blockDim.y + threadIdx.y;
    if (i >= w || j >= h) return;
    const float Density = 0.3f, Decay = 0.95f, Exposure = 0.7f;
    const float f = (float)(1.0 / 16.0) * Density;
    const float uvx = ((float)i + 0.5f) / (float)w, uvy = ((float)j + 0.5f) / (float)h;
    float cx = uvx, cy = uvy;
    float dx = uvx - 0.5f, dy = uvy - 0.5f;
    dx = dx * f; dy = dy * f;
    float illum = 1.0f;
    float color = linear_fetch4(mask, Wm, Hm, uvx, uvy).w;
#pragma unroll 1
    for (int k = 0; k < 16; ++k) {
        cx = cx - dx; cy = cy - dy;
        const float col = linear_fetch4(mask, Wm, Hm, cx, cy).w;
        color = color + (col * illum) * weight;
        illum = illum * Decay;
    }
    out[(size_t)j * w + i] = color * Exposure;
}

// blurShader S:478-494 + blurVertexShader S:461-476 on the one-channel sunrays texture
__global__ void __launch_bounds__(256) blur3_kernel(const float* __restrict__ src, float* __restrict__ dst, int w, int h,
                                                    float tsx, float tsy) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y * blockDim.y + threadIdx.y;
    if (i >= w || j >= h) return;
    const float off = 1.33333333f;
    const float uvx = ((float)i + 0.5f) / (float)w, uvy = ((float)j + 0.5f) / (float)h;
    const float c = linear_fetch1(src, w, h, uvx, uvy);
    const float l = linear_fetch1(src, w, h, uvx - tsx * off, uvy - tsy * off);
    const float r = linear_fetch1(src, w, h, uvx + tsx * off, uvy + tsy * off);
    float sum = c * 0.29411764f;
    sum = sum + l * 0.35294117f;
    sum = sum + r * 0.35294117f;
    dst[(size_t)j * w + i] = sum;
}

// displayShaderSource S:549-612 compiled with the keywords updateKeywords picks (S:1160-1166), over
// the background of render(), premultiplied blend.  One instantiation per keyword set with BLOOM or
// SUNRAYS; the sets with neither use display_kernel (passes.cuh).  The inputs of a keyword that is
// off are never read (pass nullptr).  Out: the output policy (passes.cuh), the fp32 frame of render()
// or the 8-bit image of captureScreenshot.
template <bool SHADING, bool BLOOM, bool SUNRAYS, class Out = StoreFrame>
__global__ void __launch_bounds__(256) display_full_kernel(const float4* __restrict__ dye, int Wd, int Hd,
                                                           const float4* __restrict__ bloom, int bw, int bh,
                                                           const float* __restrict__ sun, int sw, int sh,
                                                           const float* __restrict__ dither, int dw, int dh,
                                                           typename Out::T* __restrict__ out, int w, int h, float br_, float bg_,
                                                           float bb_, int bg_mode, float aspect, float4 ts) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y * blockDim.y + threadIdx.y;
    if (i >= w || j >= h) return;
    const float tsx = ts.x, tsy = ts.y;     // 1/width, 1/height (S:1337) and getTextureScale (S:1626-1631): JS doubles, narrowed on the host
    const float dsx = ts.z, dsy = ts.w;
    const float uvx = ((float)i + 0.5f) / (float)w, uvy = ((float)j + 0.5f) / (float)h;
    const float4 c = linear_fetch4(dye, Wd, Hd, uvx, uvy);
    float cc[3] = {c.x, c.y, c.z};
    if constexpr (SHADING) {
        const float4 lc = linear_fetch4(dye, Wd, Hd, uvx - tsx, uvy), rc = linear_fetch4(dye, Wd, Hd, uvx + tsx, uvy);
        const float4 tc = linear_fetch4(dye, Wd, Hd, uvx, uvy + tsy), bc = linear_fetch4(dye, Wd, Hd, uvx, uvy - tsy);
        const float dx = len3(rc) - len3(lc), dy = len3(tc) - len3(bc);
        const float nz = sqrtf(tsx * tsx + tsy * tsy);
        const float nl = sqrtf((dx * dx + dy * dy) + nz * nz);
        const float d = ((dx / nl) * 0.0f + (dy / nl) * 0.0f) + (nz / nl) * 1.0f;
        const float diffuse = fminf(fmaxf(d + 0.7f, 0.7f), 1.0f);
#pragma unroll
        for (int k = 0; k < 3; ++k) cc[k] = cc[k] * diffuse;
    }
    float bl[3] = {0.0f, 0.0f, 0.0f};
    if constexpr (BLOOM) {
        const float4 b = linear_fetch4(bloom, bw, bh, uvx, uvy);
        bl[0] = b.x; bl[1] = b.y; bl[2] = b.z;
    }
    if constexpr (SUNRAYS) {
        const float s = linear_fetch1(sun, sw, sh, uvx, uvy);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            cc[k] = cc[k] * s;
            if constexpr (BLOOM) bl[k] = bl[k] * s;
        }
    }
    if constexpr (BLOOM) {
        const float noise = linear_fetch_rgb_r_repeat(dither, dw, dh, uvx * dsx, uvy * dsy) * 2.0f - 1.0f;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            float bk = bl[k] + noise / 255.0f;
            bk = fmaxf(bk, 0.0f);
            bk = fmaxf(1.055f * powf(bk, 0.416666667f) - 0.055f, 0.0f);     // linearToGamma S:565-568
            cc[k] = cc[k] + bk;
        }
    }
    const float a = fmaxf(cc[0], fmaxf(cc[1], cc[2]));
    out[(size_t)Out::row(j, h) * w + i] =
        Out::pack(blend_over_background(cc[0], cc[1], cc[2], a, bg_mode, br_, bg_, bb_, aspect, uvx, uvy));
}

}  // namespace fk
