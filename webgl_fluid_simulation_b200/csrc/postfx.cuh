// postfx.cuh — the display side of render() and captureScreenshot() (SURVEY §8f rank 1, second half):
// the post-FX chains of bloom (applyBloom S:1350-1394; shaders S:614-674) and sunrays (applySunrays +
// blur S:1396-1419; shaders S:461-494, S:676-724), and the display shader (S:549-612) for all eight
// keyword sets, drawn over the background into the fp32 frame of render(), the 8-bit image of
// captureScreenshot, or the RGBA8 canvas of render(null).
//
// Every kernel is one reference blit: one thread per target texel, sources fetched through the sampler
// policy Smp of passes.cuh: Linear (the GL_LINEAR formula, linear_fetch) or, with
// FLUID_FLAG_NEAREST_FILTERING, Nearest (nearest_fetch).  The dithering texture is LINEAR + REPEAT
// either way (createTextureAsync S:1131-1134).  Arithmetic order follows the GLSL; with the
// library's --fmad=false / IEEE div+sqrt build everything is bit-identical to the CPU oracle except
// the display's pow() (linearToGamma), which is tolerance-checked like splat's exp().
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include "half_passes.cuh"
#include "looks.h"
#include "passes.cuh"

namespace fk {

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

// The chain kernels are templates on storage policies (passes.cuh StoreF32, half_passes.cuh
// hs::StoreHalf): Sd is the dye's, which the sunrays mask shares because it is drawn into dye.write;
// St is the bloom FBO's, the pyramid's and the sunrays FBOs' (FLUID_FLAG_HALF_POSTFX: fp16, every
// blit's fp32 result rounded to nearest even when it is stored, like the reference's RGBA16F / R16F
// targets).  Fetches widen the stored texels exactly and run the same fp32 LINEAR arithmetic.  Smp is
// the sampler of every texture a chain reads (S:1017, S:1039: the filter of dye, bloom, pyramid and
// sunrays follows ext.supportLinearFiltering).
//
// BATCH: a batch handle's draw, blockIdx.z the image.  Every array a kernel reads or writes holds the members
// back to back, as a dense (B, h, w[, C]) array of its own size, so member m of a w x h array starts
// member_offset(w, h) texels in.  The pointers move before any tap, so the sampler's clamp keeps every tap
// inside the member.  Image z draws dye member members[z] when a member list is given (a subset draw), member z
// otherwise; the post-FX targets stay dense by image.  A draw with a look per image (fluid_render_canvas_looks)
// also gives the batch forms a table of looks (looks.h ImageLook): image z then reads looks[z] where the other
// draws read the call's scalars, which only the batch forms take.

// texels before member blockIdx.z of a dense (B, h, w) array, in 64 bits
__device__ __forceinline__ size_t member_offset(int w, int h) { return (size_t)blockIdx.z * w * h; }
// texels before the dye member image blockIdx.z draws: members[blockIdx.z], or blockIdx.z without a list
__device__ __forceinline__ size_t dye_member_offset(const int* members, int w, int h) {
    return (members ? (size_t)__ldg(members + blockIdx.z) : (size_t)blockIdx.z) * w * h;
}
// p as T texels, at member blockIdx.z of a w x h array when BATCH
template <bool BATCH, class T>
__device__ __forceinline__ const T* member_of(const void* p, int w, int h) {
    const T* q = static_cast<const T*>(p);
    if constexpr (BATCH) q += member_offset(w, h);
    return q;
}

// bloomPrefilterShader S:614-631, on rows [j_lo, j_hi) of the w x h bloom FBO.  The dye's first row is global
// row dye_row_off: a slab rank draws its band of the FBO from its own dye rows (+ ghost rows); one GPU draws
// every row from the whole dye.
template <class Sd, class St, class Smp, bool BATCH = false>
__global__ void __launch_bounds__(256) bloom_prefilter_kernel(const typename Sd::T4* __restrict__ dye, int Wd, int Hd,
                                                              int dye_row_off, typename St::T4* __restrict__ out, int w,
                                                              int h, int j_lo, int j_hi, float curve0, float curve1,
                                                              float curve2, float threshold,
                                                              const int* __restrict__ members = nullptr,
                                                              const ImageLook* __restrict__ looks = nullptr) {
    if constexpr (BATCH) {
        dye += dye_member_offset(members, Wd, Hd); out += member_offset(w, h);
        if (looks) {
            const float* c = looks[blockIdx.z].curve;
            curve0 = __ldg(c); curve1 = __ldg(c + 1); curve2 = __ldg(c + 2); threshold = __ldg(c + 3);
        }
    }
    const int i = blockIdx.x * blockDim.x + threadIdx.x, j = j_lo + blockIdx.y * blockDim.y + threadIdx.y;
    if (i >= w || j >= j_hi) return;
    const float uvx = ((float)i + 0.5f) / (float)w, uvy = ((float)j + 0.5f) / (float)h;
    const float4 c = Smp::template fetch<Sd>(dye, Wd, Hd, uvx, uvy, dye_row_off);
    const float br = fmaxf(c.x, fmaxf(c.y, c.z));
    float rq = fminf(fmaxf(br - curve0, 0.0f), curve1);
    rq = (curve2 * rq) * rq;
    const float f = fmaxf(rq, br - threshold) / fmaxf(br, 0.0001f);
    St::st(out, (size_t)j * w + i, make_float4(c.x * f, c.y * f, c.z * f, 0.0f));
}

// bloomBlurShader S:633-651 / bloomFinalShader S:653-674; add = blendFunc(ONE, ONE) (S:1374-1375): the
// fragment plus the widened destination texel, rounded once by the store.  BATCH: the final pass of a draw with
// a look per image takes image z's intensity as its scale.
template <class St, class Smp, bool BATCH = false>
__global__ void __launch_bounds__(256) box4_kernel(const typename St::T4* __restrict__ src, int ws, int hs,
                                                   typename St::T4* __restrict__ dst, int w, int h, float scale, int add,
                                                   const ImageLook* __restrict__ looks = nullptr) {
    if constexpr (BATCH) {
        src += member_offset(ws, hs); dst += member_offset(w, h);
        if (looks) scale = __ldg(&looks[blockIdx.z].intensity);
    }
    const int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y * blockDim.y + threadIdx.y;
    if (i >= w || j >= h) return;
    const float tsx = (float)(1.0 / (double)ws), tsy = (float)(1.0 / (double)hs);
    const float uvx = ((float)i + 0.5f) / (float)w, uvy = ((float)j + 0.5f) / (float)h;
    const float4 L = Smp::template fetch<St>(src, ws, hs, uvx - tsx, uvy), R = Smp::template fetch<St>(src, ws, hs, uvx + tsx, uvy);
    const float4 T = Smp::template fetch<St>(src, ws, hs, uvx, uvy + tsy), B = Smp::template fetch<St>(src, ws, hs, uvx, uvy - tsy);
    float4 s;
    s.x = ((((0.0f + L.x) + R.x) + T.x) + B.x) * 0.25f * scale;
    s.y = ((((0.0f + L.y) + R.y) + T.y) + B.y) * 0.25f * scale;
    s.z = ((((0.0f + L.z) + R.z) + T.z) + B.z) * 0.25f * scale;
    s.w = ((((0.0f + L.w) + R.w) + T.w) + B.w) * 0.25f * scale;
    const size_t o = (size_t)j * w + i;
    if (add) { const float4 d = St::ld(dst, o); s.x = s.x + d.x; s.y = s.y + d.y; s.z = s.z + d.z; s.w = s.w + d.w; }
    St::st(dst, o, s);
}

// sunraysMaskShader S:676-691 (target = dye.write, like the reference: S:1300, so stored as the dye is), on dye
// rows [j_lo, j_hi); dye and mask are buffers whose first row is global row row_off.  alpha, when not null, also
// receives the mask's alpha at global row j of a dense Wd x Hd array: the band a slab rank gathers (fp32 dye only).
// BATCH: the mask goes into the drawn member's own dye.write.
template <class Sd, class Smp, bool BATCH = false>
__global__ void __launch_bounds__(256) sunrays_mask_kernel(const typename Sd::T4* __restrict__ dye,
                                                           typename Sd::T4* __restrict__ mask, int Wd, int Hd,
                                                           int j_lo, int j_hi, int row_off, float* __restrict__ alpha,
                                                           const int* __restrict__ members = nullptr) {
    if constexpr (BATCH) {
        const size_t mo = dye_member_offset(members, Wd, Hd);
        dye += mo; mask += mo;
    }
    const int i = blockIdx.x * blockDim.x + threadIdx.x, j = j_lo + blockIdx.y * blockDim.y + threadIdx.y;
    if (i >= Wd || j >= j_hi) return;
    const float uvx = ((float)i + 0.5f) / (float)Wd, uvy = ((float)j + 0.5f) / (float)Hd;
    float4 c = Smp::template fetch<Sd>(dye, Wd, Hd, uvx, uvy, row_off);
    const float br = fmaxf(c.x, fmaxf(c.y, c.z));
    c.w = 1.0f - fminf(fmaxf(br * 20.0f, 0.0f), 0.8f);
    Sd::st(mask, (size_t)(j - row_off) * Wd + i, c);
    if (alpha) alpha[(size_t)j * Wd + i] = c.w;
}

// the mask value the sunrays shader reads: .a of the RGBA mask, or the one-channel gathered alpha.  LINEAR and
// NEAREST filter each channel on its own, so both give the same bits.
__device__ __forceinline__ float mask_alpha(float4 v) { return v.w; }
__device__ __forceinline__ float mask_alpha(float v) { return v; }

// sunraysShader S:693-724.  M: the mask's texel type, Sd::T4 (the mask in dye.write) or float (a slab's
// gathered alpha).  BATCH: the mask of the drawn member, in its dye.write, and image z's weight with looks.
template <class Sd, class St, class Smp, bool BATCH = false, class M = typename Sd::T4>
__global__ void __launch_bounds__(256) sunrays_kernel(const M* __restrict__ mask, int Wm, int Hm,
                                                      typename St::T1* __restrict__ out, int w, int h, float weight,
                                                      const int* __restrict__ members = nullptr,
                                                      const ImageLook* __restrict__ looks = nullptr) {
    if constexpr (BATCH) {
        mask += dye_member_offset(members, Wm, Hm); out += member_offset(w, h);
        if (looks) weight = __ldg(&looks[blockIdx.z].weight);
    }
    const int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y * blockDim.y + threadIdx.y;
    if (i >= w || j >= h) return;
    const float Density = 0.3f, Decay = 0.95f, Exposure = 0.7f;
    const float f = (float)(1.0 / 16.0) * Density;
    const float uvx = ((float)i + 0.5f) / (float)w, uvy = ((float)j + 0.5f) / (float)h;
    float cx = uvx, cy = uvy;
    float dx = uvx - 0.5f, dy = uvy - 0.5f;
    dx = dx * f; dy = dy * f;
    float illum = 1.0f;
    float color = mask_alpha(Smp::template fetch<Sd>(mask, Wm, Hm, uvx, uvy));
#pragma unroll 1
    for (int k = 0; k < 16; ++k) {
        cx = cx - dx; cy = cy - dy;
        const float col = mask_alpha(Smp::template fetch<Sd>(mask, Wm, Hm, cx, cy));
        color = color + (col * illum) * weight;
        illum = illum * Decay;
    }
    St::st(out, (size_t)j * w + i, color * Exposure);
}

// blurShader S:478-494 + blurVertexShader S:461-476 on the one-channel sunrays texture
template <class St, class Smp, bool BATCH = false>
__global__ void __launch_bounds__(256) blur3_kernel(const typename St::T1* __restrict__ src, typename St::T1* __restrict__ dst,
                                                    int w, int h, float tsx, float tsy) {
    if constexpr (BATCH) { src += member_offset(w, h); dst += member_offset(w, h); }
    const int i = blockIdx.x * blockDim.x + threadIdx.x, j = blockIdx.y * blockDim.y + threadIdx.y;
    if (i >= w || j >= h) return;
    const float off = 1.33333333f;
    const float uvx = ((float)i + 0.5f) / (float)w, uvy = ((float)j + 0.5f) / (float)h;
    const float c = Smp::template fetch<St>(src, w, h, uvx, uvy);
    const float l = Smp::template fetch<St>(src, w, h, uvx - tsx * off, uvy - tsy * off);
    const float r = Smp::template fetch<St>(src, w, h, uvx + tsx * off, uvy + tsy * off);
    float sum = c * 0.29411764f;
    sum = sum + l * 0.35294117f;
    sum = sum + r * 0.35294117f;
    St::st(dst, (size_t)j * w + i, sum);
}

__device__ __forceinline__ float len3(float4 v) { return sqrtf((v.x * v.x + v.y * v.y) + v.z * v.z); }

// checkerboardShader (S:531-547): v = mod(floor(uv.x * 25 * aspect) + floor(uv.y * 25), 2) * 0.1 + 0.8
__device__ __forceinline__ float checkerboard(float aspect, float uvx, float uvy) {
    const float x = floorf((uvx * 25.0f) * aspect), y = floorf((uvy * 25.0f) * 1.0f);
    const float sxy = x + y;
    const float v = sxy - 2.0f * floorf(sxy / 2.0f);
    return v * 0.1f + 0.8f;
}

// What drawDisplay is blended over (render(), S:1296-1317) with blendFunc(ONE, ONE_MINUS_SRC_ALPHA)
// (S:1305) on a float target: bg_mode 0 = drawColor(BACK_COLOR) (S:1319-1323); 1 = drawCheckerboard —
// TRANSPARENT on the screen (S:1325-1329); 2 = nothing, blending disabled — TRANSPARENT into a capture
// target (S:1307-1308): the display colour goes out as it is.
__device__ __forceinline__ float4 blend_over_background(float cr, float cg, float cb, float a, int bg_mode, float br,
                                                        float bg, float bb, float aspect, float uvx, float uvy) {
    if (bg_mode == 2) return make_float4(cr, cg, cb, a);
    if (bg_mode == 1) br = bg = bb = checkerboard(aspect, uvx, uvy);
    const float k = 1.0f - a;
    return make_float4(cr + br * k, cg + bg * k, cb + bb * k, a + 1.0f * k);
}

// normalizeTexture (S:309-327) of one channel of an RGBA half-float capture target (S:289): the value
// is first stored into the fp16 target (round to nearest even, overflow to +-Inf), then clamp01 * 255
// goes into a Uint8Array, which truncates.  An fp16 value times 255 is exact in fp32, so this is the
// JS double result.  fmaxf(NaN, 0) = 0 gives ToUint8(NaN) = 0.
__device__ __forceinline__ unsigned char capture_byte(float v) {
    const float s = __half2float(__float2half_rn(v));
    const float c = fminf(fmaxf(s, 0.0f), 1.0f);
    return (unsigned char)__float2uint_rz(c * 255.0f);
}

// The fixed-point colour buffer of the canvas (RGBA8 unsigned-normalised, S:118-119): clamp01 (NaN gives
// 0, +inf 1) and the float-to-unorm conversion, round to nearest with ties to even (GLES 3.0 §2.1.6.1).
__device__ __forceinline__ float clamp01(float x) { return fminf(fmaxf(x, 0.0f), 1.0f); }
__device__ __forceinline__ unsigned char unorm8(float x) { return (unsigned char)__float2uint_rn(__fmul_rn(clamp01(x), 255.0f)); }
// a stored byte read back as a blend destination: d8 / 255, correctly rounded
__device__ __forceinline__ float unorm8_value(unsigned char d8) { return __fdiv_rn((float)d8, 255.0f); }

// The inputs of display_kernel.  Those of a keyword that is off are never read.
struct DisplayArgs {
    const float4* dye;                  // fp32 dye; its first row is global row dye_row_off
    int Wd, Hd, dye_row_off;
    const void* bloom; int bw, bh;      // the bloom FBO (BLOOM): Sp::T4 texels
    const void* sun; int sw, sh;        // the sunrays texture (SUNRAYS): Sp::T1 texels
    const float* dither; int dw, dh;    // the RGB dithering texture (BLOOM)
    void* out;                          // Out::T texels of the rows [y0, y1) of the w x h target
    int w, h, y0, y1;
    float br, bg, bb;                   // background colour (bg_mode 0)
    int bg_mode;
    float aspect;
    float4 ts;                          // 1/w, 1/h and getTextureScale of the dithering texture (BLOOM)
    const int* members;                 // BATCH: the dye member of each image (a subset draw), or null: image z
    const ImageLook* looks;             // BATCH: each image's background (a draw with a look per image), or null
};

// Output policies of display_kernel: the element type of `out`, the row of `out` that row r of an
// n-row band goes to, and what is stored for the display fragment (c, alpha) at uv, blend included.  `look`:
// the image's entry of a batch draw with a look per image, whose background replaces the call's; null otherwise.
// StoreFrame: the fp32 RGBA frame of render(), row 0 = bottom.
struct StoreFrame {
    using T = float4;
    static __device__ __forceinline__ int row(int r, int) { return r; }
    static __device__ __forceinline__ float4 store(const float (&c)[3], float alpha, const DisplayArgs& a, float uvx, float uvy,
                                                   const ImageLook*) {
        return blend_over_background(c[0], c[1], c[2], alpha, a.bg_mode, a.br, a.bg, a.bb, a.aspect, uvx, uvy);
    }
};
// StoreCapture: captureScreenshot (S:287-327) up to the bytes toDataURL encodes: the blend of render(),
// the fp16 store, then normalizeTexture's 8-bit truncation and its flip (top row first).  A look's background is
// its fp16 BACK_COLOR, or none (bg_mode 2) when transparent.
struct StoreCapture {
    using T = uchar4;
    static __device__ __forceinline__ int row(int r, int n) { return n - 1 - r; }
    static __device__ __forceinline__ uchar4 store(const float (&c)[3], float alpha, const DisplayArgs& a, float uvx, float uvy,
                                                   const ImageLook* look) {
        float br = a.br, bg = a.bg, bb = a.bb;
        int bg_mode = a.bg_mode;
        if (look) {
            br = __ldg(&look->back16[0]); bg = __ldg(&look->back16[1]); bb = __ldg(&look->back16[2]);
            bg_mode = __ldg(&look->transparent) ? 2 : 0;
        }
        const float4 v = blend_over_background(c[0], c[1], c[2], alpha, bg_mode, br, bg, bb, a.aspect, uvx, uvy);
        return make_uchar4(capture_byte(v.x), capture_byte(v.y), capture_byte(v.z), capture_byte(v.w));
    }
};
// StoreCanvas: render(null) on the RGBA8 drawing buffer (S:1296-1317; the context has alpha: true,
// S:118-119), top row first like ImageData.  The destination holds bytes: u8(BACK_COLOR) (bg_mode 0) or
// u8(checkerboard) (bg_mode 1), alpha byte 255.  A fixed-point buffer clamps the source and the blend
// factors before blending (GLES 3.0 §4.1.7), so ONE, ONE_MINUS_SRC_ALPHA is clamp01(c) + d * (1 -
// clamp01(a)) on d = d8 / 255, rounded once more to a byte.  Every operation is rounded on its own.  A look's
// destination is its u8(BACK_COLOR), or the checkerboard when transparent.
struct StoreCanvas {
    using T = uchar4;
    static __device__ __forceinline__ int row(int r, int n) { return n - 1 - r; }
    static __device__ __forceinline__ uchar4 store(const float (&c)[3], float alpha, const DisplayArgs& a, float uvx, float uvy,
                                                   const ImageLook* look) {
        // the empty asm, which takes alpha, keeps the look's loads below the shading's IEEE div / sqrt slow paths:
        // hoisted above them, their values spill (the SHADING | SUNRAYS canvas)
        if (look) asm volatile("" : "+l"(look) : "f"(alpha));
        float d[3];
        if (look ? __ldg(&look->transparent) != 0 : a.bg_mode == 1) {
            d[0] = d[1] = d[2] = unorm8_value(unorm8(checkerboard(a.aspect, uvx, uvy)));
        } else if (look) {
            d[0] = unorm8_value(__ldg(&look->back8[0])); d[1] = unorm8_value(__ldg(&look->back8[1]));
            d[2] = unorm8_value(__ldg(&look->back8[2]));
        } else {
            d[0] = unorm8_value(unorm8(a.br)); d[1] = unorm8_value(unorm8(a.bg)); d[2] = unorm8_value(unorm8(a.bb));
        }
        const float ca = clamp01(alpha), k = __fsub_rn(1.0f, ca);
        // the destination alpha is u8(1) / 255 = 1 over either background
        return make_uchar4(unorm8(__fadd_rn(clamp01(c[0]), __fmul_rn(d[0], k))), unorm8(__fadd_rn(clamp01(c[1]), __fmul_rn(d[1], k))),
                           unorm8(__fadd_rn(clamp01(c[2]), __fmul_rn(d[2], k))), unorm8(__fadd_rn(ca, __fmul_rn(1.0f, k))));
    }
};

// displayShaderSource S:549-612 compiled with the keywords updateKeywords picks (S:1160-1166), over
// the background of render() (the output policy's store() blends).  Out: the output policy; Sp: the storage policy
// of the bloom and sunrays targets (post_fx_chains' St); Smp: the sampler of the dye, bloom and sunrays
// taps (the dithering tap is LINEAR + REPEAT whatever Smp is).  A slab rank draws the band [y0, y1) of the
// target from its own dye rows (+ ghost rows); one GPU draws the whole target.  BATCH: image blockIdx.z reads
// its member's dye (a.members) and its own bloom FBO and sunrays texture, and draws its own image over its own
// background when the draw has a look per image (a.looks); the dithering texture is shared.
template <bool SHADING, bool BLOOM, bool SUNRAYS, class Out, class Sp, class Smp, bool BATCH = false>
__global__ void __launch_bounds__(256) display_kernel(DisplayArgs a) {
    // the bloom FBO and the sunrays texture are offset where they are read: a member pointer kept across the
    // shading's IEEE div / sqrt slow paths spills the SHADING | SUNRAYS capture.  For the same reason a listed
    // member's dye is reached by a signed step taken before member z's offset (dye_member_offset, or the step
    // taken after it, spills that capture)
    if constexpr (BATCH) {
        if (a.members) a.dye += (ptrdiff_t)(__ldg(a.members + blockIdx.z) - (int)blockIdx.z) * a.Wd * a.Hd;
        a.dye += member_offset(a.Wd, a.Hd);
        a.out = static_cast<typename Out::T*>(a.out) + member_offset(a.w, a.y1 - a.y0);
    }
    const int i = blockIdx.x * blockDim.x + threadIdx.x, j = a.y0 + blockIdx.y * blockDim.y + threadIdx.y;
    if (i >= a.w || j >= a.y1) return;
    const float tsx = a.ts.x, tsy = a.ts.y;     // 1/width, 1/height (S:1337) and getTextureScale (S:1626-1631): JS doubles, narrowed on the host
    const float dsx = a.ts.z, dsy = a.ts.w;
    // the destination is formed up front: fewer values live across the IEEE div / sqrt slow paths
    // (the capture instantiation spills otherwise)
    typename Out::T* const o = static_cast<typename Out::T*>(a.out) + (size_t)Out::row(j - a.y0, a.y1 - a.y0) * a.w + i;
    const float uvx = ((float)i + 0.5f) / (float)a.w, uvy = ((float)j + 0.5f) / (float)a.h;
    const float4 c = Smp::fetch(a.dye, a.Wd, a.Hd, uvx, uvy, a.dye_row_off);
    float cc[3] = {c.x, c.y, c.z};
    if constexpr (SHADING) {
        const float4 lc = Smp::fetch(a.dye, a.Wd, a.Hd, uvx - tsx, uvy, a.dye_row_off);
        const float4 rc = Smp::fetch(a.dye, a.Wd, a.Hd, uvx + tsx, uvy, a.dye_row_off);
        const float4 tc = Smp::fetch(a.dye, a.Wd, a.Hd, uvx, uvy + tsy, a.dye_row_off);
        const float4 bc = Smp::fetch(a.dye, a.Wd, a.Hd, uvx, uvy - tsy, a.dye_row_off);
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
        const float4 b = Smp::template fetch<Sp>(member_of<BATCH, typename Sp::T4>(a.bloom, a.bw, a.bh), a.bw, a.bh, uvx, uvy);
        bl[0] = b.x; bl[1] = b.y; bl[2] = b.z;
    }
    if constexpr (SUNRAYS) {
        const float s = Smp::template fetch<Sp>(member_of<BATCH, typename Sp::T1>(a.sun, a.sw, a.sh), a.sw, a.sh, uvx, uvy);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            cc[k] = cc[k] * s;
            if constexpr (BLOOM) bl[k] = bl[k] * s;
        }
    }
    if constexpr (BLOOM) {
        const float noise = linear_fetch_rgb_r_repeat(a.dither, a.dw, a.dh, uvx * dsx, uvy * dsy) * 2.0f - 1.0f;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            float bk = bl[k] + noise / 255.0f;
            bk = fmaxf(bk, 0.0f);
            bk = fmaxf(1.055f * powf(bk, 0.416666667f) - 0.055f, 0.0f);     // linearToGamma S:565-568
            cc[k] = cc[k] + bk;
        }
    }
    const float alpha = fmaxf(cc[0], fmaxf(cc[1], cc[2]));
    const ImageLook* look = nullptr;
    if constexpr (BATCH) { if (a.looks) look = a.looks + blockIdx.z; }
    *o = Out::store(cc, alpha, a, uvx, uvy, look);
}

}  // namespace fk
