// looks.h — the look of one image of a batch draw: the post-FX sliders and the background that
// fluid_render_canvas_looks / fluid_capture_looks give each image (include/fluid.h fluid_look), as the
// values the batch post-FX and display kernels read (postfx.cuh).  Derived on the host exactly as the
// single-handle draws derive their per-call scalars.  Host code and a plain struct only, so the
// derivation compiles and can be checked without a GPU.
#pragma once
#include <cmath>

#include <cuda_fp16.h>

#include "../../include/fluid.h"

namespace fk {

// applyBloom's prefilter uniforms (S:1358-1363): knee = threshold * soft_knee + 0.0001 and the curve are JS
// doubles, each narrowed once to float by gl.uniform*f: curve0 = threshold - knee, curve1 = 2 knee,
// curve2 = 0.25 / knee, and the threshold itself.
inline void prefilter_curve(double threshold, double soft_knee, float curve[4]) {
    const double knee = threshold * soft_knee + 0.0001;
    curve[0] = (float)(threshold - knee);
    curve[1] = (float)(knee * 2);
    curve[2] = (float)(0.25 / knee);
    curve[3] = (float)threshold;
}

// unorm8 of postfx.cuh on the host: clamp01 (NaN gives 0, +inf 1), times 255 in fp32, rounded to the nearest
// integer with ties to even
inline unsigned char unorm8_host(float x) {
    return (unsigned char)std::nearbyint(std::fmin(std::fmax(x, 0.0f), 1.0f) * 255.0f);
}

// One image's entry of a batch handle's look table: the per-call scalars of the batch kernels, image by image.
// Both backgrounds are kept, so one table serves either output policy.
struct ImageLook {
    float curve[4];                 // bloom_prefilter_kernel: prefilter_curve of BLOOM_THRESHOLD, BLOOM_SOFT_KNEE
    float intensity;                // the final box4_kernel pass: BLOOM_INTENSITY
    float weight;                   // sunrays_kernel: SUNRAYS_WEIGHT
    float back16[3];                // StoreCapture: BACK_COLOR / 255 as drawColor stores it in the fp16 target
    unsigned char back8[3];         // StoreCanvas: u8(BACK_COLOR / 255), the bytes drawColor leaves on the canvas
    unsigned char transparent;      // 1: the capture stores the display bare, the canvas blends it over the checkerboard
};

// What the single-handle draw of fluid_render_canvas / fluid_capture derives from the same sliders and background
inline ImageLook image_look(const fluid_look& l) {
    ImageLook e{};
    prefilter_curve(l.bloom_threshold, l.bloom_soft_knee, e.curve);
    e.intensity = (float)l.bloom_intensity;
    e.weight = (float)l.sunrays_weight;
    const float back[3] = {l.back_r, l.back_g, l.back_b};
    for (int k = 0; k < 3; ++k) {
        e.back16[k] = __half2float(__float2half_rn(back[k]));
        e.back8[k] = unorm8_host(back[k]);
    }
    e.transparent = l.transparent != 0;
    return e;
}

}  // namespace fk
