/*
 * fluid_oracle.c — CPU restatement (plain C + OpenMP) of script.js's simulation passes.
 * TEST INFRASTRUCTURE ONLY — see fluid_oracle.h.  Build: make -C oracle  (-ffp-contract=off).
 *
 * Every function is a literal restatement of one GLSL fragment shader of the reference, written
 * from the shader text, with the operation order of the GLSL expression kept (fp32 is not
 * associative and the GPU parity tests are bitwise for every pass but splat).
 * Geometry (baseVertexShader S:440-459): a fragment at cell (i,j) has vUv = ((i+.5)/W,(j+.5)/H)
 * and vL/vR/vT/vB one texel away; with CLAMP_TO_EDGE (S:1051-1052) an off-grid neighbour of an
 * edge cell is the edge cell itself.
 */
#include "fluid_oracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>
#ifdef _OPENMP
#include <omp.h>
#endif

static inline int clampi(int a, int lo, int hi) { return a < lo ? lo : (a > hi ? hi : a); }

/* torchrun exports OMP_NUM_THREADS=1 to its workers; the CPU-baseline legs of bench.py widen the
 * team again to the cores the process may actually use. */
void oracle_set_num_threads(int n) {
#ifdef _OPENMP
    if (n > 0) omp_set_num_threads(n);
#else
    (void)n;
#endif
}

int oracle_num_threads(void) {
#ifdef _OPENMP
    return omp_get_max_threads();
#else
    return 1;
#endif
}

/* S:814-833.  L,R = velocity.y left/right; T,B = velocity.x top/bottom;
 * vorticity = R - L - T + B; out = 0.5 * vorticity. */
void oracle_curl(const float* v, float* curl, int W, int H) {
#pragma omp parallel for schedule(static)
    for (int j = 0; j < H; ++j) {
        const int jb = clampi(j - 1, 0, H - 1), jt = clampi(j + 1, 0, H - 1);
        for (int i = 0; i < W; ++i) {
            const int il = clampi(i - 1, 0, W - 1), ir = clampi(i + 1, 0, W - 1);
            const float L = v[2 * ((size_t)j * W + il) + 1];
            const float R = v[2 * ((size_t)j * W + ir) + 1];
            const float T = v[2 * ((size_t)jt * W + i) + 0];
            const float B = v[2 * ((size_t)jb * W + i) + 0];
            const float vort = ((R - L) - T) + B;
            curl[(size_t)j * W + i] = 0.5f * vort;
        }
    }
}

/* S:835-866.  force = 0.5*vec2(|T|-|B|, |R|-|L|); force /= length(force)+0.0001;
 * force *= curl*C; force.y *= -1; velocity += force*dt; clamp to [-1000,1000]. */
void oracle_vorticity(const float* v, const float* curl, float* vout, int W, int H, float curl_k,
                      float dt) {
#pragma omp parallel for schedule(static)
    for (int j = 0; j < H; ++j) {
        const int jb = clampi(j - 1, 0, H - 1), jt = clampi(j + 1, 0, H - 1);
        for (int i = 0; i < W; ++i) {
            const int il = clampi(i - 1, 0, W - 1), ir = clampi(i + 1, 0, W - 1);
            const float L = curl[(size_t)j * W + il];
            const float R = curl[(size_t)j * W + ir];
            const float T = curl[(size_t)jt * W + i];
            const float B = curl[(size_t)jb * W + i];
            const float C = curl[(size_t)j * W + i];
            float fx = 0.5f * (fabsf(T) - fabsf(B));
            float fy = 0.5f * (fabsf(R) - fabsf(L));
            const float len = sqrtf(fx * fx + fy * fy);
            const float den = len + 0.0001f;
            fx = fx / den;
            fy = fy / den;
            const float s = curl_k * C;
            fx = fx * s;
            fy = fy * s;
            fy = fy * -1.0f;
            float vx = v[2 * ((size_t)j * W + i) + 0];
            float vy = v[2 * ((size_t)j * W + i) + 1];
            vx = vx + fx * dt;
            vy = vy + fy * dt;
            vx = fminf(fmaxf(vx, -1000.0f), 1000.0f);
            vy = fminf(fmaxf(vy, -1000.0f), 1000.0f);
            vout[2 * ((size_t)j * W + i) + 0] = vx;
            vout[2 * ((size_t)j * W + i) + 1] = vy;
        }
    }
}

/* S:786-812.  Reflecting walls: the tests vL.x<0, vR.x>1, vT.y>1, vB.y<0 (S:804-807) hold
 * exactly for i==0, i==W-1, j==H-1, j==0.  div = 0.5*(R - L + T - B). */
void oracle_divergence(const float* v, float* div, int W, int H) {
#pragma omp parallel for schedule(static)
    for (int j = 0; j < H; ++j) {
        const int jb = clampi(j - 1, 0, H - 1), jt = clampi(j + 1, 0, H - 1);
        for (int i = 0; i < W; ++i) {
            const int il = clampi(i - 1, 0, W - 1), ir = clampi(i + 1, 0, W - 1);
            float L = v[2 * ((size_t)j * W + il) + 0];
            float R = v[2 * ((size_t)j * W + ir) + 0];
            float T = v[2 * ((size_t)jt * W + i) + 1];
            float B = v[2 * ((size_t)jb * W + i) + 1];
            const float Cx = v[2 * ((size_t)j * W + i) + 0];
            const float Cy = v[2 * ((size_t)j * W + i) + 1];
            if (i == 0) L = -Cx;
            if (i == W - 1) R = -Cx;
            if (j == H - 1) T = -Cy;
            if (j == 0) B = -Cy;
            div[(size_t)j * W + i] = 0.5f * (((R - L) + T) - B);
        }
    }
}

/* S:508-519: gl_FragColor = value * texture2D(uTexture, vUv). */
void oracle_clear(const float* in, float* out, size_t n, float value) {
#pragma omp parallel for schedule(static)
    for (long long k = 0; k < (long long)n; ++k) out[k] = value * in[k];
}

/* S:868-890: pressure = (L + R + B + T - divergence) * 0.25   (C is fetched but unused). */
void oracle_jacobi(const float* p, const float* div, float* pout, int W, int H) {
#pragma omp parallel for schedule(static)
    for (int j = 0; j < H; ++j) {
        const float* pc = p + (size_t)j * W;
        const float* pb = p + (size_t)clampi(j - 1, 0, H - 1) * W;
        const float* pt = p + (size_t)clampi(j + 1, 0, H - 1) * W;
        const float* dv = div + (size_t)j * W;
        float* o = pout + (size_t)j * W;
        for (int i = 0; i < W; ++i) {
            const float L = pc[i > 0 ? i - 1 : 0];
            const float R = pc[i < W - 1 ? i + 1 : W - 1];
            o[i] = ((((L + R) + pb[i]) + pt[i]) - dv[i]) * 0.25f;
        }
    }
}

/* Row-parallel copy with the SAME static row schedule as the passes: timing legs use it to
 * first-touch their buffers on the threads (NUMA nodes) that will later sweep those rows. */
void oracle_copy_rows(float* dst, const float* src, int W, int H) {
#pragma omp parallel for schedule(static)
    for (int j = 0; j < H; ++j) memcpy(dst + (size_t)j * W, src + (size_t)j * W, (size_t)W * sizeof(float));
}

void oracle_jacobi_iters(float* p, float* tmp, const float* div, int W, int H, int iters) {
    float *a = p, *b = tmp;
    for (int k = 0; k < iters; ++k) {
        oracle_jacobi(a, div, b, W, H);
        float* t = a; a = b; b = t; /* pressure.swap() S:1265 */
    }
    if (a != p) memcpy(p, a, (size_t)W * H * sizeof(float));
}

/* S:892-913: velocity.xy -= vec2(R - L, T - B)  (no 1/2 factor, unlike divergence). */
void oracle_gradient_subtract(const float* p, const float* v, float* vout, int W, int H) {
#pragma omp parallel for schedule(static)
    for (int j = 0; j < H; ++j) {
        const int jb = clampi(j - 1, 0, H - 1), jt = clampi(j + 1, 0, H - 1);
        for (int i = 0; i < W; ++i) {
            const int il = clampi(i - 1, 0, W - 1), ir = clampi(i + 1, 0, W - 1);
            const float L = p[(size_t)j * W + il], R = p[(size_t)j * W + ir];
            const float T = p[(size_t)jt * W + i], B = p[(size_t)jb * W + i];
            vout[2 * ((size_t)j * W + i) + 0] = v[2 * ((size_t)j * W + i) + 0] - (R - L);
            vout[2 * ((size_t)j * W + i) + 1] = v[2 * ((size_t)j * W + i) + 1] - (T - B);
        }
    }
}

/* bilerp of S:758-770:  st = uv/tsize - 0.5; iuv = floor(st); fuv = fract(st);
 * a,b,c,d = texels (iuv + {.5,1.5}) * tsize fetched NEAREST + CLAMP_TO_EDGE;
 * mix(mix(a,b,fuv.x), mix(c,d,fuv.x), fuv.y) with GLSL mix(x,y,t) = x*(1-t) + y*t. */
static inline int texel_index(float f, int n) {
    /* NEAREST lookup of coordinate (f + .5)*tsize with CLAMP_TO_EDGE == clamp(f, 0, n-1) */
    if (!(f > 0.0f)) return 0;
    if (f >= (float)(n - 1)) return n - 1;
    return (int)f;
}
static inline float mixf(float x, float y, float t) { return x * (1.0f - t) + y * t; }

static inline void bilerp(const float* tex, int W, int H, int C, float uvx, float uvy, float tsx,
                          float tsy, float* out) {
    const float stx = uvx / tsx - 0.5f, sty = uvy / tsy - 0.5f;
    const float ix = floorf(stx), iy = floorf(sty);
    const float fx = stx - ix, fy = sty - iy;
    const int i0 = texel_index(ix, W), i1 = texel_index(ix + 1.0f, W);
    const int j0 = texel_index(iy, H), j1 = texel_index(iy + 1.0f, H);
    const float* a = tex + ((size_t)j0 * W + i0) * C;
    const float* b = tex + ((size_t)j0 * W + i1) * C;
    const float* c = tex + ((size_t)j1 * W + i0) * C;
    const float* d = tex + ((size_t)j1 * W + i1) * C;
    for (int k = 0; k < C; ++k) out[k] = mixf(mixf(a[k], b[k], fx), mixf(c[k], d[k], fx), fy);
}

/* S:772-783 (MANUAL_FILTERING branch):
 *   coord  = vUv - dt * bilerp(uVelocity, vUv, texelSize).xy * texelSize;
 *   result = bilerp(uSource, coord, dyeTexelSize);
 *   gl_FragColor = result / (1.0 + dissipation * dt);
 * texelSize is the SIM texel for both passes (S:1276 is never re-set before S:1292). */
void oracle_advect(const float* vel, int W, int H, const float* src, float* out, int Ws, int Hs,
                   int C, float dt, float dissipation) {
    const float tsx = (float)(1.0 / (double)W), tsy = (float)(1.0 / (double)H);      /* S:1061-1062 */
    const float dsx = (float)(1.0 / (double)Ws), dsy = (float)(1.0 / (double)Hs);
    const float decay = 1.0f + dissipation * dt;
#pragma omp parallel for schedule(static)
    for (int J = 0; J < Hs; ++J) {
        const float uvy = ((float)J + 0.5f) / (float)Hs;
        for (int I = 0; I < Ws; ++I) {
            const float uvx = ((float)I + 0.5f) / (float)Ws;
            float vv[2];
            bilerp(vel, W, H, 2, uvx, uvy, tsx, tsy, vv);
            const float cx = uvx - (dt * vv[0]) * tsx;
            const float cy = uvy - (dt * vv[1]) * tsy;
            float r[4];
            bilerp(src, Ws, Hs, C, cx, cy, dsx, dsy, r);
            float* o = out + ((size_t)J * Ws + I) * C;
            for (int k = 0; k < C; ++k) o[k] = r[k] / decay;
        }
    }
}

/* S:726-744: p = vUv - point; p.x *= aspectRatio; splat = exp(-dot(p,p)/radius)*color;
 * gl_FragColor = vec4(base.xyz + splat, 1.0).  An RG target keeps .xy only. */
void oracle_splat(const float* base, float* out, int W, int H, int C, float aspect, float px,
                  float py, const float* color3, float radius) {
#pragma omp parallel for schedule(static)
    for (int j = 0; j < H; ++j) {
        const float uvy = ((float)j + 0.5f) / (float)H;
        for (int i = 0; i < W; ++i) {
            const float uvx = ((float)i + 0.5f) / (float)W;
            float dx = uvx - px;
            const float dy = uvy - py;
            dx = dx * aspect;
            const float d = dx * dx + dy * dy;
            const float e = expf(-d / radius);
            const float* b = base + ((size_t)j * W + i) * C;
            float* o = out + ((size_t)j * W + i) * C;
            const int n3 = C < 3 ? C : 3;
            for (int k = 0; k < n3; ++k) o[k] = b[k] + e * color3[k];
            if (C == 4) o[3] = 1.0f;
        }
    }
}

/* GL_LINEAR + CLAMP_TO_EDGE fetch as the GL ES 2.0 spec (3.7.7) writes it: u' = u*W - 0.5,
 * i0 = floor(u'), alpha = frac(u'); tau = (1-a)(1-b) t00 + a(1-b) t10 + (1-a) b t01 + a b t11. */
static inline void linear_fetch(const float* tex, int W, int H, int C, float uvx, float uvy, float* out) {
    const float u = uvx * (float)W - 0.5f, v = uvy * (float)H - 0.5f;
    const float fi = floorf(u), fj = floorf(v);
    const float a = u - fi, b = v - fj;
    const int i0 = texel_index(fi, W), i1 = texel_index(fi + 1.0f, W);
    const int j0 = texel_index(fj, H), j1 = texel_index(fj + 1.0f, H);
    const float w00 = (1.0f - a) * (1.0f - b), w10 = a * (1.0f - b), w01 = (1.0f - a) * b, w11 = a * b;
    const float* t00 = tex + ((size_t)j0 * W + i0) * C; const float* t10 = tex + ((size_t)j0 * W + i1) * C;
    const float* t01 = tex + ((size_t)j1 * W + i0) * C; const float* t11 = tex + ((size_t)j1 * W + i1) * C;
    for (int k = 0; k < C; ++k) out[k] = ((w00 * t00[k] + w10 * t10[k]) + w01 * t01[k]) + w11 * t11[k];
}

/* copyShader S:496-506 drawn into the new FBO while sampling the old texture through its
 * LINEAR filter (resizeFBO S:1108-1114): a sampler fetch, so the GL-spec weight form of
 * linear_fetch above (the same one the display pass uses), pinned by the executed copyShader
 * golden tests/golden/resample_*.npz. */
void oracle_resample(const float* src, int Ws, int Hs, float* dst, int Wd, int Hd, int C) {
#pragma omp parallel for schedule(static)
    for (int J = 0; J < Hd; ++J) {
        const float uvy = ((float)J + 0.5f) / (float)Hd;
        for (int I = 0; I < Wd; ++I) {
            const float uvx = ((float)I + 0.5f) / (float)Wd;
            linear_fetch(src, Ws, Hs, C, uvx, uvy, dst + ((size_t)J * Wd + I) * C);
        }
    }
}

/* render(target) with BLOOM and SUNRAYS off, TRANSPARENT off (S:1296-1317): drawColor(BACK_COLOR)
 * (S:1319-1323, colorShader S:521-529) then drawDisplay (S:1331-1348, displayShaderSource
 * S:549-612 with the SHADING keyword when `shading`), blended ONE / ONE_MINUS_SRC_ALPHA (S:1305).
 * dye is sampled through its LINEAR filter at the target's resolution w x h; out is w*h RGBA. */
/* What drawDisplay is blended over (render(), S:1296-1317): bg_mode 0 = drawColor(BACK_COLOR)
 * (S:1319-1323); 1 = drawCheckerboard (TRANSPARENT on the screen, S:1325-1329 + checkerboardShader
 * S:531-547: v = mod(floor(uv.x*25*aspect) + floor(uv.y*25), 2) * 0.1 + 0.8); 2 = nothing and
 * blending disabled (TRANSPARENT into a capture target): the display colour goes out as it is. */
static inline void background(int bg_mode, const float* back_rgb, float aspect, float uvx, float uvy, float* bg) {
    if (bg_mode == 1) {
        const float x = floorf((uvx * 25.0f) * aspect), y = floorf((uvy * 25.0f) * 1.0f);
        const float sxy = x + y;
        float v = sxy - 2.0f * floorf(sxy / 2.0f);                       /* GLSL mod */
        v = v * 0.1f + 0.8f;
        bg[0] = bg[1] = bg[2] = v;
    } else {
        bg[0] = back_rgb[0]; bg[1] = back_rgb[1]; bg[2] = back_rgb[2];
    }
}

void oracle_display(const float* dye, int Wd, int Hd, float* out, int w, int h, int shading,
                    const float* back_rgb, int bg_mode, float aspect) {
    const float tsx = (float)(1.0 / (double)w), tsy = (float)(1.0 / (double)h);   /* S:1337 */
#pragma omp parallel for schedule(static)
    for (int j = 0; j < h; ++j) {
        const float uvy = ((float)j + 0.5f) / (float)h;
        for (int i = 0; i < w; ++i) {
            const float uvx = ((float)i + 0.5f) / (float)w;
            float c[4];
            linear_fetch(dye, Wd, Hd, 4, uvx, uvy, c);
            if (shading) {
                float lc[4], rc[4], tc[4], bc[4];
                linear_fetch(dye, Wd, Hd, 4, uvx - tsx, uvy, lc);
                linear_fetch(dye, Wd, Hd, 4, uvx + tsx, uvy, rc);
                linear_fetch(dye, Wd, Hd, 4, uvx, uvy + tsy, tc);
                linear_fetch(dye, Wd, Hd, 4, uvx, uvy - tsy, bc);
#define LEN3(v) sqrtf(((v)[0] * (v)[0] + (v)[1] * (v)[1]) + (v)[2] * (v)[2])
                const float dx = LEN3(rc) - LEN3(lc);
                const float dy = LEN3(tc) - LEN3(bc);
                const float nz = sqrtf(tsx * tsx + tsy * tsy);               /* length(texelSize) */
                const float nl = sqrtf((dx * dx + dy * dy) + nz * nz);       /* normalize = v / length(v) */
                const float n2 = nz / nl;
                /* dot(n, vec3(0,0,1)) = n.x*0 + n.y*0 + n.z*1 */
                const float d = ((dx / nl) * 0.0f + (dy / nl) * 0.0f) + n2 * 1.0f;
                const float diffuse = fminf(fmaxf(d + 0.7f, 0.7f), 1.0f);
                c[0] = c[0] * diffuse; c[1] = c[1] * diffuse; c[2] = c[2] * diffuse;
            }
            const float a = fmaxf(c[0], fmaxf(c[1], c[2]));
            float* o = out + ((size_t)j * w + i) * 4;
            if (bg_mode == 2) { o[0] = c[0]; o[1] = c[1]; o[2] = c[2]; o[3] = a; continue; }
            float bg[3];
            background(bg_mode, back_rgb, aspect, uvx, uvy, bg);
            const float k = 1.0f - a;                                        /* ONE_MINUS_SRC_ALPHA */
            o[0] = c[0] + bg[0] * k;
            o[1] = c[1] + bg[1] * k;
            o[2] = c[2] + bg[2] * k;
            o[3] = a + 1.0f * k;
        }
    }
}

/* ---- post-FX (bloom, sunrays) and the full display: SURVEY section 8f rank 1, second half --------------------
 * ORACLE SIDE ONLY so far: the CUDA kernels for these passes are not built yet (DESIGN.md section 9). */

/* LINEAR fetch with CLAMP_TO_EDGE or REPEAT wrap, C channels */
static inline void linear_fetch_w(const float* tex, int W, int H, int C, float uvx, float uvy, int repeat, float* out) {
    if (!repeat) { linear_fetch(tex, W, H, C, uvx, uvy, out); return; }
    const float u = uvx * (float)W - 0.5f, v = uvy * (float)H - 0.5f;
    const float fi = floorf(u), fj = floorf(v);
    const float a = u - fi, b = v - fj;
    long long i0 = (long long)fi % W, j0 = (long long)fj % H;
    if (i0 < 0) i0 += W;
    if (j0 < 0) j0 += H;
    const long long i1 = (i0 + 1) % W, j1 = (j0 + 1) % H;
    const float w00 = (1.0f - a) * (1.0f - b), w10 = a * (1.0f - b), w01 = (1.0f - a) * b, w11 = a * b;
    const float* t00 = tex + ((size_t)j0 * W + i0) * C; const float* t10 = tex + ((size_t)j0 * W + i1) * C;
    const float* t01 = tex + ((size_t)j1 * W + i0) * C; const float* t11 = tex + ((size_t)j1 * W + i1) * C;
    for (int k = 0; k < C; ++k) out[k] = ((w00 * t00[k] + w10 * t10[k]) + w01 * t01[k]) + w11 * t11[k];
}

/* bloomPrefilterShader S:614-631, drawn into the bloom FBO (w x h) sampling dye.read */
void oracle_bloom_prefilter(const float* dye, int Wd, int Hd, float* out, int w, int h, float curve0,
                            float curve1, float curve2, float threshold) {
#pragma omp parallel for schedule(static)
    for (int j = 0; j < h; ++j) {
        const float uvy = ((float)j + 0.5f) / (float)h;
        for (int i = 0; i < w; ++i) {
            const float uvx = ((float)i + 0.5f) / (float)w;
            float c[4];
            linear_fetch(dye, Wd, Hd, 4, uvx, uvy, c);
            const float br = fmaxf(c[0], fmaxf(c[1], c[2]));
            float rq = fminf(fmaxf(br - curve0, 0.0f), curve1);
            rq = (curve2 * rq) * rq;
            const float f = fmaxf(rq, br - threshold) / fmaxf(br, 0.0001f);
            float* o = out + ((size_t)j * w + i) * 4;
            o[0] = c[0] * f; o[1] = c[1] * f; o[2] = c[2] * f; o[3] = 0.0f;
        }
    }
}

/* bloomBlurShader S:633-651 / bloomFinalShader S:653-674: average of the 4 LINEAR taps one SOURCE
 * texel left/right/up/down; `add`: blendFunc(ONE, ONE) onto dst (S:1374-1375); scale = intensity. */
void oracle_box4(const float* src, int ws, int hs, float* dst, int w, int h, float scale, int add) {
    const float tsx = (float)(1.0 / (double)ws), tsy = (float)(1.0 / (double)hs);
#pragma omp parallel for schedule(static)
    for (int j = 0; j < h; ++j) {
        const float uvy = ((float)j + 0.5f) / (float)h;
        for (int i = 0; i < w; ++i) {
            const float uvx = ((float)i + 0.5f) / (float)w;
            float L[4], R[4], T[4], B[4];
            linear_fetch(src, ws, hs, 4, uvx - tsx, uvy, L);
            linear_fetch(src, ws, hs, 4, uvx + tsx, uvy, R);
            linear_fetch(src, ws, hs, 4, uvx, uvy + tsy, T);
            linear_fetch(src, ws, hs, 4, uvx, uvy - tsy, B);
            float* o = dst + ((size_t)j * w + i) * 4;
            for (int k = 0; k < 4; ++k) {
                float sum = (((0.0f + L[k]) + R[k]) + T[k]) + B[k];
                sum = sum * 0.25f;
                sum = sum * scale;
                o[k] = add ? sum + o[k] : sum;
            }
        }
    }
}

/* sunraysMaskShader S:676-691 into a dye-sized RGBA target */
void oracle_sunrays_mask(const float* dye, float* mask, int Wd, int Hd) {
#pragma omp parallel for schedule(static)
    for (int j = 0; j < Hd; ++j) {
        const float uvy = ((float)j + 0.5f) / (float)Hd;
        for (int i = 0; i < Wd; ++i) {
            const float uvx = ((float)i + 0.5f) / (float)Wd;
            float c[4];
            linear_fetch(dye, Wd, Hd, 4, uvx, uvy, c);
            const float br = fmaxf(c[0], fmaxf(c[1], c[2]));
            float* o = mask + ((size_t)j * Wd + i) * 4;
            o[0] = c[0]; o[1] = c[1]; o[2] = c[2];
            o[3] = 1.0f - fminf(fmaxf(br * 20.0f, 0.0f), 0.8f);
        }
    }
}

/* sunraysShader S:693-724: 16-step march towards the centre over the mask's alpha */
void oracle_sunrays(const float* mask, int Wm, int Hm, float* out, int w, int h, float weight) {
    const float Density = 0.3f, Decay = 0.95f, Exposure = 0.7f;
    const float f = (float)(1.0 / 16.0) * Density;                 /* 1.0 / float(ITERATIONS) * Density */
#pragma omp parallel for schedule(static)
    for (int j = 0; j < h; ++j) {
        const float uvy = ((float)j + 0.5f) / (float)h;
        for (int i = 0; i < w; ++i) {
            const float uvx = ((float)i + 0.5f) / (float)w;
            float cx = uvx, cy = uvy;
            float dx = uvx - 0.5f, dy = uvy - 0.5f;
            dx = dx * f; dy = dy * f;
            float illum = 1.0f, t[4];
            linear_fetch(mask, Wm, Hm, 4, uvx, uvy, t);
            float color = t[3];
            for (int k = 0; k < 16; ++k) {
                cx = cx - dx; cy = cy - dy;
                linear_fetch(mask, Wm, Hm, 4, cx, cy, t);
                color = color + (t[3] * illum) * weight;
                illum = illum * Decay;
            }
            out[(size_t)j * w + i] = color * Exposure;
        }
    }
}

/* blurShader S:478-494 with blurVertexShader S:461-476 on a one-channel texture (sunrays) */
void oracle_blur3(const float* src, float* dst, int w, int h, float tsx, float tsy) {
    const float off = 1.33333333f;
#pragma omp parallel for schedule(static)
    for (int j = 0; j < h; ++j) {
        const float uvy = ((float)j + 0.5f) / (float)h;
        for (int i = 0; i < w; ++i) {
            const float uvx = ((float)i + 0.5f) / (float)w;
            float c, l, r;
            linear_fetch(src, w, h, 1, uvx, uvy, &c);
            linear_fetch(src, w, h, 1, uvx - tsx * off, uvy - tsy * off, &l);
            linear_fetch(src, w, h, 1, uvx + tsx * off, uvy + tsy * off, &r);
            float sum = c * 0.29411764f;
            sum = sum + l * 0.35294117f;
            sum = sum + r * 0.35294117f;
            dst[(size_t)j * w + i] = sum;
        }
    }
}

/* displayShaderSource S:549-612 with SHADING + BLOOM + SUNRAYS, over drawColor, premultiplied blend */
void oracle_display_full(const float* dye, int Wd, int Hd, const float* bloom, int bw, int bh,
                         const float* sun, int sw, int sh, const float* dither, int dw, int dh,
                         float* out, int w, int h, const float* back_rgb, int bg_mode, float aspect) {
    const float tsx = (float)(1.0 / (double)w), tsy = (float)(1.0 / (double)h);
    const float dsx = (float)((double)w / (double)dw), dsy = (float)((double)h / (double)dh);   /* S:1626-1631 */
#pragma omp parallel for schedule(static)
    for (int j = 0; j < h; ++j) {
        const float uvy = ((float)j + 0.5f) / (float)h;
        for (int i = 0; i < w; ++i) {
            const float uvx = ((float)i + 0.5f) / (float)w;
            float c[4], lc[4], rc[4], tc[4], bc[4], bl[4], s, dn[3];
            linear_fetch(dye, Wd, Hd, 4, uvx, uvy, c);
            linear_fetch(dye, Wd, Hd, 4, uvx - tsx, uvy, lc);
            linear_fetch(dye, Wd, Hd, 4, uvx + tsx, uvy, rc);
            linear_fetch(dye, Wd, Hd, 4, uvx, uvy + tsy, tc);
            linear_fetch(dye, Wd, Hd, 4, uvx, uvy - tsy, bc);
            const float dx = LEN3(rc) - LEN3(lc), dy = LEN3(tc) - LEN3(bc);
            const float nz = sqrtf(tsx * tsx + tsy * tsy);
            const float nl = sqrtf((dx * dx + dy * dy) + nz * nz);
            const float d = ((dx / nl) * 0.0f + (dy / nl) * 0.0f) + (nz / nl) * 1.0f;
            const float diffuse = fminf(fmaxf(d + 0.7f, 0.7f), 1.0f);
            linear_fetch(bloom, bw, bh, 4, uvx, uvy, bl);
            linear_fetch(sun, sw, sh, 1, uvx, uvy, &s);
            linear_fetch_w(dither, dw, dh, 3, uvx * dsx, uvy * dsy, 1, dn);
            float noise = dn[0] * 2.0f - 1.0f;
            float a = 0.0f;
            float cc[3];
            for (int k = 0; k < 3; ++k) {
                float ck = (c[k] * diffuse) * s;
                float bk = bl[k] * s;
                bk = bk + noise / 255.0f;
                bk = fmaxf(bk, 0.0f);
                bk = fmaxf(1.055f * powf(bk, 0.416666667f) - 0.055f, 0.0f);       /* linearToGamma S:565-568 */
                cc[k] = ck + bk;
            }
            a = fmaxf(cc[0], fmaxf(cc[1], cc[2]));
            float* o = out + ((size_t)j * w + i) * 4;
            if (bg_mode == 2) { o[0] = cc[0]; o[1] = cc[1]; o[2] = cc[2]; o[3] = a; continue; }
            float bg[3];
            background(bg_mode, back_rgb, aspect, uvx, uvy, bg);
            const float k1 = 1.0f - a;
            o[0] = cc[0] + bg[0] * k1; o[1] = cc[1] + bg[1] * k1; o[2] = cc[2] + bg[2] * k1;
            o[3] = a + 1.0f * k1;
        }
    }
}

void oracle_round_half(float* a, size_t n) {
#pragma omp parallel for schedule(static)
    for (long long k = 0; k < (long long)n; ++k) a[k] = (float)(_Float16)a[k];
}

/* ---------------------------------------------------------------------------------------------- */

oracle_sim* oracle_sim_create(int W, int H, int Wd, int Hd) {
    oracle_sim* s = (oracle_sim*)calloc(1, sizeof(*s));
    s->W = W; s->H = H; s->Wd = Wd; s->Hd = Hd;
    s->density_dissipation = 1.0f;      /* S:63 */
    s->velocity_dissipation = 0.2f;     /* S:64 */
    s->pressure = 0.8f;                 /* S:65 */
    s->pressure_iterations = 20;        /* S:66 */
    s->curl = 30.0f;                    /* S:67 */
    s->splat_radius = 0.25f;            /* S:68 */
    s->aspect = (float)W / (float)H;
    const size_t n = (size_t)W * H, nd = (size_t)Wd * Hd;
    s->v = (float*)calloc(2 * n, 4);   s->v2 = (float*)calloc(2 * n, 4);
    s->dye = (float*)calloc(4 * nd, 4); s->dye2 = (float*)calloc(4 * nd, 4);
    s->p = (float*)calloc(n, 4);       s->p2 = (float*)calloc(n, 4);
    s->div = (float*)calloc(n, 4);     s->curl_f = (float*)calloc(n, 4);
    /* createFBO clears to clearColor (0,0,0,1) (S:136, S:1059): dye alpha starts at 1 */
    for (size_t k = 0; k < nd; ++k) { s->dye[4 * k + 3] = 1.0f; s->dye2[4 * k + 3] = 1.0f; }
    return s;
}

void oracle_sim_destroy(oracle_sim* s) {
    if (!s) return;
    free(s->v); free(s->v2); free(s->dye); free(s->dye2);
    free(s->p); free(s->p2); free(s->div); free(s->curl_f);
    free(s);
}

#define SWAP(a, b) do { float* t_ = (a); (a) = (b); (b) = t_; } while (0)
#define ROUND(ptr, n) do { if (s->half_storage) oracle_round_half((ptr), (n)); } while (0)

/* step(dt), S:1231-1294, pass by pass in the reference's order. */
void oracle_sim_step(oracle_sim* s, float dt) {
    const int W = s->W, H = s->H;
    const size_t n = (size_t)W * H;
    oracle_curl(s->v, s->curl_f, W, H);                                   /* S:1234-1237 */
    ROUND(s->curl_f, n);
    oracle_vorticity(s->v, s->curl_f, s->v2, W, H, s->curl, dt);          /* S:1239-1246 */
    ROUND(s->v2, 2 * n); SWAP(s->v, s->v2);
    oracle_divergence(s->v, s->div, W, H);                                /* S:1248-1251 */
    ROUND(s->div, n);
    oracle_clear(s->p, s->p2, n, s->pressure);                            /* S:1253-1257 */
    ROUND(s->p2, n); SWAP(s->p, s->p2);
    for (int k = 0; k < s->pressure_iterations; ++k) {                    /* S:1259-1266 */
        oracle_jacobi(s->p, s->div, s->p2, W, H);
        ROUND(s->p2, n); SWAP(s->p, s->p2);
    }
    oracle_gradient_subtract(s->p, s->v, s->v2, W, H);                    /* S:1268-1273 */
    ROUND(s->v2, 2 * n); SWAP(s->v, s->v2);
    oracle_advect(s->v, W, H, s->v, s->v2, W, H, 2, dt, s->velocity_dissipation); /* S:1275-1285 */
    ROUND(s->v2, 2 * n); SWAP(s->v, s->v2);
    oracle_advect(s->v, W, H, s->dye, s->dye2, s->Wd, s->Hd, 4, dt,
                  s->density_dissipation);                                /* S:1287-1293 */
    ROUND(s->dye2, 4 * (size_t)s->Wd * s->Hd); SWAP(s->dye, s->dye2);
}

/* splat(x,y,dx,dy,color), S:1441-1455, radius = correctRadius(SPLAT_RADIUS/100), S:1457-1462 */
void oracle_sim_splat(oracle_sim* s, float x, float y, float dx, float dy, float r, float g,
                      float b) {
    /* JS evaluates correctRadius() in double and gl.uniform1f narrows it to fp32.  The aspect is
     * the double canvas ratio: widening the fp32 s->aspect can move the radius by an ulp (142x100). */
    double rad = (double)s->splat_radius / 100.0;
    const double aspect = (double)s->W / (double)s->H;
    if (aspect > 1.0) rad *= aspect;
    const float radius = (float)rad;
    const float cv[3] = {dx, dy, 0.0f};
    oracle_splat(s->v, s->v2, s->W, s->H, 2, s->aspect, x, y, cv, radius);
    ROUND(s->v2, 2 * (size_t)s->W * s->H); SWAP(s->v, s->v2);
    const float cd[3] = {r, g, b};
    oracle_splat(s->dye, s->dye2, s->Wd, s->Hd, 4, s->aspect, x, y, cd, radius);
    ROUND(s->dye2, 4 * (size_t)s->Wd * s->Hd); SWAP(s->dye, s->dye2);
}
