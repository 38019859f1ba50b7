/*
 * fluid_napi.c — thin N-API shim: exposes the C ABI of include/fluid.h to Node as `fluid.node`.
 * js/fluid-sim.js builds the reference's step()/splat()/config surface on top of it.
 *
 * COMPILE-CHECKED ONLY here (gcc -fsyntax-only in build()): this image has no Node, so the addon
 * cannot be linked against node or loaded.  With a Node toolchain:
 *   gcc -shared -fPIC -DFLUID_USE_SYSTEM_NODE_API -I<node>/include/node -I../../include \
 *       fluid_napi.c -L.. -lfluid_b200 -Wl,-rpath,'$ORIGIN/..' -o fluid.node
 *
 * Exports (all take the handle first):
 *   create(cfg) / createSlab(cfg, rank, world, uid) -> handle        destroy(h)
 *   step(h, dt)  splat(h, x, y, dx, dy, r, g, b)  setParam(h, key, value)  resize(h, sw, sh, dw, dh)
 *   splats(h, Float32Array of n * 7 floats: n splat() records (x, y, dx, dy, r, g, b), in order)
 *   read(h, field) -> Float32Array over PINNED host memory (one buffer per field, owned by the
 *       handle, overwritten by the next read of that field — like rebinding the same texture)
 *   write(h, field, Float32Array)  sync(h)  dims(h, field) -> {width, height, channels, row0}
 *   render(h, width, height, shading, r, g, b) -> Float32Array (RGBA, row 0 = bottom)
 *   renderKeywords(h, width, height, keywords, config, dither, dw, dh, r, g, b) -> Float32Array (any
 *       SHADING / BLOOM / SUNRAYS set, FLUID_DISPLAY_* bits)
 *   capture(h, width, height, canvasWidth, canvasHeight, keywords, transparent, config, dither, dw, dh,
 *       r, g, b) -> Uint8Array (captureScreenshot's RGBA8 image, top row first)
 *   renderCanvas(h, width, height, keywords, transparent, config, dither, dw, dh, r, g, b) -> Uint8ClampedArray
 *       (render(null) on the RGBA8 canvas, top row first: ready for new ImageData + putImageData)
 *   pressureSolveHost(h, div: Float32Array, p: Float32Array, iters)   stat(h, key)
 *   ncclUniqueId() -> ArrayBuffer(128)  p2pExport(h) -> ArrayBuffer(256)  p2pConnect(h, below, above)
 *   p2pDisable(h)  getResolution(res, cw, ch) -> {width, height}  lastError(h?) -> number-free string
 * Every non-zero status from the C ABI becomes a thrown JS Error carrying fluid_last_error().
 */
#ifdef FLUID_USE_SYSTEM_NODE_API
#include <node_api.h>
#else
#include "node_api_min.h"
#endif
#include <stdlib.h>
#include <string.h>

#include "../../include/fluid.h"

/* what the JS side holds: the library handle plus the pinned buffers read() / render() hand out */
typedef struct {
    fluid_t* h;
    float* pinned[6];      /* FLUID_FIELD_* 0..4, [5] = render target */
    size_t pinned_n[6];
} wrap_t;

#define ARGS(n)                                                   \
    size_t argc = (n); napi_value argv[(n) > 0 ? (n) : 1];        \
    if (napi_get_cb_info(env, info, &argc, argv, NULL, NULL) != napi_ok || argc < (n)) { \
        napi_throw_error(env, NULL, "wrong number of arguments"); return NULL; }

static napi_value undefined(napi_env env) { napi_value u; napi_get_undefined(env, &u); return u; }

/* NULL (with a JS exception pending) unless v is a live handle */
static wrap_t* wrap_of(napi_env env, napi_value v) {
    void* p = NULL;
    if (napi_get_value_external(env, v, &p) != napi_ok || !p || !((wrap_t*)p)->h) {
        napi_throw_error(env, NULL, "not a live fluid handle (destroyed?)");
        return NULL;
    }
    return (wrap_t*)p;
}

static int check(napi_env env, fluid_t* h, int rc) {
    if (rc == FLUID_OK) return 1;
    const char* m = fluid_last_error(h);
    napi_throw_error(env, NULL, (m && *m) ? m : "libfluid_b200 call failed");
    return 0;
}

static double num(napi_env env, napi_value v) { double d = 0; napi_get_value_double(env, v, &d); return d; }

static double prop(napi_env env, napi_value obj, const char* name, double dflt) {
    bool has = false; napi_value v;
    if (napi_has_named_property(env, obj, name, &has) != napi_ok || !has) return dflt;
    if (napi_get_named_property(env, obj, name, &v) != napi_ok) return dflt;
    return num(env, v);
}

static void release(wrap_t* w) {               /* idempotent: explicit destroy() and the GC finalizer share it */
    if (!w) return;
    if (w->h) { fluid_destroy(w->h); w->h = NULL; }
    for (int k = 0; k < 6; ++k) { fluid_host_free(w->pinned[k]); w->pinned[k] = NULL; w->pinned_n[k] = 0; }
}
static void finalize_handle(napi_env env, void* data, void* hint) { (void)env; (void)hint; release((wrap_t*)data); free(data); }
static void no_finalize(napi_env env, void* data, void* hint) { (void)env; (void)data; (void)hint; }

static float* pinned_for(wrap_t* w, int slot, size_t n) {
    if (w->pinned_n[slot] < n) {
        fluid_host_free(w->pinned[slot]);
        w->pinned[slot] = (float*)fluid_host_alloc(n * sizeof(float));
        w->pinned_n[slot] = w->pinned[slot] ? n : 0;
    }
    return w->pinned[slot];
}

static void config_from(napi_env env, napi_value o, fluid_config* c) {
    fluid_config_default(c);
    c->sim_w = (int)prop(env, o, "simWidth", c->sim_w);   c->sim_h = (int)prop(env, o, "simHeight", c->sim_h);
    c->dye_w = (int)prop(env, o, "dyeWidth", c->dye_w);   c->dye_h = (int)prop(env, o, "dyeHeight", c->dye_h);
    c->density_dissipation = (float)prop(env, o, "DENSITY_DISSIPATION", c->density_dissipation);
    c->velocity_dissipation = (float)prop(env, o, "VELOCITY_DISSIPATION", c->velocity_dissipation);
    c->pressure = (float)prop(env, o, "PRESSURE", c->pressure);
    c->pressure_iterations = (int)prop(env, o, "PRESSURE_ITERATIONS", c->pressure_iterations);
    c->curl = (float)prop(env, o, "CURL", c->curl);
    c->splat_radius = (float)prop(env, o, "SPLAT_RADIUS", c->splat_radius);
    c->aspect = (float)prop(env, o, "aspect", c->aspect);
    c->device = (int)prop(env, o, "device", -1);
    c->flags = (uint32_t)prop(env, o, "flags", 0);
    c->jacobi_block = (int)prop(env, o, "jacobiBlock", 0);
}

static napi_value wrap_new(napi_env env, fluid_t* h) {
    wrap_t* w = (wrap_t*)calloc(1, sizeof *w);
    if (!w) { fluid_destroy(h); napi_throw_error(env, NULL, "out of memory"); return NULL; }
    w->h = h;
    napi_value ext;
    if (napi_create_external(env, w, finalize_handle, NULL, &ext) != napi_ok) { release(w); free(w); return NULL; }
    return ext;
}

/* create({simWidth, simHeight, dyeWidth, dyeHeight, aspect, device, flags, jacobiBlock, ...config keys}) */
static napi_value Create(napi_env env, napi_callback_info info) {
    ARGS(1)
    fluid_config c; config_from(env, argv[0], &c);
    fluid_t* h = NULL;
    if (!check(env, NULL, fluid_create(&c, &h))) return NULL;
    return wrap_new(env, h);
}

/* createSlab(cfg, rank, world, uid: ArrayBuffer(128)) — one process per GPU, see INTEGRATION.md */
static napi_value CreateSlab(napi_env env, napi_callback_info info) {
    ARGS(4)
    fluid_config c; config_from(env, argv[0], &c);
    int32_t rank = 0, world = 1; napi_get_value_int32(env, argv[1], &rank); napi_get_value_int32(env, argv[2], &world);
    void* uid = NULL; size_t n = 0;
    if (napi_get_arraybuffer_info(env, argv[3], &uid, &n) != napi_ok) { napi_throw_error(env, NULL, "uid must be an ArrayBuffer"); return NULL; }
    fluid_t* h = NULL;
    if (!check(env, NULL, fluid_create_slab(&c, rank, world, uid, n, &h))) return NULL;
    return wrap_new(env, h);
}

static napi_value Destroy(napi_env env, napi_callback_info info) {
    ARGS(1)
    void* p = NULL;
    if (napi_get_value_external(env, argv[0], &p) == napi_ok && p) release((wrap_t*)p);   /* frees device memory NOW */
    return undefined(env);
}

static napi_value Step(napi_env env, napi_callback_info info) {
    ARGS(2)
    wrap_t* w = wrap_of(env, argv[0]); if (!w) return NULL;
    check(env, w->h, fluid_step(w->h, (float)num(env, argv[1])));
    return undefined(env);
}

static napi_value Splat(napi_env env, napi_callback_info info) {
    ARGS(8)
    wrap_t* w = wrap_of(env, argv[0]); if (!w) return NULL;
    float a[7]; for (int i = 0; i < 7; ++i) a[i] = (float)num(env, argv[i + 1]);
    check(env, w->h, fluid_splat(w->h, a[0], a[1], a[2], a[3], a[4], a[5], a[6]));
    return undefined(env);
}

static napi_value SetParam(napi_env env, napi_callback_info info) {   /* JS numbers are doubles: pass them as such */
    ARGS(3)
    wrap_t* w = wrap_of(env, argv[0]); if (!w) return NULL;
    int32_t key = 0; napi_get_value_int32(env, argv[1], &key);
    check(env, w->h, fluid_set_param_f64(w->h, key, num(env, argv[2])));
    return undefined(env);
}

static napi_value Resize(napi_env env, napi_callback_info info) {
    ARGS(5)
    wrap_t* w = wrap_of(env, argv[0]); if (!w) return NULL;
    int32_t v[4]; for (int i = 0; i < 4; ++i) napi_get_value_int32(env, argv[i + 1], &v[i]);
    check(env, w->h, fluid_resize(w->h, v[0], v[1], v[2], v[3]));
    return undefined(env);
}

static napi_value f32_view(napi_env env, float* data, size_t n) {
    napi_value ab, ta;
    if (napi_create_external_arraybuffer(env, data, n * sizeof(float), no_finalize, NULL, &ab) != napi_ok) return NULL;
    if (napi_create_typedarray(env, napi_float32_array, n, ab, 0, &ta) != napi_ok) return NULL;
    return ta;
}

static napi_value Read(napi_env env, napi_callback_info info) {
    ARGS(2)
    wrap_t* w = wrap_of(env, argv[0]); if (!w) return NULL;
    int32_t field = 0; napi_get_value_int32(env, argv[1], &field);
    const size_t n = fluid_field_elems(w->h, field);
    if (!n || field < 0 || field > 4) { napi_throw_error(env, NULL, "bad field id"); return NULL; }
    float* dst = pinned_for(w, field, n);
    if (!dst) { napi_throw_error(env, NULL, "out of pinned host memory"); return NULL; }
    if (!check(env, w->h, fluid_read(w->h, field, dst, n))) return NULL;
    return f32_view(env, dst, n);
}

static int f32_arg(napi_env env, napi_value v, float** data, size_t* len) {
    napi_typedarray_type t; napi_value ab; size_t off = 0; void* d = NULL;
    if (napi_get_typedarray_info(env, v, &t, len, &d, &ab, &off) != napi_ok || t != napi_float32_array) {
        napi_throw_error(env, NULL, "expected a Float32Array"); return 0; }
    *data = (float*)d;
    return 1;
}

static napi_value Write(napi_env env, napi_callback_info info) {
    ARGS(3)
    wrap_t* w = wrap_of(env, argv[0]); if (!w) return NULL;
    int32_t field = 0; napi_get_value_int32(env, argv[1], &field);
    float* data; size_t len;
    if (!f32_arg(env, argv[2], &data, &len)) return NULL;
    check(env, w->h, fluid_write(w->h, field, data, len));
    return undefined(env);
}

/* splats(h, Float32Array of n * 7 floats): n splat() records (x, y, dx, dy, r, g, b) in one call */
static napi_value Splats(napi_env env, napi_callback_info info) {
    ARGS(2)
    wrap_t* w = wrap_of(env, argv[0]); if (!w) return NULL;
    float* data; size_t len;
    if (!f32_arg(env, argv[1], &data, &len)) return NULL;
    if (len % 7 != 0 || len / 7 > 0x7fffffff) { napi_throw_error(env, NULL, "splats needs a whole number of 7-float records"); return NULL; }
    check(env, w->h, fluid_splats(w->h, data, (int)(len / 7)));
    return undefined(env);
}

static napi_value PressureSolveHost(napi_env env, napi_callback_info info) {
    ARGS(4)
    wrap_t* w = wrap_of(env, argv[0]); if (!w) return NULL;
    float *d, *p; size_t nd, np; int32_t iters = 0;
    if (!f32_arg(env, argv[1], &d, &nd) || !f32_arg(env, argv[2], &p, &np)) return NULL;
    napi_get_value_int32(env, argv[3], &iters);
    if (nd != np || nd != fluid_field_elems(w->h, FLUID_FIELD_PRESSURE)) { napi_throw_error(env, NULL, "array sizes must equal the pressure field"); return NULL; }
    check(env, w->h, fluid_pressure_solve_host(w->h, d, p, iters));
    return undefined(env);
}

static napi_value Render(napi_env env, napi_callback_info info) {
    ARGS(7)
    wrap_t* w = wrap_of(env, argv[0]); if (!w) return NULL;
    int32_t wd = 0, ht = 0; napi_get_value_int32(env, argv[1], &wd); napi_get_value_int32(env, argv[2], &ht);
    bool shading = true; napi_get_value_bool(env, argv[3], &shading);
    if (wd < 1 || ht < 1) { napi_throw_error(env, NULL, "bad render size"); return NULL; }
    const size_t n = (size_t)wd * ht * 4;
    float* dst = pinned_for(w, 5, n);
    if (!dst) { napi_throw_error(env, NULL, "out of pinned host memory"); return NULL; }
    if (!check(env, w->h, fluid_render(w->h, wd, ht, shading ? 1 : 0, (float)num(env, argv[4]), (float)num(env, argv[5]),
                                       (float)num(env, argv[6]), dst, n))) return NULL;
    return f32_view(env, dst, n);
}

/* The BLOOM_* / SUNRAYS_* keys of `config` (S:77-84 defaults) */
static void postfx_from(napi_env env, napi_value o, fluid_postfx* fx) {
    fx->bloom_iterations = (int32_t)prop(env, o, "BLOOM_ITERATIONS", 8);
    fx->bloom_resolution = (int32_t)prop(env, o, "BLOOM_RESOLUTION", 256);
    fx->bloom_intensity = prop(env, o, "BLOOM_INTENSITY", 0.8);
    fx->bloom_threshold = prop(env, o, "BLOOM_THRESHOLD", 0.6);
    fx->bloom_soft_knee = prop(env, o, "BLOOM_SOFT_KNEE", 0.7);
    fx->sunrays_resolution = (int32_t)prop(env, o, "SUNRAYS_RESOLUTION", 196);
    fx->sunrays_weight = prop(env, o, "SUNRAYS_WEIGHT", 1.0);
}

/* The dw x dh RGB dithering texture: a Float32Array with BLOOM, ignored (NULL) without it.  0 with a JS
 * exception pending if it is missing or the wrong size. */
static int dither_from(napi_env env, uint32_t kw, napi_value v, int32_t dw, int32_t dh, const float** dither) {
    *dither = NULL;
    if (!(kw & FLUID_DISPLAY_BLOOM)) return 1;
    float* d; size_t len;
    if (!f32_arg(env, v, &d, &len)) return 0;
    if (dw < 1 || dh < 1 || len != (size_t)dw * dh * 3) { napi_throw_error(env, NULL, "dither must hold dw * dh * 3 floats"); return 0; }
    *dither = d;
    return 1;
}

/* renderKeywords(h, width, height, keywords, config, dither, dw, dh, r, g, b): fluid_render_keywords with
 * the BLOOM_* / SUNRAYS_* keys read from `config`; dither is the dw x dh RGB Float32Array (needed with
 * BLOOM only; pass null otherwise).  Returns the frame (or a slab rank's band of it) like render(). */
static napi_value RenderKeywords(napi_env env, napi_callback_info info) {
    ARGS(11)
    wrap_t* w = wrap_of(env, argv[0]); if (!w) return NULL;
    int32_t wd = 0, ht = 0, dw = 0, dh = 0; uint32_t kw = 0;
    napi_get_value_int32(env, argv[1], &wd); napi_get_value_int32(env, argv[2], &ht);
    napi_get_value_uint32(env, argv[3], &kw);
    napi_get_value_int32(env, argv[6], &dw); napi_get_value_int32(env, argv[7], &dh);
    if (wd < 1 || ht < 1) { napi_throw_error(env, NULL, "bad render size"); return NULL; }
    fluid_postfx fx;
    postfx_from(env, argv[4], &fx);
    const float* dither;
    if (!dither_from(env, kw, argv[5], dw, dh, &dither)) return NULL;
    int y0 = 0, y1 = ht;                        /* without post-FX a slab rank draws its band only */
    if (!(kw & (FLUID_DISPLAY_BLOOM | FLUID_DISPLAY_SUNRAYS)) && !check(env, w->h, fluid_render_band(w->h, ht, &y0, &y1))) return NULL;
    const size_t n = (size_t)wd * (y1 - y0) * 4;
    float* dst = pinned_for(w, 5, n ? n : 1);
    if (!dst) { napi_throw_error(env, NULL, "out of pinned host memory"); return NULL; }
    if (!check(env, w->h, fluid_render_keywords(w->h, wd, ht, kw, &fx, dither, dw, dh, (float)num(env, argv[8]),
                                                (float)num(env, argv[9]), (float)num(env, argv[10]), dst, n, NULL, NULL))) return NULL;
    return f32_view(env, dst, n);
}

/* capture(h, width, height, canvasWidth, canvasHeight, keywords, transparent, config, dither, dw, dh, r, g, b):
 * fluid_capture, arguments as for renderKeywords.  Returns a new Uint8Array of width * height * 4 bytes, top
 * row first: what normalizeTexture (S:309-327) hands textureToCanvas. */
static napi_value Capture(napi_env env, napi_callback_info info) {
    ARGS(14)
    wrap_t* w = wrap_of(env, argv[0]); if (!w) return NULL;
    int32_t wd = 0, ht = 0, cw = 0, ch = 0, dw = 0, dh = 0; uint32_t kw = 0; bool transparent = false;
    napi_get_value_int32(env, argv[1], &wd); napi_get_value_int32(env, argv[2], &ht);
    napi_get_value_int32(env, argv[3], &cw); napi_get_value_int32(env, argv[4], &ch);
    napi_get_value_uint32(env, argv[5], &kw); napi_get_value_bool(env, argv[6], &transparent);
    napi_get_value_int32(env, argv[9], &dw); napi_get_value_int32(env, argv[10], &dh);
    if (wd < 1 || ht < 1) { napi_throw_error(env, NULL, "bad capture size"); return NULL; }
    fluid_postfx fx;
    postfx_from(env, argv[7], &fx);
    const float* dither;
    if (!dither_from(env, kw, argv[8], dw, dh, &dither)) return NULL;
    const size_t n = (size_t)wd * ht * 4;
    void* data = NULL; napi_value ab, ta;
    if (napi_create_arraybuffer(env, n, &data, &ab) != napi_ok) return NULL;
    if (!check(env, w->h, fluid_capture(w->h, wd, ht, cw, ch, kw, transparent ? 1 : 0, &fx, dither, dw, dh,
                                        (float)num(env, argv[11]), (float)num(env, argv[12]), (float)num(env, argv[13]),
                                        (uint8_t*)data, n))) return NULL;
    if (napi_create_typedarray(env, napi_uint8_array, n, ab, 0, &ta) != napi_ok) return NULL;
    return ta;
}

/* renderCanvas(h, width, height, keywords, transparent, config, dither, dw, dh, r, g, b): fluid_render_canvas
 * into host memory, arguments as for renderKeywords.  Returns a new Uint8ClampedArray of width * height * 4
 * bytes, top row first: the pixels of the drawing buffer after render(null), for new ImageData(data, width,
 * height) and putImageData. */
static napi_value RenderCanvas(napi_env env, napi_callback_info info) {
    ARGS(12)
    wrap_t* w = wrap_of(env, argv[0]); if (!w) return NULL;
    int32_t wd = 0, ht = 0, dw = 0, dh = 0; uint32_t kw = 0; bool transparent = false;
    napi_get_value_int32(env, argv[1], &wd); napi_get_value_int32(env, argv[2], &ht);
    napi_get_value_uint32(env, argv[3], &kw); napi_get_value_bool(env, argv[4], &transparent);
    napi_get_value_int32(env, argv[7], &dw); napi_get_value_int32(env, argv[8], &dh);
    if (wd < 1 || ht < 1) { napi_throw_error(env, NULL, "bad canvas size"); return NULL; }
    fluid_postfx fx;
    postfx_from(env, argv[5], &fx);
    const float* dither;
    if (!dither_from(env, kw, argv[6], dw, dh, &dither)) return NULL;
    const size_t n = (size_t)wd * ht * 4;
    void* data = NULL; napi_value ab, ta;
    if (napi_create_arraybuffer(env, n, &data, &ab) != napi_ok) return NULL;
    if (!check(env, w->h, fluid_render_canvas(w->h, wd, ht, kw, transparent ? 1 : 0, &fx, dither, dw, dh,
                                              (float)num(env, argv[9]), (float)num(env, argv[10]), (float)num(env, argv[11]),
                                              (uint8_t*)data, n, 0))) return NULL;
    if (napi_create_typedarray(env, napi_uint8_clamped_array, n, ab, 0, &ta) != napi_ok) return NULL;
    return ta;
}

static napi_value Sync(napi_env env, napi_callback_info info) {
    ARGS(1)
    wrap_t* w = wrap_of(env, argv[0]); if (!w) return NULL;
    check(env, w->h, fluid_sync(w->h));
    return undefined(env);
}

static napi_value Stat(napi_env env, napi_callback_info info) {
    ARGS(2)
    wrap_t* w = wrap_of(env, argv[0]); if (!w) return NULL;
    int32_t key = 0; napi_get_value_int32(env, argv[1], &key);
    napi_value out; napi_create_double(env, (double)fluid_stat(w->h, key), &out);
    return out;
}

static void set_int(napi_env env, napi_value obj, const char* k, int v) {
    napi_value n; napi_create_int32(env, v, &n);
    napi_set_named_property(env, obj, k, n);
}

static napi_value Dims(napi_env env, napi_callback_info info) {
    ARGS(2)
    wrap_t* w = wrap_of(env, argv[0]); if (!w) return NULL;
    int32_t field = 0; napi_get_value_int32(env, argv[1], &field);
    int wd, r, c, r0;
    if (!check(env, w->h, fluid_field_dims(w->h, field, &wd, &r, &c, &r0))) return NULL;
    napi_value obj;
    if (napi_create_object(env, &obj) != napi_ok) return NULL;
    set_int(env, obj, "width", wd); set_int(env, obj, "height", r);
    set_int(env, obj, "channels", c); set_int(env, obj, "row0", r0);
    return obj;
}

static napi_value GetResolution(napi_env env, napi_callback_info info) {
    ARGS(3)
    int32_t v[3]; for (int i = 0; i < 3; ++i) napi_get_value_int32(env, argv[i], &v[i]);
    int wd, hh; fluid_get_resolution(v[0], v[1], v[2], &wd, &hh);
    napi_value obj;
    if (napi_create_object(env, &obj) != napi_ok) return NULL;
    set_int(env, obj, "width", wd); set_int(env, obj, "height", hh);
    return obj;
}

static napi_value LastError(napi_env env, napi_callback_info info) {
    size_t argc = 1; napi_value argv[1];
    napi_get_cb_info(env, info, &argc, argv, NULL, NULL);
    fluid_t* h = NULL;
    if (argc >= 1) { void* p = NULL; if (napi_get_value_external(env, argv[0], &p) == napi_ok && p) h = ((wrap_t*)p)->h; }
    const char* m = fluid_last_error(h);
    napi_value s; napi_create_string_utf8(env, m ? m : "", NAPI_AUTO_LENGTH, &s);
    return s;
}

/* ---- slab plumbing: the launcher (one Node process per GPU) moves these blobs between ranks ---- */
static napi_value NcclUniqueId(napi_env env, napi_callback_info info) {
    (void)info;
    void* data = NULL; napi_value ab;
    if (napi_create_arraybuffer(env, 128, &data, &ab) != napi_ok) return NULL;
    if (!check(env, NULL, fluid_nccl_unique_id(data, 128))) return NULL;
    return ab;
}
static napi_value P2PExport(napi_env env, napi_callback_info info) {
    ARGS(1)
    wrap_t* w = wrap_of(env, argv[0]); if (!w) return NULL;
    void* data = NULL; napi_value ab;
    if (napi_create_arraybuffer(env, 256, &data, &ab) != napi_ok) return NULL;
    if (!check(env, w->h, fluid_p2p_export(w->h, data, 256))) return NULL;
    return ab;
}
static void* blob_or_null(napi_env env, napi_value v) {
    void* d = NULL; size_t n = 0;
    return (napi_get_arraybuffer_info(env, v, &d, &n) == napi_ok && n >= 256) ? d : NULL;
}
static napi_value P2PConnect(napi_env env, napi_callback_info info) {
    ARGS(3)
    wrap_t* w = wrap_of(env, argv[0]); if (!w) return NULL;
    check(env, w->h, fluid_p2p_connect(w->h, blob_or_null(env, argv[1]), blob_or_null(env, argv[2])));
    return undefined(env);
}
static napi_value P2PDisable(napi_env env, napi_callback_info info) {
    ARGS(1)
    wrap_t* w = wrap_of(env, argv[0]); if (!w) return NULL;
    check(env, w->h, fluid_p2p_disable(w->h));
    return undefined(env);
}

NAPI_MODULE_INIT() {
    const napi_property_descriptor props[] = {
        {"create", NULL, Create, NULL, NULL, NULL, napi_enumerable, NULL},
        {"createSlab", NULL, CreateSlab, NULL, NULL, NULL, napi_enumerable, NULL},
        {"destroy", NULL, Destroy, NULL, NULL, NULL, napi_enumerable, NULL},
        {"step", NULL, Step, NULL, NULL, NULL, napi_enumerable, NULL},
        {"splat", NULL, Splat, NULL, NULL, NULL, napi_enumerable, NULL},
        {"splats", NULL, Splats, NULL, NULL, NULL, napi_enumerable, NULL},
        {"setParam", NULL, SetParam, NULL, NULL, NULL, napi_enumerable, NULL},
        {"resize", NULL, Resize, NULL, NULL, NULL, napi_enumerable, NULL},
        {"read", NULL, Read, NULL, NULL, NULL, napi_enumerable, NULL},
        {"write", NULL, Write, NULL, NULL, NULL, napi_enumerable, NULL},
        {"pressureSolveHost", NULL, PressureSolveHost, NULL, NULL, NULL, napi_enumerable, NULL},
        {"render", NULL, Render, NULL, NULL, NULL, napi_enumerable, NULL},
        {"renderKeywords", NULL, RenderKeywords, NULL, NULL, NULL, napi_enumerable, NULL},
        {"capture", NULL, Capture, NULL, NULL, NULL, napi_enumerable, NULL},
        {"renderCanvas", NULL, RenderCanvas, NULL, NULL, NULL, napi_enumerable, NULL},
        {"sync", NULL, Sync, NULL, NULL, NULL, napi_enumerable, NULL},
        {"stat", NULL, Stat, NULL, NULL, NULL, napi_enumerable, NULL},
        {"dims", NULL, Dims, NULL, NULL, NULL, napi_enumerable, NULL},
        {"getResolution", NULL, GetResolution, NULL, NULL, NULL, napi_enumerable, NULL},
        {"lastError", NULL, LastError, NULL, NULL, NULL, napi_enumerable, NULL},
        {"ncclUniqueId", NULL, NcclUniqueId, NULL, NULL, NULL, napi_enumerable, NULL},
        {"p2pExport", NULL, P2PExport, NULL, NULL, NULL, napi_enumerable, NULL},
        {"p2pConnect", NULL, P2PConnect, NULL, NULL, NULL, napi_enumerable, NULL},
        {"p2pDisable", NULL, P2PDisable, NULL, NULL, NULL, napi_enumerable, NULL},
    };
    napi_define_properties(env, exports, sizeof props / sizeof props[0], props);
    return exports;
}
