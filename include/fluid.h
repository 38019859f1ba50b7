/*
 * fluid.h — C ABI of libfluid_b200: the drop-in boundary for the simulation path of
 * PavelDoGreat/WebGL-Fluid-Simulation (script.js step()/splat()/config).
 *
 * The reference has no FFI: its "interface" is a set of global JS functions and a global
 * `config` object inside one classic <script> (index.html:222).  Every entry point below cites
 * the reference construct (script.js = "S") it replaces; INTEGRATION.md shows the N-API / ctypes
 * binding a maintainer would add on the reference side.
 *
 * Conventions (all from the reference):
 *   - fields are row-major, x fastest, ROW 0 = BOTTOM (GL texture convention, S:452, S:1531);
 *   - velocity is float2 interleaved (RG texture, S:994-997), dye is float4 interleaved
 *     (RGBA texture, S:989-992), pressure/divergence/curl are float (R texture, S:999-1001);
 *   - uv of cell (i,j) = ((i+.5)/W, (j+.5)/H) (S:452); sampling is CLAMP_TO_EDGE (S:1051-1052);
 *   - velocity is measured in sim-texels per second (S:777 with texelSize = 1/W).
 *   - storage is fp32 (BASELINE.json asks fp32; the reference stores fp16, S:138-147).
 *
 * Error convention: every int-returning call returns FLUID_OK (0) or a negative fluid_status;
 * fluid_last_error() returns the message.  There is NO CPU fallback anywhere in this library:
 * without a CUDA device fluid_create() fails with FLUID_ERR_NO_DEVICE.
 *
 * Threading: a handle is single-threaded like the JS it replaces.  step/splat/pass calls enqueue
 * work on the handle's CUDA stream and return; fluid_read()/fluid_sync() block.
 */
#ifndef FLUID_B200_H
#define FLUID_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FLUID_ABI_VERSION 2

typedef struct fluid fluid_t; /* opaque; owns device buffers, streams, events, graphs, NCCL comm */

typedef enum fluid_status {
    FLUID_OK = 0,
    FLUID_ERR_INVALID = -1,      /* bad argument / bad field id / size mismatch            */
    FLUID_ERR_NO_DEVICE = -2,    /* no CUDA device or device is not sm_90                  */
    FLUID_ERR_CUDA = -3,         /* a CUDA runtime/driver call failed                      */
    FLUID_ERR_NCCL = -4,         /* NCCL could not be loaded or a NCCL call failed         */
    FLUID_ERR_HALO = -5,         /* multi-GPU: an advection back-trace left the ghost zone */
    FLUID_ERR_NOMEM = -6
} fluid_status;

/* Field ids.  S:950-954: `dye, velocity, divergence, curl, pressure` globals. */
typedef enum fluid_field {
    FLUID_FIELD_VELOCITY = 0,   /* velocity.read   float2  sim_w x sim_h */
    FLUID_FIELD_DYE = 1,        /* dye.read        float4  dye_w x dye_h */
    FLUID_FIELD_PRESSURE = 2,   /* pressure.read   float   sim_w x sim_h */
    FLUID_FIELD_DIVERGENCE = 3, /* divergence      float   sim_w x sim_h */
    FLUID_FIELD_CURL = 4        /* curl            float   sim_w x sim_h */
} fluid_field;

/* Scalar parameter keys = the simulation keys of the reference `config` object (S:59-69, S:73).
 * The reference reads config live on every call; the host mirror pushes changed keys with
 * fluid_set_param() before step()/splat(). */
typedef enum fluid_param {
    FLUID_DENSITY_DISSIPATION = 0,  /* S:63 default 1     */
    FLUID_VELOCITY_DISSIPATION = 1, /* S:64 default 0.2   */
    FLUID_PRESSURE = 2,             /* S:65 default 0.8   */
    FLUID_PRESSURE_ITERATIONS = 3,  /* S:66 default 20    */
    FLUID_CURL = 4,                 /* S:67 default 30    */
    FLUID_SPLAT_RADIUS = 5,         /* S:68 default 0.25  */
    FLUID_ASPECT = 6,               /* canvas.width/canvas.height, S:1444, S:1457-1462 */
    FLUID_JACOBI_BLOCK = 7,         /* build-only tunable: max temporal-block depth, 1 = naive */
    FLUID_BACKGROUND = 8            /* what fluid_render* draws the display over (render(), S:1296-1317):
                                       0 = drawColor(BACK_COLOR); 1 = drawCheckerboard — config.TRANSPARENT on
                                       the screen (S:1325-1329, checkerboardShader S:531-547, aspect = ASPECT);
                                       2 = nothing, blending off — TRANSPARENT into a capture target          */
} fluid_param;

/* Creation flags */
#define FLUID_FLAG_UNFUSED   0x1u /* run curl / vorticity / divergence as 3 separate passes      */
#define FLUID_FLAG_NO_GRAPH  0x2u /* launch step() pass by pass instead of as one CUDA graph     */
#define FLUID_FLAG_NAIVE_JACOBI 0x4u /* one Jacobi sweep per launch (the literal S:1262 loop)    */
#define FLUID_FLAG_HALF_STORAGE 0x10u /* store every field as fp16 like the reference's textures (S:138-147,
                                         S:986-1006): fp32 arithmetic, round-to-nearest-even on every pass
                                         write, one launch per reference blit; single GPU; the ABI still
                                         speaks fp32 (fluid_read widens, fluid_write narrows)              */
#define FLUID_FLAG_HALF_POSTFX 0x20u /* the bloom FBO and pyramid, sunrays and sunraysTemp of fluid_render_keywords /
                                        fluid_capture are fp16 like the reference's RGBA16F / R16F FBOs (S:1012-1043):
                                        every blit's fp32 result is rounded to nearest even when stored, the additive
                                        up-pass rounds fragment + widened destination once.  The sunrays mask follows
                                        the dye's storage.  HALF_STORAGE | HALF_POSTFX is the reference's desktop frame.
                                        Single GPU; the render() frame stays fp32, host_bloom / host_sunrays widen  */
#define FLUID_FLAG_NEAREST_FILTERING 0x40u /* the reference on a device without float linear filtering
                                        (`!ext.supportLinearFiltering`: OES_texture_float_linear on WebGL2,
                                        OES_texture_half_float_linear on WebGL1, S:127-134): dye and velocity
                                        (S:990), the bloom FBO and pyramid (S:1017), sunrays and sunraysTemp
                                        (S:1039) are sampled NEAREST + CLAMP_TO_EDGE, texel clamp(floor(uv * n),
                                        0, n - 1), by fluid_render*, fluid_capture and fluid_resize's copy
                                        (resizeFBO S:1108-1114).  The dithering texture stays LINEAR + REPEAT.
                                        step(), splats, every fluid_pass_* and the host solves do not change:
                                        advection is the MANUAL_FILTERING shader on every handle created
                                        without FLUID_FLAG_LINEAR_ADVECTION, which is exactly this device's.
                                        The config override of S:109-114 (DYE_RESOLUTION 512, SHADING / BLOOM /
                                        SUNRAYS off) is the host's (default_config).  Combines with HALF_STORAGE
                                        and HALF_POSTFX; single GPU                                            */
#define FLUID_FLAG_LINEAR_ADVECTION 0x80u /* step() advects like the reference on a device WITH float linear
                                        filtering (every desktop browser): the advectionShader's #else branch
                                        (S:776-779) samples uVelocity and uSource through the LINEAR samplers
                                        of dye and velocity (S:990).  Without this flag advection is the
                                        MANUAL_FILTERING branch (bilerp S:758-770 over NEAREST fetches) on
                                        every handle.  fluid_step (graph and pass by pass),
                                        fluid_pass_advect_velocity and fluid_pass_advect_dye compute, in fp32
                                        with every operation rounded on its own:
                                          L(tex, n_x, n_y, uv): u = uv.x*n_x - .5, v = uv.y*n_y - .5,
                                            i0 = floor(u), a = u - i0 (b likewise), taps clamped to the grid,
                                            ((w00 t00 + w10 t10) + w01 t01) + w11 t11 with w00 = (1-a)(1-b),
                                            w10 = a(1-b), w01 = (1-a)b, w11 = ab, taps widened from storage;
                                          velocity: uv = cell centre, c = uv - (dt * L(vel, W, H, uv)) * ts,
                                            out = L(vel, W, H, c) / (1 + VELOCITY_DISSIPATION * dt);
                                          dye: uv = dye cell centre, c = uv - (dt * L(vel, W, H, uv)) * ts
                                            (ts = the SIM texel size, S:1276),
                                            out = L(dye, Wd, Hd, c) / (1 + DENSITY_DISSIPATION * dt);
                                        rounded to fp16 when stored with HALF_STORAGE.  Splats, every other
                                        pass, the host solves, resize and the display do not change.
                                        HALF_STORAGE | HALF_POSTFX | LINEAR_ADVECTION is the desktop browser's
                                        frame and step.  FLUID_ERR_INVALID with NEAREST_FILTERING (a device
                                        without linear filtering runs MANUAL_FILTERING) and on slab handles  */
#define FLUID_FLAG_TILED_PASSES 0x8u /* generation-1 kernels (one thread per fragment / smem tile) for
                                        curl-vorticity-divergence and gradientSubtract instead of the
                                        row-streaming ones (comparison + fallback path)              */

typedef struct fluid_config {
    int32_t sim_w, sim_h;           /* getResolution(SIM_RESOLUTION)  S:983, S:1612-1624 */
    int32_t dye_w, dye_h;           /* getResolution(DYE_RESOLUTION)  S:984              */
    float density_dissipation;      /* S:63 */
    float velocity_dissipation;     /* S:64 */
    float pressure;                 /* S:65 */
    int32_t pressure_iterations;    /* S:66 */
    float curl;                     /* S:67 */
    float splat_radius;             /* S:68 */
    float aspect;                   /* canvas.width / canvas.height; <=0 means sim_w/sim_h */
    int32_t device;                 /* CUDA ordinal; -1 = current device */
    uint32_t flags;                 /* FLUID_FLAG_* */
    int32_t jacobi_block;           /* 0 = library default */
} fluid_config;

/* Per-pass device timing of the last fluid_step() (milliseconds, CUDA events on the handle's
 * stream).  Only recorded when FLUID_FLAG_NO_GRAPH is set. */
typedef struct fluid_timing {
    float curl_vort_div_ms, jacobi_ms, gradient_ms, advect_velocity_ms, advect_dye_ms, total_ms;
    int32_t jacobi_launches;        /* kernels launched for the pressure loop */
    int32_t total_launches;         /* kernels launched by the step */
} fluid_timing;

/* ---- lifetime -------------------------------------------------------------------------------- */

/* Fills *cfg with the reference defaults (S:59-69): SIM 128, DYE 1024, dissipation 1 / 0.2,
 * PRESSURE 0.8, 20 iterations, CURL 30, SPLAT_RADIUS 0.25, aspect 1. */
void fluid_config_default(fluid_config* cfg);

/* getResolution(resolution) of S:1612-1624 for a canvas_w x canvas_h drawing buffer. */
void fluid_get_resolution(int resolution, int canvas_w, int canvas_h, int* out_w, int* out_h);

/* initFramebuffers() of S:982-1010 on first call (dye == null branch): allocates velocity, dye,
 * pressure (double-buffered) and divergence, curl; all zero, dye alpha = 1 (clearColor S:136
 * + gl.clear in createFBO S:1059). */
int fluid_create(const fluid_config* cfg, fluid_t** out);

/* Same, for rank `rank` of `world` row-slab ranks (one process per GPU).  `nccl_uid` is the
 * 128-byte ncclUniqueId obtained on rank 0 from fluid_nccl_unique_id() and broadcast by the
 * caller (torch.distributed in this repo).  The rank owns sim rows [rank*H/world,(rank+1)*H/world)
 * and the matching dye rows; fluid_read()/fluid_write() address the OWNED rows only. */
int fluid_create_slab(const fluid_config* cfg, int rank, int world, const void* nccl_uid,
                      size_t uid_bytes, fluid_t** out);
int fluid_nccl_unique_id(void* out_uid, size_t uid_bytes); /* uid_bytes must be >= 128 */

/* Optional peer-memory halo path for slab handles on one NVLink/NVSwitch box (no reference
 * counterpart).  Every handle keeps all its fields in one device allocation, its arena.  Every rank
 * exports a 256-byte blob (a CUDA IPC handle of that arena + its layout),
 * the launcher all-gathers them, and each rank connects to rank-1 / rank+1 (NULL at the ends).
 * Afterwards halo rows are stored straight into the neighbours' ghost rows by one kernel that
 * also carries the free/ready handshake (system-scope release/acquire flag words, bounded spins);
 * without it the NCCL send/recv path is used. */
int fluid_p2p_export(fluid_t* h, void* blob, size_t blob_bytes);   /* blob_bytes >= 256 */
int fluid_p2p_connect(fluid_t* h, const void* blob_below, const void* blob_above);
int fluid_p2p_disable(fluid_t* h);   /* back to NCCL; call on every rank if any rank failed to connect */

/* Batch handles (no reference counterpart): B = `members` independent simulations of cfg's sizes, scalars
 * and flags in one handle, stepped and splatted together through the same launches.  Member m ends every call
 * with the bits an ordinary handle given member m's inputs would hold.  All fields start zero with dye alpha
 * 1 in every member, as after fluid_create.
 *  - fluid_step steps every member with one dt (a CUDA graph unless FLUID_FLAG_NO_GRAPH); fluid_set_param and
 *    fluid_set_param_f64 set the key for every member, and fluid_get_param returns member 0's value.
 *  - Parameter sweeps: fluid_set_param_members gives each member its own DENSITY_DISSIPATION,
 *    VELOCITY_DISSIPATION, PRESSURE, CURL or SPLAT_RADIUS, and fluid_step_members its own dt (below).
 *  - fluid_field_elems is B x w x rows x channels, and fluid_field_dims gives one member's w, rows and
 *    channels with row0 = 0.  fluid_read, fluid_write, fluid_read_device and fluid_write_device move all
 *    members in member order as a (B, H, W[, C]) C-contiguous array; fluid_device_ptr is member 0's .read,
 *    the other members following it contiguously.
 *  - fluid_sync, fluid_stat, fluid_launch_count, fluid_mark, fluid_elapsed_ms, fluid_timing_last,
 *    fluid_last_error and fluid_destroy behave as on any handle.
 *  - fluid_render_canvas_batch and fluid_capture_batch draw every member's canvas or capture in one call;
 *    fluid_render_canvas_looks and fluid_capture_looks give each image its own post-FX sliders and background.
 *  - Member subsets (below): fluid_read_members and fluid_write_members move, fluid_reset_members resets, and
 *    fluid_render_canvas_members and fluid_capture_members draw, only the members a list names.
 *  - Every other entry point refuses a batch handle with FLUID_ERR_INVALID and leaves it usable: the fp32
 *    frames (fluid_render, fluid_render_keywords, fluid_render_postfx), fluid_capture, fluid_capture_device
 *    and fluid_render_canvas (use the batch calls), fluid_render_band, fluid_resize, fluid_pass_*,
 *    fluid_pressure_solve_host, fluid_splat, fluid_splats and fluid_splats_device (use fluid_splats_batch or
 *    fluid_splats_batch_device) and the p2p calls.
 * fluid_create_batch refuses with FLUID_ERR_INVALID: members < 1 or > FLUID_MAX_MEMBERS (the member is the
 * kernels' grid z index); any flag but FLUID_FLAG_NO_GRAPH; sizes that are not powers of two, a sim or dye
 * width under 128 or a height under 2.  The reference default 128^2 / 1024^2 qualifies.  FLUID_ERR_NOMEM:
 * the fields of B members do not fit; nothing is left allocated. */
#define FLUID_MAX_MEMBERS 65535
int fluid_create_batch(const fluid_config* cfg, int members, fluid_t** out);
/* B of a batch handle; 1 for ordinary and slab handles (0 for NULL). */
int fluid_members(fluid_t* h);
/* Per-member values of a batch handle.  values[m] becomes member m's value of `key`, narrowed as
 * fluid_set_param_f64 narrows it; SPLAT_RADIUS stays a double until correctRadius, with the batch's ASPECT.  Only
 * FLUID_DENSITY_DISSIPATION, FLUID_VELOCITY_DISSIPATION, FLUID_PRESSURE, FLUID_CURL and FLUID_SPLAT_RADIUS have
 * per-member values: PRESSURE_ITERATIONS and JACOBI_BLOCK choose the launches all members share, ASPECT and
 * BACKGROUND are canvas-wide.  fluid_step_members is fluid_step with member m stepped by dt[m].  After every call
 * member m holds the bits of an ordinary handle created with the batch's config, given member m's values through
 * fluid_set_param_f64 and stepped with member m's dt.  fluid_set_param / fluid_set_param_f64 of a key later set it
 * for every member again.  Neither per-member values nor dts recapture a step graph.  n must be B: n != B, a NULL
 * array, another key, or an ordinary or slab handle is FLUID_ERR_INVALID, with every value and field untouched.
 * fluid_get_param_members returns the B values as fluid_get_param would return them. */
int fluid_set_param_members(fluid_t* h, int key, const double* values, int n);
int fluid_get_param_members(fluid_t* h, int key, float* values, int n);
int fluid_step_members(fluid_t* h, const float* dt, int n);

/* Member subsets of a batch handle: `members` is a host array of n DISTINCT member indices in [0, B), in any
 * order, and slot (or image) k of the caller's buffer is member members[k].  The list is checked on the host, then
 * copied, stream-ordered, into a list buffer of B int32 the handle allocates at creation outside the field arena;
 * the caller may reuse `members` as soon as the call returns.
 *  - n == 0 does nothing and launches nothing.
 *  - Refused with FLUID_ERR_INVALID before any work, every field and buffer untouched and the handle usable: an
 *    index outside [0, B); an index listed twice; n < 0, or members == NULL with n > 0; a buffer whose size does not
 *    match n; a bad field; an ordinary or slab handle; a device buffer fluid_read_device refuses.
 *  - No call recaptures a step graph.
 * fluid_read_members / fluid_write_members: fluid_read / fluid_write of the listed members.  buf is a C-contiguous
 * (n, H, W[, C]) array, n_floats == n * w * rows * channels.
 *  - In host memory (on_device == 0): one copy per listed member, straight between its block of the arena and the
 *    caller's memory, then a stream sync.
 *  - In device memory (on_device != 0): one launch, stream-ordered and returning without a sync, with the rules of
 *    fluid_read_device / fluid_write_device.
 *  - fluid_write_members writes the listed members' .read only; every other member keeps every byte.
 * fluid_reset_members: the listed members return to the state fluid_create_batch leaves (both slots of velocity,
 * pressure and dye zero, dye alpha 1, divergence and curl zero), in one launch.  Their per-member values
 * (fluid_set_param_members) are config, not state, and stay. */
int fluid_read_members(fluid_t* h, int field, const int32_t* members, int n, float* dst, size_t n_floats,
                       int dst_on_device);
int fluid_write_members(fluid_t* h, int field, const int32_t* members, int n, const float* src, size_t n_floats,
                        int src_on_device);
int fluid_reset_members(fluid_t* h, const int32_t* members, int n);

void fluid_destroy(fluid_t* h);

/* initFramebuffers() on a live simulation (S:982-1010 else-branches + resizeDoubleFBO S:1116-1126):
 * the handle's fields move to a new arena.  Velocity and dye are bilinearly resampled to the new size
 * (copyShader through a LINEAR sampler); one whose size did not change is kept bit for bit.  Pressure /
 * divergence / curl are re-created zeroed.  Old and new arena coexist during the call.
 * FLUID_ERR_NOMEM: the new arena does not fit; the handle is left exactly as it was.
 * On a slab handle the call is collective (same sizes on every rank): ghost rows of the old velocity and
 * dye are refreshed, the rank's new rows are resampled, and the peer-memory mappings of the old arena
 * are dropped (export / connect again, or stay on NCCL).  FLUID_ERR_HALO: the factor needs more ghost
 * rows than the slab keeps. */
int fluid_resize(fluid_t* h, int sim_w, int sim_h, int dye_w, int dye_h);

/* ---- the hot path ---------------------------------------------------------------------------- */

/* step(dt) of S:1231-1294: curl -> vorticity -> divergence -> clear(pressure) ->
 * PRESSURE_ITERATIONS x Jacobi -> gradientSubtract -> advect velocity -> advect dye. */
int fluid_step(fluid_t* h, float dt);

/* splat(x, y, dx, dy, color) of S:1441-1455: velocity += exp(-|p|^2/radius)*(dx,dy), then
 * dye.rgb += exp(..)*(r,g,b), dye.a = 1; radius = correctRadius(SPLAT_RADIUS/100) (S:1457-1462). */
int fluid_splat(fluid_t* h, float x, float y, float dx, float dy, float r, float g, float b);

/* n calls of fluid_splat(h, s[7k+0], ..., s[7k+6]), k = 0..n-1, in that order, with the same bits, in
 * ceil(n/128) launches (fluid_splat itself is one): records are (x, y, dx, dy, r, g, b); radius and
 * aspect come from the handle's config, read once.  A frame that produces several splats (a burst of
 * multipleSplats, one per moved pointer) should hand them over in one call.  The array is copied
 * before the call returns.  n == 0 does nothing (dye alpha included); n < 0, or splats == NULL with
 * n > 0, is FLUID_ERR_INVALID and leaves the fields untouched. */
int fluid_splats(fluid_t* h, const float* splats, int n);

/* fluid_splats for a batch handle: record k (the 7 floats of fluid_splats) goes to member member[k].  Each
 * member receives its records in call order, with the bits fluid_splats would give an ordinary handle;
 * a member named by no record is not touched (dye alpha included).  The records are applied in place on the
 * named members' .read, in launches of at most 128 records for at most 64 members; no other member costs a
 * block.  n == 0 does nothing.  n < 0, a NULL array with n > 0, a member index outside [0, B) or an
 * ordinary handle is FLUID_ERR_INVALID, with every field untouched. */
int fluid_splats_batch(fluid_t* h, const int32_t* member, const float* splats, int n);

/* fluid_splats and fluid_splats_batch with the arrays in CUDA memory (for example torch tensors), for pipelines
 * that make their splats on the GPU: no host copy, and each call reads and writes each field once whatever n is.
 *  - fluid_splats_device(h, splats, n) gives the bits of fluid_splats(h, host copy, n): the same .read -> .write
 *    and swap of velocity and dye, the same rows written.  One launch for every n >= 1.  Ordinary handles of every
 *    flag; a batch handle is refused (use fluid_splats_batch_device).
 *  - fluid_splats_batch_device(h, member, splats, n): member m ends with the bits fluid_splats_batch gives with
 *    the same arrays on the host: its own records in call order, in place on its .read, with its own
 *    SPLAT_RADIUS.  A member no record names is not touched.  Two launches whatever n, B or the spread of the
 *    records (one orders the records by member, one splats).  An ordinary handle is refused.
 *  - Stream-ordered with the rules of fluid_write_device: work of other streams that writes the arrays must be
 *    complete before the call, and the caller calls fluid_sync before reusing them.
 *  - A member index outside [0, B) cannot be checked on the host without a sync.  The call then splats no member
 *    and changes nothing, and the next fluid_sync (or fluid_read) returns FLUID_ERR_INVALID once, with a message;
 *    calls after it work normally.
 *  - fluid_splats_batch_device keeps the grouped records in a scratch buffer outside the field arena.  It grows
 *    on demand, never during a graph capture (FLUID_ERR_INVALID there); FLUID_ERR_NOMEM when it does not fit,
 *    with the handle usable.
 * n == 0 launches nothing and touches nothing.  Refused with FLUID_ERR_INVALID, every field and buffer untouched
 * and the handle usable: n < 0; a NULL array with n > 0; an array fluid_read_device refuses (host memory, another
 * device's memory, not 4-byte aligned, overlapping the field arena), `member` and `splats` alike; slab handles. */
int fluid_splats_device(fluid_t* h, const float* splats, int n);
int fluid_splats_batch_device(fluid_t* h, const int32_t* member, const float* splats, int n);

/* config.<KEY> = value (S:59-69).  PRESSURE_ITERATIONS / JACOBI_BLOCK are rounded to int. */
int fluid_set_param(fluid_t* h, int key, float value);
int fluid_get_param(fluid_t* h, int key, float* value);
/* Same as fluid_set_param, at the precision the JS `config` values have.  SPLAT_RADIUS and ASPECT
 * enter DOUBLE arithmetic on the host (correctRadius(config.SPLAT_RADIUS / 100.0), S:1447 +
 * S:1457-1462) before the one narrowing of gl.uniform1f; host mirrors should use this entry point. */
int fluid_set_param_f64(fluid_t* h, int key, double value);

/* ---- individual passes (the reference's one-blit-per-program granularity; used by the parity
 *      tests and by callers that drive the loop themselves).  Each reads the `.read` buffers and
 *      performs the same swap() the reference does after its blit. ------------------------------ */
int fluid_pass_curl(fluid_t* h);                       /* S:1234-1237, curlShader S:814-833        */
int fluid_pass_vorticity(fluid_t* h, float dt);        /* S:1239-1246, vorticityShader S:835-866   */
int fluid_pass_divergence(fluid_t* h);                 /* S:1248-1251, divergenceShader S:786-812  */
int fluid_pass_clear_pressure(fluid_t* h);             /* S:1253-1257, clearShader S:508-519       */
int fluid_pass_jacobi(fluid_t* h, int iters);          /* S:1259-1266, pressureShader S:868-890    */
int fluid_pass_pressure_solve(fluid_t* h);             /* clear + PRESSURE_ITERATIONS Jacobi, fused */
int fluid_pass_gradient_subtract(fluid_t* h);          /* S:1268-1273, gradientSubtractShader S:892-913 */
int fluid_pass_advect_velocity(fluid_t* h, float dt);  /* S:1275-1285, advectionShader S:746-784   */
int fluid_pass_advect_dye(fluid_t* h, float dt);       /* S:1287-1293                              */
int fluid_pass_curl_vorticity_divergence(fluid_t* h, float dt); /* the three above in one kernel  */

/* ---- data in / out ---------------------------------------------------------------------------- */

/* Element count (floats) of the rows of `field` this handle owns: w*h*channels. */
size_t fluid_field_elems(fluid_t* h, int field);
int fluid_field_dims(fluid_t* h, int field, int* w, int* h_rows, int* channels, int* row0);

/* framebufferToTexture() of S:301-307 (gl.readPixels FLOAT) generalised to every field: copies
 * the `.read` buffer to host memory (blocks until the stream has drained). */
int fluid_read(fluid_t* h, int field, float* host, size_t n_floats);
/* Test / checkpoint hook with no reference counterpart: overwrites the `.read` buffer. */
int fluid_write(fluid_t* h, int field, const float* host, size_t n_floats);

/* fluid_read / fluid_write with the caller's DEVICE memory in place of host memory (for example a torch
 * float32 CUDA tensor), for pipelines whose data already lives on the GPU: no PCIe transfer, no host stall.
 *  - Layout, element count and bits are those of fluid_read / fluid_write: fp32, owned rows, row 0 at the
 *    bottom, channels interleaved.  On a half-storage handle fluid_read_device widens exactly and
 *    fluid_write_device narrows to nearest even (overflow to +-inf), on the device, allocating nothing.
 *  - Written divergence rebuilds the blocked Jacobi solve's tiny-divergence map on the stream, as
 *    fluid_write does: the solve that follows gives the same bits either way.
 *  - Stream-ordered on the handle's stream; the calls return without synchronising, like
 *    fluid_render_canvas(..., dst_on_device = 1).  The handle's stream is non-blocking: work of other
 *    streams that uses the buffer must be complete before the call (sim.py's readField / writeField wait
 *    for it), and the caller must call fluid_sync before it reads `dst` or reuses `src`.
 * Refused with FLUID_ERR_INVALID, the buffer and every field untouched and the handle usable: n_floats !=
 * fluid_field_elems; a NULL buffer; a bad field id; pageable or pinned host memory; memory of another
 * device (managed memory of the handle's device is accepted); a buffer not 4-byte aligned; a buffer whose
 * [ptr, ptr + 4 * n_floats) overlaps the handle's field arena (such as fluid_device_ptr of a field);
 * slab handles (single-GPU entry points). */
int fluid_read_device(fluid_t* h, int field, float* dst, size_t n_floats);
int fluid_write_device(fluid_t* h, int field, const float* src, size_t n_floats);

/* End-to-end form of the pressure solve for callers that keep fields in HOST memory: uploads
 * divergence and pressure, runs clear + `iters` Jacobi sweeps, downloads pressure.  All three
 * copies are inside the call (this is what bench.py's `e2e` times).  On a single-GPU handle the grid
 * is cut into up to 16 row bands that are solved and downloaded while later bands still upload (same
 * bits as the one-piece solve, which grids too short for two bands take); pass pinned buffers
 * (fluid_host_alloc) for the copies to overlap.  The divergence and pressure fields of the handle
 * hold the uploaded divergence and the result afterwards. */
int fluid_pressure_solve_host(fluid_t* h, const float* div_host, float* pressure_host_inout,
                              int iters);

/* The consumer on the far side of the path ("next" row of SURVEY §8f):
 * render(target) of S:1296-1317 with config.BLOOM = config.SUNRAYS = false and TRANSPARENT = false —
 * drawColor(BACK_COLOR) (S:1319-1323) then drawDisplay (S:1331-1348, displayShaderSource S:549-612,
 * SHADING keyword when `shading` != 0) blended ONE / ONE_MINUS_SRC_ALPHA.  Writes width*height RGBA
 * floats (row 0 = bottom, not quantised to 8 bits: fluid_render_canvas draws the RGBA8 canvas) to host
 * memory.  back_* are BACK_COLOR / 255. */
int fluid_render(fluid_t* h, int width, int height, int shading, float back_r, float back_g,
                 float back_b, float* host_rgba, size_t n_floats);
/* On a slab handle every draw — fluid_render, fluid_render_keywords and fluid_render_postfx with any of the
 * eight keyword sets, fluid_capture, fluid_capture_device and fluid_render_canvas into host or device memory —
 * draws (and returns) only the band of target rows [*y0, *y1) that corresponds to the dye rows the rank owns,
 * after one refresh of the dye ghost rows the frame's taps reach; on a single GPU the band is the whole target.
 *  - Size: n_floats / n_bytes must be 4 * width * (*y1 - *y0).
 *  - Row order: the fp32 frame is bottom row first, so the bands concatenate in rank order.  Captures and
 *    canvases are top row first, each band too, so the whole image is the bands in REVERSE rank order.
 *  - With BLOOM or SUNRAYS the call is collective, like fluid_resize: every rank calls it with the same
 *    arguments.  Each rank prefilters its band of the bloom FBO and draws the sunrays mask on its own dye rows;
 *    the bands are all-gathered over NCCL (FLUID_STAT_GATHERS), and every rank then holds the bloom FBO and the
 *    sunrays texture one GPU computes, bit for bit.  host_bloom / host_sunrays, when given, receive them whole
 *    on every rank.
 *  - Every argument check comes before the first exchange, so a refused call is refused on every rank with
 *    nothing sent.  A frame whose taps need more dye ghost rows than the slab keeps (slab.py
 *    draw_ghost_rows) returns FLUID_ERR_HALO on every rank.
 *  - Slab handles are fp32 with LINEAR samplers: the half-storage, half-post-FX and NEAREST flags are refused
 *    by fluid_create_slab. */
int fluid_render_band(fluid_t* h, int height, int* y0, int* y1);

/* The same with the reference's desktop defaults SHADING = BLOOM = SUNRAYS = true (S:70-84):
 * applyBloom (S:1350-1394), applySunrays + blur (S:1396-1419), then the display shader with all three
 * keywords.  fx = the BLOOM_* / SUNRAYS_* keys of `config`; dither_rgb = the dw x dh RGB dithering
 * texture (LDR_LLL1_0.png / 255, first image row first, S:1128-1158).  host_bloom (bloom FBO,
 * getResolution(BLOOM_RESOLUTION) x RGBA) and host_sunrays (getResolution(SUNRAYS_RESOLUTION) x R)
 * may be NULL. */
typedef struct fluid_postfx {
    int32_t bloom_iterations;    /* S:77 default 8    */
    int32_t bloom_resolution;    /* S:78 default 256  */
    double bloom_intensity;      /* S:79 default 0.8  (double: knee / curve are derived in double like the JS) */
    double bloom_threshold;      /* S:80 default 0.6  */
    double bloom_soft_knee;      /* S:81 default 0.7  */
    int32_t sunrays_resolution;  /* S:83 default 196  */
    double sunrays_weight;       /* S:84 default 1.0  */
} fluid_postfx;
int fluid_render_postfx(fluid_t* h, int width, int height, const fluid_postfx* fx, const float* dither_rgb,
                        int dw, int dh, float back_r, float back_g, float back_b, float* host_rgba,
                        size_t n_floats, float* host_bloom, float* host_sunrays);

/* Any of the eight display variants: `keywords` is the set updateKeywords (S:1160-1166) builds from
 * config.SHADING / BLOOM / SUNRAYS, as FLUID_DISPLAY_* bits.  render() runs applyBloom only with BLOOM and
 * applySunrays + blur only with SUNRAYS (S:1297-1302), and binds the bloom, dithering and sunrays
 * textures only for the keywords that are on (S:1339-1346).  The background follows FLUID_BACKGROUND.
 *  - Without BLOOM and SUNRAYS this is fluid_render(…, keywords & FLUID_DISPLAY_SHADING, …): slab bands
 *    and half storage work, and fx / dither_rgb may be NULL.
 *  - With BLOOM or SUNRAYS the handle must have fp32 storage or FLUID_FLAG_HALF_POSTFX (FLUID_ERR_INVALID
 *    otherwise; a slab handle draws its band, fluid_render_band), fx is required, and dither_rgb only with BLOOM.  host_bloom / host_sunrays (as for
 *    fluid_render_postfx, may be NULL) are written only when their keyword is on.
 * The bloom FBO + pyramid, the sunrays FBOs and the dithering texture live in the handle: made on first
 * use, made again only when a size changes (FLUID_ERR_NOMEM if that fails; the handle stays usable), and
 * freed by fluid_destroy.  fluid_render_postfx is this call with all three keywords. */
#define FLUID_DISPLAY_SHADING 0x1u
#define FLUID_DISPLAY_BLOOM 0x2u
#define FLUID_DISPLAY_SUNRAYS 0x4u
int fluid_render_keywords(fluid_t* h, int width, int height, uint32_t keywords, const fluid_postfx* fx,
                          const float* dither_rgb, int dw, int dh, float back_r, float back_g, float back_b,
                          float* host_rgba, size_t n_floats, float* host_bloom, float* host_sunrays);

/* captureScreenshot() of S:287-299 up to the bytes toDataURL encodes (normalizeTexture S:309-327):
 * render(target) with `keywords` into a width x height RGBA half-float target — width x height is
 * getResolution(CAPTURE_RESOLUTION) of the canvas — returned as 4 * width * height bytes.
 *  - fp16 target: the background is drawColor(BACK_COLOR) stored in fp16 (back_* = BACK_COLOR / 255,
 *    rounded to nearest even); the display is blended over it ONE / ONE_MINUS_SRC_ALPHA in fp32 and every
 *    channel is then rounded to fp16 (nearest even, overflow to +-Inf).  transparent != 0: the display
 *    is stored bare with blending off (S:1307-1309).  The checkerboard is never drawn and
 *    FLUID_BACKGROUND is not consulted.
 *  - Post-FX: the bloom and sunrays FBOs keep the sizes render(null) gives them on a canvas_w x canvas_h
 *    drawing buffer (S:1012-1043), and share the handle's targets with fluid_render_keywords, so a
 *    capture on the canvas render() draws does not remake them.  texelSize and ditherScale use
 *    width x height (S:1332-1344).
 *  - Bytes: clamp01(v) * 255 truncated to uint8 (NaN gives 0), rows flipped so the TOP row comes
 *    first.  One device-to-host copy of n_bytes, then a stream sync.
 * Refused with FLUID_ERR_INVALID, the handle staying usable: unknown keyword bits; n_bytes !=
 * 4 * width * height; width, height, canvas_w or canvas_h < 1; BLOOM without dither_rgb; fx == NULL with
 * BLOOM or SUNRAYS; half-storage handles with BLOOM or SUNRAYS unless created with
 * FLUID_FLAG_HALF_POSTFX (without them half storage works, as in fluid_render).  A slab handle draws its band
 * (fluid_render_band): n_bytes = 4 * width * (y1 - y0). */
int fluid_capture(fluid_t* h, int width, int height, int canvas_w, int canvas_h, uint32_t keywords,
                  int transparent, const fluid_postfx* fx, const float* dither_rgb, int dw, int dh,
                  float back_r, float back_g, float back_b, uint8_t* host_rgba8, size_t n_bytes);
/* fluid_capture into the caller's device memory (for example a torch uint8 CUDA tensor): the same bytes,
 * stored by the display kernel itself, with the same launches and no device-to-host copy.  Stream-ordered
 * and returning without synchronising, with the ordering rules of fluid_read_device: work of other streams
 * that uses dst complete before the call, fluid_sync before reading dst.  Refused with FLUID_ERR_INVALID, dst
 * untouched and the handle usable: everything fluid_capture refuses, and dst as fluid_read_device refuses it
 * (NULL, host memory, another device, not 4-byte aligned, overlapping the field arena). */
int fluid_capture_device(fluid_t* h, int width, int height, int canvas_w, int canvas_h, uint32_t keywords,
                         int transparent, const fluid_postfx* fx, const float* dither_rgb, int dw, int dh,
                         float back_r, float back_g, float back_b, uint8_t* dst, size_t n_bytes);

/* render(null) of S:1296-1317 on the canvas: what a width x height drawing buffer holds after the frame.
 * The context is created with alpha: true (S:118-119), so the buffer is RGBA8 unsigned-normalised.  The
 * post-FX FBOs are sized from width x height as in fluid_render_keywords, and texelSize / ditherScale use
 * it (S:1332-1344).  FLUID_BACKGROUND is not consulted: on the screen blending is always on.
 * The rule, per channel, in fp32 with every operation rounded on its own (no contraction):
 *  - (c, a): the display fragment of fluid_render_keywords before any blend (FLUID_BACKGROUND 2).
 *  - clamp(x) = min(max(x, 0), 1): NaN gives 0, +inf gives 1.
 *    u8(x) = clamp(x) * 255 rounded to the nearest integer, ties to even (GLES 3.0 §2.1.6.1).
 *  - Destination byte d8: u8(back_*) (drawColor(BACK_COLOR), S:1319-1323); with transparent != 0,
 *    u8(v) of drawCheckerboard (S:1325-1329, v = mod(floor(uv.x * 25 * aspect) + floor(uv.y * 25), 2)
 *    * 0.1 + 0.8 in fp32, aspect = FLUID_ASPECT).  Alpha byte 255 either way.  d = d8 / 255.0f.
 *  - blendFunc(ONE, ONE_MINUS_SRC_ALPHA) (S:1305-1306) on a fixed-point buffer clamps first (GLES 3.0
 *    §4.1.7): out = clamp(c) + d * (1 - clamp(a)); alpha clamp(a) + 1 * (1 - clamp(a)).  Stored u8(out).
 *  - Rows top row first: the order of ImageData, putImageData and PNG (as fluid_capture).
 * Destination:
 *  - dst_on_device == 0: dst is host memory.  One device-to-host copy of n_bytes, then a stream sync.
 *  - dst_on_device != 0: dst is device or managed memory of the handle's device, 4-byte aligned (for
 *    example a torch uint8 CUDA tensor).  The display kernel stores into it directly; the call is
 *    stream-ordered and returns without synchronising, like fluid_step: fluid_sync before reading it.
 *    The handle's stream is non-blocking: work of other streams that uses dst must be complete first
 *    (sim.py's render_canvas waits for it).
 * Refused with FLUID_ERR_INVALID, dst untouched and the handle usable: n_bytes != 4 * width * height;
 * width or height < 1; unknown keyword bits; BLOOM without dither_rgb; fx == NULL with BLOOM or SUNRAYS;
 * half-storage handles with BLOOM or SUNRAYS unless created with FLUID_FLAG_HALF_POSTFX; dst_on_device with
 * host memory, memory of another device, a misaligned dst, or a dst overlapping the field arena.  A slab
 * handle draws its band (fluid_render_band): n_bytes = 4 * width * (y1 - y0). */
int fluid_render_canvas(fluid_t* h, int width, int height, uint32_t keywords, int transparent,
                        const fluid_postfx* fx, const float* dither_rgb, int dw, int dh,
                        float back_r, float back_g, float back_b,
                        uint8_t* dst, size_t n_bytes, int dst_on_device);

/* fluid_render_canvas and fluid_capture for a batch handle (fluid_create_batch): every member drawn through
 * the launches one draw of an ordinary handle makes, each launch one layer of blocks per member.
 *  - Member m's image is the bytes fluid_render_canvas, or fluid_capture / fluid_capture_device, give an
 *    ordinary handle of the batch's config whose dye equals member m's.  Keywords, sliders, background and
 *    sizes apply to every member (fluid_render_canvas_looks / fluid_capture_looks, below, give each image its
 *    own sliders and background).
 *  - dst is one C-contiguous (B, height, width, 4) array, member by member, each image top row first;
 *    n_bytes == B * 4 * width * height.
 *  - dst_on_device == 0: host memory, one device-to-host copy, then a stream sync.  dst_on_device != 0:
 *    device memory with the rules and ordering of fluid_render_canvas(..., dst_on_device = 1).
 *  - The post-FX targets hold B members each (the bloom FBO and pyramid, the sunrays FBOs), and the sunrays
 *    mask goes into every member's dye.write, as on an ordinary handle.  The dithering texture is shared.
 * Refused with FLUID_ERR_INVALID, dst untouched and the handle usable: an ordinary or slab handle; every
 * argument the single-handle call refuses; a device dst fluid_render_canvas refuses.  FLUID_ERR_NOMEM, the
 * handle usable: the post-FX targets of B members, or the host path's frame buffer of B images, do not fit. */
int fluid_render_canvas_batch(fluid_t* h, int width, int height, uint32_t keywords, int transparent,
                              const fluid_postfx* fx, const float* dither_rgb, int dw, int dh,
                              float back_r, float back_g, float back_b,
                              uint8_t* dst, size_t n_bytes, int dst_on_device);
int fluid_capture_batch(fluid_t* h, int width, int height, int canvas_w, int canvas_h, uint32_t keywords,
                        int transparent, const fluid_postfx* fx, const float* dither_rgb, int dw, int dh,
                        float back_r, float back_g, float back_b,
                        uint8_t* dst, size_t n_bytes, int dst_on_device);
/* fluid_render_canvas_batch and fluid_capture_batch for the n members a list names, with the list rules of the
 * member-subset calls (fluid_read_members): dst holds n images, n_bytes == n * 4 * width * height, and image k is
 * byte for byte image members[k] of the whole-batch call.  The same launches as one whole-batch draw, each n
 * layers of blocks deep, in the same post-FX targets (sized for B), so subset and whole draws alternate without
 * remaking them.  With SUNRAYS the mask goes into the listed members' dye.write only.  Refused with
 * FLUID_ERR_INVALID, dst untouched and the handle usable: everything the whole-batch call refuses (n_bytes checked
 * against n images) and every bad list. */
int fluid_render_canvas_members(fluid_t* h, int width, int height, uint32_t keywords, int transparent,
                                const fluid_postfx* fx, const float* dither_rgb, int dw, int dh,
                                float back_r, float back_g, float back_b,
                                uint8_t* dst, size_t n_bytes, int dst_on_device, const int32_t* members, int n);
int fluid_capture_members(fluid_t* h, int width, int height, int canvas_w, int canvas_h, uint32_t keywords,
                          int transparent, const fluid_postfx* fx, const float* dither_rgb, int dw, int dh,
                          float back_r, float back_g, float back_b,
                          uint8_t* dst, size_t n_bytes, int dst_on_device, const int32_t* members, int n);
/* The look of one image of a batch draw: the post-FX sliders of fluid_postfx and the background of the draw calls. */
typedef struct fluid_look {
    double bloom_intensity, bloom_threshold, bloom_soft_knee, sunrays_weight;  /* as in fluid_postfx */
    float back_r, back_g, back_b;                                              /* BACK_COLOR / 255   */
    int32_t transparent;                                                       /* as the draw calls'  */
} fluid_look;
/* Batch draws with a look per image: a contact sheet of one frame under many slider settings, or a dataset that
 * varies the look per sample, in the launches of one shared-look draw.
 *  - Which images: with members == NULL, n must be B and image k is member k (fluid_render_canvas_batch /
 *    fluid_capture_batch); otherwise the list follows the rules of the member-subset calls (fluid_read_members)
 *    and image k is member members[k] (fluid_render_canvas_members / fluid_capture_members).
 *  - Image k is byte for byte what fluid_render_canvas, or fluid_capture, give an ordinary handle of the batch's
 *    config whose dye equals its member's, called with fx's four sliders replaced by looks[k]'s and with
 *    looks[k]'s back_* and transparent.  fx still supplies BLOOM_ITERATIONS, BLOOM_RESOLUTION and
 *    SUNRAYS_RESOLUTION; keywords, the dithering texture, the canvas and the target sizes are shared.  As there,
 *    fx and the sliders are read only with BLOOM or SUNRAYS, and any slider or background value is taken.
 *  - The launches of the shared-look draw, plus one stream-ordered copy of the n images' looks, derived on the
 *    host (the prefilter's knee and curve in double, narrowed once), into a table of B looks the handle
 *    allocates at creation outside the field arena.  The caller may reuse `looks` as soon as the call returns.
 * Refused with FLUID_ERR_INVALID, dst untouched and the handle usable: everything the _batch / _members calls
 * refuse; members == NULL with n != B; looks == NULL with n > 0. */
int fluid_render_canvas_looks(fluid_t* h, int width, int height, uint32_t keywords, const fluid_postfx* fx,
                              const float* dither_rgb, int dw, int dh, const fluid_look* looks,
                              uint8_t* dst, size_t n_bytes, int dst_on_device, const int32_t* members, int n);
int fluid_capture_looks(fluid_t* h, int width, int height, int canvas_w, int canvas_h, uint32_t keywords,
                        const fluid_postfx* fx, const float* dither_rgb, int dw, int dh, const fluid_look* looks,
                        uint8_t* dst, size_t n_bytes, int dst_on_device, const int32_t* members, int n);

int fluid_sync(fluid_t* h);
int fluid_timing_last(fluid_t* h, fluid_timing* out);

/* Page-locked host memory for the buffers a binding hands to fluid_read / fluid_write /
 * fluid_pressure_solve_host / fluid_render (DMA without a staging copy).  The N-API shim wraps these in
 * external ArrayBuffers (readPixels' destination, S:301-307), so it needs no CUDA headers itself. */
void* fluid_host_alloc(size_t bytes);
void fluid_host_free(void* p);

/* Device time (ms) between two fluid_mark() calls on the handle's stream; slot is 0 or 1.
 * bench.py uses it because torch.cuda.Event cannot see this library's stream. */
int fluid_mark(fluid_t* h, int slot);
int fluid_elapsed_ms(fluid_t* h, float* ms);

/* Number of CUDA kernels this handle has launched since creation (graph replays count their
 * kernel nodes). */
uint64_t fluid_launch_count(fluid_t* h);

/* Counters since creation (no reference counterpart; bench.py and the tests read them). */
typedef enum fluid_stat_key {
    FLUID_STAT_LAUNCHES = 0,         /* == fluid_launch_count                                        */
    FLUID_STAT_JACOBI_LAUNCHES = 1,  /* Jacobi kernels only (graph replays count their kernel nodes)  */
    FLUID_STAT_HALO_LAUNCHES = 2,    /* halo_push / halo_wait kernels of the peer-memory transport    */
    FLUID_STAT_HALO_EXCHANGES = 3,   /* halo exchanges issued (either transport)                      */
    FLUID_STAT_GRAPH_CAPTURES = 4,   /* step() graphs captured + instantiated                         */
    FLUID_STAT_GRAPH_LAUNCHES = 5,   /* step() graphs replayed                                        */
    FLUID_STAT_HALO_TRANSPORT_P2P = 6, /* 1 when the peer-memory halo path is active                   */
    FLUID_STAT_CVD_STREAM_LAUNCHES = 7,      /* row-streaming curl-vorticity-divergence kernels executed */
    FLUID_STAT_GRADIENT_STREAM_LAUNCHES = 8, /* row-streaming gradientSubtract kernels executed          */
    FLUID_STAT_JACOBI_EXACT_STREAMS = 9,     /* blocked Jacobi warps that ran the un-contracted tail:
                                                tiny divergence, or inputs near FLT_MAX (synchronises)  */
    FLUID_STAT_ADVECT4_LAUNCHES = 10,        /* 4-cell advection kernels executed (velocity or dye, MANUAL
                                                or LINEAR filter): fp32, power-of-two, width >= 128     */
    FLUID_STAT_GATHERS = 11                  /* row-band all-gathers of a slab's post-FX: one per frame for
                                                BLOOM (with >= 2 pyramid levels), one for SUNRAYS        */
} fluid_stat_key;
uint64_t fluid_stat(fluid_t* h, int key);

/* Raw device pointer of a field's `.read` buffer (for zero-copy interop, e.g. torch.as_tensor
 * through __cuda_array_interface__); valid until the next call that swaps that field. */
void* fluid_device_ptr(fluid_t* h, int field);

const char* fluid_last_error(fluid_t* h); /* h may be NULL: last error of a failed create */
int fluid_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* FLUID_B200_H */
