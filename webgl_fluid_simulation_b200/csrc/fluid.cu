// fluid.cu — libfluid_b200: the C ABI of include/fluid.h over the sm_90a kernels.
//
// Host-side structure mirrors the reference's globals (script.js S:950-954): five fields, three of
// them DoubleFBO-style read/write pairs with swap() (S:1079-1106).  There is no CPU fallback:
// every entry point either launches CUDA kernels on the handle's stream or fails.
#include "../../include/fluid.h"

#include <cuda.h>            // CUtensorMap types only: the encoder is fetched through cudaGetDriverEntryPoint
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <type_traits>
#include <vector>

#include "jacobi.cuh"
#include "nccl_dl.h"
#include "passes.cuh"
#include "stream_passes.cuh"
#include "postfx.cuh"
#include "half_passes.cuh"
#include "members.cuh"

namespace {

thread_local std::string g_create_error;

// Byte offsets of every field in a handle's arena: both slots of the velocity / pressure / dye pairs,
// divergence, curl and the peer-memory flag words, and the arena's size.  Fixed-width: it travels in P2PBlob.
struct FieldLayout {
    uint64_t v[2], p[2], dye[2], div, curl, flags, bytes;
};

struct Pair {              // createDoubleFBO, S:1079-1106
    void* read = nullptr;
    void* write = nullptr;
    int par = 0;           // arena slot of .read (toggles with swap(); SPMD-identical on a slab)
    void swap() { std::swap(read, write); par ^= 1; }
    void place(char* arena, const uint64_t (&slot)[2]) { read = arena + slot[par]; write = arena + slot[par ^ 1]; }
};

// Row ownership and ghost-zone heights of a handle (slab_geometry).  Single GPU: all rows, no ghost rows.
struct SlabGeometry {
    int G = 0, Gd = 0;               // ghost rows kept below and above the owned rows (sim / dye)
    int row0 = 0, row1 = 0;          // owned sim rows  [row0, row1)
    int drow0 = 0, drow1 = 0;        // owned dye rows  [drow0, drow1)
    int roff = 0, droff = 0;         // global row index of local row 0  (row0 - G, drow0 - Gd)
    int lrows() const { return row1 - row0 + 2 * G; }
    int ldrows() const { return drow1 - drow0 + 2 * Gd; }
};

// Kernel launches of a handle by kind (fluid_stat).  A step graph holds the counts of the step it captured
// and adds them at every replay.
struct LaunchCounts {
    uint64_t all = 0;
    uint64_t jacobi = 0;            // Jacobi kernels only (FLUID_STAT_JACOBI_LAUNCHES)
    uint64_t halo = 0;              // halo_push / halo_wait kernels of the peer-memory transport
    uint64_t cvd_stream = 0;        // cvd_stream_kernel / gradient_stream_kernel (FLUID_STAT_*_STREAM_LAUNCHES):
    uint64_t gradient_stream = 0;   // which of a pass's kernels the grid size picked
    uint64_t advect4 = 0;           // 4-cell advection kernels, either filter (FLUID_STAT_ADVECT4_LAUNCHES)
    LaunchCounts& operator+=(const LaunchCounts& o) {
        all += o.all; jacobi += o.jacobi; halo += o.halo;
        cvd_stream += o.cvd_stream; gradient_stream += o.gradient_stream; advect4 += o.advect4;
        return *this;
    }
    LaunchCounts operator-(const LaunchCounts& o) const {
        LaunchCounts d = *this;
        d.all -= o.all; d.jacobi -= o.jacobi; d.halo -= o.halo;
        d.cvd_stream -= o.cvd_stream; d.gradient_stream -= o.gradient_stream; d.advect4 -= o.advect4;
        return d;
    }
};

}  // namespace

struct fluid : SlabGeometry {
    fluid_config cfg{};
    int device = 0;
    int sm_count = 132;
    cudaStream_t stream = nullptr;
    cudaEvent_t mark[2] = {nullptr, nullptr};
    cudaEvent_t tev[8] = {};
    Pair velocity, dye, pressure;    // float2 / float4 / float
    float* divergence = nullptr;
    float* curl = nullptr;
    int* halo_flag = nullptr;        // device flag set by advection when a tap leaves the ghost zone
    unsigned long long* exact_streams = nullptr;   // device counter: blocked Jacobi warps that ran the exact tail
    LaunchCounts launches;
    uint64_t div_epoch = 1, div_sent_epoch = 0;   // slab: the divergence ghost rows are re-sent only after divergence was rewritten
    int div_sent_rows = 0;
    bool capturing = false;                // inside the stream capture of a step graph
    bool half = false;                     // FLUID_FLAG_HALF_STORAGE: fields are fp16 (half_passes.cuh), single GPU only
    bool half_fx = false;                  // FLUID_FLAG_HALF_POSTFX: the bloom and sunrays targets are fp16, single GPU only
    bool nearest = false;                  // FLUID_FLAG_NEAREST_FILTERING: display, post-FX and resize sample NEAREST, single GPU only
    bool linear_adv = false;               // FLUID_FLAG_LINEAR_ADVECTION: advection samples LINEAR (passes.cuh LinearSampler), single GPU only
    // fluid_create_batch: `members` simulations of one size and config.  Every slot of the arena holds them as a
    // dense (B, H, W) array, the tiny map one region per member, and the step kernels take the member as blockIdx.z
    bool batch = false;
    int members = 1;
    float* scratch = nullptr;              // half mode: fp32 staging of fluid_read / fluid_write / render
    size_t scratch_floats = 0;
    int* splat_scratch = nullptr;          // fluid_splats_batch_device: grouped order, per-member offsets, staged records
    size_t splat_scratch_bytes = 0;        // (outside the arena, grown on demand)
    // step()'s dt lives in device memory: one graph serves every dt.  On a batch handle this is the member table
    // (jacobi.cuh), whose first row is every member's dt; member_host is its host copy, and member_radius_d each
    // member's SPLAT_RADIUS as the JS double it is (MP_RADIUS is correctRadius of it and aspect_d)
    float* dt_dev = nullptr;
    std::vector<float> member_host;
    std::vector<double> member_radius_d;
    int* member_list = nullptr;            // the member-subset calls' list (fluid_read_members ...): B int32, outside the arena
    fk::ImageLook* look_table = nullptr;   // the looks of fluid_render_canvas_looks / fluid_capture_looks: B entries, outside the arena
    unsigned char* tiny_map = nullptr;     // where divergence has 0 < |d| < 2^-123 (jacobi.cuh): 1 byte per 128x32 cells, GLOBAL rows
    size_t tiny_map_bytes = 0;
    // 2-D tensor maps the blocked Jacobi kernel stages through: m[k] maps pressure slot k and divergence
    struct Tmaps { fk::TmapPair m[2]; } tmaps;
    double splat_radius_d = 0.25;          // config.SPLAT_RADIUS and the canvas aspect as the JS doubles they are
    double aspect_d = 1.0;                 // (correctRadius S:1457-1462 is double arithmetic, narrowed once)
    int background = 0;                    // FLUID_BACKGROUND: what render() draws the display over (0 colour, 1 checkerboard, 2 none)
    fluid_timing timing{};
    bool have_timing = false;
    std::string err;

    // every field lives in ONE allocation, laid out by `layout`: a single CUDA IPC handle maps all that a
    // slab neighbour may write into
    char* arena = nullptr;
    FieldLayout layout{};
    // ---- row-slab decomposition (SURVEY §8e; the geometry is the SlabGeometry base).  Single GPU: rank 0 of 1
    int rank = 0, world = 1;
    ncdl::ncclComm_t comm = nullptr;
    bool v_ghost_valid = true;       // velocity valid on owned rows +-3 (what the next step needs)
    uint64_t halo_groups = 0;        // halo exchanges issued (diagnostics)
    uint64_t gathers = 0;            // row-band all-gathers issued (post-FX on slabs, halo.cuh gather_bands)
    // ---- peer-memory halo path (fluid_p2p_export / fluid_p2p_connect) -------------------------------
    struct Peer {
        bool present = false;
        char* base = nullptr;        // neighbour's arena mapped here through CUDA IPC
        int roff = 0, droff = 0;     // neighbour's local-row-0 global row indices
        FieldLayout layout{};
    } peer[2];                       // [0] = rank-1 (below), [1] = rank+1 (above)
    bool p2p = false;
    uint32_t p2p_seq = 0;
    // fluid_pressure_solve_host pipelined over row bands (single GPU): copy streams, per-band events and the
    // band-private ping-pong rows of the intermediate launches
    struct HostPipe {
        cudaStream_t up = nullptr, down = nullptr;
        cudaEvent_t ev_start = nullptr, ev_up[16] = {}, ev_done[16] = {};
        float* s[2] = {nullptr, nullptr};
        size_t s_floats = 0;
    } hp;
    // divergence ghost rows of the exchange about to be issued: the peer-memory wait kernel scans them (halo.cuh)
    struct { const float* div; unsigned char* map; int W, row_off, lo0, hi0, lo1, hi1; } scan{};
    bool scan_pending = false;
    // ---- step() as a CUDA graph (single GPU): one instantiated graph per (dt, config scalars, parity)
    struct StepGraph {
        cudaGraphExec_t exec = nullptr;
        int flip_v = 0, flip_p = 0, flip_dye = 0;
        LaunchCounts launches;       // what one replay launches
    };
    std::map<std::string, StepGraph> graphs;
    uint64_t graph_launches = 0, graph_captures = 0;
    float4* frame = nullptr;         // render target of fluid_render (w x h RGBA fp32), grown on demand
    size_t frame_cells = 0;
    // post-FX targets of render() (initBloomFramebuffers / initSunraysFramebuffers, S:1012-1043): made on
    // first use, made again only when a size changes, kept across frames like the reference's FBOs
    struct PostFxTargets {
        void* bloom = nullptr;       // the bloom FBO, then its `levels` pyramid levels, in one allocation (T4 texels)
        int bw = 0, bh = 0, levels = 0;
        void* sun = nullptr;         // sunrays, then sunraysTemp (sw x sh T1 texels each)
        int sw = 0, sh = 0;
        float* dither = nullptr;     // dw x dh RGB dithering texture, uploaded every BLOOM frame
        int dw = 0, dh = 0;
        float* mask = nullptr;       // slab SUNRAYS: the mask's alpha, Wd x Hd, every rank's band gathered
        int mw = 0, mh = 0;
    } pfx;
    bool slab() const { return world > 1; }
};

namespace {

using namespace fk;

void drop_graphs(fluid_t* h) {
    if (!h->graphs.empty() && h->stream) cudaStreamSynchronize(h->stream);   // an exec may still be in flight
    for (auto& kv : h->graphs) if (kv.second.exec) cudaGraphExecDestroy(kv.second.exec);
    h->graphs.clear();
}

int fail(fluid_t* h, int code, const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    if (h) h->err = buf; else g_create_error = buf;
    return code;
}

#define CU(call)                                                                              \
    do {                                                                                      \
        cudaError_t e_ = (call);                                                              \
        if (e_ != cudaSuccess)                                                                \
            return fail(h, FLUID_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), \
                        __FILE__, __LINE__);                                                  \
    } while (0)

inline bool is_pow2(int n) { return n > 0 && (n & (n - 1)) == 0; }

// z: one layer of blocks per member of a batch handle (the kernels take the member from blockIdx.z)
inline dim3 grid2d(int W, int rows, dim3 b, int z = 1) {
    return dim3((W + b.x - 1) / b.x, (rows + b.y - 1) / b.y, z);
}

Grid sim_grid(const fluid_t* h) { return Grid{h->cfg.sim_w, h->cfg.sim_h, h->roff, h->row0, h->row1}; }
Grid dye_grid(const fluid_t* h) { return Grid{h->cfg.dye_w, h->cfg.dye_h, h->droff, h->drow0, h->drow1}; }
// same grid, producing rows [row0-e, row1+e) clipped to the domain (redundant ghost-zone compute)
Grid sim_grid_ext(const fluid_t* h, int e) {
    Grid g = sim_grid(h);
    g.j_lo = std::max(h->row0 - e, 0); g.j_hi = std::min(h->row1 + e, h->cfg.sim_h);
    return g;
}

// LOCAL cell counts (owned + ghost rows): what the device buffers hold
size_t sim_cells(const fluid_t* h) { return (size_t)h->cfg.sim_w * h->lrows(); }
size_t dye_cells(const fluid_t* h) { return (size_t)h->cfg.dye_w * h->ldrows(); }

int check_launch(fluid_t* h, const char* what, int n = 1) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess)
        return fail(h, FLUID_ERR_CUDA, "launch of %s failed: %s", what, cudaGetErrorString(e));
    h->launches.all += n;
    return FLUID_OK;
}

// Row k of a batch handle's member table from its host copy: a stream-ordered upload from pageable memory (the
// driver stages it before returning), issued outside any capture like set_dt's.
int upload_member_row(fluid_t* h, int k) {
    const size_t B = h->members;
    CU(cudaMemcpyAsync(h->dt_dev + k * B, h->member_host.data() + k * B, B * sizeof(float), cudaMemcpyHostToDevice, h->stream));
    return FLUID_OK;
}

// dt of the current step()/pass, in device memory.  Stream-ordered 4-byte upload from a pageable
// host word (the driver stages it before returning), issued OUTSIDE any capture: an instantiated
// step graph therefore never bakes dt in, and the reference's calcDeltaTime() (S:1188-1194, a new
// dt every frame) replays the same graph.  A batch handle: every member's dt.
int set_dt(fluid_t* h, float dt) {
    if (h->batch) {
        std::fill_n(h->member_host.begin() + MP_DT * h->members, h->members, dt);
        return upload_member_row(h, MP_DT);
    }
    CU(cudaMemcpyAsync(h->dt_dev, &dt, sizeof(float), cudaMemcpyHostToDevice, h->stream));
    return FLUID_OK;
}

// correctRadius(config.SPLAT_RADIUS / 100.0), S:1457-1462: JS double arithmetic, narrowed by gl.uniform1f
float splat_radius(double splat_radius_d, double aspect_d) {
    double rad = splat_radius_d / 100.0;
    if (aspect_d > 1.0) rad *= aspect_d;
    return (float)rad;
}

// the member table row of a key a batch member can hold a value of its own for; -1 for every other key
int member_row(int key) {
    switch (key) {
        case FLUID_DENSITY_DISSIPATION: return MP_DENSITY_DISSIPATION;
        case FLUID_VELOCITY_DISSIPATION: return MP_VELOCITY_DISSIPATION;
        case FLUID_PRESSURE: return MP_PRESSURE;
        case FLUID_CURL: return MP_CURL;
        case FLUID_SPLAT_RADIUS: return MP_RADIUS;
    }
    return -1;
}
// member m's value of row `row` in the host copy, narrowed as fluid_set_param_f64 narrows it (upload_member_row
// makes it the device's)
void set_member_value(fluid_t* h, int row, int m, double v) {
    const size_t at = (size_t)row * h->members + m;
    if (row == MP_RADIUS) {
        h->member_radius_d[m] = v;
        h->member_host[at] = splat_radius(v, h->aspect_d);
    } else {
        h->member_host[at] = (float)v;
    }
}
// what fluid_get_param returns for member m's value of row `row`
float member_value(const fluid_t* h, int row, int m) {
    return row == MP_RADIUS ? (float)h->member_radius_d[m] : h->member_host[(size_t)row * h->members + m];
}

// A batch handle's member table, every member holding the config's values and dt 0.  Outside the field arena,
// so the arena layout is an ordinary handle's; FLUID_ERR_NOMEM when it does not fit.
int alloc_member_table(fluid_t* h) {
    const size_t B = h->members;
    if (cudaMalloc((void**)&h->dt_dev, MP_KEYS * B * sizeof(float)) != cudaSuccess) {
        cudaGetLastError();                      // not sticky: keep it out of the next launch check
        return fail(h, FLUID_ERR_NOMEM, "out of device memory for the member table of %d members", h->members);
    }
    h->member_host.assign(MP_KEYS * B, 0.0f);
    h->member_radius_d.assign(B, 0.0);
    const fluid_config& c = h->cfg;
    const double init[][2] = {{FLUID_DENSITY_DISSIPATION, c.density_dissipation}, {FLUID_VELOCITY_DISSIPATION, c.velocity_dissipation},
                              {FLUID_PRESSURE, c.pressure}, {FLUID_CURL, c.curl}, {FLUID_SPLAT_RADIUS, h->splat_radius_d}};
    for (const auto& kv : init)
        for (size_t m = 0; m < B; ++m) set_member_value(h, member_row((int)kv[0]), (int)m, kv[1]);
    CU(cudaMemcpyAsync(h->dt_dev, h->member_host.data(), MP_KEYS * B * sizeof(float), cudaMemcpyHostToDevice, h->stream));
    return FLUID_OK;
}

#include "halo.cuh"

// bytes per cell of each field: fp32 storage (float2 / float4 / float) or half storage (S:986-1006)
inline size_t vbytes(const fluid_t* h) { return h->half ? 4 : 8; }
inline size_t dbytes(const fluid_t* h) { return h->half ? 8 : 16; }
inline size_t sbytes(const fluid_t* h) { return h->half ? 2 : 4; }
int need_scratch(fluid_t* h, size_t floats) {
    if (floats <= h->scratch_floats) return FLUID_OK;
    CU(cudaStreamSynchronize(h->stream));
    cudaFree(h->scratch); h->scratch = nullptr; h->scratch_floats = 0;
    CU(cudaMalloc((void**)&h->scratch, floats * sizeof(float)));
    h->scratch_floats = floats;
    return FLUID_OK;
}
// f(StoreF32{}) or f(hs::StoreHalf{}): a launch written once, instantiated for the handle's storage format
template <class F>
auto with_storage(const fluid_t* h, F&& f) {
    return h->half ? f(hs::StoreHalf{}) : f(StoreF32{});
}

// Which advection kernel a pass runs, for the handle's filter policy F and storage S (passes.cuh), when
// the sim grid and the advected grid are powers of two (p2) and the advected grid is w cells wide:
//   4-cell    fp32 storage, p2, w >= 128 and no FLUID_FLAG_TILED_PASSES.  SLAB only on slab handles, which are
//             always MANUAL.
//   one-cell  otherwise; the POW2 form when p2, except for MANUAL half storage (pow2_form), which runs the
//             !POW2 forms: the reference's coordinates and bilerp on every sample.
// The cell-centre velocity sample without a coordinate (centre taps), and SAME (dye grid == sim grid) with it,
// only with F::kOwnTexel.
bool advect4_runs(const fluid_t* h, bool p2, int w) {
    return p2 && !h->half && w >= 128 && !(h->cfg.flags & FLUID_FLAG_TILED_PASSES);
}
template <class S, class F>
constexpr bool pow2_form = std::is_same<S, StoreF32>::value || !F::kOwnTexel;
// f(LinearSampler{}) or f(ManualBilerp{}): an advection launch written once for the handle's filter policy
template <class Fn>
auto with_filter(const fluid_t* h, Fn&& f) {
    return h->linear_adv ? f(LinearSampler{}) : f(ManualBilerp{});
}

// ---- the tiny-divergence map (jacobi.cuh): one byte per 128 x 32 cells of the GLOBAL grid -------------
int alloc_tiny_map(fluid_t* h) {
    cudaFree(h->tiny_map); h->tiny_map = nullptr;
    h->tiny_map_bytes = (size_t)tiny_map_w(h->cfg.sim_w) * tiny_map_h(h->cfg.sim_h) * h->members;
    CU(cudaMalloc((void**)&h->tiny_map, h->tiny_map_bytes));
    CU(cudaMemsetAsync(h->tiny_map, 0, h->tiny_map_bytes, h->stream));
    return FLUID_OK;
}
// before a pass that recomputes divergence everywhere (the pass then flags cells itself)
int clear_tiny_map(fluid_t* h) {
    CU(cudaMemsetAsync(h->tiny_map, 0, h->tiny_map_bytes, h->stream));
    ++h->div_epoch;                       // every writer of divergence comes through here
    return FLUID_OK;
}
// divergence rows [j_lo, j_hi) came from outside (host write, neighbour rank): flag their cells.  A batch
// handle scans those rows of every member into the member's region of the map.
int scan_tiny(fluid_t* h, int j_lo, int j_hi) {
    if (j_hi <= j_lo) return FLUID_OK;
    dim3 b(256), g((h->cfg.sim_w + 255) / 256, j_hi - j_lo);
    const size_t region = h->tiny_map_bytes / h->members;
    for (int m = 0; m < h->members; ++m)
        tiny_scan_kernel<<<g, b, 0, h->stream>>>(h->divergence + m * sim_cells(h), h->tiny_map + m * region, h->cfg.sim_w,
                                                 h->roff, j_lo, j_hi);
    return check_launch(h, "tiny_scan_kernel", h->members);
}

// ---- Jacobi dispatch -----------------------------------------------------------------------------

// Temporal-block depths, at most KMAX (slab.py mirrors both): the depth-13 instantiation fits 255
// registers without spills.  A single-GPU in-place solve defaults to KMAX: on an H100 at 4096^2 x 50 4
// launches of 13 / 12 sweeps take 0.500 ms per solve and 5 launches of 10 take 0.524 (80 GB HBM3 card, 400 W
// power limit; DESIGN §5).  Iteration counts that split into the same number of launches either way (20, 30,
// 40) keep depth 10 launches.  Row slabs and the banded host solve default to K_DEFAULT, the depth they have
// been run at.
constexpr int KMAX = 13;
constexpr int K_DEFAULT = 10;

bool tb_eligible(const fluid_t* h) {
    return !h->half && (h->cfg.sim_w % 4 == 0) && h->cfg.sim_w >= 16 && h->cfg.sim_h >= 2;
}

// depth of a solve (slab.py SlabPlan.block, host_bands): config.JACOBI_BLOCK or the default, and on a slab
// below its ghost rows.  banded: the bands of fluid_pressure_solve_host.
int block_depth(const fluid_t* h, bool banded) {
    const int kb = std::min(h->cfg.jacobi_block > 0 ? h->cfg.jacobi_block : (h->slab() || banded ? K_DEFAULT : KMAX), KMAX);
    return h->slab() ? std::max(1, std::min(kb, h->G - 1)) : kb;
}

// a solve of depth kb runs the blocked kernel; otherwise one sweep per launch
bool blocked(const fluid_t* h, int kb) {
    return tb_eligible(h) && !(h->cfg.flags & FLUID_FLAG_NAIVE_JACOBI) && kb != 1;
}

// Balanced split of iters > 0 sweeps into ceil(iters/kb) launches (slab.py jacobi_launches): launch k
// runs depth(k) sweeps, and after(k) sweeps of the solve follow it.
struct JacobiPlan {
    int n, base, extra;
    JacobiPlan(int iters, int kb) : n((iters + kb - 1) / kb), base(iters / n), extra(iters % n) {}
    int depth(int k) const { return base + (k < extra ? 1 : 0); }
    int after(int k) const { return (n - 1 - k) * base + std::max(extra - 1 - k, 0); }
};

// JacobiArgs of a launch whose local row 0 is global row row_off; the caller sets pin, pout and the rows
JacobiArgs jacobi_args(const fluid_t* h, const float* div, int row_off) {
    JacobiArgs a{};
    a.div = div; a.row_off = row_off; a.W = h->cfg.sim_w; a.H = h->cfg.sim_h;
    a.scale = h->cfg.pressure;
    a.err = h->halo_flag; a.tiny_map = h->tiny_map; a.exact_streams = h->exact_streams;
    return a;
}

// cuTensorMapEncodeTiled through the runtime (no link-time dependency on libcuda)
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_tiled_fn() {
    static EncodeTiledFn fn = []() -> EncodeTiledFn {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
            q != cudaDriverEntryPointSuccess) { cudaGetLastError(); return nullptr; }
        return (EncodeTiledFn)p;
    }();
    return fn;
}

// fp32 field of `rows` x W from `base` as a 2-D tensor map (`tm`: TmapPair::p or ::d); box = TB_BOX columns
// x 3 rows, no swizzle, out-of-range elements read as zero (the blocked kernel never lets them reach a
// valid output)
int encode_rows_map(fluid_t* h, unsigned char (&tm)[128], const void* base, int W, int rows) {
    static_assert(sizeof(CUtensorMap) == sizeof(tm), "TmapPair holds CUtensorMap images");
    EncodeTiledFn enc = encode_tiled_fn();
    const cuuint64_t dims[2] = {(cuuint64_t)W, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)W * sizeof(float)};
    const cuuint32_t box[2] = {TB_BOX, 3};
    const cuuint32_t estr[2] = {1, 1};
    if (!enc || enc(reinterpret_cast<CUtensorMap*>(tm), CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(base), dims,
                    strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
        return fail(h, FLUID_ERR_CUDA, "cuTensorMapEncodeTiled of a %d x %d fp32 field failed", W, rows);
    return FLUID_OK;
}

// The B members of a batch handle's fp32 field at `base` as a 3-D tensor map (W, H, B); box = TB_BOX columns x
// 3 rows x 1 member, so that a box reaching past a member's first or last row reads zeros, as on a 2-D map.
int encode_members_map(fluid_t* h, unsigned char (&tm)[128], const void* base, int W, int H, int B) {
    EncodeTiledFn enc = encode_tiled_fn();
    const cuuint64_t dims[3] = {(cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)B};
    const cuuint64_t strides[2] = {(cuuint64_t)W * sizeof(float), (cuuint64_t)W * H * sizeof(float)};
    const cuuint32_t box[3] = {TB_BOX, 3, 1};
    const cuuint32_t estr[3] = {1, 1, 1};
    if (!enc || enc(reinterpret_cast<CUtensorMap*>(tm), CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<void*>(base), dims,
                    strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                    CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
        return fail(h, FLUID_ERR_CUDA, "cuTensorMapEncodeTiled of %d members of a %d x %d fp32 field failed", B, W, H);
    return FLUID_OK;
}

// (re)build the tensor maps after the pressure / divergence buffers were allocated.  The blocked kernel
// stages only through them, so a handle that runs it cannot do without.
int build_tmaps(fluid_t* h) {
    h->tmaps = {};
    if (!tb_eligible(h)) return FLUID_OK;
    const int W = h->cfg.sim_w;
    for (int k = 0; k < 2; ++k) {
        fk::TmapPair& m = h->tmaps.m[k];
        const void* p = h->arena + h->layout.p[k];
        int rc = h->batch ? encode_members_map(h, m.p, p, W, h->cfg.sim_h, h->members) : encode_rows_map(h, m.p, p, W, h->lrows());
        if (!rc) rc = h->batch ? encode_members_map(h, m.d, h->divergence, W, h->cfg.sim_h, h->members)
                               : encode_rows_map(h, m.d, h->divergence, W, h->lrows());
        if (rc) return rc;
    }
    return FLUID_OK;
}

// kTb[K - 1]: jacobi_tb_kernel<K, SCALE> as kernel[SCALE], its batch-handle form as batch[SCALE], and the TB<K>
// constants their launches need
typedef void (*TbKernel)(JacobiArgs, TmapPair, const float*);
struct TbEntry {
    TbKernel kernel[2];
    int valid, u, smem;
    TbKernel batch[2];
};
template <int K>
constexpr TbEntry tb_entry() {
    return {{jacobi_tb_kernel<K, false>, jacobi_tb_kernel<K, true>}, TB<K>::VALID, TB<K>::U, TB<K>::SMEM,
            {jacobi_tb_kernel<K, false, true>, jacobi_tb_kernel<K, true, true>}};
}
static const TbEntry kTb[KMAX] = {tb_entry<1>(), tb_entry<2>(), tb_entry<3>(), tb_entry<4>(), tb_entry<5>(),
                                  tb_entry<6>(), tb_entry<7>(), tb_entry<8>(), tb_entry<9>(), tb_entry<10>(),
                                  tb_entry<11>(), tb_entry<12>(), tb_entry<13>()};

// rows per warp stream of a depth-K launch: enough chunks that every SM holds its full complement of
// resident warps (single wave) across the members x windows x chunks, rounded so that a stream's step count
// R + 2K is a multiple of the unroll U.  Both SCALE instantiations are sized from the occupancy of the
// SCALE = false one.
int tb_rows(const fluid_t* h, const TbEntry& e, int K, int W, int rows) {
    const int nxw = (W + e.valid - 1) / e.valid * h->members;     // windows of all members
    int occ = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, h->batch ? e.batch[0] : e.kernel[0], 32, e.smem);
    if (occ < 1) occ = 1;
    const int resident_warps = std::max(nxw, h->sm_count * occ);
    const int nch = std::max(1, resident_warps / nxw);
    int r = (rows + nch - 1) / nch;
    r = std::max(r, 4 * K);                 // keep the 2K warm-up rows a bounded fraction
    // round R up so that (R + 2K) % U == 0: no partially wasted unrolled block
    const int rem = (r + 2 * K) % e.u;
    if (rem) r += e.u - rem;
    return std::min(r, rows);
}

// One blocked launch of depth K, global rows [a.out_lo, a.out_hi); `maps` describe a.pin and a.div from their
// local row 0.  scale: the clear pass fused into the loads.  chained: programmatic dependent launch behind the
// previous kernel on the stream (jacobi.cuh), never while a graph is being captured.
int launch_tb(fluid_t* h, int K, bool scale, bool chained, JacobiArgs a, const TmapPair& maps) {
    if (K < 1 || K > KMAX) return fail(h, FLUID_ERR_INVALID, "temporal block depth %d out of range", K);
    const TbEntry& e = kTb[K - 1];
    a.rows_per_chunk = tb_rows(h, e, K, a.W, a.out_hi - a.out_lo);
    const int nxw = (a.W + e.valid - 1) / e.valid;
    const int nch = (a.out_hi - a.out_lo + a.rows_per_chunk - 1) / a.rows_per_chunk;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cudaLaunchConfig_t lc{};
    lc.gridDim = dim3(nxw * nch, 1, h->members); lc.blockDim = dim3(32); lc.stream = h->stream;   // one warp per CTA
    lc.attrs = attr; lc.numAttrs = (chained && !h->capturing) ? 1 : 0;
    lc.dynamicSmemBytes = e.smem;
    const float* member_table = h->batch ? h->dt_dev : nullptr;
    cudaLaunchKernelEx(&lc, h->batch ? e.batch[scale] : e.kernel[scale], a, maps, member_table);
    ++h->launches.jacobi;
    return check_launch(h, "jacobi_tb_kernel");
}

// One sweep without temporal blocking, rows [a.out_lo, a.out_hi).  scale: the clear pass fused into the
// loads (never in half storage, which clears in a launch of its own).
int launch_sweep(fluid_t* h, const JacobiArgs& a, bool scale) {
    const int W = a.W, H = a.H;
    const char* what = "jacobi_sweep_kernel";
    if (tb_eligible(h)) {
        dim3 b(32, 8);
        dim3 g((W / 4 + b.x - 1) / b.x, (a.out_hi - a.out_lo + b.y - 1) / b.y);
        if (scale) jacobi_sweep_kernel<true><<<g, b, 0, h->stream>>>(a);
        else jacobi_sweep_kernel<false><<<g, b, 0, h->stream>>>(a);
    } else if (h->half && W % 8 == 0 && W >= 64) {
        dim3 b(32, 8), g((W / 8 + 31) / 32, (H + 7) / 8);
        hs::jacobi8_kernel<<<g, b, 0, h->stream>>>((const hs::h1*)a.pin, (const hs::h1*)a.div, (hs::h1*)a.pout, W, H);
        what = "hs::jacobi8_kernel";
    } else {
        dim3 b(64, 4);
        with_storage(h, [&](auto s) {
            jacobi_scalar_kernel<decltype(s)><<<grid2d(W, a.out_hi - a.out_lo, b), b, 0, h->stream>>>(a, scale);
        });
        what = "jacobi_scalar_kernel";
    }
    ++h->launches.jacobi;
    return check_launch(h, what);
}

// `iters` sweeps reading pressure.read, result in pressure.read (swaps like S:1265).
// scale_first: fold p <- PRESSURE*p (clear pass) into the first sweep's loads.
// On a slab: before a launch of depth K the neighbours' K rows of p are exchanged (K+1 for the last
// launch, which also produces one row beyond each slab edge so that gradientSubtract needs no
// message of its own); divergence ghosts are exchanged once per solve (it is constant in the loop).
int run_jacobi(fluid_t* h, int iters, bool scale_first, int* launches_out) {
    int nl = 0;
    const int W = h->cfg.sim_w, H = h->cfg.sim_h;
    // clear pass alone (owned + ghost rows; ghosts are refreshed before use anyway).  Half storage always
    // clears in a launch of its own: the reference rounds the cleared field to fp16 before the first sweep.
    if (scale_first && (iters <= 0 || h->half)) {
        const size_t n = sim_cells(h) * h->members;
        int rc;
        if (h->batch) {                                  // each member by its own PRESSURE
            const size_t nm = sim_cells(h);
            scale_members_kernel<<<dim3((unsigned)((nm + 255) / 256), 1, h->members), 256, 0, h->stream>>>(
                (const float*)h->pressure.read, (float*)h->pressure.write, nm, h->dt_dev);
            rc = check_launch(h, "scale_members_kernel");
        } else {
            rc = with_storage(h, [&](auto s) {
                using S = decltype(s);
                scale_kernel<S><<<(unsigned)((n + 255) / 256), 256, 0, h->stream>>>(
                    (const typename S::T1*)h->pressure.read, (typename S::T1*)h->pressure.write, n, h->cfg.pressure);
                return check_launch(h, "scale_kernel");
            });
        }
        if (rc) return rc;
        h->pressure.swap(); ++nl;
        scale_first = false;
    }
    if (iters <= 0) {
        if (launches_out) *launches_out = nl;
        return FLUID_OK;
    }
    const int kb = block_depth(h, false);
    const bool tb = h->batch || blocked(h, kb);          // a batch runs the blocked kernel at every depth, 1 included
    const JacobiPlan plan(iters, tb ? kb : 1);
    // Slab halos.  Communication-avoiding form (deep): ONE group per solve carries iters+1 rows of
    // pressure and iters rows of divergence; launch i then produces owned rows +- (sweeps still to
    // come + 1), so later launches find their input already there (~1 % redundant rows instead of
    // one latency-bound message per launch).  If the ghost zone is too thin for that (iterations
    // raised after creation) fall back to one K-row message per launch.
    const bool deep = h->slab() && (iters + 1 <= h->G) && (iters + 1 <= h->row1 - h->row0);
    if (h->slab()) {
        if (deep) {
            // divergence is constant during a solve and often across solves (a host that iterates the solve on
            // one right-hand side, bench.py's loop): its ghost rows — and their tiny-value flags — are still in
            // place unless some pass rewrote divergence since they were last received (SPMD-identical decision)
            const bool send_div = h->div_sent_epoch != h->div_epoch || h->div_sent_rows < iters;
            const HaloItem it[2] = {{HB_PRESSURE, iters + 1}, {HB_DIVERGENCE, iters}};
            // the neighbours' divergence rows get their tiny values flagged like the local producers do:
            // inside the wait kernel on the peer-memory path, by a scan kernel after the NCCL group
            h->scan.div = h->divergence; h->scan.map = h->tiny_map; h->scan.W = W; h->scan.row_off = h->roff;
            h->scan.lo0 = std::max(h->row0 - iters, 0); h->scan.hi0 = h->row0;
            h->scan.lo1 = h->row1; h->scan.hi1 = std::min(h->row1 + iters, H);
            h->scan_pending = h->p2p && send_div;
            int rc = exchange_many(h, it, send_div ? 2 : 1);
            if (send_div) { h->div_sent_epoch = h->div_epoch; h->div_sent_rows = iters; }
            if (!rc && !h->p2p && send_div) {
                rc = scan_tiny(h, h->scan.lo0, h->scan.hi0);
                if (!rc) rc = scan_tiny(h, h->scan.lo1, h->scan.hi1);
            }
            h->scan_pending = false;
            if (rc) return rc;
        } else {
            const int kmax = plan.depth(0);
            int rc = exchange_rows(h, HB_DIVERGENCE, kmax);
            if (rc) return rc;
            if ((rc = scan_tiny(h, std::max(h->row0 - kmax, 0), h->row0))) return rc;
            if ((rc = scan_tiny(h, h->row1, std::min(h->row1 + kmax, H)))) return rc;
        }
    }
    JacobiArgs a = jacobi_args(h, h->divergence, h->roff);
    for (int k = 0; k < plan.n; ++k) {
        const int K = plan.depth(k);
        a.pin = (const float*)h->pressure.read; a.pout = (float*)h->pressure.write;
        int ext = 0;                                   // launch k produces the owned rows +- ext
        if (h->slab()) {
            if (deep) {
                ext = plan.after(k) + 1;
            } else {
                ext = (k == plan.n - 1) ? 1 : 0;
                int rc = exchange_rows(h, HB_PRESSURE, K + ext);
                if (rc) return rc;
            }
        }
        a.out_lo = std::max(h->row0 - ext, 0); a.out_hi = std::min(h->row1 + ext, H);
        const bool sc = scale_first && k == 0;
        int rc;
        if (tb) {
            // chained: behind another blocked launch of this solve, and — first launch — behind whatever kernel
            // precedes it on the stream (the previous solve's last launch in a host loop of solves; a kernel
            // without griddepcontrol.launch_dependents simply triggers at its end)
            rc = launch_tb(h, K, sc, true, a, h->tmaps.m[h->pressure.par]);
        } else {
            rc = launch_sweep(h, a, sc);
        }
        if (rc) return rc;
        h->pressure.swap(); ++nl;
    }
    if (launches_out) *launches_out = nl;
    return FLUID_OK;
}

// The arena of n sim and nd dye cells (local rows) at the handle's bytes per cell.  Every slot starts on a
// 2 MiB boundary, where a cudaMalloc of its own would put a large field.  The order (velocity, dye, pressure,
// divergence, curl) is not free: with pressure ahead of dye the 4096^2 x 50 blocked solve measured 0.4 %
// slower (H100 80GB HBM3, 700 W power limit).  The 1 KiB of peer-memory flag words come last (unused on one GPU).
FieldLayout field_layout(const fluid_t* h, size_t n, size_t nd) {
    constexpr uint64_t ALIGN = 2ull << 20;
    FieldLayout L{};
    uint64_t o = 0;
    auto slot = [&o](uint64_t bytes) { const uint64_t at = o; o += (bytes + ALIGN - 1) & ~(ALIGN - 1); return at; };
    for (int k = 0; k < 2; ++k) L.v[k] = slot(n * vbytes(h));
    for (int k = 0; k < 2; ++k) L.dye[k] = slot(nd * dbytes(h));
    for (int k = 0; k < 2; ++k) L.p[k] = slot(n * sbytes(h));
    L.div = slot(n * sbytes(h));
    L.curl = slot(n * sbytes(h));
    L.flags = o;
    L.bytes = o + 1024;
    return L;
}

// A new arena for `L`, zeroed, with dye alpha 1 in both dye slots (createFBO / createDoubleFBO, S:1004-1006).
// FLUID_ERR_NOMEM when it does not fit: nothing is allocated and the runtime keeps no error.
int make_arena(fluid_t* h, const FieldLayout& L, size_t nd, char** out) {
    char* a = nullptr;
    if (cudaMalloc((void**)&a, L.bytes) != cudaSuccess) {
        cudaGetLastError();                      // not sticky: keep it out of the next launch check
        return fail(h, FLUID_ERR_NOMEM, "out of device memory for the fields (%llu bytes)", (unsigned long long)L.bytes);
    }
    if (cudaMemsetAsync(a, 0, L.bytes, h->stream) != cudaSuccess) {
        cudaFree(a);
        return fail(h, FLUID_ERR_CUDA, "cudaMemsetAsync of the field arena failed: %s", cudaGetErrorString(cudaGetLastError()));
    }
    int rc = with_storage(h, [&](auto s) {
        using S = decltype(s);
        for (const uint64_t o : L.dye)
            fill_alpha_kernel<S><<<(unsigned)((nd + 255) / 256), 256, 0, h->stream>>>((typename S::T4*)(a + o), nd);
        return check_launch(h, "fill_alpha_kernel", 2);
    });
    if (rc) { cudaFree(a); return rc; }
    *out = a;
    return FLUID_OK;
}

// the handle's fields now live in arena `a` (each pair keeps its parity); the tiny map and the tensor maps
// follow the new addresses and sizes
int adopt_arena(fluid_t* h, char* a, const FieldLayout& L) {
    h->arena = a; h->layout = L;
    h->velocity.place(a, L.v); h->pressure.place(a, L.p); h->dye.place(a, L.dye);
    h->divergence = (float*)(a + L.div); h->curl = (float*)(a + L.curl);
    h->div_sent_epoch = 0;                               // fresh buffers: no divergence ghost rows in place yet
    int rc = alloc_tiny_map(h);
    return rc ? rc : build_tmaps(h);
}

int alloc_fields(fluid_t* h) {
    const FieldLayout L = field_layout(h, sim_cells(h) * h->members, dye_cells(h) * h->members);
    char* a = nullptr;
    int rc = make_arena(h, L, dye_cells(h) * h->members, &a);
    return rc ? rc : adopt_arena(h, a, L);
}

// One field's rows [j0, j1) of the new grid (Wn x Hn, local row 0 at global row dst_off) from the old grid
// (W x H, local row 0 at src_off): the copy of the old texture through its sampler (LINEAR, or NEAREST with
// FLUID_FLAG_NEAREST_FILTERING: resizeFBO's `filtering`, S:997 / S:1002) written in the storage format (in half
// storage the reference's blit into an RG16F / RGBA16F target rounds to fp16), or, when the size did not
// change, the rows as they are — like resizeDoubleFBO, which keeps such a field (S:1116-1126).
template <class S, class T>
int carry_field(fluid_t* h, const void* src, int W, int H, int src_off, char* dst, int Wn, int Hn, int dst_off, int j0, int j1) {
    if (W == Wn && H == Hn) {
        CU(cudaMemcpyAsync(dst + (size_t)(j0 - dst_off) * W * sizeof(T), (const char*)src + (size_t)(j0 - src_off) * W * sizeof(T),
                           (size_t)(j1 - j0) * W * sizeof(T), cudaMemcpyDeviceToDevice, h->stream));
        return FLUID_OK;
    }
    dim3 b(64, 4);
    if (h->nearest)
        resample_kernel<S, Nearest><<<grid2d(Wn, j1 - j0, b), b, 0, h->stream>>>((const T*)src, W, H, src_off, (T*)dst, Wn, Hn, dst_off, j0, j1);
    else
        resample_kernel<S, Linear><<<grid2d(Wn, j1 - j0, b), b, 0, h->stream>>>((const T*)src, W, H, src_off, (T*)dst, Wn, Hn, dst_off, j0, j1);
    return check_launch(h, "resample_kernel");
}

// back to NCCL halos: the neighbours' arenas are unmapped
void close_peers(fluid_t* h) {
    for (auto& p : h->peer) if (p.present && p.base) { cudaIpcCloseMemHandle(p.base); p.base = nullptr; p.present = false; }
    h->p2p = false;
}

// pointer to the first OWNED row of a field's .read buffer, plus its owned extent
int field_info(const fluid_t* h, int field, void** ptr, int* w, int* rows, int* ch) {
    const size_t so = (size_t)h->G * h->cfg.sim_w, doff_ = (size_t)h->Gd * h->cfg.dye_w;
    switch (field) {
        case FLUID_FIELD_VELOCITY: *ptr = (float2*)h->velocity.read + so; *w = h->cfg.sim_w; *rows = h->row1 - h->row0; *ch = 2; return 0;
        case FLUID_FIELD_DYE: *ptr = (float4*)h->dye.read + doff_; *w = h->cfg.dye_w; *rows = h->drow1 - h->drow0; *ch = 4; return 0;
        case FLUID_FIELD_PRESSURE: *ptr = (float*)h->pressure.read + so; *w = h->cfg.sim_w; *rows = h->row1 - h->row0; *ch = 1; return 0;
        case FLUID_FIELD_DIVERGENCE: *ptr = h->divergence + so; *w = h->cfg.sim_w; *rows = h->row1 - h->row0; *ch = 1; return 0;
        case FLUID_FIELD_CURL: *ptr = h->curl + so; *w = h->cfg.sim_w; *rows = h->row1 - h->row0; *ch = 1; return 0;
    }
    return -1;
}

// Multi-GPU: an advection back-trace that needed a row outside the ghost zone set the device flag;
// never clamp silently (SURVEY §7) — report it at the next synchronisation point.
int check_halo(fluid_t* h) {
    int flag = 0;
    CU(cudaMemcpyAsync(&flag, h->halo_flag, sizeof(int), cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    if (flag) CU(cudaMemsetAsync(h->halo_flag, 0, sizeof(int), h->stream));   // report once; the caller decides what to do next
    if (flag == 2)
        return fail(h, FLUID_ERR_HALO, "peer-memory halo exchange timed out waiting for a neighbour rank");
    if (flag == 3)
        return fail(h, FLUID_ERR_CUDA, "jacobi_tb_kernel: a TMA staging barrier never completed");
    if (flag == DEV_ERR_MEMBER)
        return fail(h, FLUID_ERR_INVALID, "fluid_splats_batch_device: a record named a member outside [0, %d); "
                    "that call splatted nothing", h->members);
    if (flag)
        return fail(h, FLUID_ERR_HALO, "advection back-trace left the %d-row ghost zone: |v|*dt exceeds it; "
                    "re-create the slab handle with a taller halo (FLUID_HALO_ROWS)", h->G);
    return FLUID_OK;
}

int not_on_slab(fluid_t* h, const char* what) {
    return fail(h, FLUID_ERR_INVALID, "%s is a single-GPU test entry point; a slab handle supports "
                "fluid_step / fluid_splat / fluid_pass_pressure_solve / fluid_pass_jacobi / read / write / the draw calls", what);
}

// what a batch handle refuses: everything but fluid_step, fluid_splats_batch[_device], the config, field I/O, the stats and
// the batch draw calls
int not_on_batch(fluid_t* h, const char* what) {
    return fail(h, FLUID_ERR_INVALID, "%s does not take a batch handle; one supports fluid_step / fluid_splats_batch[_device] / "
                "read / write / the *_members calls / set_param / stat / fluid_render_canvas_batch / fluid_capture_batch", what);
}

// Row ownership + ghost-zone heights of rank `rank` of `world` for a sim_h / dye_h grid (DESIGN.md §7).
// Returns false when the slabs are too short for the minimum 14-row halo.
bool slab_geometry(SlabGeometry* h, int rank, int world, int H, int Hd, int iters) {
    h->row0 = (int)((long long)H * rank / world);  h->row1 = (int)((long long)H * (rank + 1) / world);
    h->drow0 = (int)((long long)Hd * rank / world); h->drow1 = (int)((long long)Hd * (rank + 1) / world);
    h->G = h->Gd = 0;
    if (world > 1) {
        // ghost rows: enough for the advection back-trace (3 ghost-compute rows + dt*|v|max + 2)
        // and for the deep Jacobi halo (iterations + 1).
        // 64 rows: a back-trace of up to (64 - 5) rows per step, i.e. |v| up to 3540 texels/s at the reference's
        // dt <= 1/60 (vorticity clamps |v| to 1000, a pointer flick of half the canvas splats 3000); the rows
        // cost ~4 MB of halo traffic per step per neighbour at 4096 columns, microseconds on NVLink
        int g = std::max(64, iters + 2);
        if (const char* e = getenv("FLUID_HALO_ROWS")) g = std::max(14, atoi(e));
        // every rank must arrive at the SAME halo height (message sizes must match), so clip with
        // the height of the shortest slab, which all ranks can compute: floor(H / world)
        const int per = std::max(1, (Hd + H - 1) / H);
        g = std::min(g, std::min(H / world, (Hd / world) / per));
        h->G = g;
        h->Gd = g * per;                              // same physical reach on the dye grid
        if (g < 14) return false;
    }
    h->roff = h->row0 - h->G; h->droff = h->drow0 - h->Gd;
    return true;
}

// shared by fluid_create, fluid_create_slab and fluid_create_batch (batch_members > 0, checked by the caller)
int create_common(const fluid_config* cfg, int rank, int world, const void* uid, fluid_t** out, int batch_members = 0) {
    fluid_t* h = nullptr;
    if (!cfg || !out) return fail(h, FLUID_ERR_INVALID, "null argument");
    *out = nullptr;
    if (cfg->sim_w < 1 || cfg->sim_h < 1 || cfg->dye_w < 1 || cfg->dye_h < 1)
        return fail(h, FLUID_ERR_INVALID, "bad resolution %dx%d / %dx%d", cfg->sim_w, cfg->sim_h,
                    cfg->dye_w, cfg->dye_h);
    if (world < 1 || rank < 0 || rank >= world) return fail(h, FLUID_ERR_INVALID, "bad rank %d of %d", rank, world);
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) {
        cudaGetLastError();
        return fail(h, FLUID_ERR_NO_DEVICE, "no CUDA device: libfluid_b200 has no CPU path");
    }
    int dev = cfg->device;
    if (dev < 0) { if (cudaGetDevice(&dev) != cudaSuccess) dev = 0; }
    if (dev >= ndev) return fail(h, FLUID_ERR_INVALID, "device %d of %d", dev, ndev);
    cudaDeviceProp prop{};
    if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess || prop.major != 9 || prop.minor != 0)
        return fail(h, FLUID_ERR_NO_DEVICE, "device %d is sm_%d%d; this library is built for sm_90a only",
                    dev, prop.major, prop.minor);
    if (cudaSetDevice(dev) != cudaSuccess) return fail(h, FLUID_ERR_CUDA, "cudaSetDevice(%d)", dev);

    h = new fluid();
    h->cfg = *cfg;
    h->device = dev;
    h->sm_count = prop.multiProcessorCount;
    if (!(h->cfg.aspect > 0.0f)) h->cfg.aspect = (float)((double)cfg->sim_w / (double)cfg->sim_h);
    h->aspect_d = (cfg->aspect > 0.0f) ? (double)cfg->aspect : (double)cfg->sim_w / (double)cfg->sim_h;
    h->splat_radius_d = (double)cfg->splat_radius;
    h->rank = rank; h->world = world;
    h->batch = batch_members > 0;
    h->members = std::max(batch_members, 1);
    h->half = (cfg->flags & FLUID_FLAG_HALF_STORAGE) != 0;
    if (h->half && world > 1) {
        int rc = fail(nullptr, FLUID_ERR_INVALID, "FLUID_FLAG_HALF_STORAGE is a single-GPU mode");
        delete h; return rc;
    }
    h->half_fx = (cfg->flags & FLUID_FLAG_HALF_POSTFX) != 0;
    if (h->half_fx && world > 1) {
        int rc = fail(nullptr, FLUID_ERR_INVALID, "FLUID_FLAG_HALF_POSTFX is a single-GPU mode");
        delete h; return rc;
    }
    h->nearest = (cfg->flags & FLUID_FLAG_NEAREST_FILTERING) != 0;
    if (h->nearest && world > 1) {
        int rc = fail(nullptr, FLUID_ERR_INVALID, "FLUID_FLAG_NEAREST_FILTERING is a single-GPU mode");
        delete h; return rc;
    }
    h->linear_adv = (cfg->flags & FLUID_FLAG_LINEAR_ADVECTION) != 0;
    if (h->linear_adv && h->nearest) {   // no float linear filtering means the MANUAL_FILTERING shader (S:783)
        int rc = fail(nullptr, FLUID_ERR_INVALID, "FLUID_FLAG_LINEAR_ADVECTION needs linear filtering: it cannot be "
                      "combined with FLUID_FLAG_NEAREST_FILTERING");
        delete h; return rc;
    }
    if (h->linear_adv && world > 1) {
        int rc = fail(nullptr, FLUID_ERR_INVALID, "FLUID_FLAG_LINEAR_ADVECTION is a single-GPU mode");
        delete h; return rc;
    }
    if (!slab_geometry(h, rank, world, cfg->sim_h, cfg->dye_h, cfg->pressure_iterations)) {
        int rc = fail(nullptr, FLUID_ERR_INVALID, "slabs of %d rows are too short for a 14-row halo: use fewer GPUs", cfg->sim_h / world);
        delete h; return rc;
    }
    auto body = [&]() -> int {
        CU(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
        for (auto& e : h->mark) CU(cudaEventCreate(&e));
        for (auto& e : h->tev) CU(cudaEventCreate(&e));
        CU(cudaMalloc((void**)&h->halo_flag, sizeof(int)));
        CU(cudaMemsetAsync(h->halo_flag, 0, sizeof(int), h->stream));
        CU(cudaMalloc((void**)&h->exact_streams, sizeof(unsigned long long)));
        CU(cudaMemsetAsync(h->exact_streams, 0, sizeof(unsigned long long), h->stream));
        if (h->batch) {
            int r = alloc_member_table(h); if (r) return r;
            CU(cudaMalloc((void**)&h->member_list, (size_t)h->members * sizeof(int32_t)));
            CU(cudaMalloc((void**)&h->look_table, (size_t)h->members * sizeof(fk::ImageLook)));
        } else {
            CU(cudaMalloc((void**)&h->dt_dev, sizeof(float)));
            CU(cudaMemsetAsync(h->dt_dev, 0, sizeof(float), h->stream));
        }
        int r = alloc_fields(h); if (r) return r;
        CU(cudaStreamSynchronize(h->stream));
#ifndef FLUID_TEST_LOOPBACK   // the loopback test build links its ranks in-process (tests/slab_loopback.cu)
        if (world > 1) {
            ncdl::Api& N = ncdl::api();
            if (!N.handle) return fail(h, FLUID_ERR_NCCL, "NCCL not available: %s", N.why);
            ncdl::ncclUniqueId id;
            memcpy(&id, uid, sizeof id);
            int rc = N.CommInitRank(&h->comm, world, id, rank);
            if (rc) return fail(h, FLUID_ERR_NCCL, "ncclCommInitRank failed: %s", N.GetErrorString(rc));
        }
#endif
        return FLUID_OK;
    };
    int rc = body();
    if (rc != FLUID_OK) { g_create_error = h->err; fluid_destroy(h); return rc; }
    *out = h;
    return FLUID_OK;
}

}  // namespace

// ================================================================================================
extern "C" {

int fluid_abi_version(void) { return FLUID_ABI_VERSION; }

void fluid_config_default(fluid_config* c) {
    memset(c, 0, sizeof *c);
    c->sim_w = c->sim_h = 128;            // SIM_RESOLUTION  S:60
    c->dye_w = c->dye_h = 1024;           // DYE_RESOLUTION  S:61
    c->density_dissipation = 1.0f;        // S:63
    c->velocity_dissipation = 0.2f;       // S:64
    c->pressure = 0.8f;                   // S:65
    c->pressure_iterations = 20;          // S:66
    c->curl = 30.0f;                      // S:67
    c->splat_radius = 0.25f;              // S:68
    c->aspect = 1.0f;
    c->device = -1;
    c->flags = 0;
    c->jacobi_block = 0;
}

// getResolution, S:1612-1624
void fluid_get_resolution(int resolution, int canvas_w, int canvas_h, int* out_w, int* out_h) {
    double aspect = (double)canvas_w / (double)canvas_h;
    if (aspect < 1.0) aspect = 1.0 / aspect;
    // Math.round: half away from zero for positive values == floor(x + 0.5)
    const int mn = (int)(resolution + 0.5);
    const int mx = (int)((double)resolution * aspect + 0.5);
    if (canvas_w > canvas_h) { *out_w = mx; *out_h = mn; }
    else { *out_w = mn; *out_h = mx; }
}

const char* fluid_last_error(fluid_t* h) { return h ? h->err.c_str() : g_create_error.c_str(); }

int fluid_create(const fluid_config* cfg, fluid_t** out) { return create_common(cfg, 0, 1, nullptr, out); }

// B simulations of cfg's size and config in one handle.  The step kernels take the member as blockIdx.z,
// whose grid extent caps B at FLUID_MAX_MEMBERS; they exist for power-of-two grids at least 128 columns wide
// (the 4-cell advection) and 2 rows high (the blocked Jacobi kernel), in fp32 storage with the MANUAL
// advection filter, so every flag that would pick another kernel is refused.
int fluid_create_batch(const fluid_config* cfg, int members, fluid_t** out) {
    if (!cfg || !out) return fail(nullptr, FLUID_ERR_INVALID, "null argument");
    *out = nullptr;
    if (members < 1 || members > FLUID_MAX_MEMBERS)
        return fail(nullptr, FLUID_ERR_INVALID, "a batch holds 1 to %d members, not %d", FLUID_MAX_MEMBERS, members);
    if (cfg->flags & ~(uint32_t)FLUID_FLAG_NO_GRAPH)
        return fail(nullptr, FLUID_ERR_INVALID, "a batch handle takes no flag but FLUID_FLAG_NO_GRAPH (got 0x%x)", cfg->flags);
    if (!is_pow2(cfg->sim_w) || !is_pow2(cfg->sim_h) || !is_pow2(cfg->dye_w) || !is_pow2(cfg->dye_h) ||
        cfg->sim_w < 128 || cfg->dye_w < 128 || cfg->sim_h < 2 || cfg->dye_h < 2)
        return fail(nullptr, FLUID_ERR_INVALID, "a batch needs power-of-two sizes, widths >= 128 and heights >= 2 "
                    "(got %dx%d / %dx%d)", cfg->sim_w, cfg->sim_h, cfg->dye_w, cfg->dye_h);
    return create_common(cfg, 0, 1, nullptr, out, members);
}

int fluid_members(fluid_t* h) { return h ? h->members : 0; }

int fluid_nccl_unique_id(void* out_uid, size_t uid_bytes) {
    if (!out_uid || uid_bytes < sizeof(ncdl::ncclUniqueId)) return fail(nullptr, FLUID_ERR_INVALID, "uid buffer must hold 128 bytes");
    ncdl::Api& N = ncdl::api();
    if (!N.handle) return fail(nullptr, FLUID_ERR_NCCL, "NCCL not available: %s", N.why);
    ncdl::ncclUniqueId id;
    int rc = N.GetUniqueId(&id);
    if (rc) return fail(nullptr, FLUID_ERR_NCCL, "ncclGetUniqueId failed: %s", N.GetErrorString(rc));
    memcpy(out_uid, &id, sizeof id);
    return FLUID_OK;
}

int fluid_create_slab(const fluid_config* cfg, int rank, int world, const void* nccl_uid,
                      size_t uid_bytes, fluid_t** out) {
    if (world > 1 && (!nccl_uid || uid_bytes < sizeof(ncdl::ncclUniqueId)))
        return fail(nullptr, FLUID_ERR_INVALID, "nccl_uid must be the 128 bytes from fluid_nccl_unique_id()");
    return create_common(cfg, rank, world, nccl_uid, out);
}

// ---- peer-memory halo path -------------------------------------------------------------------------
struct P2PBlob {            // what fluid_p2p_export hands to the launcher (opaque to it), 256 bytes
    cudaIpcMemHandle_t mem;
    int32_t rank, roff, droff, reserved;
    FieldLayout layout;
    char pad[256 - sizeof(cudaIpcMemHandle_t) - 16 - sizeof(FieldLayout)];
};
static_assert(sizeof(P2PBlob) == 256, "blob layout");

int fluid_p2p_export(fluid_t* h, void* blob, size_t blob_bytes) {
    if (h && h->batch) return not_on_batch(h, "fluid_p2p_export");
    if (!h || !blob || blob_bytes < sizeof(P2PBlob)) return fail(h, FLUID_ERR_INVALID, "blob must hold 256 bytes");
    if (!h->slab() || !h->arena) return fail(h, FLUID_ERR_INVALID, "fluid_p2p_export needs a slab handle");
    // halo_push_kernel moves rows as 16-byte words: every exchanged row (4*W pressure / divergence,
    // 8*W velocity, 16*Wd dye) must be a multiple of 16 bytes.  Otherwise refuse, so that the
    // launcher keeps ALL ranks on the byte-exact NCCL transport.
    if (h->cfg.sim_w % 4 != 0)
        return fail(h, FLUID_ERR_INVALID, "peer-memory halos need sim width %% 4 == 0 (got %d): staying on NCCL", h->cfg.sim_w);
    P2PBlob b{};
    CU(cudaStreamSynchronize(h->stream));
    CU(cudaIpcGetMemHandle(&b.mem, h->arena));
    b.rank = h->rank; b.roff = h->roff; b.droff = h->droff; b.layout = h->layout;
    memcpy(blob, &b, sizeof b);
    return FLUID_OK;
}

// blob_below / blob_above: the 256-byte exports of rank-1 / rank+1 (NULL at the domain ends).
// Collective in spirit: every rank of the slab group must connect before the next fluid_step.
int fluid_p2p_connect(fluid_t* h, const void* blob_below, const void* blob_above) {
    if (h && h->batch) return not_on_batch(h, "fluid_p2p_connect");
    if (!h || !h->slab() || !h->arena) return fail(h, FLUID_ERR_INVALID, "fluid_p2p_connect needs a slab handle");
    const void* blobs[2] = {blob_below, blob_above};
    for (int side = 0; side < 2; ++side) {
        const bool need = (side == 0) ? h->rank > 0 : h->rank + 1 < h->world;
        if (!need) continue;
        if (!blobs[side]) return fail(h, FLUID_ERR_INVALID, "missing neighbour blob (side %d)", side);
        P2PBlob b; memcpy(&b, blobs[side], sizeof b);
        if (b.rank != h->rank + (side == 0 ? -1 : 1)) return fail(h, FLUID_ERR_INVALID, "blob of rank %d passed as side %d of rank %d", b.rank, side, h->rank);
        void* base = nullptr;
        CU(cudaIpcOpenMemHandle(&base, b.mem, cudaIpcMemLazyEnablePeerAccess));
        h->peer[side] = fluid::Peer{true, (char*)base, b.roff, b.droff, b.layout};
    }
    h->p2p = true;
    return FLUID_OK;
}

// Back to the NCCL transport (used by launchers when ANY rank failed to map its neighbours, so
// that all ranks keep using the same one).
int fluid_p2p_disable(fluid_t* h) {
    if (!h) return FLUID_ERR_INVALID;
    if (h->batch) return not_on_batch(h, "fluid_p2p_disable");
    if (h->stream) CU(cudaStreamSynchronize(h->stream));
    close_peers(h);
    return FLUID_OK;
}

void fluid_destroy(fluid_t* h) {
    if (!h) return;
    cudaSetDevice(h->device);
    if (h->stream) cudaStreamSynchronize(h->stream);
    drop_graphs(h);
    close_peers(h);
    cudaFree(h->arena);
    cudaFree(h->tiny_map);
    cudaFree(h->halo_flag);
    cudaFree(h->exact_streams);
    cudaFree(h->dt_dev);
    cudaFree(h->member_list);
    cudaFree(h->look_table);
    cudaFree(h->scratch);
    cudaFree(h->splat_scratch);
    cudaFree(h->frame);
    cudaFree(h->pfx.bloom); cudaFree(h->pfx.sun); cudaFree(h->pfx.dither); cudaFree(h->pfx.mask);
    if (h->comm) { ncdl::api().CommDestroy(h->comm); h->comm = nullptr; }
    for (auto& e : h->mark) if (e) cudaEventDestroy(e);
    for (auto& e : h->tev) if (e) cudaEventDestroy(e);
    if (h->hp.up) { cudaStreamSynchronize(h->hp.up); cudaStreamDestroy(h->hp.up); }
    if (h->hp.down) { cudaStreamSynchronize(h->hp.down); cudaStreamDestroy(h->hp.down); }
    if (h->hp.ev_start) cudaEventDestroy(h->hp.ev_start);
    for (auto& e : h->hp.ev_up) if (e) cudaEventDestroy(e);
    for (auto& e : h->hp.ev_done) if (e) cudaEventDestroy(e);
    cudaFree(h->hp.s[0]); cudaFree(h->hp.s[1]);
    if (h->stream) cudaStreamDestroy(h->stream);
    delete h;
}

// config.<key> = v, where SPLAT_RADIUS and ASPECT keep vd, the value as the caller's double.  On a batch handle
// every member takes a per-member key's value, and ASPECT moves every member's splat radius.
static int set_param(fluid_t* h, int key, float v, double vd) {
    switch (key) {
        case FLUID_DENSITY_DISSIPATION: h->cfg.density_dissipation = v; break;
        case FLUID_VELOCITY_DISSIPATION: h->cfg.velocity_dissipation = v; break;
        case FLUID_PRESSURE: h->cfg.pressure = v; break;
        case FLUID_PRESSURE_ITERATIONS: h->cfg.pressure_iterations = (int)(v + 0.5f); break;
        case FLUID_CURL: h->cfg.curl = v; break;
        case FLUID_SPLAT_RADIUS: h->cfg.splat_radius = v; h->splat_radius_d = vd; break;
        case FLUID_ASPECT: h->cfg.aspect = v; h->aspect_d = vd; break;
        case FLUID_JACOBI_BLOCK: h->cfg.jacobi_block = (int)(v + 0.5f); break;
        case FLUID_BACKGROUND: h->background = (int)(v + 0.5f); break;
        default: return fail(h, FLUID_ERR_INVALID, "unknown param key %d", key);
    }
    if (!h->batch) return FLUID_OK;
    const int row = key == FLUID_ASPECT ? MP_RADIUS : member_row(key);
    if (row < 0) return FLUID_OK;
    for (int m = 0; m < h->members; ++m)
        set_member_value(h, row, m, key == FLUID_ASPECT ? h->member_radius_d[m] : vd);
    return upload_member_row(h, row);
}

int fluid_set_param(fluid_t* h, int key, float v) {
    if (!h) return FLUID_ERR_INVALID;
    return set_param(h, key, v, (double)v);
}

// The JS config values are doubles; two of them enter double arithmetic on the host before the
// single narrowing of gl.uniform1f (correctRadius S:1457-1462: SPLAT_RADIUS / 100 * aspectRatio),
// so a host mirror passes them at full precision.  Every other key narrows like fluid_set_param.
int fluid_set_param_f64(fluid_t* h, int key, double v) {
    if (!h) return FLUID_ERR_INVALID;
    return set_param(h, key, (float)v, v);
}

// what fluid_set_param_members, fluid_get_param_members and fluid_step_members refuse before they change anything
static int check_members(fluid_t* h, const char* what, const void* values, int n) {
    if (!h->batch) return fail(h, FLUID_ERR_INVALID, "%s needs a batch handle (fluid_create_batch)", what);
    if (!values || n != h->members)
        return fail(h, FLUID_ERR_INVALID, "%s takes one value for each of the %d members (got %d at %p)", what, h->members, n, values);
    return FLUID_OK;
}
static int check_member_key(fluid_t* h, const char* what, int key) {
    if (member_row(key) >= 0) return FLUID_OK;
    return fail(h, FLUID_ERR_INVALID, "%s: key %d has no per-member values (DENSITY_DISSIPATION, VELOCITY_DISSIPATION, "
                "PRESSURE, CURL and SPLAT_RADIUS do)", what, key);
}

int fluid_set_param_members(fluid_t* h, int key, const double* values, int n) {
    if (!h) return FLUID_ERR_INVALID;
    int rc = check_members(h, "fluid_set_param_members", values, n);
    if (!rc) rc = check_member_key(h, "fluid_set_param_members", key);
    if (rc) return rc;
    const int row = member_row(key);
    for (int m = 0; m < n; ++m) set_member_value(h, row, m, values[m]);
    return upload_member_row(h, row);
}

int fluid_get_param_members(fluid_t* h, int key, float* values, int n) {
    if (!h) return FLUID_ERR_INVALID;
    int rc = check_members(h, "fluid_get_param_members", values, n);
    if (!rc) rc = check_member_key(h, "fluid_get_param_members", key);
    if (rc) return rc;
    for (int m = 0; m < n; ++m) values[m] = member_value(h, member_row(key), m);
    return FLUID_OK;
}

int fluid_get_param(fluid_t* h, int key, float* v) {
    if (!h || !v) return FLUID_ERR_INVALID;
    if (h->batch && member_row(key) >= 0) {            // member 0's
        *v = member_value(h, member_row(key), 0);
        return FLUID_OK;
    }
    switch (key) {
        case FLUID_DENSITY_DISSIPATION: *v = h->cfg.density_dissipation; break;
        case FLUID_VELOCITY_DISSIPATION: *v = h->cfg.velocity_dissipation; break;
        case FLUID_PRESSURE: *v = h->cfg.pressure; break;
        case FLUID_PRESSURE_ITERATIONS: *v = (float)h->cfg.pressure_iterations; break;
        case FLUID_CURL: *v = h->cfg.curl; break;
        case FLUID_SPLAT_RADIUS: *v = h->cfg.splat_radius; break;
        case FLUID_ASPECT: *v = h->cfg.aspect; break;
        case FLUID_JACOBI_BLOCK: *v = (float)h->cfg.jacobi_block; break;
        case FLUID_BACKGROUND: *v = (float)h->background; break;
        default: return fail(h, FLUID_ERR_INVALID, "unknown param key %d", key);
    }
    return FLUID_OK;
}

// ---- passes ---------------------------------------------------------------------------------------
// do_*: launch on an explicit row range (owned rows, or owned +- e for redundant ghost compute on a
// slab); the public fluid_pass_* wrappers are the single-GPU, one-blit-per-call test surface.

static int do_curl(fluid_t* h, Grid g) {
    return with_storage(h, [&](auto s) {
        using S = decltype(s);
        dim3 b(64, 4);
        curl_kernel<S><<<grid2d(g.W, g.j_hi - g.j_lo, b), b, 0, h->stream>>>(
            (const typename S::T2*)h->velocity.read, (typename S::T1*)h->curl, g);
        return check_launch(h, "curl_kernel");
    });
}
static int do_vorticity(fluid_t* h, Grid g) {
    int rc = with_storage(h, [&](auto s) {
        using S = decltype(s);
        dim3 b(64, 4);
        vorticity_kernel<S><<<grid2d(g.W, g.j_hi - g.j_lo, b), b, 0, h->stream>>>(
            (const typename S::T2*)h->velocity.read, (const typename S::T1*)h->curl, (typename S::T2*)h->velocity.write, g,
            h->cfg.curl, h->dt_dev);
        return check_launch(h, "vorticity_kernel");
    });
    if (rc) return rc;
    h->velocity.swap();                          // S:1246
    return FLUID_OK;
}
static int do_divergence(fluid_t* h, Grid g) {
    // half storage never runs the contracted Jacobi tail, so it keeps no tiny-divergence map
    if (!h->half) { int rc = clear_tiny_map(h); if (rc) return rc; }
    return with_storage(h, [&](auto s) {
        using S = decltype(s);
        dim3 b(64, 4);
        divergence_kernel<S><<<grid2d(g.W, g.j_hi - g.j_lo, b), b, 0, h->stream>>>(
            (const typename S::T2*)h->velocity.read, (typename S::T1*)h->divergence, g, h->half ? nullptr : h->tiny_map);
        return check_launch(h, "divergence_kernel");
    });
}
// rows per warp stream of the row-streaming kernels: one full wave of resident warps (`warps_per_sm`
// from the occupancy calculator) across all members, at least `rmin` rows each so that the halo rows a
// stream re-reads stay a bounded fraction.  Grids too small to give every SM a warp use the tiled kernels
// instead, except on a batch handle, which always streams: its kernels have a member axis, the tiled ones do not.
static StreamArgs stream_args(const fluid_t* h, Grid g, int cols_per_window, int rmin, int warps_per_sm, int round_to) {
    StreamArgs a{};
    a.g = g;
    a.nxw = (g.W + cols_per_window - 1) / cols_per_window;
    const int rows = g.j_hi - g.j_lo;
    const int chunks = std::max(1, h->sm_count * warps_per_sm / (a.nxw * h->members));
    int r = std::max((rows + chunks - 1) / chunks, rmin);
    r = (r + round_to - 1) / round_to * round_to;
    a.rows_per_chunk = std::min(r, std::max(rows, 1));
    return a;
}
static int stream_warps(const StreamArgs& a) {
    return a.nxw * ((a.g.j_hi - a.g.j_lo + a.rows_per_chunk - 1) / a.rows_per_chunk);
}
static bool streaming_ok(const fluid_t* h) {
    return !h->half && h->cfg.sim_w % 4 == 0 && h->cfg.sim_w >= 8 && !(h->cfg.flags & FLUID_FLAG_TILED_PASSES);
}

static int do_curl(fluid_t* h, Grid g);
static int do_vorticity(fluid_t* h, Grid g);
static int do_divergence(fluid_t* h, Grid g);
static int do_cvd(fluid_t* h, Grid g) {
    if (h->half) {                                   // one launch per reference blit (each rounds to fp16)
        int rc = do_curl(h, g); if (rc) return rc;
        if ((rc = do_vorticity(h, g))) return rc;
        return do_divergence(h, g);
    }
    { int rc = clear_tiny_map(h); if (rc) return rc; }
    static int cvd_occ = 0;
    if (!cvd_occ) {
        int blocks = 0;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks, cvd_stream_kernel<false>, 32 * CVD2_WARPS, CVD2_SMEM);
        cvd_occ = std::max(1, blocks) * CVD2_WARPS;
    }
    const StreamArgs a = stream_args(h, g, CVD2_VALID, 16, cvd_occ, 1);
    const int nwarps = stream_warps(a);
    if (h->batch || (streaming_ok(h) && nwarps >= h->sm_count)) {
        const dim3 grid((nwarps + CVD2_WARPS - 1) / CVD2_WARPS, 1, h->members);
        auto* k = h->batch ? cvd_stream_kernel<true> : cvd_stream_kernel<false>;
        k<<<grid, 32 * CVD2_WARPS, CVD2_SMEM, h->stream>>>(
            (const float2*)h->velocity.read, h->curl, (float2*)h->velocity.write, h->divergence, a, h->cfg.curl,
            h->dt_dev, h->tiny_map);
        int rc = check_launch(h, "cvd_stream_kernel"); if (rc) return rc;
        ++h->launches.cvd_stream;
        h->velocity.swap();
        return FLUID_OK;
    }
    dim3 b(64, 4);
    dim3 grid((g.W + CVD_TX - 1) / CVD_TX, (g.j_hi - g.j_lo + CVD_TY - 1) / CVD_TY);
    curl_vorticity_divergence_kernel<<<grid, b, 0, h->stream>>>(
        (const float2*)h->velocity.read, h->curl, (float2*)h->velocity.write, h->divergence, g,
        h->cfg.curl, h->dt_dev, h->tiny_map);
    int rc = check_launch(h, "curl_vorticity_divergence_kernel"); if (rc) return rc;
    h->velocity.swap();
    return FLUID_OK;
}
static int do_gradient(fluid_t* h, Grid g) {
    const StreamArgs a = stream_args(h, g, 128, 8, 32, GS_U);
    const int nwarps = stream_warps(a);
    if (h->batch || (streaming_ok(h) && nwarps >= h->sm_count)) {
        const dim3 grid((nwarps + GS_WARPS - 1) / GS_WARPS, 1, h->members);
        auto* k = h->batch ? gradient_stream_kernel<true> : gradient_stream_kernel<false>;
        k<<<grid, 32 * GS_WARPS, 0, h->stream>>>(
            (const float*)h->pressure.read, (const float2*)h->velocity.read, (float2*)h->velocity.write, a);
        int rc = check_launch(h, "gradient_stream_kernel"); if (rc) return rc;
        ++h->launches.gradient_stream;
        h->velocity.swap();                          // S:1273
        return FLUID_OK;
    }
    int rc = with_storage(h, [&](auto s) {
        using S = decltype(s);
        dim3 b(64, 4);
        gradient_subtract_kernel<S><<<grid2d(g.W, g.j_hi - g.j_lo, b), b, 0, h->stream>>>(
            (const typename S::T1*)h->pressure.read, (const typename S::T2*)h->velocity.read, (typename S::T2*)h->velocity.write, g);
        return check_launch(h, "gradient_subtract_kernel");
    });
    if (rc) return rc;
    h->velocity.swap();                          // S:1273
    return FLUID_OK;
}
// valid source rows of a slab buffer: owned + ghost, clipped to the domain
static void valid_rows(int r0, int r1, int g, int H, int* lo, int* hi) {
    *lo = std::max(r0 - g, 0); *hi = std::min(r1 + g, H);
}
static int do_advect_velocity(fluid_t* h, Grid out) {
    AdvectArgs a{};
    a.vel = sim_grid(h); a.src = out;
    valid_rows(h->row0, h->row1, h->G, h->cfg.sim_h, &a.vel_lo, &a.vel_hi);
    a.src_lo = a.vel_lo; a.src_hi = a.vel_hi;
    a.dtp = h->dt_dev; a.dissipation = h->cfg.velocity_dissipation; a.halo_violation = h->halo_flag;
    a.tsx = a.dsx = (float)(1.0 / (double)h->cfg.sim_w); a.tsy = a.dsy = (float)(1.0 / (double)h->cfg.sim_h);
    const bool p2 = is_pow2(h->cfg.sim_w) && is_pow2(h->cfg.sim_h);
    int rc = with_filter(h, [&](auto f) {
        using F = decltype(f);
        if (advect4_runs(h, p2, out.W)) {    // 4 cells per thread, 32 apart; a batch handle's members along z
            auto* k = h->slab()  ? advect_velocity4_kernel<true>
                    : h->batch ? advect_velocity4_kernel<false, F, true> : advect_velocity4_kernel<false, F>;
            k<<<dim3(out.W / 128, (out.j_hi - out.j_lo + 7) / 8, h->members), dim3(32, 8), 0, h->stream>>>(
                (const float2*)h->velocity.read, (float2*)h->velocity.write, a);
            ++h->launches.advect4;
        } else with_storage(h, [&](auto s) {
            using S = decltype(s);
            auto* k = p2 ? advect_velocity_kernel<S, F, pow2_form<S, F>> : advect_velocity_kernel<S, F, false>;
            const dim3 b(64, 4);
            k<<<grid2d(out.W, out.j_hi - out.j_lo, b), b, 0, h->stream>>>(
                (const typename S::T2*)h->velocity.read, (typename S::T2*)h->velocity.write, a);
        });
        return check_launch(h, "advect_velocity_kernel");
    });
    if (rc) return rc;
    h->velocity.swap();                          // S:1285
    return FLUID_OK;
}
static int do_advect_dye(fluid_t* h) {
    AdvectArgs a{};
    a.vel = sim_grid(h); a.src = dye_grid(h);
    // after the velocity advection the slab holds valid velocity on owned rows +- 3
    valid_rows(h->row0, h->row1, h->slab() ? 3 : 0, h->cfg.sim_h, &a.vel_lo, &a.vel_hi);
    valid_rows(h->drow0, h->drow1, h->Gd, h->cfg.dye_h, &a.src_lo, &a.src_hi);
    a.dtp = h->dt_dev; a.dissipation = h->cfg.density_dissipation; a.halo_violation = h->halo_flag;
    a.tsx = (float)(1.0 / (double)h->cfg.sim_w); a.tsy = (float)(1.0 / (double)h->cfg.sim_h);
    a.dsx = (float)(1.0 / (double)h->cfg.dye_w); a.dsy = (float)(1.0 / (double)h->cfg.dye_h);
    const bool p2 = is_pow2(h->cfg.sim_w) && is_pow2(h->cfg.sim_h) && is_pow2(h->cfg.dye_w) && is_pow2(h->cfg.dye_h);
    const bool same = h->cfg.sim_w == h->cfg.dye_w && h->cfg.sim_h == h->cfg.dye_h;
    const Grid& out = a.src;
    int rc = with_filter(h, [&](auto f) {
        using F = decltype(f);
        constexpr bool own = F::kOwnTexel;
        if (advect4_runs(h, p2, out.W)) {    // 4 cells per thread, 32 apart; a batch handle's members along z
            auto* k = h->slab()  ? (same ? advect_dye4_kernel<true, true> : advect_dye4_kernel<false, true>)
                    : h->batch ? (same ? advect_dye4_kernel<own, false, F, true> : advect_dye4_kernel<false, false, F, true>)
                               : (same ? advect_dye4_kernel<own, false, F> : advect_dye4_kernel<false, false, F>);
            k<<<dim3(out.W / 128, (out.j_hi - out.j_lo + 7) / 8, h->members), dim3(32, 8), 0, h->stream>>>(
                (const float2*)h->velocity.read, (const float4*)h->dye.read, (float4*)h->dye.write, a);
            ++h->launches.advect4;
        } else with_storage(h, [&](auto s) {
            using S = decltype(s);
            constexpr bool pf = pow2_form<S, F>;
            auto* k = !p2  ? advect_dye_kernel<S, F, false, false>
                    : same ? advect_dye_kernel<S, F, pf, pf && own> : advect_dye_kernel<S, F, pf, false>;
            const dim3 b(64, 4);
            k<<<grid2d(out.W, out.j_hi - out.j_lo, b), b, 0, h->stream>>>(
                (const typename S::T2*)h->velocity.read, (const typename S::T4*)h->dye.read, (typename S::T4*)h->dye.write, a);
        });
        return check_launch(h, "advect_dye_kernel");
    });
    if (rc) return rc;
    h->dye.swap();                                      // S:1293
    return FLUID_OK;
}

int fluid_pass_curl(fluid_t* h) {
    if (!h) return FLUID_ERR_INVALID;
    if (h->batch) return not_on_batch(h, "fluid_pass_curl");
    if (h->slab()) return not_on_slab(h, "fluid_pass_curl");
    return do_curl(h, sim_grid(h));
}
int fluid_pass_vorticity(fluid_t* h, float dt) {
    if (!h) return FLUID_ERR_INVALID;
    if (h->batch) return not_on_batch(h, "fluid_pass_vorticity");
    if (h->slab()) return not_on_slab(h, "fluid_pass_vorticity");
    int rc = set_dt(h, dt); if (rc) return rc;
    return do_vorticity(h, sim_grid(h));
}
int fluid_pass_divergence(fluid_t* h) {
    if (!h) return FLUID_ERR_INVALID;
    if (h->batch) return not_on_batch(h, "fluid_pass_divergence");
    if (h->slab()) return not_on_slab(h, "fluid_pass_divergence");
    return do_divergence(h, sim_grid(h));
}
int fluid_pass_curl_vorticity_divergence(fluid_t* h, float dt) {
    if (!h) return FLUID_ERR_INVALID;
    if (h->batch) return not_on_batch(h, "fluid_pass_curl_vorticity_divergence");
    if (h->slab()) return not_on_slab(h, "fluid_pass_curl_vorticity_divergence");
    int rc = set_dt(h, dt); if (rc) return rc;
    return do_cvd(h, sim_grid(h));
}
int fluid_pass_clear_pressure(fluid_t* h) {
    if (!h) return FLUID_ERR_INVALID;
    if (h->batch) return not_on_batch(h, "fluid_pass_clear_pressure");
    return run_jacobi(h, 0, true, nullptr);
}
int fluid_pass_jacobi(fluid_t* h, int iters) {
    if (!h) return FLUID_ERR_INVALID;
    if (h->batch) return not_on_batch(h, "fluid_pass_jacobi");
    if (iters < 0) return fail(h, FLUID_ERR_INVALID, "iters < 0");
    return run_jacobi(h, iters, false, nullptr);
}
int fluid_pass_pressure_solve(fluid_t* h) {
    if (!h) return FLUID_ERR_INVALID;
    if (h->batch) return not_on_batch(h, "fluid_pass_pressure_solve");
    return run_jacobi(h, h->cfg.pressure_iterations, true, nullptr);
}
int fluid_pass_gradient_subtract(fluid_t* h) {
    if (!h) return FLUID_ERR_INVALID;
    if (h->batch) return not_on_batch(h, "fluid_pass_gradient_subtract");
    if (h->slab()) return not_on_slab(h, "fluid_pass_gradient_subtract");
    return do_gradient(h, sim_grid(h));
}
int fluid_pass_advect_velocity(fluid_t* h, float dt) {
    if (!h) return FLUID_ERR_INVALID;
    if (h->batch) return not_on_batch(h, "fluid_pass_advect_velocity");
    if (h->slab()) return not_on_slab(h, "fluid_pass_advect_velocity");
    int rc = set_dt(h, dt); if (rc) return rc;
    return do_advect_velocity(h, sim_grid(h));
}
int fluid_pass_advect_dye(fluid_t* h, float dt) {
    if (!h) return FLUID_ERR_INVALID;
    if (h->batch) return not_on_batch(h, "fluid_pass_advect_dye");
    if (h->slab()) return not_on_slab(h, "fluid_pass_advect_dye");
    int rc = set_dt(h, dt); if (rc) return rc;
    return do_advect_dye(h);
}

// step(dt), S:1231-1294.
// On a slab the only messages are the Jacobi halos (inside run_jacobi) and the two advection
// halos below; curl / vorticity / divergence / gradientSubtract read ghost rows that the previous
// step's advection (velocity on owned rows +- 3) and the last Jacobi launch (pressure on owned
// rows +- 1) already computed redundantly.
static int step_enqueue(fluid_t* h, bool timed) {
    const uint64_t l0 = h->launches.all;
    int rc;
    int jl = 0;
    if (timed) cudaEventRecord(h->tev[0], h->stream);
    if (h->slab() && !h->v_ghost_valid) {   // after fluid_write(velocity): rebuild the +-3 ghost rows
        if ((rc = exchange_rows(h, HB_VELOCITY, 3))) return rc;
        h->v_ghost_valid = true;
    }
    if (h->cfg.flags & FLUID_FLAG_UNFUSED) {
        if ((rc = do_curl(h, sim_grid_ext(h, h->slab() ? 2 : 0)))) return rc;
        if ((rc = do_vorticity(h, sim_grid_ext(h, h->slab() ? 1 : 0)))) return rc;
        if ((rc = do_divergence(h, sim_grid(h)))) return rc;
    } else {
        if ((rc = do_cvd(h, sim_grid(h)))) return rc;
    }
    if (timed) cudaEventRecord(h->tev[1], h->stream);
    if ((rc = run_jacobi(h, h->cfg.pressure_iterations, true, &jl))) return rc;
    if (timed) cudaEventRecord(h->tev[2], h->stream);
    if ((rc = do_gradient(h, sim_grid(h)))) return rc;
    if (timed) cudaEventRecord(h->tev[3], h->stream);
    if (h->slab()) {   // advection halo #1: G rows of the projected velocity
        if ((rc = exchange_rows(h, HB_VELOCITY, h->G))) return rc;
    }
    if ((rc = do_advect_velocity(h, sim_grid_ext(h, h->slab() ? 3 : 0)))) return rc;
    if (timed) cudaEventRecord(h->tev[4], h->stream);
    if (h->slab()) {   // advection halo #2: Gd rows of dye
        if ((rc = exchange_rows(h, HB_DYE, h->Gd))) return rc;
    }
    if ((rc = do_advect_dye(h))) return rc;
    if (timed) cudaEventRecord(h->tev[5], h->stream);
    h->timing.jacobi_launches = jl;
    h->timing.total_launches = (int)(h->launches.all - l0);
    h->have_timing = timed;
    return FLUID_OK;
}

// The reference pays one draw call per pass (7 + PRESSURE_ITERATIONS per step) and is bound by
// that at its default 128^2 grid.  Here a step is 4 + ceil(iters/10) kernels, and on a single GPU
// they are replayed as ONE instantiated CUDA graph.  A graph bakes in kernel arguments, so the
// cache key holds everything they depend on: the config scalars, the grid sizes and which half of
// each ping-pong pair is currently `.read`.  dt is NOT part of the key: kernels read it from
// device memory (set_dt), so the reference's frame loop — calcDeltaTime() yields a different dt
// on every frame (S:1188-1194) — replays the same two graphs (one per ping-pong parity).
// A batch handle's kernels read CURL, PRESSURE and the dissipations from the member table, like dt, so they are
// not part of its key either: per-member values and dts change every step and still replay the same graphs.
static int step_after_dt(fluid_t* h) {
    const bool no_graph = (h->cfg.flags & FLUID_FLAG_NO_GRAPH) != 0;
    if (no_graph || h->slab()) return step_enqueue(h, no_graph);
    char key[256];
    const fluid_config& c = h->cfg;
    const bool b = h->batch;
    snprintf(key, sizeof key, "%a|%a|%a|%a|%d|%d|%u|%d%d%d|%dx%d|%dx%d|%d",
             b ? 0.0f : c.curl, b ? 0.0f : c.pressure, b ? 0.0f : c.velocity_dissipation, b ? 0.0f : c.density_dissipation,
             c.pressure_iterations, c.jacobi_block,
             c.flags, h->velocity.par, h->pressure.par, h->dye.par, c.sim_w, c.sim_h, c.dye_w, c.dye_h, h->members);
    auto it = h->graphs.find(key);
    if (it == h->graphs.end()) {
        if (h->graphs.size() > 64) drop_graphs(h);          // config sliders dragged for a long time: stay bounded
        const int pv = h->velocity.par, pp = h->pressure.par, pd = h->dye.par;
        const LaunchCounts n0 = h->launches;
        cudaGraph_t g = nullptr;
        CU(cudaStreamBeginCapture(h->stream, cudaStreamCaptureModeThreadLocal));
        h->capturing = true;
        int rc = step_enqueue(h, false);
        h->capturing = false;
        cudaError_t e = cudaStreamEndCapture(h->stream, &g);
        if (rc) { if (g) cudaGraphDestroy(g); return rc; }
        if (e != cudaSuccess) return fail(h, FLUID_ERR_CUDA, "stream capture of step() failed: %s", cudaGetErrorString(e));
        fluid::StepGraph sg;
        e = cudaGraphInstantiate(&sg.exec, g, 0);
        cudaGraphDestroy(g);
        if (e != cudaSuccess) return fail(h, FLUID_ERR_CUDA, "cudaGraphInstantiate failed: %s", cudaGetErrorString(e));
        sg.flip_v = pv ^ h->velocity.par; sg.flip_p = pp ^ h->pressure.par; sg.flip_dye = pd ^ h->dye.par;
        sg.launches = h->launches - n0;
        h->launches = n0;                                   // captured, not yet executed
        ++h->graph_captures;
        it = h->graphs.emplace(key, sg).first;
        // the capture already performed the host-side swaps of this step
    } else {
        const fluid::StepGraph& sg = it->second;
        if (sg.flip_v) h->velocity.swap();
        if (sg.flip_p) h->pressure.swap();
        if (sg.flip_dye) h->dye.swap();
    }
    CU(cudaGraphLaunch(it->second.exec, h->stream));
    h->launches += it->second.launches;
    h->timing.jacobi_launches = (int)it->second.launches.jacobi;
    h->timing.total_launches = (int)it->second.launches.all;
    h->have_timing = false;
    ++h->graph_launches;
    return FLUID_OK;
}

int fluid_step(fluid_t* h, float dt) {
    if (!h) return FLUID_ERR_INVALID;
    { int rc = set_dt(h, dt); if (rc) return rc; }
    return step_after_dt(h);
}

int fluid_step_members(fluid_t* h, const float* dt, int n) {
    if (!h) return FLUID_ERR_INVALID;
    if (int rc = check_members(h, "fluid_step_members", dt, n)) return rc;
    std::copy(dt, dt + n, h->member_host.begin() + (size_t)MP_DT * n);
    if (int rc = upload_member_row(h, MP_DT)) return rc;
    return step_after_dt(h);
}

static SplatPlane splat_plane(const Grid& g) {
    SplatPlane p{};
    p.g = g; p.pow2 = is_pow2(g.W) && is_pow2(g.H);
    p.tsx = (float)(1.0 / (double)g.W); p.tsy = (float)(1.0 / (double)g.H);
    p.bx = (g.W + SPL_BW - 1) / SPL_BW;
    return p;
}
static int splat_blocks(const SplatPlane& p) { return p.bx * ((p.g.j_hi - p.g.j_lo + SPL_BH - 1) / SPL_BH); }

// what every splat launch shares: correctRadius(config.SPLAT_RADIUS / 100.0) and the aspect
static SplatsArgs splats_args(const fluid_t* h) {
    SplatsArgs a{};
    a.radius = splat_radius(h->splat_radius_d, h->aspect_d);
    a.aspect = h->cfg.aspect;
    return a;
}

// n x splat(x,y,dx,dy,color) of S:1441-1455, in order, SPLATS_PER_LAUNCH records per launch
int fluid_splats(fluid_t* h, const float* splats, int n) {
    if (!h) return FLUID_ERR_INVALID;
    if (h->batch) return not_on_batch(h, "fluid_splats");
    if (n < 0 || (n > 0 && !splats)) return fail(h, FLUID_ERR_INVALID, "fluid_splats: bad record block (%d records at %p)", n, (const void*)splats);
    if (n == 0) return FLUID_OK;
    static_assert(sizeof(SplatRec) == 7 * sizeof(float), "records are 7 packed floats");
    static_assert(sizeof(SplatsArgs) <= 4096, "the records travel in the 4 KB kernel parameter block");
    SplatsArgs a = splats_args(h);
    // a splat is point-wise, so the +-3 velocity ghost rows of a slab are simply splatted as well
    a.v = splat_plane(sim_grid_ext(h, h->slab() ? 3 : 0));
    a.d = splat_plane(dye_grid(h));
    a.blocks_v = splat_blocks(a.v);
    const int blocks = a.blocks_v + splat_blocks(a.d);
    for (int k0 = 0; k0 < n; k0 += SPLATS_PER_LAUNCH) {
        a.n = std::min(n - k0, SPLATS_PER_LAUNCH);
        memcpy(a.rec, splats + 7 * (size_t)k0, (size_t)a.n * sizeof(SplatRec));
        // the first launch reads .read; the next ones continue in place on .write
        const void* vin = k0 ? h->velocity.write : h->velocity.read;
        const void* din = k0 ? h->dye.write : h->dye.read;
        int rc = with_storage(h, [&](auto s) {
            using S = decltype(s);
            splats_kernel<S><<<blocks, 256, 0, h->stream>>>((const typename S::T2*)vin, (typename S::T2*)h->velocity.write,
                                                            (const typename S::T4*)din, (typename S::T4*)h->dye.write, a);
            return check_launch(h, "splats_kernel");
        });
        if (rc) return rc;
    }
    h->velocity.swap();                          // S:1449
    h->dye.swap();                               // S:1454
    return FLUID_OK;
}

// Record k to member[k] of a batch handle.  The records are ordered by member (stably: each member keeps
// the call order) and cut into launches of at most SPLATS_PER_LAUNCH records in SPLAT_GROUPS member groups.
// Each launch updates its members' .read in place and launches no block for any other member: a splat is
// point-wise, so the bits are those of fluid_splats' read-write-swap on an ordinary handle.
int fluid_splats_batch(fluid_t* h, const int32_t* member, const float* splats, int n) {
    if (!h) return FLUID_ERR_INVALID;
    if (!h->batch) return fail(h, FLUID_ERR_INVALID, "fluid_splats_batch needs a batch handle (fluid_create_batch)");
    if (n < 0 || (n > 0 && (!member || !splats)))
        return fail(h, FLUID_ERR_INVALID, "fluid_splats_batch: bad record block (%d records)", n);
    for (int k = 0; k < n; ++k)
        if (member[k] < 0 || member[k] >= h->members)
            return fail(h, FLUID_ERR_INVALID, "fluid_splats_batch: record %d names member %d of %d", k, member[k], h->members);
    if (n == 0) return FLUID_OK;
    std::vector<int> order(n);
    for (int k = 0; k < n; ++k) order[k] = k;
    std::stable_sort(order.begin(), order.end(), [&](int x, int y) { return member[x] < member[y]; });
    SplatsArgs a = splats_args(h);
    a.v = splat_plane(sim_grid(h));
    a.d = splat_plane(dye_grid(h));
    a.blocks_v = splat_blocks(a.v);
    const int blocks = a.blocks_v + splat_blocks(a.d);
    SplatGroups g{};
    int ng = 0;
    a.n = 0;
    auto flush = [&]() {
        g.start[ng] = (unsigned char)a.n;
        splats_batch_kernel<<<dim3(blocks, ng), 256, 0, h->stream>>>((float2*)h->velocity.read, (float4*)h->dye.read, a, g,
                                                                     h->dt_dev + (size_t)MP_RADIUS * h->members);
        a.n = 0; ng = 0;
        return check_launch(h, "splats_batch_kernel");
    };
    for (int k = 0; k < n; ++k) {
        const int r = order[k], m = member[r];
        const bool new_group = ng == 0 || g.member[ng - 1] != m;
        if (a.n == SPLATS_PER_LAUNCH || (new_group && ng == SPLAT_GROUPS)) {
            if (int rc = flush()) return rc;
        }
        if (ng == 0 || g.member[ng - 1] != m) { g.member[ng] = m; g.start[ng] = (unsigned char)a.n; ++ng; }
        memcpy(&a.rec[a.n++], splats + 7 * (size_t)r, sizeof(SplatRec));
    }
    return flush();
}

static int check_device_buf(fluid_t* h, const char* what, const void* p, size_t bytes);   // data in / out, below

// fluid_splats from device memory: one launch applies all n records, each tile reading and writing its texels once
int fluid_splats_device(fluid_t* h, const float* splats, int n) {
    const char* what = "fluid_splats_device";
    if (!h) return FLUID_ERR_INVALID;
    if (h->batch) return not_on_batch(h, what);
    if (h->slab()) return not_on_slab(h, what);
    if (n < 0 || (n > 0 && !splats)) return fail(h, FLUID_ERR_INVALID, "%s: bad record block (%d records at %p)", what, n, (const void*)splats);
    if (n == 0) return FLUID_OK;
    if (int rc = check_device_buf(h, what, splats, 7 * sizeof(float) * (size_t)n)) return rc;
    SplatsDeviceArgs a{};
    a.radius = splat_radius(h->splat_radius_d, h->aspect_d);
    a.aspect = h->cfg.aspect;
    a.v = splat_plane(sim_grid(h));
    a.d = splat_plane(dye_grid(h));
    a.blocks_v = splat_blocks(a.v);
    a.n = n;
    a.rec = splats;
    const int blocks = a.blocks_v + splat_blocks(a.d);
    int rc = with_storage(h, [&](auto s) {
        using S = decltype(s);
        splats_device_kernel<S><<<blocks, 256, 0, h->stream>>>((const typename S::T2*)h->velocity.read, (typename S::T2*)h->velocity.write,
                                                               (const typename S::T4*)h->dye.read, (typename S::T4*)h->dye.write, a);
        return check_launch(h, "splats_device_kernel");
    });
    if (rc) return rc;
    h->velocity.swap();                          // S:1449
    h->dye.swap();                               // S:1454
    return FLUID_OK;
}

// The scratch of fluid_splats_batch_device, at least `bytes`.  It grows outside any capture: a graph must not
// hold an allocation, and the old buffer may still be in use by queued launches.
static int need_splat_scratch(fluid_t* h, size_t bytes) {
    if (bytes <= h->splat_scratch_bytes) return FLUID_OK;
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    CU(cudaStreamIsCapturing(h->stream, &cs));
    if (h->capturing || cs != cudaStreamCaptureStatusNone)
        return fail(h, FLUID_ERR_INVALID, "fluid_splats_batch_device: the splat scratch cannot grow during a graph capture");
    CU(cudaStreamSynchronize(h->stream));
    cudaFree(h->splat_scratch); h->splat_scratch = nullptr; h->splat_scratch_bytes = 0;
    bytes = std::max(bytes, (size_t)64 << 10);
    if (cudaMalloc((void**)&h->splat_scratch, bytes) != cudaSuccess) {
        cudaGetLastError();                      // not sticky: keep it out of the next launch check
        h->splat_scratch = nullptr;
        return fail(h, FLUID_ERR_NOMEM, "fluid_splats_batch_device: out of device memory for %zu bytes of splat scratch", bytes);
    }
    h->splat_scratch_bytes = bytes;
    return FLUID_OK;
}

// fluid_splats_batch from device memory in two launches whatever n, B or the spread of the records: a grouping
// launch (splat_group_kernel) checks the member indices and orders the records by member, and one splat launch
// applies each named member's records in place on its .read.  An index outside [0, B) cannot be seen here without
// a sync: the grouping launch then names no member, so nothing is splatted, and sets the device error word that
// the next fluid_sync reports.
int fluid_splats_batch_device(fluid_t* h, const int32_t* member, const float* splats, int n) {
    const char* what = "fluid_splats_batch_device";
    if (!h) return FLUID_ERR_INVALID;
    if (!h->batch) return fail(h, FLUID_ERR_INVALID, "%s needs a batch handle (fluid_create_batch)", what);
    if (n < 0 || (n > 0 && (!member || !splats)))
        return fail(h, FLUID_ERR_INVALID, "%s: bad record block (%d records)", what, n);
    if (n == 0) return FLUID_OK;
    if (int rc = check_device_buf(h, what, member, sizeof(int32_t) * (size_t)n)) return rc;
    if (int rc = check_device_buf(h, what, splats, 7 * sizeof(float) * (size_t)n)) return rc;
    const SplatGroupLayout L = splat_group_layout(n, h->members);
    if (int rc = need_splat_scratch(h, L.ints * sizeof(int) + 7 * sizeof(float) * (size_t)n)) return rc;
    splat_group_kernel<<<1, GROUP_THREADS, 0, h->stream>>>(member, splats, n, h->members, h->splat_scratch, h->halo_flag);
    if (int rc = check_launch(h, "splat_group_kernel")) return rc;
    SplatsBatchDeviceArgs a{};
    a.aspect = h->cfg.aspect;
    a.v = splat_plane(sim_grid(h));
    a.d = splat_plane(dye_grid(h));
    a.blocks_v = splat_blocks(a.v);
    a.g = h->splat_scratch;
    a.named = L.named; a.start = L.start;
    a.rec = reinterpret_cast<const float*>(h->splat_scratch + L.ints);
    a.radius = h->dt_dev + (size_t)MP_RADIUS * h->members;
    const int tiles = a.blocks_v + splat_blocks(a.d);
    // enough member rows for about 16 blocks per SM, and never more than can be named
    const int rows = std::min({n, h->members, std::max(1, 16 * h->sm_count / tiles)});
    splats_batch_device_kernel<<<dim3(tiles, rows), 256, 0, h->stream>>>((float2*)h->velocity.read, (float4*)h->dye.read, a);
    return check_launch(h, "splats_batch_device_kernel");
}

// splat(x,y,dx,dy,color), S:1441-1455
int fluid_splat(fluid_t* h, float x, float y, float dx, float dy, float r, float g, float b) {
    const float rec[7] = {x, y, dx, dy, r, g, b};
    return fluid_splats(h, rec, 1);
}

// initFramebuffers() on a live simulation: S:982-1010 + resizeDoubleFBO S:1116-1126
int fluid_resize(fluid_t* h, int sim_w, int sim_h, int dye_w, int dye_h) {
    if (!h) return FLUID_ERR_INVALID;
    if (h->batch) return not_on_batch(h, "fluid_resize");
    if (sim_w < 1 || sim_h < 1 || dye_w < 1 || dye_h < 1) return fail(h, FLUID_ERR_INVALID, "bad size");
    const int ow = h->cfg.sim_w, oh = h->cfg.sim_h, odw = h->cfg.dye_w, odh = h->cfg.dye_h;
    int rc;
    if (h->slab()) {
        // Collective among the ranks of the group (all call it with the same sizes).  The new rows a rank
        // owns sample old rows it owns +- ceil(old/new) + 2: refresh that many ghost rows of the old
        // velocity and dye.
        const int need_v = (oh + sim_h - 1) / sim_h + 2, need_d = (odh + dye_h - 1) / dye_h + 2;
        if (need_v > h->G || need_d > h->Gd)
            return fail(h, FLUID_ERR_HALO, "resize by this factor needs %d / %d ghost rows, the slab keeps %d / %d", need_v, need_d, h->G, h->Gd);
        if ((rc = exchange_rows(h, HB_VELOCITY, need_v))) return rc;
        if ((rc = exchange_rows(h, HB_DYE, need_d))) return rc;
    }
    SlabGeometry g;
    if (!slab_geometry(&g, h->rank, h->world, sim_h, dye_h, h->cfg.pressure_iterations))
        return fail(h, FLUID_ERR_INVALID, "new slabs of %d rows are too short for a 14-row halo", sim_h / h->world);
    // the new arena first: if it does not fit, the handle stays as it was
    const FieldLayout L = field_layout(h, (size_t)sim_w * g.lrows(), (size_t)dye_w * g.ldrows());
    char* a = nullptr;
    if ((rc = make_arena(h, L, (size_t)dye_w * g.ldrows(), &a))) return rc;
    // velocity and dye of the rows this rank owns, into the slots their pairs read next; pressure, divergence
    // and curl start over at zero
    rc = with_storage(h, [&](auto s) {
        using S = decltype(s);
        const int r = carry_field<S, typename S::T2>(h, h->velocity.read, ow, oh, h->roff, a + L.v[h->velocity.par],
                                                     sim_w, sim_h, g.roff, g.row0, g.row1);
        return r ? r : carry_field<S, typename S::T4>(h, h->dye.read, odw, odh, h->droff, a + L.dye[h->dye.par],
                                                       dye_w, dye_h, g.droff, g.drow0, g.drow1);
    });
    const cudaError_t e = cudaStreamSynchronize(h->stream);
    if (!rc && e != cudaSuccess) rc = fail(h, FLUID_ERR_CUDA, "resize of the fields failed: %s", cudaGetErrorString(e));
    if (rc) { cudaFree(a); return rc; }
    drop_graphs(h);                                          // graphs hold the old buffers' addresses
    // slab: the neighbours' mappings die with the old arena, so the group is back on NCCL until the launcher
    // exports / connects again (distributed.connect_peers); the +-3 velocity ghost rows are rebuilt by the next step
    close_peers(h);
    h->v_ghost_valid = false;
    cudaFree(h->arena);
    h->cfg.sim_w = sim_w; h->cfg.sim_h = sim_h; h->cfg.dye_w = dye_w; h->cfg.dye_h = dye_h;
    static_cast<SlabGeometry&>(*h) = g;
    return adopt_arena(h, a, L);
}

// ---- data in / out --------------------------------------------------------------------------------

// a batch handle's fields hold all members: B x w x rows x channels floats
size_t fluid_field_elems(fluid_t* h, int field) {
    void* p; int w, rows, ch;
    if (!h || field_info(h, field, &p, &w, &rows, &ch)) return 0;
    return (size_t)w * rows * ch * h->members;
}

int fluid_field_dims(fluid_t* h, int field, int* w, int* rows, int* ch, int* row0) {
    void* p; int ww, rr, cc;
    if (!h || field_info(h, field, &p, &ww, &rr, &cc)) return FLUID_ERR_INVALID;
    if (w) *w = ww; if (rows) *rows = rr; if (ch) *ch = cc;
    if (row0) *row0 = (field == FLUID_FIELD_DYE) ? h->drow0 : h->row0;
    return FLUID_OK;
}

int fluid_read(fluid_t* h, int field, float* host, size_t n_floats) {
    void* p; int w, rows, ch;
    if (!h || !host || field_info(h, field, &p, &w, &rows, &ch)) return fail(h, FLUID_ERR_INVALID, "bad field %d", field);
    const size_t n = (size_t)w * rows * ch * h->members;
    if (n_floats != n) return fail(h, FLUID_ERR_INVALID, "field %d has %zu floats, caller passed %zu", field, n, n_floats);
    if (h->half) {                                   // the ABI speaks fp32: widen on the device, then copy
        int rc = need_scratch(h, n); if (rc) return rc;
        hs::widen_kernel<<<(unsigned)((n + 255) / 256), 256, 0, h->stream>>>((const hs::h1*)p, h->scratch, n);
        if ((rc = check_launch(h, "hs::widen_kernel"))) return rc;
        p = h->scratch;
    }
    CU(cudaMemcpyAsync(host, p, n * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    return check_halo(h);
}

int fluid_write(fluid_t* h, int field, const float* host, size_t n_floats) {
    void* p; int w, rows, ch;
    if (!h || !host || field_info(h, field, &p, &w, &rows, &ch)) return fail(h, FLUID_ERR_INVALID, "bad field %d", field);
    const size_t n = (size_t)w * rows * ch * h->members;
    if (n_floats != n) return fail(h, FLUID_ERR_INVALID, "field %d has %zu floats, caller passed %zu", field, n, n_floats);
    if (h->half) {                                   // narrow with round-to-nearest-even, like a texture upload would
        int rc = need_scratch(h, n); if (rc) return rc;
        CU(cudaMemcpyAsync(h->scratch, host, n * sizeof(float), cudaMemcpyHostToDevice, h->stream));
        hs::narrow_kernel<<<(unsigned)((n + 255) / 256), 256, 0, h->stream>>>(h->scratch, (hs::h1*)p, n);
        if ((rc = check_launch(h, "hs::narrow_kernel"))) return rc;
        CU(cudaStreamSynchronize(h->stream));
        return FLUID_OK;
    }
    CU(cudaMemcpyAsync(p, host, n * sizeof(float), cudaMemcpyHostToDevice, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    if (field == FLUID_FIELD_VELOCITY) h->v_ghost_valid = false;   // ghosts rebuilt by the next step
    if (field == FLUID_FIELD_DIVERGENCE) {                          // host-provided divergence: rebuild the map
        int rc = clear_tiny_map(h); if (rc) return rc;
        if ((rc = scan_tiny(h, h->row0, h->row1))) return rc;
    }
    return FLUID_OK;
}

// A caller's device buffer [p, p + bytes): device or managed memory of the handle's device, 4-byte aligned
// (float and uchar4 accesses), and outside the field arena, where it would alias a field.
static int check_device_buf(fluid_t* h, const char* what, const void* p, size_t bytes) {
    cudaPointerAttributes at{};
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
        cudaGetLastError();                      // not sticky: keep it out of the next launch check
        return fail(h, FLUID_ERR_INVALID, "%s: the buffer is not a pointer CUDA knows", what);
    }
    if ((at.type != cudaMemoryTypeDevice && at.type != cudaMemoryTypeManaged) || at.device != h->device)
        return fail(h, FLUID_ERR_INVALID, "%s needs device or managed memory of device %d (the buffer is %s memory of "
                    "device %d)", what, h->device, at.type == cudaMemoryTypeHost ? "pinned host" : at.type == cudaMemoryTypeUnregistered
                    ? "pageable host" : "device or managed", at.device);
    if ((uintptr_t)p % 4)
        return fail(h, FLUID_ERR_INVALID, "%s: a device buffer must be 4-byte aligned", what);
    const uintptr_t a = (uintptr_t)h->arena, q = (uintptr_t)p;
    if (q < a + h->layout.bytes && a < q + bytes)
        return fail(h, FLUID_ERR_INVALID, "%s: the buffer overlaps the handle's field arena", what);
    return FLUID_OK;
}

// The checks fluid_read_device / fluid_write_device share; *p / *n: the field's owned rows and their floats.
static int device_io_args(fluid_t* h, const char* what, int field, const void* buf, size_t n_floats, void** p, size_t* n) {
    int w, rows, ch;
    if (!h) return FLUID_ERR_INVALID;
    if (field_info(h, field, p, &w, &rows, &ch)) return fail(h, FLUID_ERR_INVALID, "%s: bad field %d", what, field);
    *n = (size_t)w * rows * ch * h->members;
    if (n_floats != *n) return fail(h, FLUID_ERR_INVALID, "%s: field %d has %zu floats, caller passed %zu", what, field, *n, n_floats);
    if (!buf) return fail(h, FLUID_ERR_INVALID, "%s: NULL buffer", what);
    if (h->slab()) return not_on_slab(h, what);
    return check_device_buf(h, what, buf, *n * sizeof(float));
}

// fluid_read into device memory: the same bits, stream-ordered, no host copy and no sync.  Half storage widens
// straight into the caller's buffer, so the call allocates nothing.
int fluid_read_device(fluid_t* h, int field, float* dst, size_t n_floats) {
    void* p = nullptr; size_t n = 0;
    int rc = device_io_args(h, "fluid_read_device", field, dst, n_floats, &p, &n);
    if (rc) return rc;
    if (h->half) {
        hs::widen_kernel<<<(unsigned)((n + 255) / 256), 256, 0, h->stream>>>((const hs::h1*)p, dst, n);
        return check_launch(h, "hs::widen_kernel");
    }
    CU(cudaMemcpyAsync(dst, p, n * sizeof(float), cudaMemcpyDeviceToDevice, h->stream));
    return FLUID_OK;
}

// fluid_write from device memory: the field ends with the bits fluid_write leaves, stream-ordered.  Written
// divergence rebuilds the tiny-divergence map on the stream, as after a host write.
int fluid_write_device(fluid_t* h, int field, const float* src, size_t n_floats) {
    void* p = nullptr; size_t n = 0;
    int rc = device_io_args(h, "fluid_write_device", field, src, n_floats, &p, &n);
    if (rc) return rc;
    if (h->half) {
        hs::narrow_kernel<<<(unsigned)((n + 255) / 256), 256, 0, h->stream>>>(src, (hs::h1*)p, n);
        return check_launch(h, "hs::narrow_kernel");
    }
    CU(cudaMemcpyAsync(p, src, n * sizeof(float), cudaMemcpyDeviceToDevice, h->stream));
    if (field == FLUID_FIELD_DIVERGENCE) {
        if ((rc = clear_tiny_map(h))) return rc;
        if ((rc = scan_tiny(h, h->row0, h->row1))) return rc;
    }
    return FLUID_OK;
}

// ---- member subsets of a batch handle ----------------------------------------------------------------------

// The member list of a member-subset call: n distinct indices in [0, B) on a batch handle, checked on the host
// before any work.  n == 0 passes; the call then does nothing.
static int check_member_list(fluid_t* h, const char* what, const int32_t* members, int n) {
    if (!h->batch) return fail(h, FLUID_ERR_INVALID, "%s needs a batch handle (fluid_create_batch)", what);
    if (n < 0 || (n > 0 && !members))
        return fail(h, FLUID_ERR_INVALID, "%s: bad member list (%d members at %p)", what, n, (const void*)members);
    std::vector<char> seen(h->members, 0);
    for (int k = 0; k < n; ++k) {
        const int32_t m = members[k];
        if (m < 0 || m >= h->members)
            return fail(h, FLUID_ERR_INVALID, "%s: members[%d] = %d is outside [0, %d)", what, k, m, h->members);
        if (seen[m]++) return fail(h, FLUID_ERR_INVALID, "%s: member %d is listed twice", what, m);
    }
    return FLUID_OK;
}

// A checked list into the handle's list buffer, which the launches of the call read: stream-ordered, from pageable
// memory like upload_member_row, so a list buffer still in use by queued work is overwritten only after it.
static int upload_member_list(fluid_t* h, const int32_t* members, int n) {
    CU(cudaMemcpyAsync(h->member_list, members, (size_t)n * sizeof(int32_t), cudaMemcpyHostToDevice, h->stream));
    return FLUID_OK;
}

// The looks of n images (looks.h image_look) into the handle's look table, which the launches of the draw read:
// one stream-ordered copy from pageable memory, like upload_member_list.
static int upload_looks(fluid_t* h, const fluid_look* looks, int n) {
    std::vector<fk::ImageLook> t(n);
    for (int k = 0; k < n; ++k) t[k] = fk::image_look(looks[k]);
    CU(cudaMemcpyAsync(h->look_table, t.data(), (size_t)n * sizeof(fk::ImageLook), cudaMemcpyHostToDevice, h->stream));
    return FLUID_OK;
}

// The checks fluid_read_members / fluid_write_members share, all before any work; *p: the field's .read, *per:
// the floats of one member
static int members_io_args(fluid_t* h, const char* what, int field, const int32_t* members, int n, const void* buf,
                           size_t n_floats, int on_device, float** p, size_t* per) {
    void* q; int w, rows, ch;
    if (!h) return FLUID_ERR_INVALID;
    if (field_info(h, field, &q, &w, &rows, &ch)) return fail(h, FLUID_ERR_INVALID, "%s: bad field %d", what, field);
    if (int rc = check_member_list(h, what, members, n)) return rc;
    *p = (float*)q;
    *per = (size_t)w * rows * ch;
    if (n_floats != *per * n)
        return fail(h, FLUID_ERR_INVALID, "%s: %d members of field %d have %zu floats, caller passed %zu", what, n, field,
                    *per * n, n_floats);
    if (n == 0) return FLUID_OK;
    if (!buf) return fail(h, FLUID_ERR_INVALID, "%s: NULL buffer", what);
    return on_device ? check_device_buf(h, what, buf, n_floats * sizeof(float)) : FLUID_OK;
}

// One launch moving the listed members' blocks of `per` floats between a field and the caller's device buffer,
// in 16-byte words when the buffer is 16-byte aligned (the member blocks always are)
static int launch_member_copy(fluid_t* h, bool to_buf, float* field, float* buf, size_t per, int n) {
    const bool v4 = (uintptr_t)buf % 16 == 0;
    const size_t units = v4 ? per / 4 : per;
    const dim3 g((unsigned)std::min<size_t>((units + 255) / 256, 1024), 1, n);
    if (v4 && to_buf) member_copy_kernel<float4, true><<<g, 256, 0, h->stream>>>((const float4*)field, (float4*)buf, h->member_list, units);
    else if (v4) member_copy_kernel<float4, false><<<g, 256, 0, h->stream>>>((const float4*)buf, (float4*)field, h->member_list, units);
    else if (to_buf) member_copy_kernel<float, true><<<g, 256, 0, h->stream>>>(field, buf, h->member_list, units);
    else member_copy_kernel<float, false><<<g, 256, 0, h->stream>>>(buf, field, h->member_list, units);
    return check_launch(h, "member_copy_kernel");
}

// fluid_read for the listed members: slot k of dst is member members[k].  Into host memory one copy per member
// straight from the arena, then a sync; into device memory one gather launch, stream-ordered.
int fluid_read_members(fluid_t* h, int field, const int32_t* members, int n, float* dst, size_t n_floats, int dst_on_device) {
    float* p = nullptr; size_t per = 0;
    int rc = members_io_args(h, "fluid_read_members", field, members, n, dst, n_floats, dst_on_device, &p, &per);
    if (rc || n == 0) return rc;
    if (dst_on_device) {
        if ((rc = upload_member_list(h, members, n))) return rc;
        return launch_member_copy(h, true, p, dst, per, n);
    }
    for (int k = 0; k < n; ++k)
        CU(cudaMemcpyAsync(dst + k * per, p + (size_t)members[k] * per, per * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    return check_halo(h);
}

// fluid_write for the listed members, .read only; every other member keeps every byte.  Written divergence
// leaves the tiny-divergence map alone: every batch step clears and rebuilds it (cvd_stream_kernel<true>) before
// the blocked solve reads it, and no other batch call reads it.
int fluid_write_members(fluid_t* h, int field, const int32_t* members, int n, const float* src, size_t n_floats, int src_on_device) {
    float* p = nullptr; size_t per = 0;
    int rc = members_io_args(h, "fluid_write_members", field, members, n, src, n_floats, src_on_device, &p, &per);
    if (rc || n == 0) return rc;
    if (src_on_device) {
        if ((rc = upload_member_list(h, members, n))) return rc;
        return launch_member_copy(h, false, p, const_cast<float*>(src), per, n);
    }
    for (int k = 0; k < n; ++k)
        CU(cudaMemcpyAsync(p + (size_t)members[k] * per, src + k * per, per * sizeof(float), cudaMemcpyHostToDevice, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    return FLUID_OK;
}

// The listed members back to the state fluid_create_batch leaves, both slots of every pair, in one launch.  Their
// per-member values are config and stay; no step graph is recaptured (a reset member's slots are alike).
int fluid_reset_members(fluid_t* h, const int32_t* members, int n) {
    if (!h) return FLUID_ERR_INVALID;
    int rc = check_member_list(h, "fluid_reset_members", members, n);
    if (rc || n == 0) return rc;
    if ((rc = upload_member_list(h, members, n))) return rc;
    const size_t sv = sim_cells(h) / 2, ss = sim_cells(h) / 4, sd = dye_cells(h);   // float4 per member
    const MemberSlots s{{(float4*)h->dye.read, (float4*)h->dye.write, (float4*)h->velocity.read, (float4*)h->velocity.write,
                         (float4*)h->pressure.read, (float4*)h->pressure.write, (float4*)h->divergence, (float4*)h->curl},
                        {sd, sd, sv, sv, ss, ss, ss, ss}};
    const dim3 g((unsigned)std::min<size_t>((sd + 255) / 256, 1024), 1, n);
    member_reset_kernel<<<g, 256, 0, h->stream>>>(s, h->member_list);
    return check_launch(h, "member_reset_kernel");
}

// fluid_pressure_solve_host on one GPU is PCIe-bound (4096^2: 128 MiB up, 64 MiB down per call), so
// the solve is hidden behind the copies: the grid is cut into row bands, band b is solved as soon as its rows
// (+ `iters` rows beyond it) have arrived and is copied back while the later bands still upload — the slab
// decomposition of section 7 applied in time instead of across GPUs, the host standing in for the
// neighbours.  Communication-avoiding schedule as on a slab: launch k of a band produces its rows +- (sweeps
// still to come), out of band-private ping-pong rows; the first launch reads the uploaded field, the last one
// writes the band's rows of the result field.  Bit-identical to the one-piece solve (same kernel, same
// per-cell arithmetic; which rows a launch covers does not enter the values).
int solve_host_banded(fluid_t* h, const float* div_host, float* p_host, int iters, int nb) {
    const int W = h->cfg.sim_w, H = h->cfg.sim_h;
    fluid::HostPipe& hp = h->hp;
    if (!hp.up) {
        CU(cudaStreamCreateWithFlags(&hp.up, cudaStreamNonBlocking));
        CU(cudaStreamCreateWithFlags(&hp.down, cudaStreamNonBlocking));
        CU(cudaEventCreateWithFlags(&hp.ev_start, cudaEventDisableTiming));
        for (auto& e : hp.ev_up) CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        for (auto& e : hp.ev_done) CU(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    }
    const JacobiPlan plan(iters, block_depth(h, true));
    const int band = (H + nb - 1) / nb, halo = iters;
    // band-private rows [loc, loc + band + 2*halo): every row a launch of band [b_lo, b_hi) reads or writes lies
    // in [max(b_lo - halo, 0), b_hi + halo).  Boxes staged beyond a map's rows read as zero, and rows past what
    // a launch wrote never reach a valid output, as on the whole grid.
    const size_t need = (size_t)(band + 2 * halo) * W;
    if (hp.s_floats < need) {
        cudaFree(hp.s[0]); cudaFree(hp.s[1]); hp.s[0] = hp.s[1] = nullptr; hp.s_floats = 0;
        CU(cudaMalloc((void**)&hp.s[0], need * sizeof(float)));
        CU(cudaMalloc((void**)&hp.s[1], need * sizeof(float)));
        hp.s_floats = need;
    }
    float* const p_in = (float*)h->pressure.read;
    float* const result = (float*)h->pressure.write;
    // tensor maps of what the launches of a band read, all from the band's local row 0: launch 0 reads the
    // uploaded field (m[0]), launch k > 0 the band-private rows s[(k-1)&1] (m[1 + ((k-1)&1)]); the band's
    // divergence maps are filled in per band
    TmapPair m[3];
    int rc = FLUID_OK;
    for (int k = 0; k < 2 && !rc; ++k) rc = encode_rows_map(h, m[1 + k].p, hp.s[k], W, band + 2 * halo);
    if (rc) return rc;
    if ((rc = clear_tiny_map(h))) return rc;
    CU(cudaEventRecord(hp.ev_start, h->stream));          // the copies overwrite fields earlier work on the stream may still read
    CU(cudaStreamWaitEvent(hp.up, hp.ev_start, 0));
    for (int b = 0; b < nb; ++b) {
        const int b_lo = std::min(b * band, H), b_hi = std::min(b_lo + band, H);
        if (b_hi <= b_lo) break;
        // upload chunk b = what band b needs beyond what the earlier chunks brought: rows up to b_hi + halo
        const int up_lo = b == 0 ? 0 : std::min(b_lo + halo, H), up_hi = (b_hi == H) ? H : std::min(b_hi + halo, H);
        if (up_hi > up_lo) {
            const size_t o = (size_t)up_lo * W, n = (size_t)(up_hi - up_lo) * W * sizeof(float);
            CU(cudaMemcpyAsync(h->divergence + o, div_host + o, n, cudaMemcpyHostToDevice, hp.up));
            CU(cudaMemcpyAsync(p_in + o, p_host + o, n, cudaMemcpyHostToDevice, hp.up));
        }
        CU(cudaEventRecord(hp.ev_up[b], hp.up));
        CU(cudaStreamWaitEvent(h->stream, hp.ev_up[b], 0));
        if ((rc = scan_tiny(h, up_lo, up_hi))) return rc;
        // global row of local row 0 of the band-private rows.  No launch of the band reads a row below
        // b_lo - halo, or below row 0, so every field is passed from a row inside its allocation.
        const int loc = std::max(b_lo - halo, 0);
        if ((rc = encode_rows_map(h, m[0].p, p_in + (ptrdiff_t)loc * W, W, H - loc))) return rc;
        if ((rc = encode_rows_map(h, m[0].d, h->divergence + (ptrdiff_t)loc * W, W, H - loc))) return rc;
        memcpy(m[1].d, m[0].d, sizeof m[0].d);
        memcpy(m[2].d, m[0].d, sizeof m[0].d);
        for (int k = 0; k < plan.n; ++k) {
            // the kernel addresses all three fields as "local row 0 + (row - row_off)": a whole-grid field G is
            // passed as G + loc*W
            JacobiArgs a = jacobi_args(h, h->divergence + (ptrdiff_t)loc * W, loc);
            a.out_lo = std::max(b_lo - plan.after(k), 0); a.out_hi = std::min(b_hi + plan.after(k), H);
            a.pin = (k == 0) ? p_in + (ptrdiff_t)loc * W : hp.s[(k - 1) & 1];
            a.pout = (k == plan.n - 1) ? result + (ptrdiff_t)loc * W : hp.s[k & 1];
            // chained only behind the band's previous launch
            if ((rc = launch_tb(h, plan.depth(k), k == 0, k > 0, a, m[k == 0 ? 0 : 1 + ((k - 1) & 1)]))) return rc;
        }
        CU(cudaEventRecord(hp.ev_done[b], h->stream));
        CU(cudaStreamWaitEvent(hp.down, hp.ev_done[b], 0));
        const size_t o = (size_t)b_lo * W;
        CU(cudaMemcpyAsync(p_host + o, result + o, (size_t)(b_hi - b_lo) * W * sizeof(float), cudaMemcpyDeviceToHost, hp.down));
    }
    h->pressure.swap();                                   // pressure.read = the result, like S:1265 after the loop
    CU(cudaStreamSynchronize(hp.down));
    CU(cudaStreamSynchronize(h->stream));
    return FLUID_OK;
}

int fluid_pressure_solve_host(fluid_t* h, const float* div_host, float* p_host, int iters) {
    if (h && h->batch) return not_on_batch(h, "fluid_pressure_solve_host");
    if (!h || !div_host || !p_host || iters < 0) return fail(h, FLUID_ERR_INVALID, "bad argument");
    if (h->half) {
        int rc = fluid_write(h, FLUID_FIELD_DIVERGENCE, div_host, (size_t)h->cfg.sim_w * h->cfg.sim_h);
        if (!rc) rc = fluid_write(h, FLUID_FIELD_PRESSURE, p_host, (size_t)h->cfg.sim_w * h->cfg.sim_h);
        if (!rc) rc = run_jacobi(h, iters, true, nullptr);
        if (!rc) rc = fluid_read(h, FLUID_FIELD_PRESSURE, p_host, (size_t)h->cfg.sim_w * h->cfg.sim_h);
        return rc;
    }
    // one GPU, blocked kernel: solve band by band behind the copies, unless the grid is too short for two bands
    if (!h->slab() && iters > 0 && blocked(h, block_depth(h, true))) {
        const int nb = std::min(16, h->cfg.sim_h / std::max(256, 4 * iters));
        if (nb >= 2) return solve_host_banded(h, div_host, p_host, iters, nb);
    }
    const size_t n = (size_t)h->cfg.sim_w * (h->row1 - h->row0);   // owned rows
    const size_t go = (size_t)h->G * h->cfg.sim_w;
    // Host buffers may be pageable; pinned ones (cudaHostAlloc / cudaHostRegister by the caller)
    // make the copies asynchronous DMA.  Either way all three copies are inside this call.
    CU(cudaMemcpyAsync(h->divergence + go, div_host, n * sizeof(float), cudaMemcpyHostToDevice, h->stream));
    CU(cudaMemcpyAsync((float*)h->pressure.read + go, p_host, n * sizeof(float), cudaMemcpyHostToDevice, h->stream));
    int rc = clear_tiny_map(h); if (rc) return rc;
    if ((rc = scan_tiny(h, h->row0, h->row1))) return rc;
    rc = run_jacobi(h, iters, true, nullptr); if (rc) return rc;
    CU(cudaMemcpyAsync(p_host, (float*)h->pressure.read + go, n * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
    CU(cudaStreamSynchronize(h->stream));
    return FLUID_OK;
}

// The band of a width x height target this handle draws: the whole target on one GPU, rows
// [height*rank/world, height*(rank+1)/world) on a slab rank (the same fractions as the dye rows it owns).
int fluid_render_band(fluid_t* h, int height, int* y0, int* y1) {
    if (h && h->batch) return not_on_batch(h, "fluid_render_band");
    if (!h || height < 1 || !y0 || !y1) return FLUID_ERR_INVALID;
    *y0 = (int)((long long)height * h->rank / h->world);
    *y1 = (int)((long long)height * (h->rank + 1) / h->world);
    return FLUID_OK;
}

// The fp32 dye the display kernels sample: dye.read, or in half storage its widened copy in the scratch
// buffer (the sampler widens fp16 texels exactly; shading is fp32 as in the shader).
static int display_source(fluid_t* h, const float4** src) {
    *src = (const float4*)h->dye.read;
    if (!h->half) return FLUID_OK;
    const size_t nd = (size_t)h->cfg.dye_w * h->cfg.dye_h * 4;
    int rc = need_scratch(h, nd); if (rc) return rc;
    hs::widen_kernel<<<(unsigned)((nd + 255) / 256), 256, 0, h->stream>>>((const hs::h1*)h->dye.read, h->scratch, nd);
    if ((rc = check_launch(h, "hs::widen_kernel"))) return rc;
    *src = (const float4*)h->scratch;
    return FLUID_OK;
}

// (Re)allocates one post-FX target once the stream has drained.  Out of memory leaves it empty, so the
// handle stays usable and the next call tries again.
static int remake_target(fluid_t* h, void** p, size_t bytes, const char* what) {
    CU(cudaStreamSynchronize(h->stream));
    cudaFree(*p); *p = nullptr;
    if (cudaMalloc(p, bytes) != cudaSuccess) {
        cudaGetLastError();                      // not sticky: keep it out of the next launch check
        *p = nullptr;
        return fail(h, FLUID_ERR_NOMEM, "out of device memory for %s (%zu bytes)", what, bytes);
    }
    return FLUID_OK;
}

// grows the render target to at least `cells` RGBA texels (a batch draw's B images into host memory pass through
// it, so it is made like a post-FX target: out of memory leaves the handle usable)
static int need_frame(fluid_t* h, size_t cells) {
    if (cells <= h->frame_cells) return FLUID_OK;
    h->frame_cells = 0;
    if (int rc = remake_target(h, (void**)&h->frame, cells * sizeof(float4), "the frame buffer")) return rc;
    h->frame_cells = cells;
    return FLUID_OK;
}

// bytes per texel of the RGBA bloom targets and of the one-channel sunrays targets (fp16 with
// FLUID_FLAG_HALF_POSTFX, like the reference's RGBA16F / R16F FBOs)
inline size_t fx4bytes(const fluid_t* h) { return h->half_fx ? 8 : 16; }
inline size_t fx1bytes(const fluid_t* h) { return h->half_fx ? 2 : 4; }

// The bloom FBO and its pyramid (initBloomFramebuffers S:1012-1032), cleared like createFBO (S:1059).
// A pyramid shorter than 2 levels leaves the FBO as cleared (applyBloom returns early, S:1351-1352).
// A batch handle's FBO and each of its levels hold the B members back to back.
static int need_bloom_targets(fluid_t* h, int bw, int bh, int levels) {
    auto& t = h->pfx;
    if (t.bloom && t.bw == bw && t.bh == bh && t.levels == levels) return FLUID_OK;
    size_t n = (size_t)bw * bh;
    for (int i = 0; i < levels; ++i) n += (size_t)(bw >> (i + 1)) * (bh >> (i + 1));
    n *= h->members;
    t.bw = t.bh = t.levels = 0;
    if (int rc = remake_target(h, &t.bloom, n * fx4bytes(h), "the bloom FBO and pyramid")) return rc;
    t.bw = bw; t.bh = bh; t.levels = levels;
    const unsigned blocks = (unsigned)((n + 255) / 256);
    if (h->half_fx) fill_alpha_kernel<hs::StoreHalf><<<blocks, 256, 0, h->stream>>>((hs::h4*)t.bloom, n);   // (0,0,0,1) is exact in fp16
    else fill_alpha_kernel<<<blocks, 256, 0, h->stream>>>((float4*)t.bloom, n);
    return check_launch(h, "fill_alpha_kernel");
}

// sunrays + sunraysTemp (initSunraysFramebuffers S:1034-1043): one-channel FBOs, cleared to 0 (all-zero
// bits in fp32 and fp16 alike); on a batch handle each holds the B members back to back
static int need_sunrays_targets(fluid_t* h, int sw, int sh) {
    auto& t = h->pfx;
    if (t.sun && t.sw == sw && t.sh == sh) return FLUID_OK;
    const size_t bytes = 2 * (size_t)sw * sh * h->members * fx1bytes(h);
    t.sw = t.sh = 0;
    if (int rc = remake_target(h, &t.sun, bytes, "the sunrays FBOs")) return rc;
    t.sw = sw; t.sh = sh;
    CU(cudaMemsetAsync(t.sun, 0, bytes, h->stream));
    return FLUID_OK;
}

static int need_dither_target(fluid_t* h, int dw, int dh) {
    auto& t = h->pfx;
    if (t.dither && t.dw == dw && t.dh == dh) return FLUID_OK;
    t.dw = t.dh = 0;
    if (int rc = remake_target(h, (void**)&t.dither, (size_t)dw * dh * 3 * sizeof(float), "the dithering texture")) return rc;
    t.dw = dw; t.dh = dh;
    return FLUID_OK;
}

// slab SUNRAYS: the one-channel Wd x Hd buffer the ranks gather the mask's alpha into; made like a post-FX target
static int need_mask_target(fluid_t* h, int w, int hh) {
    auto& t = h->pfx;
    if (t.mask && t.mw == w && t.mh == hh) return FLUID_OK;
    t.mw = t.mh = 0;
    if (int rc = remake_target(h, (void**)&t.mask, (size_t)w * hh * sizeof(float), "the gathered sunrays mask")) return rc;
    t.mw = w; t.mh = hh;
    return FLUID_OK;
}

// Dye ghost rows a slab frame samples beyond the rows a rank owns (slab.py draw_ghost_rows).  A band starts at
// floor(n * rank / world) on every grid, so a target band may begin up to one target row before the dye rows it
// covers: the display + shading taps of a `height`-row target reach less than 1.5 Hd / height + 1.5 rows, the
// bloom prefilter's taps of a bh-row FBO less than Hd / (2 bh) + 1.5, the sunrays mask's (at dye texel centres)
// one.  bh = 0: no prefilter.  The same on every rank: the exchange sizes must match.
int draw_ghost_rows(int Hd, int height, int bh, bool mask) {
    long long need = (3LL * Hd + 2LL * height - 1) / (2LL * height) + 2;
    if (bh > 0) need = std::max(need, ((long long)Hd + 2LL * bh - 1) / (2LL * bh) + 2);
    if (mask) need = std::max(need, 1LL);
    return (int)std::min<long long>(need, 1 << 30);
}

// The FBO sizes of a frame's post-FX chains (initBloomFramebuffers / initSunraysFramebuffers, S:1012-1043, sized
// from the canvas_w x canvas_h drawing buffer) and the bloom pyramid's depth
struct PostFXOut { int bw, bh, sw, sh, levels; };
static int post_fx_sizes(fluid_t* h, uint32_t keywords, const fluid_postfx* fx, int canvas_w, int canvas_h, PostFXOut* o) {
    const bool bloom_on = keywords & FLUID_DISPLAY_BLOOM, sun_on = keywords & FLUID_DISPLAY_SUNRAYS;
    int bw = 1, bh = 1, sw = 1, sh = 1, levels = 0;
    if (bloom_on) fluid_get_resolution(fx->bloom_resolution, canvas_w, canvas_h, &bw, &bh);
    if (sun_on) fluid_get_resolution(fx->sunrays_resolution, canvas_w, canvas_h, &sw, &sh);
    if (bw < 1 || bh < 1 || sw < 1 || sh < 1) return fail(h, FLUID_ERR_INVALID, "bad post-FX resolution");
    if (bloom_on)
        while (levels < fx->bloom_iterations && (bw >> (levels + 1)) >= 2 && (bh >> (levels + 1)) >= 2) ++levels;
    *o = {bw, bh, sw, sh, levels};
    return FLUID_OK;
}

// The targets of the chains that are on, and the dithering texture's upload (BLOOM); a slab's gathered mask (SUNRAYS)
static int post_fx_targets(fluid_t* h, uint32_t keywords, const PostFXOut& o, const float* dither_rgb, int dw, int dh) {
    int rc;
    if (keywords & FLUID_DISPLAY_BLOOM) {
        if ((rc = need_bloom_targets(h, o.bw, o.bh, o.levels)) || (rc = need_dither_target(h, dw, dh))) return rc;
        CU(cudaMemcpyAsync(h->pfx.dither, dither_rgb, (size_t)dw * dh * 3 * sizeof(float), cudaMemcpyHostToDevice, h->stream));
    }
    if (keywords & FLUID_DISPLAY_SUNRAYS) {
        if ((rc = need_sunrays_targets(h, o.sw, o.sh))) return rc;
        if (h->slab() && (rc = need_mask_target(h, h->cfg.dye_w, h->cfg.dye_h))) return rc;
    }
    return FLUID_OK;
}

// The post-FX chains of render() for the keywords that are on, into the targets post_fx_targets made: applyBloom
// (S:1350-1394) with BLOOM, applySunrays + blur(…, 1) (S:1396-1419; the mask is drawn into dye.write exactly like
// S:1300) with SUNRAYS.  Sd: the dye's storage policy (the mask is drawn in it), St: the targets', Smp: the sampler
// of every texture the chains read (postfx.cuh).  BATCH: `images` images of a batch handle, each target a dense
// (B, h, w) array of which image z takes slot z, and each launch `images` layers of blocks deep; image z draws
// member members[z] (a subset draw's list in device memory), or member z when members is null; with `looks` (a
// draw with a look per image, in device memory) image z takes its sliders from looks[z] and fx's are not read.
// Arguments checked by the caller.
// A slab rank (fp32, LINEAR) prefilters its band of the bloom FBO's rows and draws the mask on the dye rows it
// owns; the bands are gathered (halo.cuh gather_bands), so every rank runs the pyramid, the sunrays and the blurs
// on the inputs one GPU has and ends with its bits.  The dye ghost rows must be fresh (draw_ghost_rows).
extern "C++" {
template <class Sd, class St, class Smp, bool BATCH = false>
static int post_fx_chains(fluid_t* h, uint32_t keywords, const fluid_postfx* fx, const PostFXOut& o, int images,
                          const int* members, const ImageLook* looks) {
    using D4 = typename Sd::T4;
    using T4 = typename St::T4;
    using T1 = typename St::T1;
    constexpr bool kSlab = !BATCH && std::is_same<Sd, StoreF32>::value && std::is_same<St, StoreF32>::value &&
                           std::is_same<Smp, Linear>::value;
    if (h->slab() && !kSlab) return fail(h, FLUID_ERR_INVALID, "post-FX on a slab handle is fp32 and LINEAR only");
    const bool bloom_on = keywords & FLUID_DISPLAY_BLOOM, sun_on = keywords & FLUID_DISPLAY_SUNRAYS;
    const int bw = o.bw, bh = o.bh, sw = o.sw, sh = o.sh, levels = o.levels;
    const int Wd = h->cfg.dye_w, Hd = h->cfg.dye_h, B = h->members, Z = images;
    T4* bloom = static_cast<T4*>(h->pfx.bloom);
    T1 *sun = static_cast<T1*>(h->pfx.sun), *sun2 = sun ? sun + (size_t)sw * sh * B : nullptr;
    dim3 b(32, 8);
    int nk = 0, rc;
    // ---- applyBloom(dye.read, bloom) ----------------------------------------------------------------
    if (bloom_on && levels >= 2) {
        struct Lv { T4* p; int w, h; };
        std::vector<Lv> pyr;
        T4* p = bloom + (size_t)bw * bh * B;
        for (int i = 0; i < levels; ++i) {
            const int pw = bw >> (i + 1), ph = bh >> (i + 1);
            pyr.push_back({p, pw, ph});
            p += (size_t)pw * ph * B;
        }
        float curve[4];
        prefilter_curve(fx->bloom_threshold, fx->bloom_soft_knee, curve);
        const int j_lo = band_row(bh, h->rank, h->world), j_hi = band_row(bh, h->rank + 1, h->world);
        if (j_hi > j_lo) {
            bloom_prefilter_kernel<Sd, St, Smp, BATCH><<<grid2d(bw, j_hi - j_lo, b, Z), b, 0, h->stream>>>(
                (const D4*)h->dye.read, Wd, Hd, h->droff, bloom, bw, bh, j_lo, j_hi, curve[0], curve[1], curve[2], curve[3],
                members, looks);
            ++nk;
        }
        if ((rc = gather_bands(h, GB_BLOOM))) return rc;
        Lv last{bloom, bw, bh};
        for (auto& d : pyr) {
            box4_kernel<St, Smp, BATCH><<<grid2d(d.w, d.h, b, Z), b, 0, h->stream>>>(last.p, last.w, last.h, d.p, d.w, d.h, 1.0f, 0);
            last = d; ++nk;
        }
        for (int i = (int)pyr.size() - 2; i >= 0; --i) {
            box4_kernel<St, Smp, BATCH><<<grid2d(pyr[i].w, pyr[i].h, b, Z), b, 0, h->stream>>>(last.p, last.w, last.h, pyr[i].p, pyr[i].w, pyr[i].h, 1.0f, 1);
            last = pyr[i]; ++nk;
        }
        box4_kernel<St, Smp, BATCH><<<grid2d(bw, bh, b, Z), b, 0, h->stream>>>(last.p, last.w, last.h, bloom, bw, bh, (float)fx->bloom_intensity, 0,
                                                                           looks);
        ++nk;
    }
    // ---- applySunrays(dye.read, dye.write, sunrays); blur(sunrays, sunraysTemp, 1) -------------------
    if (sun_on) {
        bool gathered = false;
        if constexpr (kSlab) {
            if (h->slab()) {
                sunrays_mask_kernel<Sd, Smp><<<grid2d(Wd, h->drow1 - h->drow0, b), b, 0, h->stream>>>(
                    (const D4*)h->dye.read, (D4*)h->dye.write, Wd, Hd, h->drow0, h->drow1, h->droff, h->pfx.mask);
                if ((rc = gather_bands(h, GB_MASK))) return rc;
                sunrays_kernel<Sd, St, Smp, false, float><<<grid2d(sw, sh, b), b, 0, h->stream>>>(h->pfx.mask, Wd, Hd, sun, sw, sh, (float)fx->sunrays_weight);
                gathered = true;
            }
        }
        if (!gathered) {
            sunrays_mask_kernel<Sd, Smp, BATCH><<<grid2d(Wd, Hd, b, Z), b, 0, h->stream>>>((const D4*)h->dye.read, (D4*)h->dye.write, Wd, Hd, 0, Hd, 0, nullptr, members);
            sunrays_kernel<Sd, St, Smp, BATCH><<<grid2d(sw, sh, b, Z), b, 0, h->stream>>>((const D4*)h->dye.write, Wd, Hd, sun, sw, sh, (float)fx->sunrays_weight, members,
                                                                                    looks);
        }
        blur3_kernel<St, Smp, BATCH><<<grid2d(sw, sh, b, Z), b, 0, h->stream>>>(sun, sun2, sw, sh, (float)(1.0 / (double)sw), 0.0f);
        blur3_kernel<St, Smp, BATCH><<<grid2d(sw, sh, b, Z), b, 0, h->stream>>>(sun2, sun, sw, sh, 0.0f, (float)(1.0 / (double)sh));
        nk += 4;
    }
    return check_launch(h, "post-FX kernels", nk);
}

// post_fx_chains<Sd, St, Smp> of a handle: the dye's and the targets' storage, and the sampler.  A batch handle
// is fp32 and LINEAR.
using Chains = int (*)(fluid_t*, uint32_t, const fluid_postfx*, const PostFXOut&, int, const int*, const ImageLook*);
template <class Smp>
static Chains chains_for(const fluid_t* h) {
    return !h->half_fx ? post_fx_chains<StoreF32, StoreF32, Smp>
         : !h->half    ? post_fx_chains<StoreF32, hs::StoreHalf, Smp>
                       : post_fx_chains<hs::StoreHalf, hs::StoreHalf, Smp>;
}
static Chains chains_of(const fluid_t* h) {
    return h->batch ? post_fx_chains<StoreF32, StoreF32, Linear, true> : h->nearest ? chains_for<Nearest>(h) : chains_for<Linear>(h);
}

// display_kernel<SHADING, BLOOM, SUNRAYS, Out, Sp, Smp> for the eight FLUID_DISPLAY_* masks.  The sets
// without BLOOM and SUNRAYS read no post-FX target: one instantiation.
using DisplayKernel = void (*)(DisplayArgs);
using F32 = StoreF32;
using F16 = hs::StoreHalf;
template <class Out, class Sp, class Smp, bool BATCH = false>
struct DisplaySet {
    static constexpr DisplayKernel k[8] = {
        display_kernel<false, false, false, Out, F32, Smp, BATCH>, display_kernel<true, false, false, Out, F32, Smp, BATCH>,
        display_kernel<false, true, false, Out, Sp, Smp, BATCH>,   display_kernel<true, true, false, Out, Sp, Smp, BATCH>,
        display_kernel<false, false, true, Out, Sp, Smp, BATCH>,   display_kernel<true, false, true, Out, Sp, Smp, BATCH>,
        display_kernel<false, true, true, Out, Sp, Smp, BATCH>,    display_kernel<true, true, true, Out, Sp, Smp, BATCH>};
};
// What a draw() produces: the output policy of its display kernel
enum DisplayOut { OUT_FRAME = 0, OUT_CAPTURE = 1, OUT_CANVAS = 2 };
// indexed by [sampler == Nearest][DisplayOut][Sp == hs::StoreHalf][FLUID_DISPLAY_* mask]
static const DisplayKernel* const kDisplay[2][3][2] = {
    {{DisplaySet<StoreFrame, F32, Linear>::k, DisplaySet<StoreFrame, F16, Linear>::k},
     {DisplaySet<StoreCapture, F32, Linear>::k, DisplaySet<StoreCapture, F16, Linear>::k},
     {DisplaySet<StoreCanvas, F32, Linear>::k, DisplaySet<StoreCanvas, F16, Linear>::k}},
    {{DisplaySet<StoreFrame, F32, Nearest>::k, DisplaySet<StoreFrame, F16, Nearest>::k},
     {DisplaySet<StoreCapture, F32, Nearest>::k, DisplaySet<StoreCapture, F16, Nearest>::k},
     {DisplaySet<StoreCanvas, F32, Nearest>::k, DisplaySet<StoreCanvas, F16, Nearest>::k}},
};
// a batch handle's (fp32, LINEAR; no fp32 frame), indexed by [DisplayOut][FLUID_DISPLAY_* mask]
static const DisplayKernel* const kDisplayBatch[3] = {
    nullptr, DisplaySet<StoreCapture, F32, Linear, true>::k, DisplaySet<StoreCanvas, F32, Linear, true>::k};
}  // extern "C++"

// Queues the copy of n values of a post-FX target into the caller's fp32 array.  An fp16 target goes
// into `stage` instead, which widen_staged() widens exactly once the stream has synchronised: no launch.
static int read_target(fluid_t* h, float* host, const void* dev, size_t n, std::vector<__half>& stage) {
    if (!h->half_fx) {
        CU(cudaMemcpyAsync(host, dev, n * sizeof(float), cudaMemcpyDeviceToHost, h->stream));
        return FLUID_OK;
    }
    stage.resize(n);
    CU(cudaMemcpyAsync(stage.data(), dev, n * sizeof(__half), cudaMemcpyDeviceToHost, h->stream));
    return FLUID_OK;
}
static void widen_staged(float* host, const std::vector<__half>& stage) {
    for (size_t k = 0; k < stage.size(); ++k) host[k] = __half2float(stage[k]);
}

// One frame of render(), captureScreenshot() or render(null) on the canvas, as the entry points below ask
// for it.
struct DrawRequest {
    const char* what;                  // the entry point, for error messages
    int width, height;                 // the target
    int canvas_w, canvas_h;            // the drawing buffer the post-FX FBOs are sized from
    uint32_t keywords;                 // FLUID_DISPLAY_*
    const fluid_postfx* fx;            // BLOOM or SUNRAYS
    const float* dither; int dw, dh;   // BLOOM
    float back[3]; int bg_mode;        // the background the output policy blends over (postfx.cuh)
    DisplayOut out;                    // the fp32 frame, the 8-bit capture image or the RGBA8 canvas
    bool on_device;                    // dst is the caller's device memory: no copy, no sync
    void* dst; size_t n;               // where the image goes: n floats (frame) or n bytes (capture, canvas)
    float* host_bloom;                 // the bloom FBO / sunrays texture, read back when given
    float* host_sunrays;
    bool batch;                        // a batch handle's call: one image per member, member by member in dst
    bool subset;                       // a batch call for the listed members only: image k is member members[k]
    const int32_t* members; int n_members;
    bool per_image;                    // a batch call with a look per image: image k's is looks[k], n_members images
    const fluid_look* looks;
};

// render(target) of S:1296-1317: the post-FX chains of the keywords that are on, then the background and
// drawDisplay in one display_kernel launch, read back to the host (or, for a capture or canvas into device
// memory, left on the stream for the caller's fluid_sync).  A slab handle draws its band of the target
// (fluid_render_band) after one refresh of the dye ghost rows the frame samples; with BLOOM or SUNRAYS the
// call is collective (post_fx_chains gathers), so every argument check comes before the first exchange.
// Half storage draws from a widened copy of dye; its post-FX needs FLUID_FLAG_HALF_POSTFX, and then the
// chains read the fp16 dye directly and draw the mask into the fp16 dye.write.  A batch request draws every
// member of a batch handle through the same launches, each launch B layers of blocks deep, or with `subset` the
// n_members listed members, n_members layers deep; only batch requests take a batch handle.  With `per_image`
// each image's sliders and background come from its look, uploaded into the look table before the launches.
static int draw(fluid_t* h, const DrawRequest& r) {
    if (!h) return FLUID_ERR_INVALID;
    if (h->batch && !r.batch) return not_on_batch(h, r.what);
    if (r.batch && !h->batch) return fail(h, FLUID_ERR_INVALID, "%s takes a batch handle (fluid_create_batch)", r.what);
    if (r.subset) { if (int rc = check_member_list(h, r.what, r.members, r.n_members)) return rc; }
    if (r.per_image && !r.subset && r.n_members != h->members)
        return fail(h, FLUID_ERR_INVALID, "%s: n = %d without a member list, the batch has %d members", r.what,
                    r.n_members, h->members);
    if (r.per_image && !r.looks && r.n_members > 0) return fail(h, FLUID_ERR_INVALID, "%s: NULL looks", r.what);
    if (r.keywords & ~(uint32_t)(FLUID_DISPLAY_SHADING | FLUID_DISPLAY_BLOOM | FLUID_DISPLAY_SUNRAYS))
        return fail(h, FLUID_ERR_INVALID, "unknown display keyword bits 0x%x", r.keywords);
    const bool bloom_on = r.keywords & FLUID_DISPLAY_BLOOM, sun_on = r.keywords & FLUID_DISPLAY_SUNRAYS;
    const bool postfx = bloom_on || sun_on, bytes = r.out != OUT_FRAME;
    const size_t images = r.subset ? (size_t)r.n_members : (size_t)h->members;
    if ((!r.dst && images > 0) || r.width < 1 || r.height < 1 || r.canvas_w < 1 || r.canvas_h < 1 || (postfx && !r.fx) ||
        (bloom_on && (!r.dither || r.dw < 1 || r.dh < 1)))
        return fail(h, FLUID_ERR_INVALID, "bad argument");
    int y0 = 0, y1 = r.height;
    if (h->slab()) fluid_render_band(h, r.height, &y0, &y1);
    const size_t cells = (size_t)r.width * (y1 - y0);
    if (r.batch && r.n != 4 * cells * images)
        return fail(h, FLUID_ERR_INVALID, "%s: the targets of %zu images have %zu bytes, caller passed %zu", r.what,
                    images, 4 * cells * images, r.n);
    if (r.n != 4 * cells * images)
        return fail(h, FLUID_ERR_INVALID, "%s: the target%s has %zu %s, caller passed %zu", r.what, h->slab() ? " band" : "",
                    4 * cells, bytes ? "bytes" : "floats", r.n);
    if (images == 0) return FLUID_OK;
    if (cells == 0 && !h->slab()) return FLUID_OK;      // a slab rank with no rows still takes part in the exchanges
    if (h->half && !h->half_fx && postfx)
        return fail(h, FLUID_ERR_INVALID, "%s with BLOOM or SUNRAYS is not built for FLUID_FLAG_HALF_STORAGE "
                    "(the reference's bloom / sunrays FBOs are fp16 too: add FLUID_FLAG_HALF_POSTFX)", r.what);
    PostFXOut o{};
    int rc = postfx ? post_fx_sizes(h, r.keywords, r.fx, r.canvas_w, r.canvas_h, &o) : FLUID_OK;
    if (rc) return rc;
    rc = r.on_device ? check_device_buf(h, r.what, r.dst, r.n)
                     : need_frame(h, bytes ? (cells * images + 3) / 4 : cells);     // uchar4 images live in the frame
    if (rc) return rc;
    if (postfx && (rc = post_fx_targets(h, r.keywords, o, r.dither, r.dw, r.dh))) return rc;
    if (h->slab()) {
        // refresh the dye ghost rows the frame's taps reach (those of dye.read are stale after advection); every
        // rank computes the same depth
        const int need = draw_ghost_rows(h->cfg.dye_h, r.height, bloom_on && o.levels >= 2 ? o.bh : 0, sun_on);
        if ((rc = exchange_rows(h, HB_DYE, std::min(h->Gd, need)))) return rc;
        if (need > h->Gd)
            return fail(h, FLUID_ERR_HALO, "a frame of a %d-row target needs %d dye ghost rows, the slab keeps %d", r.height, need, h->Gd);
    }
    if (r.subset && (rc = upload_member_list(h, r.members, r.n_members))) return rc;
    if (r.per_image && (rc = upload_looks(h, r.looks, r.n_members))) return rc;
    const int* list = r.subset ? h->member_list : nullptr;
    const ImageLook* looks = r.per_image ? h->look_table : nullptr;
    if (postfx && (rc = chains_of(h)(h, r.keywords, r.fx, o, (int)images, list, looks))) return rc;
    const float4* dye_src;
    if ((rc = display_source(h, &dye_src))) return rc;
    // texelSize = 1 / width, 1 / height (S:1337) and getTextureScale (S:1626-1631) are JS doubles, narrowed here
    const float4 ts = make_float4((float)(1.0 / (double)r.width), (float)(1.0 / (double)r.height),
                                  bloom_on ? (float)((double)r.width / (double)r.dw) : 0.0f,
                                  bloom_on ? (float)((double)r.height / (double)r.dh) : 0.0f);
    const DisplayArgs a{dye_src, h->cfg.dye_w, h->cfg.dye_h, h->droff, bloom_on ? h->pfx.bloom : nullptr, o.bw, o.bh,
                        sun_on ? h->pfx.sun : nullptr, o.sw, o.sh, bloom_on ? h->pfx.dither : nullptr, r.dw, r.dh,
                        r.on_device ? r.dst : h->frame, r.width, r.height, y0, y1, r.back[0], r.back[1], r.back[2], r.bg_mode,
                        h->cfg.aspect, ts, list, looks};
    dim3 b(32, 8);
    const DisplayKernel k = h->batch ? kDisplayBatch[r.out][r.keywords] : kDisplay[h->nearest][r.out][h->half_fx][r.keywords];
    if (cells > 0) {
        k<<<grid2d(r.width, y1 - y0, b, (int)images), b, 0, h->stream>>>(a);
        if ((rc = check_launch(h, "display_kernel"))) return rc;
    }
    if (r.on_device) return FLUID_OK;
    CU(cudaMemcpyAsync(r.dst, h->frame, r.n * (bytes ? 1 : sizeof(float)), cudaMemcpyDeviceToHost, h->stream));
    std::vector<__half> bloom16, sun16;
    if (bloom_on && r.host_bloom && (rc = read_target(h, r.host_bloom, h->pfx.bloom, (size_t)o.bw * o.bh * 4, bloom16))) return rc;
    if (sun_on && r.host_sunrays && (rc = read_target(h, r.host_sunrays, h->pfx.sun, (size_t)o.sw * o.sh, sun16))) return rc;
    CU(cudaStreamSynchronize(h->stream));
    widen_staged(r.host_bloom, bloom16);
    widen_staged(r.host_sunrays, sun16);
    return FLUID_OK;
}

// render(target) for config.BLOOM = config.SUNRAYS = false: the background selected by FLUID_BACKGROUND
// (colour / checkerboard / none), then the display shader (optionally SHADING) blended over it.
int fluid_render(fluid_t* h, int width, int height, int shading, float back_r, float back_g,
                 float back_b, float* host_rgba, size_t n_floats) {
    return draw(h, {.what = "fluid_render", .width = width, .height = height, .canvas_w = width, .canvas_h = height,
                    .keywords = shading ? (uint32_t)FLUID_DISPLAY_SHADING : 0u, .back = {back_r, back_g, back_b},
                    .bg_mode = h ? h->background : 0, .dst = host_rgba, .n = n_floats});
}

// render() with the display keywords of updateKeywords (S:1160-1166); the post-FX FBOs are sized from
// the target.
int fluid_render_keywords(fluid_t* h, int width, int height, uint32_t keywords, const fluid_postfx* fx,
                          const float* dither_rgb, int dw, int dh, float back_r, float back_g, float back_b,
                          float* host_rgba, size_t n_floats, float* host_bloom, float* host_sunrays) {
    return draw(h, {.what = "fluid_render_keywords", .width = width, .height = height, .canvas_w = width,
                    .canvas_h = height, .keywords = keywords, .fx = fx, .dither = dither_rgb, .dw = dw, .dh = dh,
                    .back = {back_r, back_g, back_b}, .bg_mode = h ? h->background : 0, .dst = host_rgba,
                    .n = n_floats, .host_bloom = host_bloom, .host_sunrays = host_sunrays});
}

// render(null) with the reference's desktop defaults SHADING = BLOOM = SUNRAYS = true (S:70-84)
int fluid_render_postfx(fluid_t* h, int width, int height, const fluid_postfx* fx, const float* dither_rgb,
                        int dw, int dh, float back_r, float back_g, float back_b, float* host_rgba,
                        size_t n_floats, float* host_bloom, float* host_sunrays) {
    return draw(h, {.what = "fluid_render_postfx", .width = width, .height = height, .canvas_w = width,
                    .canvas_h = height, .keywords = FLUID_DISPLAY_SHADING | FLUID_DISPLAY_BLOOM | FLUID_DISPLAY_SUNRAYS,
                    .fx = fx, .dither = dither_rgb, .dw = dw, .dh = dh, .back = {back_r, back_g, back_b},
                    .bg_mode = h ? h->background : 0, .dst = host_rgba, .n = n_floats, .host_bloom = host_bloom,
                    .host_sunrays = host_sunrays});
}

// captureScreenshot (S:287-299) up to normalizeTexture (S:309-327): render(target) into a width x height
// RGBA half-float target.  The post-FX chains run on the canvas-sized FBOs of render(null); the display
// draws at the target's size over drawColor(BACK_COLOR) stored in fp16 (not TRANSPARENT) or bare with
// blending off (TRANSPARENT), never over the checkerboard (S:1303-1314).  The display kernel's epilogue
// does the fp16 store, the 8-bit truncation and the flip; the fp32 frame never reaches memory.
static int capture(fluid_t* h, const char* what, int width, int height, int canvas_w, int canvas_h, uint32_t keywords,
                   int transparent, const fluid_postfx* fx, const float* dither_rgb, int dw, int dh,
                   float back_r, float back_g, float back_b, uint8_t* dst, size_t n_bytes, bool on_device,
                   bool batch = false, bool subset = false, const int32_t* members = nullptr, int n_members = 0,
                   bool per_image = false, const fluid_look* looks = nullptr) {
    // drawColor's store of normalizeColor(BACK_COLOR) into the half-float target
    const float b16[3] = {__half2float(__float2half_rn(back_r)), __half2float(__float2half_rn(back_g)),
                          __half2float(__float2half_rn(back_b))};
    return draw(h, {.what = what, .width = width, .height = height, .canvas_w = canvas_w,
                    .canvas_h = canvas_h, .keywords = keywords, .fx = fx, .dither = dither_rgb, .dw = dw, .dh = dh,
                    .back = {b16[0], b16[1], b16[2]}, .bg_mode = transparent ? 2 : 0, .out = OUT_CAPTURE,
                    .on_device = on_device, .dst = dst, .n = n_bytes, .batch = batch, .subset = subset,
                    .members = members, .n_members = n_members, .per_image = per_image, .looks = looks});
}

int fluid_capture(fluid_t* h, int width, int height, int canvas_w, int canvas_h, uint32_t keywords,
                  int transparent, const fluid_postfx* fx, const float* dither_rgb, int dw, int dh,
                  float back_r, float back_g, float back_b, uint8_t* host_rgba8, size_t n_bytes) {
    return capture(h, "fluid_capture", width, height, canvas_w, canvas_h, keywords, transparent, fx, dither_rgb, dw, dh,
                   back_r, back_g, back_b, host_rgba8, n_bytes, false);
}

// The same image stored by the display kernel's StoreCapture epilogue straight into the caller's device memory,
// stream-ordered.
int fluid_capture_device(fluid_t* h, int width, int height, int canvas_w, int canvas_h, uint32_t keywords,
                         int transparent, const fluid_postfx* fx, const float* dither_rgb, int dw, int dh,
                         float back_r, float back_g, float back_b, uint8_t* dst, size_t n_bytes) {
    return capture(h, "fluid_capture_device", width, height, canvas_w, canvas_h, keywords, transparent, fx, dither_rgb,
                   dw, dh, back_r, back_g, back_b, dst, n_bytes, true);
}

// The captures of every member of a batch handle, member by member into dst, through the launches of one capture.
int fluid_capture_batch(fluid_t* h, int width, int height, int canvas_w, int canvas_h, uint32_t keywords,
                        int transparent, const fluid_postfx* fx, const float* dither_rgb, int dw, int dh,
                        float back_r, float back_g, float back_b, uint8_t* dst, size_t n_bytes, int dst_on_device) {
    return capture(h, "fluid_capture_batch", width, height, canvas_w, canvas_h, keywords, transparent, fx, dither_rgb,
                   dw, dh, back_r, back_g, back_b, dst, n_bytes, dst_on_device != 0, true);
}

// render(null) (S:1296-1317) on a width x height RGBA8 drawing buffer: the post-FX chains on the canvas-sized
// FBOs, then the display over drawColor(BACK_COLOR) or drawCheckerboard (TRANSPARENT, S:1304-1315), blended
// on the fixed-point buffer by the display kernel's StoreCanvas epilogue.  Into host memory through the
// frame buffer, or straight into the caller's device memory, stream-ordered.
static int canvas(fluid_t* h, const char* what, int width, int height, uint32_t keywords, int transparent,
                  const fluid_postfx* fx, const float* dither_rgb, int dw, int dh, float back_r, float back_g,
                  float back_b, uint8_t* dst, size_t n_bytes, int dst_on_device, bool batch, bool subset = false,
                  const int32_t* members = nullptr, int n_members = 0, bool per_image = false,
                  const fluid_look* looks = nullptr) {
    return draw(h, {.what = what, .width = width, .height = height, .canvas_w = width,
                    .canvas_h = height, .keywords = keywords, .fx = fx, .dither = dither_rgb, .dw = dw, .dh = dh,
                    .back = {back_r, back_g, back_b}, .bg_mode = transparent ? 1 : 0, .out = OUT_CANVAS,
                    .on_device = dst_on_device != 0, .dst = dst, .n = n_bytes, .batch = batch, .subset = subset,
                    .members = members, .n_members = n_members, .per_image = per_image, .looks = looks});
}

int fluid_render_canvas(fluid_t* h, int width, int height, uint32_t keywords, int transparent,
                        const fluid_postfx* fx, const float* dither_rgb, int dw, int dh,
                        float back_r, float back_g, float back_b,
                        uint8_t* dst, size_t n_bytes, int dst_on_device) {
    return canvas(h, "fluid_render_canvas", width, height, keywords, transparent, fx, dither_rgb, dw, dh,
                  back_r, back_g, back_b, dst, n_bytes, dst_on_device, false);
}

// The canvases of every member of a batch handle, member by member into dst, through the launches of one canvas.
int fluid_render_canvas_batch(fluid_t* h, int width, int height, uint32_t keywords, int transparent,
                              const fluid_postfx* fx, const float* dither_rgb, int dw, int dh,
                              float back_r, float back_g, float back_b,
                              uint8_t* dst, size_t n_bytes, int dst_on_device) {
    return canvas(h, "fluid_render_canvas_batch", width, height, keywords, transparent, fx, dither_rgb, dw, dh,
                  back_r, back_g, back_b, dst, n_bytes, dst_on_device, true);
}

// fluid_capture_batch and fluid_render_canvas_batch for the listed members: image k is member members[k]'s, through
// the launches of one whole-batch draw, each n layers of blocks deep, in the same post-FX targets.
int fluid_capture_members(fluid_t* h, int width, int height, int canvas_w, int canvas_h, uint32_t keywords,
                          int transparent, const fluid_postfx* fx, const float* dither_rgb, int dw, int dh,
                          float back_r, float back_g, float back_b, uint8_t* dst, size_t n_bytes, int dst_on_device,
                          const int32_t* members, int n) {
    return capture(h, "fluid_capture_members", width, height, canvas_w, canvas_h, keywords, transparent, fx, dither_rgb,
                   dw, dh, back_r, back_g, back_b, dst, n_bytes, dst_on_device != 0, true, true, members, n);
}
int fluid_render_canvas_members(fluid_t* h, int width, int height, uint32_t keywords, int transparent,
                                const fluid_postfx* fx, const float* dither_rgb, int dw, int dh,
                                float back_r, float back_g, float back_b,
                                uint8_t* dst, size_t n_bytes, int dst_on_device, const int32_t* members, int n) {
    return canvas(h, "fluid_render_canvas_members", width, height, keywords, transparent, fx, dither_rgb, dw, dh,
                  back_r, back_g, back_b, dst, n_bytes, dst_on_device, true, true, members, n);
}

// The batch draws with a look per image: the whole batch (members == NULL, n == B) or the listed members, image k
// drawn with looks[k]'s sliders and background through the launches of the shared-look draw.  The call's own
// background arguments are placeholders the look table replaces.
int fluid_capture_looks(fluid_t* h, int width, int height, int canvas_w, int canvas_h, uint32_t keywords,
                        const fluid_postfx* fx, const float* dither_rgb, int dw, int dh, const fluid_look* looks,
                        uint8_t* dst, size_t n_bytes, int dst_on_device, const int32_t* members, int n) {
    return capture(h, "fluid_capture_looks", width, height, canvas_w, canvas_h, keywords, 0, fx, dither_rgb, dw, dh,
                   0.0f, 0.0f, 0.0f, dst, n_bytes, dst_on_device != 0, true, members != nullptr, members, n, true, looks);
}
int fluid_render_canvas_looks(fluid_t* h, int width, int height, uint32_t keywords, const fluid_postfx* fx,
                              const float* dither_rgb, int dw, int dh, const fluid_look* looks,
                              uint8_t* dst, size_t n_bytes, int dst_on_device, const int32_t* members, int n) {
    return canvas(h, "fluid_render_canvas_looks", width, height, keywords, 0, fx, dither_rgb, dw, dh, 0.0f, 0.0f, 0.0f,
                  dst, n_bytes, dst_on_device, true, members != nullptr, members, n, true, looks);
}

void* fluid_host_alloc(size_t bytes) {
    void* p = nullptr;
    if (bytes == 0 || cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return p;
}
void fluid_host_free(void* p) { if (p) cudaFreeHost(p); }

int fluid_sync(fluid_t* h) {
    if (!h) return FLUID_ERR_INVALID;
    CU(cudaStreamSynchronize(h->stream));
    return check_halo(h);
}

int fluid_timing_last(fluid_t* h, fluid_timing* out) {
    if (!h || !out) return FLUID_ERR_INVALID;
    if (!h->have_timing) return fail(h, FLUID_ERR_INVALID, "per-pass timing needs FLUID_FLAG_NO_GRAPH");
    CU(cudaStreamSynchronize(h->stream));
    float ms[5];
    for (int k = 0; k < 5; ++k) CU(cudaEventElapsedTime(&ms[k], h->tev[k], h->tev[k + 1]));
    h->timing.curl_vort_div_ms = ms[0]; h->timing.jacobi_ms = ms[1]; h->timing.gradient_ms = ms[2];
    h->timing.advect_velocity_ms = ms[3]; h->timing.advect_dye_ms = ms[4];
    CU(cudaEventElapsedTime(&h->timing.total_ms, h->tev[0], h->tev[5]));
    *out = h->timing;
    return FLUID_OK;
}

int fluid_mark(fluid_t* h, int slot) {
    if (!h || slot < 0 || slot > 1) return FLUID_ERR_INVALID;
    CU(cudaEventRecord(h->mark[slot], h->stream));
    return FLUID_OK;
}

int fluid_elapsed_ms(fluid_t* h, float* ms) {
    if (!h || !ms) return FLUID_ERR_INVALID;
    CU(cudaEventSynchronize(h->mark[1]));
    CU(cudaEventElapsedTime(ms, h->mark[0], h->mark[1]));
    return FLUID_OK;
}

uint64_t fluid_launch_count(fluid_t* h) { return h ? h->launches.all : 0; }

uint64_t fluid_stat(fluid_t* h, int key) {
    if (!h) return 0;
    switch (key) {
        case FLUID_STAT_LAUNCHES: return h->launches.all;
        case FLUID_STAT_JACOBI_LAUNCHES: return h->launches.jacobi;
        case FLUID_STAT_HALO_LAUNCHES: return h->launches.halo;
        case FLUID_STAT_HALO_EXCHANGES: return h->halo_groups;
        case FLUID_STAT_GRAPH_CAPTURES: return h->graph_captures;
        case FLUID_STAT_GRAPH_LAUNCHES: return h->graph_launches;
        case FLUID_STAT_HALO_TRANSPORT_P2P: return h->p2p ? 1 : 0;
        case FLUID_STAT_CVD_STREAM_LAUNCHES: return h->launches.cvd_stream;
        case FLUID_STAT_GRADIENT_STREAM_LAUNCHES: return h->launches.gradient_stream;
        case FLUID_STAT_ADVECT4_LAUNCHES: return h->launches.advect4;
        case FLUID_STAT_GATHERS: return h->gathers;
        case FLUID_STAT_JACOBI_EXACT_STREAMS: {          // counted on the device: waits for the handle's work
            unsigned long long n = 0;
            if (cudaMemcpyAsync(&n, h->exact_streams, sizeof n, cudaMemcpyDeviceToHost, h->stream) != cudaSuccess ||
                cudaStreamSynchronize(h->stream) != cudaSuccess) return 0;
            return n;
        }
    }
    return 0;
}

void* fluid_device_ptr(fluid_t* h, int field) {
    void* p; int w, rows, ch;
    if (!h || field_info(h, field, &p, &w, &rows, &ch)) return nullptr;
    return p;
}

}  // extern "C"
