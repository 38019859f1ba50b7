// stage_probe.cu — is a depth-13 blocked launch bound by how it stages p and divergence?
//
// Standalone timing harness, not part of the library (tools/stage_probe.py compiles and runs it).  At the
// geometry of one depth-13 launch of the 4096^2 solve (40 windows x 26 chunks of 160 output rows, 186
// steps per stream, 8 warps per SM) it times, with CUDA events over many launches, alternated, repeated:
//   stage G=1  today's staging: one-warp CTAs, each running its own TMA ring (TB<K>::NS stages) of a 136-column x
//              3-row box of p and of div per 3 steps, refilled after a __syncwarp; per row it loads its
//              float4 of p and div from shared memory and stores their sum to the output row.  No
//              Jacobi arithmetic.
//   stage G=2/4 the same work with G adjacent windows per CTA (one warp each) sharing ONE box per field
//              per stage, (G-1)*104 + 136 columns wide (two side-by-side boxes where that exceeds the
//              256-element TMA limit), with a full mbarrier (1 arrival + bytes) and an empty mbarrier
//              (one arrival per warp) per stage; one elected lane waits on empty before refilling.
//   real       jacobi_tb_kernel<13, false> from csrc/jacobi.cuh on the same fields.
// Every staging variant is padded with dynamic shared memory to exactly 8 warps per SM, as the real kernel
// runs at 255 registers.  Prints one line per variant and repeat, then a summary.
#include <cuda.h>
#include <cuda_runtime.h>
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include "../webgl_fluid_simulation_b200/csrc/jacobi.cuh"

using namespace fk;

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { \
    fprintf(stderr, "%s:%d %s: %s\n", __FILE__, __LINE__, #x, cudaGetErrorString(e_)); exit(1); } } while (0)

constexpr int K = 13;

template <int G>
struct SG {
    static constexpr int HX = TB<K>::HX, VALID = TB<K>::VALID;
    static constexpr int WB = (G - 1) * VALID + TB_BOX;          // columns the CTA's windows span
    static constexpr int NSUB = (WB + 255) / 256;                // side-by-side boxes per field
    static constexpr int BW = ((WB + NSUB - 1) / NSUB + 3) / 4 * 4;   // columns per box
    static constexpr int FIELD4 = (NSUB * 3 * BW / 4 + 7) / 8 * 8;    // float4 per field per stage (128 B multiple)
    static constexpr int STAGE4 = 2 * FIELD4;
    static constexpr int NS = TB<K>::NS;
    static constexpr int TX = 2 * NSUB * 3 * BW * (int)sizeof(float);
    static constexpr int RING = NS * STAGE4 * (int)sizeof(float4) + 2 * NS * 8;
};

struct Maps { TmapPair m[3]; };   // box shape of G = 1, 2, 4

template <int G>
__global__ void __launch_bounds__(32 * G, 1) stage_kernel(JacobiArgs a, const __grid_constant__ TmapPair maps) {
    using S = SG<G>;
    extern __shared__ __align__(128) float4 smem4[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int W = a.W, W4 = W >> 2;
    const int nxw = (W + S::VALID - 1) / S::VALID, ngx = (nxw + G - 1) / G;
    const int gxi = blockIdx.x % ngx, cy = blockIdx.x / ngx;
    const int live = min(G, nxw - gxi * G);
    const int wx = gxi * G + warp;
    const int xb = gxi * G * S::VALID - S::HX - 4;                // first column of the CTA box
    const int x0 = wx * S::VALID - S::HX;
    const int gx = x0 + 4 * lane;
    int lc = gx < 0 ? -gx - 4 : (gx >= W ? 2 * W - 4 - gx : gx);
    lc = min(max(lc, 0), W - 4);
    const int col = min(max(lc, x0), x0 + 124) - xb;             // in [0, WB)
    const float4* ring = smem4 + ((col / S::BW) * 3 * S::BW + col % S::BW) / 4;
    const bool lane_out = lane >= S::HX / 4 && lane < 32 - S::HX / 4 && gx >= 0 && gx < W;
    const int y0 = a.out_lo + cy * a.rows_per_chunk, y1 = min(y0 + a.rows_per_chunk, a.out_hi);
    const int ys = max(y0 - K, 0);
    const int nsteps = y1 - ys + K;
    unsigned long long* full = reinterpret_cast<unsigned long long*>(smem4 + S::NS * S::STAGE4);
    unsigned long long* empty = full + S::NS;
    const void* tp = &maps.p;
    const void* td = &maps.d;
    auto fill = [&](int q, int yrow) {
        float4* dst = smem4 + q * S::STAGE4;
        mbar_expect_tx(full + q, (unsigned)S::TX);
#pragma unroll
        for (int b = 0; b < S::NSUB; ++b) {
            tma_load_2d(dst + b * 3 * S::BW / 4, td, xb + b * S::BW, yrow, full + q);
            tma_load_2d(dst + S::FIELD4 + b * 3 * S::BW / 4, tp, xb + b * S::BW, yrow, full + q);
        }
    };
    if (threadIdx.x == 0) {
        for (int q = 0; q < S::NS; ++q) { mbar_init(full + q, 1); mbar_init(empty + q, live); }
        mbar_fence_init();
    }
    __syncthreads();
    if (warp >= live) return;
    int yfill = ys - a.row_off;
    if (threadIdx.x == 0)
        for (int q = 0; q < S::NS - 1; ++q) fill(q, yfill + 3 * q);
    yfill += 3 * (S::NS - 1);
    float4* op = reinterpret_cast<float4*>(a.pout) + (lane_out ? gx / 4 : 0);
    int stg = 0;
    unsigned phase = 0;
    unsigned ephase = 0;    // parity of the empty barrier of the stage refilled next
#pragma unroll 1
    for (int s0 = 0; s0 < nsteps; s0 += 3) {
        mbar_wait(full + stg, phase, a.err);
        const float4* srow = ring + stg * S::STAGE4;
#pragma unroll
        for (int ph = 0; ph < 3; ++ph) {
            const float4 d = lds128(srow + ph * S::BW / 4);
            const float4 p = lds128(srow + S::FIELD4 + ph * S::BW / 4);
            const int r = ys + s0 + ph;     // the row just staged
            if (lane_out && (unsigned)(r - y0) < (unsigned)(y1 - y0))
                op[(size_t)(r - a.row_off) * W4] = make_float4(p.x + d.x, p.y + d.y, p.z + d.z, p.w + d.w);
        }
        // the stage consumed one block ago is refilled with the box NS-1 blocks ahead
        const int q = (stg == 0) ? S::NS - 1 : stg - 1;
        __syncwarp();
        if (G == 1 || s0 == 0) {            // one warp, or stage NS-1, which nobody has read yet
            if (threadIdx.x == 0) fill(q, yfill);
        } else {
            if (lane == 0) asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(empty + q)) : "memory");
            if (threadIdx.x == 0) {
                mbar_wait(empty + q, (ephase >> q) & 1u, a.err);
                fill(q, yfill);
            }
            ephase ^= 1u << q;
        }
        yfill += 3;
        if (stg + 1 == S::NS) { stg = 0; phase ^= 1u; } else { ++stg; }
    }
    // drain the over-fetched tail before the CTA (and its shared memory) goes away
#pragma unroll
    for (int q = 0; q < S::NS - 1; ++q) {
        mbar_wait(full + stg, phase, a.err);
        if (stg + 1 == S::NS) { stg = 0; phase ^= 1u; } else { ++stg; }
    }
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static void encode(EncodeTiledFn enc, unsigned char (&tm)[128], void* base, int W, int H, int bw) {
    const cuuint64_t dims[2] = {(cuuint64_t)W, (cuuint64_t)H};
    const cuuint64_t strides[1] = {(cuuint64_t)W * sizeof(float)};
    const cuuint32_t box[2] = {(cuuint32_t)bw, 3}, estr[2] = {1, 1};
    if (enc(reinterpret_cast<CUtensorMap*>(tm), CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, base, dims, strides, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS) { fprintf(stderr, "encode failed (box %d)\n", bw); exit(1); }
}

template <class F>
static float time_launches(F launch, int n, cudaEvent_t e0, cudaEvent_t e1) {
    CK(cudaEventRecord(e0));
    for (int i = 0; i < n; ++i) launch();
    CK(cudaEventRecord(e1));
    CK(cudaEventSynchronize(e1));
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, e0, e1));
    CK(cudaGetLastError());
    return 1000.0f * ms / n;
}

int main(int argc, char** argv) {
    const int N = argc > 1 ? atoi(argv[1]) : 1000, REPS = argc > 2 ? atoi(argv[2]) : 3;
    const int W = 4096, H = 4096;
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, 0));
    const int sms = prop.multiProcessorCount;
    const size_t n = (size_t)W * H;
    float *p, *d, *o;
    int* err;
    CK(cudaMalloc(&p, n * 4)); CK(cudaMalloc(&d, n * 4)); CK(cudaMalloc(&o, n * 4)); CK(cudaMalloc(&err, 4));
    std::vector<float> hbuf(n);
    srand(1);
    for (auto& v : hbuf) v = (float)rand() / RAND_MAX - 0.5f;
    CK(cudaMemcpy(p, hbuf.data(), n * 4, cudaMemcpyHostToDevice));
    for (auto& v : hbuf) v = 0.01f * ((float)rand() / RAND_MAX - 0.5f);
    CK(cudaMemcpy(d, hbuf.data(), n * 4, cudaMemcpyHostToDevice));
    CK(cudaMemset(err, 0, 4));

    void* fn = nullptr;
    cudaDriverEntryPointQueryResult q;
    CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
    EncodeTiledFn enc = (EncodeTiledFn)fn;
    Maps maps;
    const int bws[3] = {SG<1>::BW, SG<2>::BW, SG<4>::BW};
    for (int k = 0; k < 3; ++k) { encode(enc, maps.m[k].p, p, W, H, bws[k]); encode(enc, maps.m[k].d, d, W, H, bws[k]); }

    // the chunking of tb_rows() for depth 13 at 8 warps per SM
    const int valid = TB<K>::VALID, nxw = (W + valid - 1) / valid;
    const int nch0 = std::max(1, std::max(nxw, sms * 8) / nxw);
    int R = std::max((H + nch0 - 1) / nch0, 4 * K);
    if ((R + 2 * K) % 3) R += 3 - (R + 2 * K) % 3;
    const int nch = (H + R - 1) / R;
    JacobiArgs a{};
    a.pin = p; a.div = d; a.pout = o; a.W = W; a.H = H; a.row_off = 0; a.out_lo = 0; a.out_hi = H;
    a.rows_per_chunk = R; a.scale = 1.0f; a.err = err; a.tiny_map = nullptr; a.exact_streams = nullptr;
    printf("device %s, %d SMs; depth %d: %d windows x %d chunks of %d rows\n", prop.name, sms, K, nxw, nch, R);

    // one SM holds 8 warps of every variant: pad each CTA's shared memory to G/8 of what an SM offers
    const int per_sm = (int)prop.sharedMemPerMultiprocessor, reserve = (int)prop.reservedSharedMemPerBlock;
    auto pad = [&](int G) { return per_sm / (8 / G) - reserve - 64; };
    CK(cudaFuncSetAttribute(stage_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, pad(1)));
    CK(cudaFuncSetAttribute(stage_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, pad(2)));
    CK(cudaFuncSetAttribute(stage_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, pad(4)));
    CK(cudaFuncSetAttribute(jacobi_tb_kernel<K, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, TB<K>::SMEM));
    int occ[4];
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ[0], stage_kernel<1>, 32, pad(1)));
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ[1], stage_kernel<2>, 64, pad(2)));
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ[2], stage_kernel<4>, 128, pad(4)));
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ[3], jacobi_tb_kernel<K, false>, 32, TB<K>::SMEM));
    printf("warps per SM: stage G=1 %d, G=2 %d, G=4 %d, real %d; box columns %d / %d / %dx%d\n",
           occ[0], 2 * occ[1], 4 * occ[2], occ[3], SG<1>::BW, SG<2>::BW, SG<4>::NSUB, SG<4>::BW);

    const char* names[4] = {"stage G=1", "stage G=2", "stage G=4", "real"};
    auto launch = [&](int v) {
        if (v == 0) stage_kernel<1><<<nxw * nch, 32, pad(1)>>>(a, maps.m[0]);
        if (v == 1) stage_kernel<2><<<(nxw + 1) / 2 * nch, 64, pad(2)>>>(a, maps.m[1]);
        if (v == 2) stage_kernel<4><<<(nxw + 3) / 4 * nch, 128, pad(4)>>>(a, maps.m[2]);
        if (v == 3) jacobi_tb_kernel<K, false><<<nxw * nch, 32, TB<K>::SMEM>>>(a, maps.m[0], nullptr);
    };
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    // the staged rows reach the output unchanged: every variant must store p + d on every output cell
    std::vector<float> ref(n), got(n), pin(n), dv(n);
    CK(cudaMemcpy(pin.data(), p, n * 4, cudaMemcpyDeviceToHost));
    CK(cudaMemcpy(dv.data(), d, n * 4, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < n; ++i) ref[i] = pin[i] + dv[i];
    for (int v = 0; v < 3; ++v) {
        CK(cudaMemset(o, 0xff, n * 4));
        launch(v);
        CK(cudaDeviceSynchronize());
        CK(cudaMemcpy(got.data(), o, n * 4, cudaMemcpyDeviceToHost));
        size_t bad = 0;
        for (size_t i = 0; i < n; ++i) bad += got[i] != ref[i];
        printf("%s: %zu of %zu output cells differ from p + d\n", names[v], bad, n);
    }
    for (int v = 0; v < 4; ++v) time_launches([&] { launch(v); }, 50, e0, e1);   // warm-up
    std::vector<float> us[4];
    for (int r = 0; r < REPS; ++r)
        for (int v = 0; v < 4; ++v) {
            us[v].push_back(time_launches([&] { launch(v); }, N, e0, e1));
            printf("repeat %d %-10s %7.2f us per launch\n", r, names[v], us[v].back());
            fflush(stdout);
        }
    int herr = 0;
    CK(cudaMemcpy(&herr, err, 4, cudaMemcpyDeviceToHost));
    for (int v = 0; v < 4; ++v) {
        std::sort(us[v].begin(), us[v].end());
        printf("%-10s min %7.2f  median %7.2f  max %7.2f us per launch over %d x %d launches\n", names[v],
               us[v].front(), us[v][us[v].size() / 2], us[v].back(), REPS, N);
    }
    printf("error word %d\n", herr);
    return herr != 0;
}
