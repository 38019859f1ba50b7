// halo.cuh — slab halo exchange: the peer-memory transport (IPC-mapped arenas, one push kernel with
// the free/ready handshake) and the NCCL send/recv fallback; and the all-gather of row bands that
// post-FX on slabs runs (NCCL only).  Included by fluid.cu inside its anonymous namespace, after
// `struct fluid`, fail(), CU() and check_launch() are defined.
#pragma once

// ---- halo exchange (NCCL point-to-point; all buffers and both neighbours in ONE group) ------------
// For each item: sends my top `n` owned rows up and my bottom `n` owned rows down, receives the
// neighbours' rows into my ghost rows.  Halo messages are latency-bound (a 4096-float row is 16 KiB),
// so everything that can travel together does.
// `which` names the buffer: velocity.read, pressure.read, dye.read or divergence.
enum { HB_VELOCITY = 0, HB_PRESSURE = 1, HB_DYE = 2, HB_DIVERGENCE = 3 };
struct HaloItem { int which, n; };

// Buffer `which` in the arena of `side` (this rank's own, or a neighbour's mapped through CUDA IPC): local
// row 0 at `base`, which is global row `off`.  The neighbour's copy of a pair's .read is in the same slot as
// mine (SPMD-identical swap parity).  r0, r1: the rows THIS rank owns in that grid.
struct HaloRows { char* base; size_t row_bytes; int off, r0, r1; };
HaloRows halo_rows(const fluid_t* h, const fluid::Peer& side, int which) {
    const FieldLayout& L = side.layout;
    const size_t W = h->cfg.sim_w, Wd = h->cfg.dye_w;
    switch (which) {
        case HB_VELOCITY: return {side.base + L.v[h->velocity.par], W * sizeof(float2), side.roff, h->row0, h->row1};
        case HB_PRESSURE: return {side.base + L.p[h->pressure.par], W * sizeof(float), side.roff, h->row0, h->row1};
        case HB_DYE: return {side.base + L.dye[h->dye.par], Wd * sizeof(float4), side.droff, h->drow0, h->drow1};
        default: return {side.base + L.div, W * sizeof(float), side.roff, h->row0, h->row1};
    }
}
fluid::Peer own_arena(const fluid_t* h) { return {true, h->arena, h->roff, h->droff, h->layout}; }

struct ScanArgs { const float* div; unsigned char* map; int W, row_off, lo0, hi0, lo1, hi1; };
struct PushSeg { const float4* src; float4* dst; unsigned long long n4; };
struct PushArgs {
    PushSeg seg[8];
    int count;
    unsigned seq;
    unsigned* my_flags;        // [0] ready-from-below [1] ready-from-above [2] free-from-below [3] free-from-above
    unsigned* peer_flags[2];   // the same four words in the neighbours' arenas (IPC-mapped); [0] below, [1] above
    int present[2];
    unsigned* counter;         // block-completion counter (local)
    int* err;                  // set when a bounded spin times out (reported as FLUID_ERR_HALO)
    ScanArgs scan;             // divergence ghost strips to scan for tiny values once they have arrived (W == 0: none)
};

__device__ __forceinline__ unsigned ld_acquire_sys(const unsigned* p) {
    unsigned v; asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v;
}
__device__ __forceinline__ void st_release_sys(unsigned* p, unsigned v) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ unsigned long long global_ns() {
    unsigned long long t; asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t)); return t;
}
// bounded spin: a neighbour that never arrives costs 4 s and an error flag, never a hung GPU
__device__ __forceinline__ void spin_until(const unsigned* flag, unsigned seq, int* err) {
    const unsigned long long t0 = global_ns();
    while ((int)(ld_acquire_sys(flag) - seq) < 0) {
        if (global_ns() - t0 > 4000000000ull) { *err = 2; break; }
        __nanosleep(100);
    }
}

// One halo exchange in ONE kernel, producer and consumer side:
//   (a) tell the neighbours my ghost rows may be overwritten (this kernel is stream-ordered after
//       every kernel of mine that read them), (b) wait until theirs are free, (c) store my boundary
//       rows straight into their ghost rows — dst pointers are the neighbours' arenas mapped through
//       CUDA IPC, so the stores travel over NVLink / NVSwitch — and (d) once the last block is
//       done, release-store "ready = seq" into the neighbours' flag words.
__global__ void __launch_bounds__(256) halo_push_kernel(PushArgs a) {
    if (threadIdx.x == 0) {
        if (blockIdx.x == 0) {
            for (int side = 0; side < 2; ++side)
                if (a.present[side]) st_release_sys(a.peer_flags[side] + (side == 0 ? 3 : 2), a.seq);
        }
        for (int side = 0; side < 2; ++side)
            if (a.present[side]) spin_until(a.my_flags + (side == 0 ? 2 : 3), a.seq, a.err);
    }
    __syncthreads();
    for (int k = 0; k < a.count; ++k) {
        const float4* __restrict__ s = a.seg[k].src;
        float4* __restrict__ d = a.seg[k].dst;
        const unsigned long long n4 = a.seg[k].n4;
        for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
             i += (unsigned long long)gridDim.x * blockDim.x)
            d[i] = s[i];
    }
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x == 0) {
        const unsigned done = atomicAdd(a.counter, 1u);
        if (done == gridDim.x - 1) {
            *a.counter = 0;
            __threadfence_system();
            for (int side = 0; side < 2; ++side)
                if (a.present[side]) st_release_sys(a.peer_flags[side] + (side == 0 ? 1 : 0), a.seq);
        }
    }
    // (e) consumer side in the SAME kernel (every block is resident: the grid is at most 2 blocks per SM):
    // acquire the neighbours' "ready" words, then (f) flag tiny values in the divergence strips that arrived.
    if (threadIdx.x == 0) {
        if (a.present[0]) spin_until(a.my_flags + 0, a.seq, a.err);
        if (a.present[1]) spin_until(a.my_flags + 1, a.seq, a.err);
    }
    __syncthreads();
    if (a.scan.W > 0) {
        const ScanArgs& sc = a.scan;
        const int n0 = max(sc.hi0 - sc.lo0, 0) * sc.W, n1 = max(sc.hi1 - sc.lo1, 0) * sc.W;
        const int mw = fk::tiny_map_w(sc.W);
        for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < n0 + n1; k += gridDim.x * blockDim.x) {
            const int q = k < n0 ? k : k - n0;
            const int j = (k < n0 ? sc.lo0 : sc.lo1) + q / sc.W, i = q % sc.W;
            if (fk::is_tiny_div(sc.div[(size_t)(j - sc.row_off) * sc.W + i])) sc.map[(j / fk::TINY_CH) * mw + i / fk::TINY_CW] = 1;
        }
    }
}

int exchange_p2p(fluid_t* h, const HaloItem* it, int count) {
    PushArgs pa{};
    pa.seq = ++h->p2p_seq;
    pa.my_flags = (unsigned*)(h->arena + h->layout.flags);
    pa.counter = pa.my_flags + 8;
    pa.err = h->halo_flag;
    unsigned long long total4 = 0;
    for (int side = 0; side < 2; ++side) {
        const fluid::Peer& P = h->peer[side];
        pa.present[side] = P.present ? 1 : 0;
        pa.peer_flags[side] = P.present ? (unsigned*)(P.base + P.layout.flags) : nullptr;
    }
    for (int k = 0; k < count; ++k) {
        const HaloItem& q = it[k];
        if (q.n <= 0) continue;
        const HaloRows me = halo_rows(h, own_arena(h), q.which);
        for (int side = 0; side < 2; ++side) {
            if (!h->peer[side].present) continue;
            const HaloRows nb = halo_rows(h, h->peer[side], q.which);
            const int g0 = (side == 1) ? me.r1 - q.n : me.r0;         // my owned rows that the neighbour needs
            const char* src = me.base + (size_t)(g0 - me.off) * me.row_bytes;
            char* dst = nb.base + (size_t)(g0 - nb.off) * me.row_bytes;
            if (pa.count >= 8) return fail(h, FLUID_ERR_INVALID, "too many halo segments");
            PushSeg& sg = pa.seg[pa.count++];
            sg.src = (const float4*)src; sg.dst = (float4*)dst; sg.n4 = (unsigned long long)q.n * me.row_bytes / 16;
            total4 = std::max(total4, sg.n4);
        }
    }
    const unsigned blocks = (unsigned)std::min<unsigned long long>(std::max<unsigned long long>((total4 + 255) / 256, 1), (unsigned long long)h->sm_count * 2);
    if (h->scan_pending) {          // this exchange carries divergence ghost rows: their tiny-value scan rides along
        pa.scan = ScanArgs{h->scan.div, h->scan.map, h->scan.W, h->scan.row_off, h->scan.lo0, h->scan.hi0, h->scan.lo1, h->scan.hi1};
        h->scan_pending = false;
    }
    halo_push_kernel<<<blocks, 256, 0, h->stream>>>(pa);     // push + handshake + wait + scan: one launch per exchange
    int rc = check_launch(h, "halo_push_kernel"); if (rc) return rc;
    h->launches.halo += 1;
    ++h->halo_groups;
    return FLUID_OK;
}

#ifdef FLUID_TEST_LOOPBACK
// tests/slab_loopback.cu: the ranks of one process on one device, rows moved by stream-ordered device copies
int exchange_loopback(fluid_t* h, const HaloItem* it, int count);
#endif

int exchange_many(fluid_t* h, const HaloItem* it, int count) {
    if (!h->slab()) return FLUID_OK;
    for (int k = 0; k < count; ++k) {
        const HaloRows me = halo_rows(h, own_arena(h), it[k].which);
        if (it[k].n > me.r1 - me.r0)
            return fail(h, FLUID_ERR_HALO, "halo of %d rows exceeds the slab height %d (use fewer GPUs or a taller grid)",
                        it[k].n, me.r1 - me.r0);
    }
    if (h->p2p) return exchange_p2p(h, it, count);
#ifdef FLUID_TEST_LOOPBACK
    return exchange_loopback(h, it, count);
#endif
    ncdl::Api& N = ncdl::api();
    int rc = N.GroupStart();
    for (int k = 0; k < count && !rc; ++k) {
        const HaloItem& q = it[k];
        if (q.n <= 0) continue;
        const HaloRows me = halo_rows(h, own_arena(h), q.which);
        auto at = [&](int grow) { return me.base + (size_t)(grow - me.off) * me.row_bytes; };
        const size_t bytes = (size_t)q.n * me.row_bytes;
        if (h->rank + 1 < h->world) {
            if (!rc) rc = N.Send(at(me.r1 - q.n), bytes, ncdl::ncclInt8, h->rank + 1, h->comm, h->stream);
            if (!rc) rc = N.Recv(at(me.r1), bytes, ncdl::ncclInt8, h->rank + 1, h->comm, h->stream);
        }
        if (h->rank > 0) {
            if (!rc) rc = N.Send(at(me.r0), bytes, ncdl::ncclInt8, h->rank - 1, h->comm, h->stream);
            if (!rc) rc = N.Recv(at(me.r0 - q.n), bytes, ncdl::ncclInt8, h->rank - 1, h->comm, h->stream);
        }
    }
    const int rc2 = N.GroupEnd();
    if (rc || rc2) return fail(h, FLUID_ERR_NCCL, "NCCL halo exchange failed: %s", N.GetErrorString(rc ? rc : rc2));
    ++h->halo_groups;
    return FLUID_OK;
}

int exchange_rows(fluid_t* h, int which, int n) {
    const HaloItem it{which, n};
    return exchange_many(h, &it, 1);
}


// ---- all-gather of row bands (post-FX on slabs) ----------------------------------------------------------
// A dense `rows` x row_bytes buffer of which rank k computed the band [rows*k/world, rows*(k+1)/world) (the
// fractions of the rows a rank owns): afterwards every rank holds every band.  One NCCL group in which each rank
// sends its band to every other rank and receives theirs in place.  NCCL even when the peer-memory halo path is
// on: its IPC mappings reach only the two neighbours.
// `which` names the buffer: the bloom FBO (prefiltered) or the sunrays mask's one-channel alpha.
enum { GB_BLOOM = 0, GB_MASK = 1 };
struct GatherRows { char* base; size_t row_bytes; int rows; };
GatherRows gather_rows(const fluid_t* h, int which) {
    if (which == GB_BLOOM) return {(char*)h->pfx.bloom, (size_t)h->pfx.bw * sizeof(float4), h->pfx.bh};
    return {(char*)h->pfx.mask, (size_t)h->cfg.dye_w * sizeof(float), h->cfg.dye_h};
}
inline int band_row(int rows, int k, int world) { return (int)((long long)rows * k / world); }

#ifdef FLUID_TEST_LOOPBACK_GATHER
// tests/slab_loopback_gather.cu: the ranks of one process on one device, bands moved by stream-ordered device copies
int gather_loopback(fluid_t* h, int which);
#endif

int gather_bands(fluid_t* h, int which) {
    if (!h->slab()) return FLUID_OK;
#ifdef FLUID_TEST_LOOPBACK
#ifdef FLUID_TEST_LOOPBACK_GATHER
    const int lrc = gather_loopback(h, which);
    if (!lrc) ++h->gathers;
    return lrc;
#else
    return fail(h, FLUID_ERR_INVALID, "this loopback build has no row-band gather (build it with FLUID_TEST_LOOPBACK_GATHER)");
#endif
#endif
    const GatherRows g = gather_rows(h, which);
    ncdl::Api& N = ncdl::api();
    int rc = N.GroupStart();
    for (int k = 0; k < h->world && !rc; ++k) {
        if (k == h->rank) continue;
        const int my0 = band_row(g.rows, h->rank, h->world), my1 = band_row(g.rows, h->rank + 1, h->world);
        const int k0 = band_row(g.rows, k, h->world), k1 = band_row(g.rows, k + 1, h->world);
        if (my1 > my0) rc = N.Send(g.base + (size_t)my0 * g.row_bytes, (size_t)(my1 - my0) * g.row_bytes, ncdl::ncclInt8, k, h->comm, h->stream);
        if (!rc && k1 > k0) rc = N.Recv(g.base + (size_t)k0 * g.row_bytes, (size_t)(k1 - k0) * g.row_bytes, ncdl::ncclInt8, k, h->comm, h->stream);
    }
    const int rc2 = N.GroupEnd();
    if (rc || rc2) return fail(h, FLUID_ERR_NCCL, "NCCL row-band gather failed: %s", N.GetErrorString(rc ? rc : rc2));
    ++h->gathers;
    return FLUID_OK;
}
