// slab_loopback_gather.cu — the loopback test build of slab_loopback.cu with the row-band all-gather that a slab's
// post-FX runs (halo.cuh gather_bands): BLOOM and SUNRAYS frames, canvases and captures on N slab ranks of one
// process on one device (tests/test_gpu_slab_draw.py).  Not part of the product: the real transport is NCCL.
//
// One gather, per rank, with the group, events and barrier of slab_loopback.cu:
//   1. record `ready` on my stream (my band of the buffer is final up to here);
//   2. host barrier across the group;
//   3. my stream waits for every other rank's `ready`;
//   4. device copies of every other rank's band of its buffer into the same rows of mine;
//   5. record `consumed` on my stream;
//   6. host barrier;
//   7. my stream waits for every other rank's `consumed` before anything later may overwrite my band.
#define FLUID_TEST_LOOPBACK_GATHER 1
#include "slab_loopback.cu"

namespace {

int gather_loopback(fluid_t* h, int which) {
    std::shared_ptr<LoopGroup> g = group_of(h);
    if (!g) return fail(h, FLUID_ERR_HALO, "slab rank %d of %d is not linked into a loopback group", h->rank, h->world);
    CU(cudaEventRecord(g->ready[h->rank], h->stream));
    if (!barrier(*g)) return fail(h, FLUID_ERR_HALO, "loopback gather: a rank did not arrive within 60 s");
    // between the two barriers every rank is inside this function: the other ranks' buffers hold still
    for (const fluid_t* n : g->ranks)
        if (n != h) CU(cudaStreamWaitEvent(h->stream, g->ready[n->rank], 0));
    const GatherRows me = gather_rows(h, which);
    int rc = FLUID_OK;
    for (const fluid_t* n : g->ranks) {
        if (n == h) continue;
        const GatherRows src = gather_rows(n, which);
        if (src.rows != me.rows || src.row_bytes != me.row_bytes || !src.base || !me.base) {
            rc = fail(h, FLUID_ERR_HALO, "gather %d: rank %d holds %d rows of %zu bytes, rank %d %d of %zu", which, n->rank,
                      src.rows, src.row_bytes, h->rank, me.rows, me.row_bytes);
            break;
        }
        const int k0 = band_row(me.rows, n->rank, h->world), k1 = band_row(me.rows, n->rank + 1, h->world);
        if (k1 <= k0) continue;
        const cudaError_t e = cudaMemcpyAsync(me.base + (size_t)k0 * me.row_bytes, src.base + (size_t)k0 * me.row_bytes,
                                              (size_t)(k1 - k0) * me.row_bytes, cudaMemcpyDeviceToDevice, h->stream);
        if (e != cudaSuccess) { rc = fail(h, FLUID_ERR_CUDA, "loopback gather copy: %s", cudaGetErrorString(e)); break; }
    }
    // the second half runs even after a failed copy, so that the other ranks are not left at the barrier
    CU(cudaEventRecord(g->consumed[h->rank], h->stream));
    if (!barrier(*g)) return fail(h, FLUID_ERR_HALO, "loopback gather: a rank did not arrive within 60 s");
    for (const fluid_t* n : g->ranks)
        if (n != h) CU(cudaStreamWaitEvent(h->stream, g->consumed[n->rank], 0));
    return rc;
}

}  // namespace
