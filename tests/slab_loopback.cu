// slab_loopback.cu — a test build of libfluid_b200 whose row-slab ranks are handles of ONE process on ONE
// device.  It is fluid.cu compiled with FLUID_TEST_LOOPBACK, which (a) skips NCCL when a slab handle is
// created and (b) routes every halo exchange to exchange_loopback below.  Everything else — the step, the
// Jacobi plan and launches, the splats, resize and render bands, the ghost-zone checks — is the library's own
// code, so N slab handles on one GPU can be compared row for row with an ordinary handle
// (tests/test_gpu_slab_loopback.py).  Not part of the product: the real transports are NCCL and the
// peer-memory push of halo.cuh, which this build does not run.
//
// Each rank is driven from its own host thread.  One exchange, per rank:
//   1. record `ready` on my stream (my owned rows are final up to here);
//   2. host barrier across the group;
//   3. my stream waits for the neighbours' `ready`;
//   4. device copies of the neighbours' owned boundary rows into my ghost rows;
//   5. record `consumed` on my stream (my copies out of the neighbours' rows are queued before it);
//   6. host barrier;
//   7. my stream waits for the neighbours' `consumed` before anything later may overwrite my owned rows.
// Every wait names an event that is already recorded: the device never waits for work that has not been
// enqueued.  A barrier that does not complete within 60 s fails the exchange with FLUID_ERR_HALO and marks the
// group broken, so that the other ranks fail at once instead of blocking.
#define FLUID_TEST_LOOPBACK 1
#include "../webgl_fluid_simulation_b200/csrc/fluid.cu"

#include <chrono>
#include <condition_variable>
#include <memory>
#include <mutex>

namespace {

struct LoopGroup {
    std::vector<fluid_t*> ranks;
    std::vector<cudaEvent_t> ready, consumed;      // one of each per rank, re-recorded at every exchange
    std::mutex m;
    std::condition_variable cv;
    int arrived = 0;
    uint64_t generation = 0;
    bool broken = false;
    ~LoopGroup() {
        for (cudaEvent_t e : ready) if (e) cudaEventDestroy(e);
        for (cudaEvent_t e : consumed) if (e) cudaEventDestroy(e);
    }
};

std::mutex g_groups_mu;
std::map<const fluid_t*, std::shared_ptr<LoopGroup>> g_groups;    // rank handle -> the group it was linked into

std::shared_ptr<LoopGroup> group_of(const fluid_t* h) {
    std::lock_guard<std::mutex> lk(g_groups_mu);
    auto it = g_groups.find(h);
    if (it == g_groups.end() || it->second->ranks[h->rank] != h) return nullptr;
    return it->second;
}

bool barrier(LoopGroup& g) {
    std::unique_lock<std::mutex> lk(g.m);
    if (g.broken) return false;
    const uint64_t gen = g.generation;
    if (++g.arrived == (int)g.ranks.size()) {
        g.arrived = 0;
        ++g.generation;
        g.cv.notify_all();
        return true;
    }
    if (!g.cv.wait_for(lk, std::chrono::seconds(60), [&] { return g.generation != gen || g.broken; }) || g.broken) {
        g.broken = true;
        g.cv.notify_all();
        return false;
    }
    return true;
}

// The NCCL branch of exchange_many with device copies: for each item, my ghost rows [row0 - n, row0) and
// [row1, row1 + n) receive the rows the neighbour below / above owns there, all items in one group.
int exchange_loopback(fluid_t* h, const HaloItem* it, int count) {
    std::shared_ptr<LoopGroup> g = group_of(h);
    if (!g) return fail(h, FLUID_ERR_HALO, "slab rank %d of %d is not linked into a loopback group", h->rank, h->world);
    const fluid_t* nb[2] = {h->rank > 0 ? g->ranks[h->rank - 1] : nullptr,
                            h->rank + 1 < h->world ? g->ranks[h->rank + 1] : nullptr};
    CU(cudaEventRecord(g->ready[h->rank], h->stream));
    if (!barrier(*g)) return fail(h, FLUID_ERR_HALO, "loopback halo exchange: a rank did not arrive within 60 s");
    // between the two barriers every rank is inside this function: the neighbours' handles hold still
    for (const fluid_t* n : nb)
        if (n) CU(cudaStreamWaitEvent(h->stream, g->ready[n->rank], 0));
    int rc = FLUID_OK;
    for (int k = 0; k < count && !rc; ++k) {
        const HaloItem& q = it[k];
        if (q.n <= 0) continue;
        const HaloRows me = halo_rows(h, own_arena(h), q.which);
        for (int side = 0; side < 2 && !rc; ++side) {
            const fluid_t* n = nb[side];
            if (!n) continue;
            // the neighbour's buffer in the slot MY pair reads, as the peer-memory push addresses it: the swap
            // parity of a pair must be the same on every rank
            const HaloRows src = halo_rows(h, fluid::Peer{true, n->arena, n->roff, n->droff, n->layout}, q.which);
            const HaloRows own = halo_rows(n, own_arena(n), q.which);
            if (src.base != own.base) {
                rc = fail(h, FLUID_ERR_HALO, "halo item %d: rank %d reads the other slot of the pair than rank %d", q.which, n->rank, h->rank);
                break;
            }
            const int g0 = (side == 0) ? me.r0 - q.n : me.r1;    // rows the neighbour owns that I keep as ghosts
            const char* s = src.base + (size_t)(g0 - src.off) * me.row_bytes;
            char* d = me.base + (size_t)(g0 - me.off) * me.row_bytes;
            const cudaError_t e = cudaMemcpyAsync(d, s, (size_t)q.n * me.row_bytes, cudaMemcpyDeviceToDevice, h->stream);
            if (e != cudaSuccess) rc = fail(h, FLUID_ERR_CUDA, "loopback halo copy: %s", cudaGetErrorString(e));
        }
    }
    // the second half runs even after a failed copy, so that the other ranks are not left at the barrier
    CU(cudaEventRecord(g->consumed[h->rank], h->stream));
    if (!barrier(*g)) return fail(h, FLUID_ERR_HALO, "loopback halo exchange: a rank did not arrive within 60 s");
    for (const fluid_t* n : nb)
        if (n) CU(cudaStreamWaitEvent(h->stream, g->consumed[n->rank], 0));
    if (rc) return rc;
    ++h->halo_groups;
    return FLUID_OK;
}

}  // namespace

extern "C" {

// Links ranks[0..world) — slab handles rank k of `world` on one device, made by fluid_create_slab of this
// build — into one group.  Every rank must be linked before its first call that exchanges halos; linking a
// handle again moves it to the new group.
int fluid_loopback_link(fluid_t** ranks, int world) {
    if (!ranks || world < 2) return fail(nullptr, FLUID_ERR_INVALID, "a loopback group has at least 2 ranks");
    for (int k = 0; k < world; ++k) {
        const fluid_t* h = ranks[k];
        if (!h || h->rank != k || h->world != world || h->batch)
            return fail(nullptr, FLUID_ERR_INVALID, "ranks[%d] is not slab rank %d of %d", k, k, world);
        if (h->device != ranks[0]->device)
            return fail(nullptr, FLUID_ERR_INVALID, "loopback ranks share one device (rank %d is on %d, rank 0 on %d)",
                        k, h->device, ranks[0]->device);
    }
    auto g = std::make_shared<LoopGroup>();
    g->ranks.assign(ranks, ranks + world);
    g->ready.assign(world, nullptr);
    g->consumed.assign(world, nullptr);
    if (cudaSetDevice(ranks[0]->device) != cudaSuccess) return fail(nullptr, FLUID_ERR_CUDA, "cudaSetDevice");
    for (int k = 0; k < world; ++k)
        if (cudaEventCreateWithFlags(&g->ready[k], cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&g->consumed[k], cudaEventDisableTiming) != cudaSuccess)
            return fail(nullptr, FLUID_ERR_CUDA, "cudaEventCreate");
    std::lock_guard<std::mutex> lk(g_groups_mu);
    for (int k = 0; k < world; ++k) g_groups[ranks[k]] = g;
    return FLUID_OK;
}

}  // extern "C"
