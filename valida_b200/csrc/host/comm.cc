// Multi-GPU plumbing: ONE proof split across the GPUs of one box (SURVEY.md §8(e)).
// Data path: trace columns shard across the ranks for the coset LDE, the LDE is exchanged ONCE into contiguous row shards
// (kernels storing through peer pointers over NVLink, exchange.cu), and from there every sweep — Keccak leaves and
// sub-trees, quotient, reduced openings, FRI folds — is local to a rank's rows; what crosses ranks afterwards are
// 32-byte sub-roots, per-rank partial sums and the 40 opened rows.
// Two transports behind one interface:
//   * processes (one rank per GPU, torchrun style): NCCL for the small all-gathers / barriers, CUDA IPC for the peer
//     pointers of the symmetric heap.  NCCL is resolved at run time (dlopen of libnccl.so.2 — the copy torch already
//     loaded when the caller is a torchrun rank), so a single-GPU user of the library needs no NCCL at all;
//   * threads of one process (vgpu_comm_init_local — what a Rust host with one worker thread per GPU would use): a host
//     barrier, events across streams and direct peer pointers (cudaDeviceEnablePeerAccess); several ranks may share one
//     device, which is how the split-proof tests run on a one-GPU box.
#include "../ctx.h"
#include <nccl.h>
#include <dlfcn.h>
#include <atomic>
#include <chrono>
#include <cstring>
#include <mutex>
#include <thread>

namespace {

struct Nccl {
    void* lib = nullptr;
    ncclResult_t (*GetUniqueId)(ncclUniqueId*) = nullptr;
    ncclResult_t (*CommInitRank)(ncclComm_t*, int, ncclUniqueId, int) = nullptr;
    ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
    const char* (*GetErrorString)(ncclResult_t) = nullptr;
    ncclResult_t (*AllGather)(const void*, void*, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*Broadcast)(const void*, void*, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
    ncclResult_t (*GroupStart)() = nullptr;
    ncclResult_t (*GroupEnd)() = nullptr;
    std::string why;
};

Nccl& nccl() {
    static Nccl n;
    static std::once_flag once;
    std::call_once(once, [] {
        n.lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
        if (!n.lib) n.lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
        if (!n.lib) { n.why = std::string("cannot load libnccl.so.2: ") + dlerror(); return; }
        auto sym = [&](const char* name) { void* p = dlsym(n.lib, name); if (!p && n.why.empty()) n.why = std::string("libnccl lacks ") + name; return p; };
        n.GetUniqueId = (decltype(n.GetUniqueId))sym("ncclGetUniqueId");
        n.CommInitRank = (decltype(n.CommInitRank))sym("ncclCommInitRank");
        n.CommDestroy = (decltype(n.CommDestroy))sym("ncclCommDestroy");
        n.GetErrorString = (decltype(n.GetErrorString))sym("ncclGetErrorString");
        n.AllGather = (decltype(n.AllGather))sym("ncclAllGather");
        n.Broadcast = (decltype(n.Broadcast))sym("ncclBroadcast");
        n.GroupStart = (decltype(n.GroupStart))sym("ncclGroupStart");
        n.GroupEnd = (decltype(n.GroupEnd))sym("ncclGroupEnd");
        if (!n.why.empty()) n.lib = nullptr;
    });
    return n;
}

#define VG_NCCL(ctx, expr) do { ncclResult_t _r = (expr); if (_r != ncclSuccess) VG_FAIL(ctx, "%s failed: %s", #expr, nccl().GetErrorString(_r)); } while (0)

constexpr size_t SCRATCH_WORDS = 4096;   // barrier tokens + IPC handles of up to 16 ranks

}  // namespace

// ---- in-process ranks ------------------------------------------------------------------------------------
struct VgLocalGroup {
    int n = 0;
    std::vector<vgpu_ctx*> ctx;
    std::atomic<int> arrived{0};
    std::atomic<uint32_t> generation{0};
    std::atomic<int> refs{0};
    std::atomic<bool> broken{false};                 // a rank failed or timed out: every later wait fails at once
    std::vector<const void*> slot;                    // per-rank pointer published before a barrier
    std::vector<cudaEvent_t> ev[2];                   // per-rank barrier events (two alternating slots)
    int timeout_s = 120;
};

namespace {

// sense-reversing barrier over the group's threads; a rank that never arrives turns into an error, not a hang
int32_t host_barrier(vgpu_ctx* ctx) {
    VgLocalGroup* g = (VgLocalGroup*)ctx->local_group;
    if (g->broken.load()) VG_FAIL(ctx, "comm: another rank of the in-process group failed");
    const uint32_t gen = g->generation.load(std::memory_order_acquire);
    if (g->arrived.fetch_add(1, std::memory_order_acq_rel) + 1 == g->n) {
        g->arrived.store(0, std::memory_order_relaxed);
        g->generation.fetch_add(1, std::memory_order_acq_rel);
        return 0;
    }
    const auto t0 = std::chrono::steady_clock::now();
    uint32_t spins = 0;
    while (g->generation.load(std::memory_order_acquire) == gen) {
        if (g->broken.load()) VG_FAIL(ctx, "comm: another rank of the in-process group failed");
        if (++spins > 200) {
            std::this_thread::yield();
            if ((spins & 1023) == 0 && std::chrono::steady_clock::now() - t0 > std::chrono::seconds(g->timeout_s)) {
                g->broken.store(true);
                VG_FAIL(ctx, "comm: rank %d waited %d s at a barrier (a rank left the common call sequence)", ctx->comm_rank, g->timeout_s);
            }
        }
    }
    return 0;
}

int32_t local_barrier(vgpu_ctx* ctx) {
    VgLocalGroup* g = (VgLocalGroup*)ctx->local_group;
    const uint32_t s = ctx->bar_slot; ctx->bar_slot ^= 1;
    VG_CUDA(ctx, cudaEventRecord(g->ev[s][ctx->comm_rank], ctx->stream));
    VG_TRY(host_barrier(ctx));
    for (int p = 0; p < g->n; p++) if (p != ctx->comm_rank) VG_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, g->ev[s][p], 0));
    return 0;
}

}  // namespace

int32_t vg_comm_group_begin(vgpu_ctx* ctx) { if (ctx->nccl) VG_NCCL(ctx, nccl().GroupStart()); return 0; }
int32_t vg_comm_group_end(vgpu_ctx* ctx) { if (ctx->nccl) VG_NCCL(ctx, nccl().GroupEnd()); return 0; }

int32_t vg_comm_barrier(vgpu_ctx* ctx) {
    if (ctx->comm_size <= 1) return 0;
    ctx->stat_barrier.calls++;
    KScope ks(ctx, KC_COLLECTIVE, 0.0);
    if (ctx->local_group) return local_barrier(ctx);
    // an all-gather of one word per rank: completes on a rank only after every rank has enqueued it behind its earlier work
    VG_NCCL(ctx, nccl().AllGather(ctx->comm_scratch + ctx->comm_rank, ctx->comm_scratch, 1, ncclUint32, (ncclComm_t)ctx->nccl, ctx->stream));
    return 0;
}

int32_t vg_comm_allgather_inplace(vgpu_ctx* ctx, uint32_t* buf, uint64_t words_per_rank) {
    if (ctx->comm_size <= 1 || !words_per_rank) return 0;
    ctx->stat_allgather.calls++; ctx->stat_allgather.bytes += 4.0 * (double)words_per_rank * (ctx->comm_size - 1);
    KScope ks(ctx, KC_COLLECTIVE, 4.0 * (double)words_per_rank * (ctx->comm_size - 1));
    if (ctx->nccl) {
        VG_NCCL(ctx, nccl().AllGather(buf + (uint64_t)ctx->comm_rank * words_per_rank, buf, words_per_rank, ncclUint32, (ncclComm_t)ctx->nccl, ctx->stream));
        return 0;
    }
    VgLocalGroup* g = (VgLocalGroup*)ctx->local_group;
    g->slot[ctx->comm_rank] = buf;
    VG_TRY(local_barrier(ctx));                       // every block is written, every pointer published
    for (int p = 0; p < g->n; p++) {
        if (p == ctx->comm_rank) continue;
        const uint32_t* src = (const uint32_t*)g->slot[p] + (uint64_t)p * words_per_rank;
        VG_CUDA(ctx, cudaMemcpyAsync(buf + (uint64_t)p * words_per_rank, src, words_per_rank * 4, cudaMemcpyDefault, ctx->stream));
    }
    return local_barrier(ctx);                        // nobody reuses its block (or the slot table) before all have read it
}

// Uneven runs are gathered at their own offsets (no padding): processes broadcast each rank's run in place, in one NCCL group;
// in-process ranks copy each peer's run from its published buffer.
int32_t vg_comm_allgather_runs(vgpu_ctx* ctx, uint32_t* buf, uint64_t n, uint64_t words) {
    const int G = ctx->comm_size;
    if (G <= 1 || !n || !words) return 0;
    if (vg_run_max(n, G) * (uint64_t)G == n) return vg_comm_allgather_inplace(ctx, buf, n / G * words);    // equal runs, in rank order
    const VgRun mine = vg_run(n, G, ctx->comm_rank, true);
    ctx->stat_allgather.calls++; ctx->stat_allgather.bytes += 4.0 * (double)words * (double)(n - mine.count);
    KScope ks(ctx, KC_COLLECTIVE, 4.0 * (double)words * (double)(n - mine.count));
    if (ctx->nccl) {
        VG_NCCL(ctx, nccl().GroupStart());
        for (int d = 0; d < G; d++) {
            const VgRun run = vg_run(n, G, d, true);
            uint32_t* at = buf + run.begin * words;
            VG_NCCL(ctx, nccl().Broadcast(at, at, run.count * words, ncclUint32, d, (ncclComm_t)ctx->nccl, ctx->stream));
        }
        VG_NCCL(ctx, nccl().GroupEnd());
        return 0;
    }
    VgLocalGroup* g = (VgLocalGroup*)ctx->local_group;
    g->slot[ctx->comm_rank] = buf;
    VG_TRY(local_barrier(ctx));                       // every run is written, every pointer published
    for (int d = 0; d < G; d++) {
        if (d == ctx->comm_rank) continue;
        const VgRun run = vg_run(n, G, d, true);
        VG_CUDA(ctx, cudaMemcpyAsync(buf + run.begin * words, (const uint32_t*)g->slot[d] + run.begin * words, run.count * words * 4, cudaMemcpyDefault, ctx->stream));
    }
    return local_barrier(ctx);
}

// ---- symmetric heap ----------------------------------------------------------------------------------------
static int32_t symm_exchange_bases(vgpu_ctx* ctx) {
    const int G = ctx->comm_size;
    ctx->peer_base.assign(G, nullptr);
    ctx->peer_base[ctx->comm_rank] = ctx->symm_base;
    if (ctx->local_group) {
        VgLocalGroup* g = (VgLocalGroup*)ctx->local_group;
        g->slot[ctx->comm_rank] = ctx->symm_base;
        VG_TRY(host_barrier(ctx));
        for (int p = 0; p < G; p++) ctx->peer_base[p] = (uint8_t*)g->slot[p];
        return host_barrier(ctx);
    }
    // processes: all-gather the IPC handles through the device scratch, open the peers' heaps
    static_assert(sizeof(cudaIpcMemHandle_t) == 64, "IPC handle size");
    cudaIpcMemHandle_t mine;
    VG_CUDA(ctx, cudaIpcGetMemHandle(&mine, ctx->symm_base));
    uint32_t* area = ctx->comm_scratch + 64;          // past the barrier tokens
    VG_CUDA(ctx, cudaMemcpyAsync(area + 16 * ctx->comm_rank, &mine, 64, cudaMemcpyHostToDevice, ctx->stream));
    VG_NCCL(ctx, nccl().AllGather(area + 16 * ctx->comm_rank, area, 16, ncclUint32, (ncclComm_t)ctx->nccl, ctx->stream));
    std::vector<cudaIpcMemHandle_t> all(G);
    VG_CUDA(ctx, cudaMemcpyAsync(all.data(), area, 64 * (size_t)G, cudaMemcpyDeviceToHost, ctx->stream));
    VG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    for (int p = 0; p < G; p++) {
        if (p == ctx->comm_rank) continue;
        void* q = nullptr;
        cudaError_t e = cudaIpcOpenMemHandle(&q, all[p], cudaIpcMemLazyEnablePeerAccess);
        if (e != cudaSuccess) VG_FAIL(ctx, "comm: cudaIpcOpenMemHandle of rank %d's heap failed: %s (the split proof needs peer access between the GPUs)", p, cudaGetErrorString(e));
        ctx->peer_base[p] = (uint8_t*)q;
    }
    return 0;
}

static void symm_release(vgpu_ctx* ctx) {
    if (!ctx->symm_base) return;
    cudaStreamSynchronize(ctx->stream);
    if (!ctx->local_group)
        for (int p = 0; p < (int)ctx->peer_base.size(); p++) if (p != ctx->comm_rank && ctx->peer_base[p]) cudaIpcCloseMemHandle(ctx->peer_base[p]);
    ctx->peer_base.clear();
    cudaFree(ctx->symm_base);
    ctx->symm_base = nullptr; ctx->symm_bytes = 0;
    ctx->symm_free.clear(); ctx->symm_live.clear(); ctx->symm_live_bytes = 0;
}

int32_t vg_symm_reserve(vgpu_ctx* ctx, size_t extra_bytes) {
    if (ctx->comm_size <= 1) VG_FAIL(ctx, "symmetric heap: no communicator");
    const size_t need = ctx->symm_live_bytes + extra_bytes + (1u << 20);
    if (need <= ctx->symm_bytes) {
        // room in total; a fragmented heap is caught by vg_symm_alloc
        return 0;
    }
    if (!ctx->symm_live.empty())
        VG_FAIL(ctx, "symmetric heap: %zu MB live + %zu MB requested exceed the %zu MB heap and it cannot grow while buffers are live (set VGPU_SYMM_HEAP_MB)",
                ctx->symm_live_bytes >> 20, extra_bytes >> 20, ctx->symm_bytes >> 20);
    size_t bytes = need + need / 8;
    size_t floor_mb = 512;                                            // floor: small commits one after the other never regrow
    if (const char* e = getenv("VGPU_SYMM_HEAP_MIN_MB")) floor_mb = (size_t)atoll(e);
    if (bytes < (floor_mb << 20)) bytes = floor_mb << 20;
    if (const char* e = getenv("VGPU_SYMM_HEAP_MB")) { const size_t v = (size_t)atoll(e) << 20; if (v > bytes) bytes = v; }
    bytes = (bytes + (2u << 20) - 1) & ~(size_t)((2u << 20) - 1);
    // quiesce: peers may still be reading the old heap
    VG_TRY(vg_comm_barrier(ctx));
    VG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    if (ctx->local_group) VG_TRY(host_barrier(ctx));
    symm_release(ctx);
    // the caching allocator may hold what the heap needs
    cudaError_t e = cudaMalloc((void**)&ctx->symm_base, bytes);
    if (e != cudaSuccess) {
        cudaGetLastError();
        for (auto& kv : ctx->free_bufs) cudaFree(kv.second);
        ctx->free_bufs.clear(); ctx->cached_bytes = 0;
        e = cudaMalloc((void**)&ctx->symm_base, bytes);
    }
    if (e != cudaSuccess) { ctx->symm_base = nullptr; VG_FAIL(ctx, "symmetric heap: cudaMalloc(%zu MB) failed: %s", bytes >> 20, cudaGetErrorString(e)); }
    ctx->symm_bytes = bytes;
    ctx->symm_free.clear(); ctx->symm_free[0] = bytes;
    return symm_exchange_bases(ctx);
}

int32_t vg_symm_alloc(vgpu_ctx* ctx, void** p, size_t bytes) {
    bytes = vg_symm_round(bytes ? bytes : 1);
    for (auto it = ctx->symm_free.begin(); it != ctx->symm_free.end(); ++it) {    // first fit: deterministic across ranks
        if (it->second < bytes) continue;
        const size_t off = it->first, len = it->second;
        ctx->symm_free.erase(it);
        if (len > bytes) ctx->symm_free[off + bytes] = len - bytes;
        *p = ctx->symm_base + off;
        ctx->symm_live[*p] = bytes;
        ctx->symm_live_bytes += bytes;
        if (ctx->symm_live_bytes > ctx->symm_peak_bytes) ctx->symm_peak_bytes = ctx->symm_live_bytes;
        return 0;
    }
    VG_FAIL(ctx, "symmetric heap: no run of %zu MB left (%zu MB heap, %zu MB live); vg_symm_reserve was not called with the full need or VGPU_SYMM_HEAP_MB is too small",
            bytes >> 20, ctx->symm_bytes >> 20, ctx->symm_live_bytes >> 20);
}

void vg_symm_free(vgpu_ctx* ctx, void* p) {
    if (!p) return;
    auto it = ctx->symm_live.find(p);
    if (it == ctx->symm_live.end()) return;
    size_t off = (uint8_t*)p - ctx->symm_base, len = it->second;
    ctx->symm_live.erase(it);
    ctx->symm_live_bytes -= len;
    auto nx = ctx->symm_free.lower_bound(off);
    if (nx != ctx->symm_free.end() && off + len == nx->first) { len += nx->second; nx = ctx->symm_free.erase(nx); }
    if (nx != ctx->symm_free.begin()) {
        auto pv = std::prev(nx);
        if (pv->first + pv->second == off) { off = pv->first; len += pv->second; ctx->symm_free.erase(pv); }
    }
    ctx->symm_free[off] = len;
}

void vg_comm_free(vgpu_ctx* ctx) {
    symm_release(ctx);
    if (ctx->comm_scratch) { cudaFree(ctx->comm_scratch); ctx->comm_scratch = nullptr; }
    if (ctx->nccl) { nccl().CommDestroy((ncclComm_t)ctx->nccl); ctx->nccl = nullptr; }
    if (ctx->local_group) {
        VgLocalGroup* g = (VgLocalGroup*)ctx->local_group;
        g->broken.store(true);                        // a rank that leaves ends the group for the others
        if (g->refs.fetch_sub(1) == 1) {
            for (int s = 0; s < 2; s++) for (auto e : g->ev[s]) if (e) cudaEventDestroy(e);
            delete g;
        }
        ctx->local_group = nullptr;
    }
    ctx->comm_size = 1; ctx->comm_rank = 0; ctx->sharding = false;
}

extern "C" {

int32_t vgpu_comm_unique_id(uint8_t out[VGPU_COMM_ID_BYTES]) {
    static_assert(sizeof(ncclUniqueId) == VGPU_COMM_ID_BYTES, "ncclUniqueId size");
    if (!out || !nccl().lib) return -1;
    ncclUniqueId id;
    if (nccl().GetUniqueId(&id) != ncclSuccess) return -1;
    std::memcpy(out, &id, sizeof id);
    return 0;
}

int32_t vgpu_comm_init(vgpu_ctx* ctx, int32_t nranks, int32_t rank, const uint8_t unique_id[VGPU_COMM_ID_BYTES]) {
    if (!ctx) return -1;
    if (nranks < 1 || rank < 0 || rank >= nranks || !unique_id) VG_FAIL(ctx, "comm_init: bad rank %d of %d", rank, nranks);
    if (nranks > VG_MAX_RANKS) VG_FAIL(ctx, "comm_init: the number of ranks must be 1..%d, got %d", VG_MAX_RANKS, nranks);
    if (!nccl().lib) VG_FAIL(ctx, "comm_init: %s", nccl().why.c_str());
    vg_comm_free(ctx);
    VG_CUDA(ctx, cudaSetDevice(ctx->device));
    ncclUniqueId id;
    std::memcpy(&id, unique_id, sizeof id);
    ncclComm_t comm = nullptr;
    VG_NCCL(ctx, nccl().CommInitRank(&comm, nranks, id, rank));
    ctx->nccl = comm; ctx->comm_size = nranks; ctx->comm_rank = rank; ctx->sharding = nranks > 1;
    VG_CUDA(ctx, cudaMalloc((void**)&ctx->comm_scratch, SCRATCH_WORDS * 4));
    VG_CUDA(ctx, cudaMemsetAsync(ctx->comm_scratch, 0, SCRATCH_WORDS * 4, ctx->stream));
    return 0;
}

// In-process group: ctxs[i] becomes rank i.  Called ONCE by one thread before the worker threads start; afterwards every
// rank's calls must come from its own thread (the collectives block on a host barrier until all ranks arrive).
int32_t vgpu_comm_init_local(vgpu_ctx* const* ctxs, int32_t nranks) {
    if (!ctxs || nranks < 1) return -1;
    vgpu_ctx* c0 = ctxs[0];
    if (nranks > VG_MAX_RANKS) VG_FAIL(c0, "comm_init_local: the number of ranks must be 1..%d, got %d", VG_MAX_RANKS, nranks);
    VgLocalGroup* g = new VgLocalGroup();
    g->n = nranks; g->ctx.assign(ctxs, ctxs + nranks); g->slot.assign(nranks, nullptr); g->refs.store(nranks);
    if (const char* e = getenv("VGPU_COMM_TIMEOUT_S")) g->timeout_s = atoi(e) > 0 ? atoi(e) : g->timeout_s;
    for (int s = 0; s < 2; s++) g->ev[s].assign(nranks, nullptr);
    for (int r = 0; r < nranks; r++) {
        vgpu_ctx* c = ctxs[r];
        vg_comm_free(c);
        VG_CUDA(c, cudaSetDevice(c->device));
        for (int p = 0; p < nranks; p++) {
            if (ctxs[p]->device == c->device) continue;
            int can = 0;
            VG_CUDA(c, cudaDeviceCanAccessPeer(&can, c->device, ctxs[p]->device));
            if (!can) VG_FAIL(c, "comm_init_local: device %d cannot access device %d", c->device, ctxs[p]->device);
            cudaError_t e = cudaDeviceEnablePeerAccess(ctxs[p]->device, 0);
            if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) VG_FAIL(c, "cudaDeviceEnablePeerAccess(%d) failed: %s", ctxs[p]->device, cudaGetErrorString(e));
            cudaGetLastError();
        }
        for (int s = 0; s < 2; s++) VG_CUDA(c, cudaEventCreateWithFlags(&g->ev[s][r], cudaEventDisableTiming));
        c->local_group = g; c->comm_size = nranks; c->comm_rank = r; c->sharding = nranks > 1; c->bar_slot = 0;
    }
    return 0;
}

int32_t vgpu_comm_set_sharding(vgpu_ctx* ctx, int32_t on) {
    if (!ctx) return -1;
    if (on && !ctx->nccl && !ctx->local_group) VG_FAIL(ctx, "comm_set_sharding: vgpu_comm_init has not been called");
    ctx->sharding = on != 0;
    return 0;
}

// per-proof collective counters: calls[0..2] / bytes[0..2] = barriers, all-gathers, peer-store exchanges since the last reset
void vgpu_comm_stats(vgpu_ctx* ctx, uint32_t calls[3], double bytes[3], int32_t reset) {
    const vgpu_ctx::CommStat* s[3] = {&ctx->stat_barrier, &ctx->stat_allgather, &ctx->stat_exchange};
    for (int i = 0; i < 3; i++) { calls[i] = s[i]->calls; bytes[i] = s[i]->bytes; }
    if (reset) { ctx->stat_barrier = {}; ctx->stat_allgather = {}; ctx->stat_exchange = {}; }
}

// the share of a tree layer of `len` nodes that rank `rank` derives itself (merkle.cu); *split = 0 when the
// layer is above the last split one and every rank computes all of it
void vgpu_tree_share(uint64_t len, int32_t nranks, int32_t rank, uint64_t* begin, uint64_t* count, int32_t* split) {
    const VgRun run = vg_layer_run(len, nranks, rank);
    *begin = run.begin; *count = run.count; *split = run.split;
}
// the run of a matrix / vector of `n` stored rows that rank `rank` holds in a split proof of nranks ranks (ctx.h); *split = 0 when
// it is too short to be split and every rank holds all of it
void vgpu_row_share(uint64_t n, int32_t nranks, int32_t rank, uint64_t* begin, uint64_t* count, int32_t* split) {
    const VgRun run = vg_run(n, nranks, rank, vg_split_rows_n(n, nranks));
    *begin = run.begin; *count = run.count; *split = run.split;
}

void vgpu_shard_range(uint64_t total, int32_t nranks, int32_t rank, uint64_t* begin, uint64_t* end) {
    // the first (total % nranks) ranks take one extra unit
    const uint64_t q = total / (uint64_t)nranks, r = total % (uint64_t)nranks, k = (uint64_t)rank;
    *begin = k * q + (k < r ? k : r);
    *end = *begin + q + (k < r ? 1 : 0);
}

}  // extern "C"
