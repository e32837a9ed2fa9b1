// K12 — host <-> device staging: RowMajorMatrix<Val> (machine/src/config.rs:17-22 boundary type)
// to/from the device's column-major Montgomery store.  One H2D/D2H copy of the row-major image plus
// a shared-memory tile transpose: 64 rows x w words are read as one contiguous run (coalesced) and
// written as w runs of 64 consecutive rows (256 B segments).
#include "ctx.h"
#include <atomic>
#include <condition_variable>
#include <cstring>
#include <memory>
#include <mutex>
#include <thread>

namespace {
constexpr int TR = 64;      // rows per tile
constexpr int TW = 128;     // max columns per tile

__global__ void __launch_bounds__(256) rm_to_cm_kernel(const uint32_t* __restrict__ rm, uint64_t h, uint64_t w, uint32_t* __restrict__ cm, uint64_t cs, int to_monty, uint64_t c0, uint32_t wc) {
    __shared__ uint32_t tile[TR][TW + 1];
    uint64_t r0 = (uint64_t)blockIdx.x * TR;
    uint32_t rows = (uint32_t)(h - r0 < TR ? h - r0 : TR);
    if (wc == w) {   // whole rows are contiguous: one run of rows*w words
        uint32_t tot = rows * wc;
        const uint32_t* src = rm + r0 * w;
        for (uint32_t i = threadIdx.x; i < tot; i += blockDim.x) tile[i / wc][i % wc] = src[i];
    } else {
        for (uint32_t i = threadIdx.x; i < rows * wc; i += blockDim.x) { uint32_t r = i / wc, c = i % wc; tile[r][c] = rm[(r0 + r) * w + c0 + c]; }
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < rows * wc; i += blockDim.x) {
        uint32_t c = i / rows, r = i % rows;
        uint32_t v = tile[r][c];
        cm[(c0 + c) * cs + r0 + r] = to_monty ? bb::to_monty(v) : v;
    }
}
__global__ void __launch_bounds__(256) cm_to_rm_kernel(const uint32_t* __restrict__ cm, uint64_t cs, uint64_t h, uint64_t w, uint32_t* __restrict__ rm, int from_monty, uint64_t c0, uint32_t wc) {
    __shared__ uint32_t tile[TR][TW + 1];
    uint64_t r0 = (uint64_t)blockIdx.x * TR;
    uint32_t rows = (uint32_t)(h - r0 < TR ? h - r0 : TR);
    for (uint32_t i = threadIdx.x; i < rows * wc; i += blockDim.x) {
        uint32_t c = i / rows, r = i % rows;
        uint32_t v = cm[(c0 + c) * cs + r0 + r];
        tile[r][c] = from_monty ? bb::from_monty(v) : v;
    }
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < rows * wc; i += blockDim.x) { uint32_t r = i / wc, c = i % wc; rm[(r0 + r) * w + c0 + c] = tile[r][c]; }
}
}  // namespace

static int32_t transpose_in(vgpu_ctx* ctx, const uint32_t* stage, uint64_t h, uint64_t w, int32_t repr, vgpu_dmat* dst) {
    for (uint64_t c0 = 0; c0 < w; c0 += TW) {
        uint32_t wc = (uint32_t)(w - c0 < TW ? w - c0 : TW);
        KScope ks(ctx, KC_TRANSPOSE, 8.0 * (double)h * wc);
        rm_to_cm_kernel<<<(unsigned)((h + TR - 1) / TR), 256, 0, ctx->stream>>>(stage, h, w, dst->d, dst->col_stride, repr == VGPU_REPR_CANONICAL, c0, wc);
        VG_LAUNCH_CHECK(ctx);
    }
    return 0;
}

int32_t vg_upload_rowmajor(vgpu_ctx* ctx, const uint32_t* host, uint64_t h, uint64_t w, int32_t repr, vgpu_dmat* dst) {
    if (h == 0 || w == 0) return 0;
    VgBuf stage(ctx);
    VG_TRY(stage.upload(host, h * w));
    return transpose_in(ctx, stage.as<uint32_t>(), h, w, repr, dst);
}

// ---- uploads out of PAGEABLE caller memory (a Rust Vec, a numpy array) ------------------------------------------------------
// cudaMemcpyAsync from pageable memory is staged by the runtime through one bounce buffer on the calling thread (~7 GB/s measured:
// 0.3 s for the 2 GB of a 2^22-row witness, twice the proving time).  Here a few host threads copy 16 MB chunks into page-locked
// buffers of the context and enqueue the chunk copies on the copy stream themselves; the proving thread goes on enqueueing kernels
// and only waits, per matrix, until that matrix's last chunk has been ENQUEUED (vg_dmat_materialize), not until it has arrived.
namespace {
constexpr size_t STAGE_CHUNK = 16u << 20, STAGE_MIN = 8u << 20;
constexpr int STAGE_THREADS = 6;
struct StageJob {
    const uint8_t* src; uint8_t* dst; size_t bytes, first_chunk, nchunks;
    cudaEvent_t done = nullptr;
    std::atomic<size_t> left{0};
    std::atomic<bool> issued{false};
};
}  // namespace
struct VgStager {
    std::vector<std::unique_ptr<StageJob>> jobs;
    std::vector<std::thread> threads;
    std::mutex mu; std::condition_variable cv;
    uint8_t* pinned[STAGE_THREADS][2] = {};
    cudaEvent_t free_ev[STAGE_THREADS][2] = {};
    std::atomic<bool> failed{false};
    bool running = false;
};
namespace {
void stager_worker(vgpu_ctx* ctx, VgStager* st, int t) {
    cudaSetDevice(ctx->device);
    bool used[2] = {false, false};
    int b = 0;
    for (auto& jp : st->jobs) {
        StageJob& j = *jp;
        for (size_t c = 0; c < j.nchunks; c++) {
            if ((j.first_chunk + c) % STAGE_THREADS != (size_t)t) continue;
            const size_t off = c * STAGE_CHUNK, n = std::min(STAGE_CHUNK, j.bytes - off);
            bool ok = !st->failed.load();
            if (ok && used[b]) ok = cudaEventSynchronize(st->free_ev[t][b]) == cudaSuccess;
            if (ok) {
                std::memcpy(st->pinned[t][b], j.src + off, n);
                ok = cudaMemcpyAsync(j.dst + off, st->pinned[t][b], n, cudaMemcpyHostToDevice, ctx->copy_stream) == cudaSuccess &&
                     cudaEventRecord(st->free_ev[t][b], ctx->copy_stream) == cudaSuccess;
                used[b] = true; b ^= 1;
            }
            if (!ok) st->failed.store(true);
            if (j.left.fetch_sub(1) == 1) {        // the last chunk of this matrix has been enqueued (by whichever thread)
                if (cudaEventRecord(j.done, ctx->copy_stream) != cudaSuccess) st->failed.store(true);
                { std::lock_guard<std::mutex> lk(st->mu); j.issued.store(true); }
                st->cv.notify_all();
            }
        }
    }
}
bool is_pageable(const void* p) {
    cudaPointerAttributes a{};
    if (cudaPointerGetAttributes(&a, p) != cudaSuccess) { cudaGetLastError(); return true; }
    return a.type == cudaMemoryTypeUnregistered;
}
}  // namespace

// after the last vg_upload_begin of a vgpu_prove: start copying
int32_t vg_stager_start(vgpu_ctx* ctx) {
    VgStager* st = (VgStager*)ctx->stager;
    if (!st || st->jobs.empty() || st->running) return 0;
    for (int t = 0; t < STAGE_THREADS; t++)
        for (int b = 0; b < 2; b++)
            if (!st->pinned[t][b]) {
                VG_CUDA(ctx, cudaHostAlloc((void**)&st->pinned[t][b], STAGE_CHUNK, cudaHostAllocDefault));
                VG_CUDA(ctx, cudaEventCreateWithFlags(&st->free_ev[t][b], cudaEventDisableTiming));
            }
    st->failed.store(false);
    st->running = true;
    for (int t = 0; t < STAGE_THREADS; t++) st->threads.emplace_back(stager_worker, ctx, st, t);
    return 0;
}
// before vgpu_prove returns (also on its error paths): the caller's buffers are no longer read after this
int32_t vg_stager_finish(vgpu_ctx* ctx) {
    VgStager* st = (VgStager*)ctx->stager;
    if (!st) return 0;
    for (auto& th : st->threads) th.join();
    st->threads.clear();
    const bool failed = st->running && st->failed.load();
    st->running = false;
    for (auto& j : st->jobs) if (j->done) ctx->event_pool.push_back(j->done);
    st->jobs.clear();
    if (failed) VG_FAIL(ctx, "upload: a staged copy out of pageable memory failed");
    return 0;
}
void vg_stager_free(vgpu_ctx* ctx) {
    VgStager* st = (VgStager*)ctx->stager;
    if (!st) return;
    vg_stager_finish(ctx);
    for (int t = 0; t < STAGE_THREADS; t++) for (int b = 0; b < 2; b++) { if (st->pinned[t][b]) cudaFreeHost(st->pinned[t][b]); if (st->free_ev[t][b]) cudaEventDestroy(st->free_ev[t][b]); }
    delete st;
    ctx->stager = nullptr;
}

// Pipelined form used by vgpu_prove: the copy is queued on the context's copy stream (so it overlaps the kernels of
// matrices that arrived earlier) and the transpose is deferred to the matrix's first use on the compute stream.
int32_t vg_upload_begin(vgpu_ctx* ctx, const uint32_t* host, uint64_t h, uint64_t w, int32_t repr, vgpu_dmat* dst) {
    if (h == 0 || w == 0) return 0;
    if (!ctx->copy_stream) VG_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking));
    VG_TRY(vg_alloc(ctx, (void**)&dst->pend_stage, h * w * 4));
    {   // the staging block may be a cached one whose last user is still queued on the compute stream
        cudaEvent_t fence;
        VG_CUDA(ctx, vg_take_event(ctx, &fence));
        VG_CUDA(ctx, cudaEventRecord(fence, ctx->stream));
        VG_CUDA(ctx, cudaStreamWaitEvent(ctx->copy_stream, fence, 0));
        ctx->event_pool.push_back(fence);
    }
    VG_CUDA(ctx, vg_take_event(ctx, &dst->pend_ev));
    dst->pend_repr = repr;
    const size_t bytes = h * w * 4;
    if (bytes >= STAGE_MIN && is_pageable(host)) {
        if (!ctx->stager) ctx->stager = new VgStager();
        VgStager* st = (VgStager*)ctx->stager;
        if (st->running) VG_FAIL(ctx, "upload: a staged upload is already running on this context");
        std::unique_ptr<StageJob> j(new StageJob());
        j->src = (const uint8_t*)host; j->dst = (uint8_t*)dst->pend_stage; j->bytes = bytes;
        j->nchunks = (bytes + STAGE_CHUNK - 1) / STAGE_CHUNK;
        j->first_chunk = st->jobs.empty() ? 0 : st->jobs.back()->first_chunk + st->jobs.back()->nchunks;
        j->left.store(j->nchunks);
        j->done = dst->pend_ev;              // recorded by the thread that enqueues the last chunk
        dst->pend_job = j.get();
        dst->pend_ev = nullptr;              // owned by the job until it is issued
        st->jobs.push_back(std::move(j));
        return 0;
    }
    VG_CUDA(ctx, cudaMemcpyAsync(dst->pend_stage, host, bytes, cudaMemcpyHostToDevice, ctx->copy_stream));
    VG_CUDA(ctx, cudaEventRecord(dst->pend_ev, ctx->copy_stream));
    return 0;
}

// the event after which the row-major image of `m` is in pend_stage (waits, for a staged upload, until its last chunk is enqueued)
static int32_t pending_event(vgpu_ctx* ctx, vgpu_dmat* m, cudaEvent_t* ev) {
    if (m->pend_job) {
        VgStager* st = (VgStager*)ctx->stager;
        StageJob* j = (StageJob*)m->pend_job;
        if (!st || !st->running) VG_FAIL(ctx, "upload: the staged copy of this matrix was never started");
        std::unique_lock<std::mutex> lk(st->mu);
        st->cv.wait(lk, [&] { return j->issued.load(); });
        if (st->failed.load()) VG_FAIL(ctx, "upload: a staged copy out of pageable memory failed");
        *ev = j->done;
        return 0;
    }
    *ev = m->pend_ev;
    return 0;
}

int32_t vg_dmat_materialize(vgpu_ctx* ctx, const vgpu_dmat* cm) {
    vgpu_dmat* m = const_cast<vgpu_dmat*>(cm);   // completing a pending upload does not change the matrix's value
    if (!m || !m->pend_stage) return 0;
    cudaEvent_t ev = nullptr;
    VG_TRY(pending_event(ctx, m, &ev));
    VG_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ev, 0));
    int32_t rc = transpose_in(ctx, m->pend_stage, m->h, m->w, m->pend_repr, m);
    vg_free(ctx, m->pend_stage);                 // reused only by later work on the compute stream, i.e. after the transpose
    m->pend_stage = nullptr;
    if (m->pend_ev) ctx->event_pool.push_back(m->pend_ev);      // a staged upload's event goes back with its job (vg_stager_finish)
    m->pend_ev = nullptr; m->pend_job = nullptr;
    return rc;
}

int32_t vg_download_rowmajor(vgpu_ctx* ctx, const vgpu_dmat* src, int32_t repr, uint32_t* host) {
    uint64_t h = src->h, w = src->w;
    if (h == 0 || w == 0) return 0;
    VgBuf stage(ctx);
    VG_TRY(stage.alloc(h * w * 4));
    for (uint64_t c0 = 0; c0 < w; c0 += TW) {
        uint32_t wc = (uint32_t)(w - c0 < TW ? w - c0 : TW);
        KScope ks(ctx, KC_TRANSPOSE, 8.0 * (double)h * wc);
        cm_to_rm_kernel<<<(unsigned)((h + TR - 1) / TR), 256, 0, ctx->stream>>>(src->d, src->col_stride, h, w, stage.as<uint32_t>(), repr == VGPU_REPR_CANONICAL, c0, wc);
        VG_LAUNCH_CHECK(ctx);
    }
    VG_CUDA(ctx, cudaMemcpyAsync(host, stage.p, h * w * 4, cudaMemcpyDeviceToHost, ctx->stream));
    VG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return 0;
}

// ---- caller device memory (vgpu_dmat_import / _borrow / _export) -----------------------------------------------------------
// A caller matrix is any strided view: element (r, c) at v[r * rs + c * cs].  One CTA moves a tile of up to 128 columns and
// `tr` rows through shared memory: it reads along whichever stride is the unit one (row-major: runs of a row; column-major: runs
// of a column), so the loads are coalesced either way, and writes the library's columns as runs of consecutive rows.  Narrow
// matrices get taller tiles (tr = 4096 rows of one column), so every CTA moves about 8 K words.
namespace {
constexpr uint32_t IO_TILE_WORDS = TR * (TW + 1);

struct IoTiles {
    uint64_t h, w;          // rows and columns moved
    uint32_t tr;            // rows per tile (a power of two)
    uint64_t row_tiles;     // ceil(h / tr); tile t covers row tile t % row_tiles of column tile t / row_tiles
};
__device__ __forceinline__ void io_tile(const IoTiles& g, uint64_t& r0, uint64_t& c0, uint32_t& rows, uint32_t& wc, uint32_t& wp) {
    const uint64_t t = blockIdx.x;
    r0 = (t % g.row_tiles) * g.tr;
    c0 = (t / g.row_tiles) * TW;
    rows = (uint32_t)(g.h - r0 < g.tr ? g.h - r0 : g.tr);
    wc = (uint32_t)(g.w - c0 < TW ? g.w - c0 : TW);
    wp = wc | 1;            // odd row pitch: a walk down a tile column touches 32 different banks
}

// Import (STORE) and the borrow check (!STORE).  Every word must be below p in either representation; the smallest row-major
// index r * w + c of a word that is not goes to *bad with ONE atomicMin per warp that holds one (a clean matrix costs no atomic).
template <bool STORE>
__global__ void __launch_bounds__(256) import_kernel(const __grid_constant__ IoTiles g, const uint32_t* __restrict__ src, uint64_t rs, uint64_t cs,
                                                     uint32_t* __restrict__ cm, uint64_t dcs, int to_monty, unsigned long long* __restrict__ bad) {
    __shared__ uint32_t tile[IO_TILE_WORDS];
    uint64_t r0, c0; uint32_t rows, wc, wp;
    io_tile(g, r0, c0, rows, wc, wp);
    const uint32_t tot = rows * wc;
    const bool row_runs = cs <= rs;      // the unit (or smaller) stride is along a row
    unsigned long long mine = ~0ull;
    for (uint32_t i = threadIdx.x; i < tot; i += blockDim.x) {
        uint32_t r, c;
        if (row_runs) { r = i / wc; c = i % wc; } else { c = i / rows; r = i % rows; }
        const uint32_t v = src[(r0 + r) * rs + (c0 + c) * cs];
        if (v >= bb::P) mine = min(mine, (unsigned long long)((r0 + r) * g.w + c0 + c));
        if (STORE) tile[r * wp + c] = v;
    }
    const unsigned vote = __ballot_sync(0xffffffffu, mine != ~0ull);
    if (vote) {                          // rare: the warp's smallest key, then one atomic
        for (int o = 16; o; o >>= 1) mine = min(mine, __shfl_xor_sync(0xffffffffu, mine, o));
        if ((threadIdx.x & 31) == 0) atomicMin(bad, mine);
    }
    if (!STORE) return;
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < tot; i += blockDim.x) {
        const uint32_t c = i / rows, r = i % rows;
        const uint32_t v = tile[r * wp + c];
        cm[(c0 + c) * dcs + r0 + r] = to_monty ? bb::to_monty(v) : v;
    }
}

// Export: the mirror image.  Stored row r of the local part is logical row row0 + r, or reverse_bits(r) of a bit-reversed matrix.
__global__ void __launch_bounds__(256) export_kernel(const __grid_constant__ IoTiles g, const uint32_t* __restrict__ cm, uint64_t scs, int from_monty,
                                                     uint32_t* __restrict__ dst, uint64_t rs, uint64_t cs, uint64_t row0, int log_bitrev) {
    __shared__ uint32_t tile[IO_TILE_WORDS];
    uint64_t r0, c0; uint32_t rows, wc, wp;
    io_tile(g, r0, c0, rows, wc, wp);
    const uint32_t tot = rows * wc;
    for (uint32_t i = threadIdx.x; i < tot; i += blockDim.x) {
        const uint32_t c = i / rows, r = i % rows;
        const uint32_t v = cm[(c0 + c) * scs + r0 + r];
        tile[r * wp + c] = from_monty ? bb::from_monty(v) : v;
    }
    __syncthreads();
    const bool row_runs = cs <= rs;
    for (uint32_t i = threadIdx.x; i < tot; i += blockDim.x) {
        uint32_t r, c;
        if (row_runs) { r = i / wc; c = i % wc; } else { c = i / rows; r = i % rows; }
        const uint64_t lr = log_bitrev >= 0 ? (uint64_t)bb::reverse_bits((uint32_t)(r0 + r), log_bitrev) : row0 + r0 + r;
        dst[lr * rs + (c0 + c) * cs] = tile[r * wp + c];
    }
}

IoTiles io_tiles(uint64_t h, uint64_t w) {
    const uint32_t wp = (uint32_t)(w < TW ? w : TW) | 1;
    uint32_t tr = 1;
    while (tr < 4096 && 2 * tr * wp <= IO_TILE_WORDS) tr *= 2;
    return IoTiles{h, w, tr, (h + tr - 1) / tr};
}
}  // namespace

// Enqueues the import of h x w words at src (strides rs, cs) into dst (null: check only) and reads the verdict: synchronises the
// context's stream once.  *bad_key: ~0 when every word is below p, else the smallest row-major index r * w + c of one that is not.
int32_t vg_import_strided(vgpu_ctx* ctx, const uint32_t* src, uint64_t h, uint64_t w, uint64_t rs, uint64_t cs, int32_t repr, vgpu_dmat* dst,
                          unsigned long long* bad_key) {
    *bad_key = ~0ull;
    if (h == 0 || w == 0) return 0;
    VgBuf bad(ctx);
    VG_TRY(bad.alloc(sizeof(unsigned long long)));
    unsigned long long* d_bad = bad.as<unsigned long long>();
    VG_CUDA(ctx, cudaMemsetAsync(d_bad, 0xff, sizeof *d_bad, ctx->stream));
    const IoTiles g = io_tiles(h, w);
    const uint64_t tiles = g.row_tiles * ((w + TW - 1) / TW);
    if (tiles > 0x7fffffffull) VG_FAIL(ctx, "import: %llu x %llu words exceed one launch", (unsigned long long)h, (unsigned long long)w);
    {
        KScope ks(ctx, KC_DEVICE_IO, (dst ? 8.0 : 4.0) * (double)h * (double)w);
        if (dst) import_kernel<true><<<(unsigned)tiles, 256, 0, ctx->stream>>>(g, src, rs, cs, dst->d, dst->col_stride, repr == VGPU_REPR_CANONICAL, d_bad);
        else import_kernel<false><<<(unsigned)tiles, 256, 0, ctx->stream>>>(g, src, rs, cs, nullptr, 0, 0, d_bad);
        VG_LAUNCH_CHECK(ctx);
    }
    VG_CUDA(ctx, cudaMemcpyAsync(bad_key, d_bad, sizeof *d_bad, cudaMemcpyDeviceToHost, ctx->stream));
    VG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return 0;
}

// The local rows of src into the caller's view at dst (strides rs, cs; logical row i at dst[i * rs]), on the context's stream.
int32_t vg_export_strided(vgpu_ctx* ctx, const vgpu_dmat* src, int32_t repr, uint32_t* dst, uint64_t rs, uint64_t cs) {
    const uint64_t h = src->h, w = src->w;
    if (h == 0 || w == 0) return 0;
    int lg = -1;
    if (src->bitrev_rows) { lg = 0; while ((1ull << lg) < h) lg++; }
    const IoTiles g = io_tiles(h, w);
    const uint64_t tiles = g.row_tiles * ((w + TW - 1) / TW);
    if (tiles > 0x7fffffffull) VG_FAIL(ctx, "export: %llu x %llu words exceed one launch", (unsigned long long)h, (unsigned long long)w);
    KScope ks(ctx, KC_DEVICE_IO, 8.0 * (double)h * (double)w);
    export_kernel<<<(unsigned)tiles, 256, 0, ctx->stream>>>(g, src->d, src->col_stride, repr == VGPU_REPR_CANONICAL, dst, rs, cs, src->row0, lg);
    VG_LAUNCH_CHECK(ctx);
    return 0;
}
