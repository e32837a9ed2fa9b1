// C ABI entry points (include/valida_b200.h): context, device matrices, NTT/LDE, commit.
#include "ctx.h"
#include "merkle.h"
#include <algorithm>
#include <cstring>
#include <new>
#include <utility>

// ---- memory ------------------------------------------------------------------------------------
int32_t vg_alloc(vgpu_ctx* ctx, void** p, size_t bytes) {
    bytes = (bytes + 511) & ~(size_t)511;
    if (bytes == 0) bytes = 512;
    auto it = ctx->free_bufs.find(bytes);
    if (it != ctx->free_bufs.end()) {
        *p = it->second;
        ctx->free_bufs.erase(it);
        ctx->cached_bytes -= bytes;
    } else {
        cudaError_t e = cudaMalloc(p, bytes);
        if (e != cudaSuccess && !ctx->free_bufs.empty()) {   // out of memory: drop the cache and retry once
            cudaGetLastError();
            cudaStreamSynchronize(ctx->stream);
            for (auto& kv : ctx->free_bufs) cudaFree(kv.second);
            ctx->free_bufs.clear(); ctx->cached_bytes = 0;
            e = cudaMalloc(p, bytes);
        }
        if (e != cudaSuccess) VG_FAIL(ctx, "cudaMalloc(%zu bytes) failed: %s (live %zu MB)", bytes, cudaGetErrorString(e), ctx->live_bytes >> 20);
    }
    ctx->live_bufs[*p] = bytes;
    ctx->live_bytes += bytes;
    if (ctx->live_bytes > ctx->peak_bytes) ctx->peak_bytes = ctx->live_bytes;
    return 0;
}
void vg_free(vgpu_ctx* ctx, void* p) {
    if (!p) return;
    auto it = ctx->live_bufs.find(p);
    if (it == ctx->live_bufs.end()) return;
    size_t bytes = it->second;
    ctx->live_bufs.erase(it);
    ctx->live_bytes -= bytes;
    ctx->free_bufs.emplace(bytes, p);
    ctx->cached_bytes += bytes;
}

int32_t vg_dmat_alloc_run(vgpu_ctx* ctx, uint64_t gh, uint64_t gw, bool split, bool symm, VgMat* out) {
    vgpu_dmat* m = new (std::nothrow) vgpu_dmat();
    if (!m) VG_FAIL(ctx, "out of host memory");
    const VgRun run = vg_run(gh, ctx->comm_size, ctx->comm_rank, split);
    m->ctx = ctx; m->gh = gh; m->gw = gw; m->dist = split ? VG_ROWS : VG_FULL; m->owns = true; m->symm = symm;
    m->h = run.count; m->w = gw; m->row0 = run.begin;
    m->col_stride = symm && split ? vg_run_max(gh, ctx->comm_size) : run.count;
    const size_t bytes = m->col_stride * m->w * 4;
    int32_t rc = symm ? vg_symm_alloc(ctx, (void**)&m->d, bytes) : vg_alloc(ctx, (void**)&m->d, bytes);
    if (rc) { delete m; return rc; }
    out->reset(m);
    return 0;
}

static int32_t build_pow_table(vgpu_ctx* ctx, uint32_t base_monty, uint32_t scale_monty, uint64_t max_exp, PowTable* t) {
    uint64_t hi_len = (max_exp >> VG_POW_LO_BITS) + 1;
    std::vector<uint32_t> lo(VG_POW_LO), hi(hi_len);
    uint32_t a = bb::R1;
    for (uint32_t j = 0; j < VG_POW_LO; j++) { lo[j] = a; a = bb::mul(a, base_monty); }
    uint32_t step = a;  // base^4096
    a = scale_monty;
    for (uint64_t j = 0; j < hi_len; j++) { hi[j] = a; a = bb::mul(a, step); }
    VgBuf dlo(ctx), dhi(ctx);
    VG_TRY(dlo.upload(lo.data(), lo.size()));
    VG_TRY(dhi.upload(hi.data(), hi.size()));
    VG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));   // host vectors go out of scope
    t->lo = (uint32_t*)dlo.release();                    // the caller's table owns them from here on
    t->hi = (uint32_t*)dhi.release();
    t->hi_len = (uint32_t)hi_len;
    t->base = base_monty;
    return 0;
}

int32_t vg_get_shift_table(vgpu_ctx* ctx, uint32_t shift_canonical, uint32_t scale_canonical, uint64_t max_exp, const PowTable** out) {
    auto key = std::make_pair(shift_canonical, scale_canonical);
    auto it = ctx->shift_tables.find(key);
    if (it == ctx->shift_tables.end() || (uint64_t)it->second.hi_len * VG_POW_LO <= max_exp) {
        PowTable t;
        VG_TRY(build_pow_table(ctx, bb::to_monty(shift_canonical), bb::to_monty(scale_canonical), max_exp, &t));
        if (it != ctx->shift_tables.end()) { vg_free(ctx, it->second.lo); vg_free(ctx, it->second.hi); }
        ctx->shift_tables[key] = t;
        it = ctx->shift_tables.find(key);
    }
    *out = &it->second;
    return 0;
}

void vg_host_state_free(vgpu_ctx* ctx);

// Every entry point runs on the context's device whatever the calling thread's current device is (a thread per GPU in
// one process, or torch having switched devices).
int32_t vg_enter(vgpu_ctx* ctx) {
    int cur = -1;
    if (cudaGetDevice(&cur) != cudaSuccess || cur != ctx->device) VG_CUDA(ctx, cudaSetDevice(ctx->device));
    return 0;
}

extern "C" {

int32_t vgpu_ctx_create(int32_t device, void* cuda_stream, vgpu_ctx** out) {
    if (!out) return -1;
    *out = nullptr;
    vgpu_ctx* ctx = new (std::nothrow) vgpu_ctx();
    if (!ctx) return -1;
    ctx->device = device;
    *out = ctx;   // returned even on failure so the caller can read vgpu_last_error
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) { ctx->err = "no CUDA device available: valida_b200 has no CPU fallback"; return -2; }
    VG_CUDA(ctx, cudaSetDevice(device));
    if (cuda_stream) { ctx->stream = (cudaStream_t)cuda_stream; ctx->own_stream = false; }
    else { VG_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking)); ctx->own_stream = true; }
    cudaDeviceProp prop;
    VG_CUDA(ctx, cudaGetDeviceProperties(&prop, device));
    ctx->sm_count = prop.multiProcessorCount;
    VG_TRY(build_pow_table(ctx, bb::two_adic_generator_monty(VG_LOG_NMAX), bb::R1, (1ull << VG_LOG_NMAX) - 1, &ctx->root_table));
    {   // three-level table (9 + 9 + 9 exponent bits)
        std::vector<uint32_t> t(3 * 512);
        uint32_t base = bb::two_adic_generator_monty(VG_LOG_NMAX);
        for (int lvl = 0; lvl < 3; lvl++) {
            uint32_t a = bb::R1;
            for (int i = 0; i < 512; i++) { t[lvl * 512 + i] = a; a = bb::mul(a, base); }
            base = a;   // base^512
        }
        VG_TRY(vg_alloc(ctx, (void**)&ctx->root3, t.size() * 4));
        VG_CUDA(ctx, cudaMemcpy(ctx->root3, t.data(), t.size() * 4, cudaMemcpyHostToDevice));
    }
    return 0;
}

void vgpu_ctx_destroy(vgpu_ctx* ctx) {
    if (!ctx) return;
    vg_host_state_free(ctx);
    vg_stager_free(ctx);
    vg_comm_free(ctx);
    if (ctx->stream) {
        cudaStreamSynchronize(ctx->stream);
        vg_free(ctx, ctx->root_table.lo); vg_free(ctx, ctx->root_table.hi);
        for (auto& kv : ctx->shift_tables) { vg_free(ctx, kv.second.lo); vg_free(ctx, kv.second.hi); }
        cudaStreamSynchronize(ctx->stream);
        for (auto& kv : ctx->free_bufs) cudaFree(kv.second);
        for (auto& kv : ctx->live_bufs) cudaFree(kv.first);
        for (auto e : ctx->event_pool) cudaEventDestroy(e);
        if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
        if (ctx->xfer_stream) { cudaStreamDestroy(ctx->xfer_stream); for (auto e : ctx->xfer_ev) if (e) cudaEventDestroy(e); }
        if (ctx->own_stream) cudaStreamDestroy(ctx->stream);
    }
    delete ctx;
}

const char* vgpu_last_error(const vgpu_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }
int32_t vgpu_ctx_synchronize(vgpu_ctx* ctx) { VG_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); return 0; }
int32_t vgpu_ctx_wait_event(vgpu_ctx* ctx, void* cuda_event) {
    if (!cuda_event) VG_FAIL(ctx, "ctx_wait_event: null event");
    VG_TRY(vg_enter(ctx));
    VG_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, (cudaEvent_t)cuda_event, 0));
    return 0;
}
int32_t vgpu_ctx_record_event(vgpu_ctx* ctx, void* cuda_event) {
    if (!cuda_event) VG_FAIL(ctx, "ctx_record_event: null event");
    VG_TRY(vg_enter(ctx));
    VG_CUDA(ctx, cudaEventRecord((cudaEvent_t)cuda_event, ctx->stream));
    return 0;
}
uint64_t vgpu_ctx_launch_count(const vgpu_ctx* ctx) { return ctx->launches; }
int32_t vgpu_ctx_release_cached(vgpu_ctx* ctx) {
    VG_TRY(vg_enter(ctx));
    VG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));   // a cached block may still be read by queued work
    for (auto& kv : ctx->free_bufs) cudaFree(kv.second);
    ctx->free_bufs.clear(); ctx->cached_bytes = 0;
    return 0;
}
int32_t vgpu_ctx_memory_stats(vgpu_ctx* ctx, uint64_t out[4], int32_t reset) {
    out[0] = ctx->live_bytes; out[1] = ctx->peak_bytes; out[2] = ctx->cached_bytes; out[3] = ctx->symm_peak_bytes;
    if (reset) { ctx->peak_bytes = ctx->live_bytes; ctx->symm_peak_bytes = ctx->symm_live_bytes; }
    return 0;
}

int32_t vgpu_ctx_set_kernel_timing(vgpu_ctx* ctx, int32_t on) { ctx->ktiming = on != 0; return 0; }
int32_t vgpu_ctx_set_merkle_hash(vgpu_ctx* ctx, int32_t hash) {
    if (!ctx) return -1;
    if (hash != VGPU_MERKLE_KECCAK256 && hash != VGPU_MERKLE_POSEIDON16) VG_FAIL(ctx, "set_merkle_hash: unknown hash %d", hash);
    ctx->merkle_hash = hash;
    return 0;
}
static const char* KCLASS_NAMES[KC_COUNT] = {"ntt_pass_kernel", "leaf_hash_kernel", "compress_layer_kernel", "fri_leaf_hash_kernel", "transpose (rm<->cm)",
                                             "perm trace kernels", "quotient_kernel", "inverse denominators", "bary_kernel", "reduced_opening_kernel", "fri_fold_kernel", "peer-store exchange", "all-gathers + barriers (incl. waiting for the slowest rank)", "other",
                                             "check_kernel", "query_path_kernel", "p16_leaf_kernel", "p16_layer_kernel + p16_tail_kernel", "p16_fri_leaf_kernel",
                                             "p16_path_kernel", "import_kernel / export_kernel (caller device memory)"};
uint32_t vgpu_ctx_kernel_stats(vgpu_ctx* ctx, const char** names, uint32_t* launches, float* ms, double* bytes, uint32_t cap) {
    cudaStreamSynchronize(ctx->stream);
    uint32_t n[KC_COUNT] = {0}; float t[KC_COUNT] = {0}; double b[KC_COUNT] = {0};
    for (auto& k : ctx->ktimers) {
        float e = 0;
        if (cudaEventElapsedTime(&e, k.a, k.b) == cudaSuccess) { n[k.cls]++; t[k.cls] += e; b[k.cls] += k.bytes; }
        else cudaGetLastError();   // do not leave the error for the caller's next CUDA call
        ctx->event_pool.push_back(k.a); ctx->event_pool.push_back(k.b);
    }
    ctx->ktimers.clear();
    uint32_t out = 0;
    for (int c = 0; c < KC_COUNT && out < cap; c++) if (n[c]) { names[out] = KCLASS_NAMES[c]; launches[out] = n[c]; ms[out] = t[c]; bytes[out] = b[c]; out++; }
    return out;
}

// ---- caller memory ---------------------------------------------------------------------------------
// vgpu_prove copies the traces out of the caller's buffers on a copy stream while the commits of earlier matrices run.  From
// PAGEABLE memory (a Rust Vec, a numpy array) the CUDA runtime stages every copy through its own bounce buffer and the copy call
// blocks the host; page-locking the buffers once lets the same call overlap for real.
int32_t vgpu_host_register(vgpu_ctx* ctx, const void* p, uint64_t bytes) {
    VG_TRY(vg_enter(ctx));
    cudaError_t e = cudaHostRegister(const_cast<void*>(p), bytes, cudaHostRegisterDefault);
    if (e == cudaErrorHostMemoryAlreadyRegistered) { cudaGetLastError(); return 0; }
    if (e != cudaSuccess) VG_FAIL(ctx, "cudaHostRegister(%llu bytes) failed: %s", (unsigned long long)bytes, cudaGetErrorString(e));
    return 0;
}
int32_t vgpu_host_unregister(vgpu_ctx* ctx, const void* p) {
    VG_TRY(vg_enter(ctx));
    cudaError_t e = cudaHostUnregister(const_cast<void*>(p));
    if (e != cudaSuccess) { cudaGetLastError(); VG_FAIL(ctx, "cudaHostUnregister failed: %s", cudaGetErrorString(e)); }
    return 0;
}

// ---- device matrices -----------------------------------------------------------------------------
int32_t vgpu_dmat_upload(vgpu_ctx* ctx, const vgpu_matrix* host, int32_t repr, vgpu_dmat** out) {
    if (!host || !out) VG_FAIL(ctx, "dmat_upload: null argument");
    VG_TRY(vg_enter(ctx));
    VgMat m;
    VG_TRY(vg_dmat_alloc(ctx, host->height, host->width, &m));
    VG_TRY(vg_upload_rowmajor(ctx, host->data, host->height, host->width, repr, m.get()));
    *out = m.release();
    return 0;
}
// Split proof: a rank keeps only ITS run of rows of a trace tall enough to be split (every rank passes the same host
// matrix, or at least its own rows of it); shorter traces are uploaded whole.  The handle reports the logical dimensions.
int32_t vgpu_dmat_upload_rows(vgpu_ctx* ctx, const vgpu_matrix* host, int32_t repr, vgpu_dmat** out) {
    if (!host || !out) VG_FAIL(ctx, "dmat_upload_rows: null argument");
    if (!vg_trace_run(ctx, host->height).split) return vgpu_dmat_upload(ctx, host, repr, out);
    VG_TRY(vg_enter(ctx));
    VgMat m;
    VG_TRY(vg_dmat_alloc_run(ctx, host->height, host->width, true, false, &m));
    VG_TRY(vg_upload_rowmajor(ctx, host->data + m->row0 * host->width, m->h, m->w, repr, m.get()));
    *out = m.release();
    return 0;
}
// Writes the rows this rank holds (all of them unless the matrix is a row shard) at their place in the caller's
// gh x gw row-major buffer, in natural row order: stored row s of a matrix with bit-reversed rows (quotient chunks, also their row
// shards) lands at row reverse_bits(s, log2 gh).  Rows another rank holds are left untouched.
int32_t vgpu_dmat_download(vgpu_ctx* ctx, const vgpu_dmat* m, int32_t repr, uint32_t* host_row_major_out) {
    VG_TRY(vg_enter(ctx));
    VG_TRY(vg_dmat_materialize(ctx, m));
    if (!m->bitrev_rows || m->gh < 2) return vg_download_rowmajor(ctx, m, repr, host_row_major_out + m->row0 * m->gw);
    std::vector<uint32_t> stored;
    try { stored.resize(m->h * m->w); } catch (const std::bad_alloc&) { VG_FAIL(ctx, "out of host memory"); }
    VG_TRY(vg_download_rowmajor(ctx, m, repr, stored.data()));
    int lg = 0; while ((1ull << lg) < m->gh) lg++;
    for (uint64_t i = 0; i < m->h; i++)
        std::memcpy(host_row_major_out + bb::reverse_bits((uint32_t)(m->row0 + i), lg) * m->w, stored.data() + i * m->w, m->w * 4);
    return 0;
}
// ---- caller device memory ----------------------------------------------------------------------------
// A caller's view must lie in device memory of the context's device (first and last word), hold whole words, and address its h x w
// elements, their row-major index r * w + c and their bytes without 64-bit overflow.  Checked before anything is enqueued.
static int32_t check_device_view(vgpu_ctx* ctx, const char* what, const uint32_t* p, uint64_t h, uint64_t w, uint64_t rs, uint64_t cs) {
    uint64_t a, b, last, n;
    if (__builtin_mul_overflow(h - 1, rs, &a) || __builtin_mul_overflow(w - 1, cs, &b) || __builtin_add_overflow(a, b, &last) ||
        last > (UINT64_MAX >> 2) || (uintptr_t)p + 4 * last < (uintptr_t)p || __builtin_mul_overflow(h, w, &n) || n > (UINT64_MAX >> 2))
        VG_FAIL(ctx, "%s: a %llu x %llu view with strides (%llu, %llu) overflows 64-bit addressing", what, (unsigned long long)h, (unsigned long long)w,
                (unsigned long long)rs, (unsigned long long)cs);
    if ((uintptr_t)p % 4) VG_FAIL(ctx, "%s: the device pointer %p is not 4-byte aligned", what, (const void*)p);
    for (const uint32_t* q : {p, p + last}) {
        cudaPointerAttributes at{};
        if (cudaPointerGetAttributes(&at, q) != cudaSuccess) { cudaGetLastError(); at.type = cudaMemoryTypeUnregistered; }
        if (at.type != cudaMemoryTypeDevice || at.device != ctx->device)
            VG_FAIL(ctx, "%s: %p is not device memory of the context's device %d", what, (const void*)q, ctx->device);
    }
    return 0;
}
// The rows this rank holds of a trace of height h: vg_trace_run, the rule of vgpu_dmat_upload_rows.
static int32_t check_local_height(vgpu_ctx* ctx, const char* what, uint64_t view_rows, uint64_t h) {
    const VgRun run = vg_trace_run(ctx, h);
    if (view_rows != run.count)
        VG_FAIL(ctx, "%s: the view has %llu rows, but of a matrix of height %llu rank %d holds rows = %llu starting at row0 = %llu", what,
                (unsigned long long)view_rows, (unsigned long long)h, ctx->comm_rank, (unsigned long long)run.count, (unsigned long long)run.begin);
    return 0;
}
// rows: keep this rank's run of a trace tall enough to be split.  local: `src` views those rows only (of a matrix of height h);
// otherwise it views the whole matrix (h == src->height).
static int32_t import_view(vgpu_ctx* ctx, const char* what, const vgpu_dev_matrix* src, uint64_t h, int32_t repr, bool rows, bool local, vgpu_dmat** out) {
    if (!src || !out) VG_FAIL(ctx, "%s: null argument", what);
    VG_TRY(vg_enter(ctx));
    const uint64_t w = src->width;
    if (local) VG_TRY(check_local_height(ctx, what, src->height, h));
    if (src->height && w) VG_TRY(check_device_view(ctx, what, src->data, src->height, w, src->row_stride, src->col_stride));
    VgMat m;
    VG_TRY(vg_dmat_alloc_run(ctx, h, w, rows && vg_trace_run(ctx, h).split, false, &m));
    unsigned long long bad = ~0ull;
    const uint32_t* first = local ? src->data : src->data + m->row0 * src->row_stride;
    VG_TRY(vg_import_strided(ctx, first, m->h, m->w, src->row_stride, src->col_stride, repr, m.get(), &bad));
    if (bad != ~0ull)
        VG_FAIL(ctx, "%s: the word at row %llu, column %llu is not below p = %u (neither a canonical nor a Montgomery BabyBear word)", what,
                (unsigned long long)(m->row0 + bad / w), (unsigned long long)(bad % w), bb::P);
    *out = m.release();
    return 0;
}
int32_t vgpu_dmat_import(vgpu_ctx* ctx, const vgpu_dev_matrix* src, int32_t repr, vgpu_dmat** out) {
    return import_view(ctx, "dmat_import", src, src ? src->height : 0, repr, false, false, out);
}
int32_t vgpu_dmat_import_rows(vgpu_ctx* ctx, const vgpu_dev_matrix* src, int32_t repr, vgpu_dmat** out) {
    return import_view(ctx, "dmat_import_rows", src, src ? src->height : 0, repr, true, false, out);
}
int32_t vgpu_dmat_import_local(vgpu_ctx* ctx, const vgpu_dev_matrix* local, uint64_t height, int32_t repr, vgpu_dmat** out) {
    return import_view(ctx, "dmat_import_local", local, height, repr, true, true, out);
}
// local: `data` holds this rank's rows of a matrix of height `height` (a VG_ROWS shard when the matrix is split), else all of it.
static int32_t borrow_view(vgpu_ctx* ctx, const char* what, uint32_t* data, uint64_t height, uint64_t width, uint64_t col_stride, bool local, vgpu_dmat** out) {
    if (!out) VG_FAIL(ctx, "%s: null argument", what);
    VG_TRY(vg_enter(ctx));
    const VgRun run = local ? vg_trace_run(ctx, height) : VgRun{0, height, false};
    const uint64_t row0 = run.begin, rows = run.count;
    if (col_stride < rows) VG_FAIL(ctx, "%s: column stride %llu is below the height %llu", what, (unsigned long long)col_stride, (unsigned long long)rows);
    if (rows && width) {
        VG_TRY(check_device_view(ctx, what, data, rows, width, 1, col_stride));
        unsigned long long bad = ~0ull;
        VG_TRY(vg_import_strided(ctx, data, rows, width, 1, col_stride, VGPU_REPR_MONTY_R32, nullptr, &bad));
        if (bad != ~0ull)
            VG_FAIL(ctx, "%s: the word at row %llu, column %llu is not below p = %u (not a Montgomery BabyBear word)", what,
                    (unsigned long long)(row0 + bad / width), (unsigned long long)(bad % width), bb::P);
    }
    vgpu_dmat* m = new (std::nothrow) vgpu_dmat();
    if (!m) VG_FAIL(ctx, "out of host memory");
    m->ctx = ctx; m->d = data; m->h = rows; m->gh = height; m->w = m->gw = width; m->col_stride = col_stride;
    m->row0 = row0; m->dist = run.split ? VG_ROWS : VG_FULL;
    m->owns = false;
    *out = m;
    return 0;
}
int32_t vgpu_dmat_borrow(vgpu_ctx* ctx, uint32_t* data, uint64_t height, uint64_t width, uint64_t col_stride, vgpu_dmat** out) {
    return borrow_view(ctx, "dmat_borrow", data, height, width, col_stride, false, out);
}
int32_t vgpu_dmat_borrow_local(vgpu_ctx* ctx, uint32_t* data, uint64_t height, uint64_t width, uint64_t col_stride, vgpu_dmat** out) {
    return borrow_view(ctx, "dmat_borrow_local", data, height, width, col_stride, true, out);
}
// local: the view holds this rank's rows only (local row i at view row i); otherwise the whole matrix, each row at its logical place.
static int32_t export_view(vgpu_ctx* ctx, const char* what, const vgpu_dmat* m, int32_t repr, const vgpu_dev_matrix* dst, bool local) {
    if (!m || !dst) VG_FAIL(ctx, "%s: null argument", what);
    VG_TRY(vg_enter(ctx));
    if (m->dist == VG_ROWS && m->bitrev_rows) VG_FAIL(ctx, "%s: a bit-reversed row shard has no contiguous natural-order image", what);
    if (local && (dst->height != m->h || dst->width != m->w))
        VG_FAIL(ctx, "%s: the view is %llu x %llu, but of the %llu x %llu matrix rank %d holds rows = %llu starting at row0 = %llu", what,
                (unsigned long long)dst->height, (unsigned long long)dst->width, (unsigned long long)m->gh, (unsigned long long)m->gw, ctx->comm_rank,
                (unsigned long long)m->h, (unsigned long long)m->row0);
    if (!local && (dst->height != m->gh || dst->width != m->gw))
        VG_FAIL(ctx, "%s: the view is %llu x %llu, the matrix %llu x %llu", what, (unsigned long long)dst->height, (unsigned long long)dst->width,
                (unsigned long long)m->gh, (unsigned long long)m->gw);
    if (m->h == 0 || m->w == 0) return 0;
    VG_TRY(check_device_view(ctx, what, dst->data, dst->height, dst->width, dst->row_stride, dst->col_stride));
    VG_TRY(vg_dmat_materialize(ctx, m));
    vgpu_dmat at = *m;                  // export_kernel writes stored row r at view row at.row0 + r
    if (local) at.row0 = 0;
    return vg_export_strided(ctx, &at, repr, const_cast<uint32_t*>(dst->data), dst->row_stride, dst->col_stride);
}
int32_t vgpu_dmat_export(vgpu_ctx* ctx, const vgpu_dmat* m, int32_t repr, const vgpu_dev_matrix* dst) {
    return export_view(ctx, "dmat_export", m, repr, dst, false);
}
int32_t vgpu_dmat_export_local(vgpu_ctx* ctx, const vgpu_dmat* m, int32_t repr, const vgpu_dev_matrix* dst) {
    return export_view(ctx, "dmat_export_local", m, repr, dst, true);
}
int32_t vgpu_ctx_local_rows(const vgpu_ctx* ctx, uint64_t height, uint64_t* row0, uint64_t* rows) {
    if (!ctx || !row0 || !rows) return -1;
    const VgRun run = vg_trace_run(ctx, height);
    *row0 = run.begin; *rows = run.count;
    return 0;
}
int32_t vgpu_dmat_dims(const vgpu_dmat* m, uint64_t* height, uint64_t* width) { *height = m->gh; *width = m->gw; return 0; }
int32_t vgpu_dmat_local_rows(const vgpu_dmat* m, uint64_t* row0, uint64_t* rows) { *row0 = m->row0; *rows = m->h; return m->dist; }
void vgpu_dmat_free(vgpu_dmat* m) {
    if (!m) return;
    if (m->pend_stage) {   // an upload that was never consumed: let the copy finish, then release
        if (m->pend_job) vg_stager_finish(m->ctx);       // joins the staging threads: every chunk is enqueued
        if (m->pend_ev) cudaEventSynchronize(m->pend_ev);
        else if (m->ctx->copy_stream) cudaStreamSynchronize(m->ctx->copy_stream);
        vg_free(m->ctx, m->pend_stage);
        if (m->pend_ev) m->ctx->event_pool.push_back(m->pend_ev);
    }
    if (m->owns) { if (m->symm) vg_symm_free(m->ctx, m->d); else vg_free(m->ctx, m->d); }
    delete m;
}

// ---- NTT / LDE -------------------------------------------------------------------------------------
int32_t vgpu_ntt_batch(vgpu_ctx* ctx, vgpu_dmat* m, int32_t inverse) {
    VG_TRY(vg_enter(ctx));
    if (m->dist != VG_FULL) VG_FAIL(ctx, "ntt_batch: the matrix is a shard of a split proof");
    if (!m->owns) VG_FAIL(ctx, "ntt_batch: the matrix is a borrowed caller buffer, which the library never writes");
    int log_n = 0;
    while ((1ull << log_n) < m->h) log_n++;
    if ((1ull << log_n) != m->h) VG_FAIL(ctx, "ntt_batch: height %llu is not a power of two", (unsigned long long)m->h);
    if (log_n > VG_LOG_NMAX) VG_FAIL(ctx, "ntt_batch: height exceeds two-adicity");
    if (m->bitrev_rows) VG_FAIL(ctx, "ntt_batch: matrix rows are stored bit-reversed");
    VG_TRY(vg_dmat_materialize(ctx, m));
    VgBuf tmp(ctx);
    VG_TRY(tmp.alloc(m->h * m->w * 4));
    return vg_ntt_nat2nat(ctx, m->d, m->col_stride, m->d, m->col_stride, log_n, m->w, inverse != 0, nullptr, tmp.as<uint32_t>(), m->h);
}

int32_t vgpu_coset_lde_batch(vgpu_ctx* ctx, const vgpu_dmat* in, uint32_t log_blowup, uint32_t shift_canonical, int32_t bit_reversed, vgpu_dmat** out) {
    if (log_blowup < 1 || log_blowup > 4) VG_FAIL(ctx, "coset_lde: log_blowup must be 1..4");
    VG_TRY(vg_enter(ctx));
    if (in->dist != VG_FULL) VG_FAIL(ctx, "coset_lde: the matrix is a shard of a split proof");
    VG_TRY(vg_dmat_materialize(ctx, in));
    VgMat o;
    VG_TRY(vg_dmat_alloc(ctx, in->h << log_blowup, in->w, &o));
    VG_TRY(vg_coset_lde(ctx, in->d, in->col_stride, in->h, in->w, shift_canonical, o->d, o->col_stride, bit_reversed != 0, in->bitrev_rows, log_blowup));
    *out = o.release();
    return 0;
}

int32_t vgpu_ntt_batch_host(vgpu_ctx* ctx, uint32_t* row_major, uint64_t height, uint64_t width, int32_t repr, int32_t inverse) {
    vgpu_matrix hm{row_major, height, width};
    vgpu_dmat* raw = nullptr;
    VG_TRY(vgpu_dmat_upload(ctx, &hm, repr, &raw));
    VgMat m(raw);
    VG_TRY(vgpu_ntt_batch(ctx, m.get(), inverse));
    return vgpu_dmat_download(ctx, m.get(), repr, row_major);
}

// ---- commit ------------------------------------------------------------------------------------------
// TwoAdicFriPcs::commit_shifted_batches per matrix: shift = generator / coset_shift_i; LDE; bit-reversed rows.
static uint32_t lde_shift_of(const uint32_t* coset_shifts_or_null, uint32_t i) {
    const uint32_t cs = coset_shifts_or_null ? coset_shifts_or_null[i] : 1;
    return bb::from_monty(bb::mul(bb::to_monty(bb::GEN_CANON), bb::inv(bb::to_monty(cs))));
}

// Which rank extends which columns of the tall matrices of one commit: contiguous column ranges per rank, sized by water-filling
// over the whole commit — tallest matrix first, every column goes to the rank with the least work so far (a column of height h
// weighs h) — so that a rank that had to take two of the ten columns of a 2^24-row matrix takes fewer columns of the others.
// (An even split of every matrix on its own leaves the first ranks with up to 60 % more LDE work than the mean at 8 ranks.)
struct ColPlan { uint32_t begin[17]; uint32_t widest; };
static std::vector<ColPlan> plan_columns(const int G, const std::vector<std::pair<uint64_t, uint64_t>>& dims /* (height, width) of the tall matrices */) {
    std::vector<size_t> order(dims.size());
    for (size_t k = 0; k < dims.size(); k++) order[k] = k;
    std::stable_sort(order.begin(), order.end(), [&](size_t a, size_t b) { return dims[a].first > dims[b].first; });
    std::vector<uint64_t> load(G, 0);
    std::vector<ColPlan> plan(dims.size());
    for (size_t k : order) {
        uint32_t count[16] = {0};
        for (uint64_t c = 0; c < dims[k].second; c++) {
            int best = 0;
            for (int r = 1; r < G; r++) if (load[r] < load[best]) best = r;
            count[best]++; load[best] += dims[k].first;
        }
        ColPlan& p = plan[k];
        p.begin[0] = 0; p.widest = 0;
        for (int r = 0; r < G; r++) { p.begin[r + 1] = p.begin[r] + count[r]; p.widest = std::max(p.widest, count[r]); }
    }
    return plan;
}

// Symmetric-heap bytes of one split commit of the tall matrices dims[k] = (height, width), columns planned by `plan`: the row shard
// of every LDE, and the column buffer of every matrix that arrives as row shards (as_rows[k]).
static size_t commit_symm_bytes(int G, const std::vector<std::pair<uint64_t, uint64_t>>& dims, const std::vector<ColPlan>& plan, const std::vector<bool>& as_rows) {
    size_t need = 0;
    for (size_t k = 0; k < dims.size(); k++) {
        need += vg_symm_round(vg_run_max(2 * dims[k].first, (uint64_t)G) * dims[k].second * 4);
        if (as_rows[k]) need += vg_symm_round(dims[k].first * plan[k].widest * 4);
    }
    return need;
}
// The same for matrices with these (height, width), all arriving as row shards when tall enough to be split (prover.cc sizes the
// heap for a whole proof with it).
extern "C++" size_t vg_commit_symm_need(const vgpu_ctx* ctx, const std::vector<std::pair<uint64_t, uint64_t>>& dims_all) {
    std::vector<std::pair<uint64_t, uint64_t>> dims;
    for (auto& d : dims_all) if (vg_trace_run(ctx, d.first).split) dims.push_back(d);
    return commit_symm_bytes(ctx->comm_size, dims, plan_columns(ctx->comm_size, dims), std::vector<bool>(dims.size(), true));
}

// The column plan of a commit as data (tests; a host program that wants to know which rank extends what): matrices i = 0..n-1 of
// heights[i] x widths[i], all tall enough to be split; begin_out[i * (nranks + 1) + r] = first column of rank r, ... + nranks] = width.
void vgpu_split_column_plan(int32_t nranks, uint32_t n, const uint64_t* heights, const uint64_t* widths, uint32_t* begin_out) {
    std::vector<std::pair<uint64_t, uint64_t>> dims;
    for (uint32_t i = 0; i < n; i++) dims.push_back({heights[i], widths[i]});
    const std::vector<ColPlan> plan = plan_columns(nranks, dims);
    for (uint32_t i = 0; i < n; i++) for (int r = 0; r <= nranks; r++) begin_out[(size_t)i * (nranks + 1) + r] = plan[i].begin[r];
}

// Split proof: the tall matrices of a commit.  (1) a matrix that arrives as row shards is handed to the ranks that extend
// its columns; (2) every rank extends its column share and stores, through peer pointers, each rank's run of the committed
// rows into that rank's shard.  After the closing barrier pd->ldes[i] holds this rank's run of the H committed rows of all columns.
static int32_t extend_split(vgpu_ctx* ctx, vgpu_prover_data* pd, const vgpu_dmat* const* mats, const std::vector<size_t>& tall, const uint32_t* coset_shifts_or_null) {
    std::vector<std::pair<uint64_t, uint64_t>> dims;
    std::vector<bool> as_rows;
    for (size_t i : tall) { dims.push_back({mats[i]->gh, mats[i]->gw}); as_rows.push_back(mats[i]->dist == VG_ROWS); }
    const std::vector<ColPlan> plan = plan_columns(ctx->comm_size, dims);
    VG_TRY(vg_symm_reserve(ctx, commit_symm_bytes(ctx->comm_size, dims, plan, as_rows)));
    std::vector<uint32_t*> cols(tall.size(), nullptr);      // column buffers of the matrices that arrive as row shards (symmetric heap)
    struct Guard { vgpu_ctx* c; std::vector<uint32_t*>& v; ~Guard() { for (auto* p : v) vg_symm_free(c, p); } } guard{ctx, cols};
    bool moved = false;
    for (size_t k = 0; k < tall.size(); k++) {
        const vgpu_dmat* m = mats[tall[k]];
        VG_TRY(vg_dmat_materialize(ctx, m));
        if (!as_rows[k]) continue;
        VG_TRY(vg_symm_alloc(ctx, (void**)&cols[k], m->gh * plan[k].widest * 4));
        VG_TRY(vg_exchange_rows_to_cols(ctx, m, cols[k], plan[k].begin));
        moved = true;
    }
    if (moved) VG_TRY(vg_comm_barrier(ctx));
    // (2) extend the column share of matrix k on the context's stream while the exchange of matrix k-1 runs on a second
    // stream: the LDE kernels are issue bound, the exchange is NVLink bound.  Two extension buffers alternate; a buffer is
    // rewritten only after its exchange has finished.  (With per-kernel timing on everything stays on one stream.)
    const bool overlap = !ctx->ktiming;
    if (overlap && !ctx->xfer_stream) {
        VG_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->xfer_stream, cudaStreamNonBlocking));
        for (auto& e : ctx->xfer_ev) VG_CUDA(ctx, cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    }
    size_t ext_words = 0;
    for (size_t k = 0; k < tall.size(); k++)
        ext_words = std::max<size_t>(ext_words, 2 * mats[tall[k]]->gh * (plan[k].begin[ctx->comm_rank + 1] - plan[k].begin[ctx->comm_rank]));
    VgBuf ext[2] = {VgBuf(ctx), VgBuf(ctx)};
    if (ext_words) { VG_TRY(ext[0].alloc(ext_words * 4)); if (overlap) VG_TRY(ext[1].alloc(ext_words * 4)); }
    bool used[2] = {false, false};
    for (size_t k = 0; k < tall.size(); k++) {
        const size_t i = tall[k];
        const vgpu_dmat* m = mats[i];
        const uint64_t h = m->gh, H = 2 * h;
        const uint64_t c0 = plan[k].begin[ctx->comm_rank], c1 = plan[k].begin[ctx->comm_rank + 1];
        VgMat lde;
        VG_TRY(vg_dmat_alloc_run(ctx, H, m->gw, true, true, &lde));
        lde->bitrev_rows = false;                // committed order IS the stored order of an LDE (rows at reverse_bits)
        pd->ldes[i] = lde.release();
        if (c1 <= c0) continue;
        const uint32_t* src; uint64_t scs;
        if (m->dist == VG_ROWS) { src = cols[k]; scs = h; }
        else { src = m->d + c0 * m->col_stride; scs = m->col_stride; }
        const int b = overlap ? (int)(k & 1) : 0;
        if (overlap && used[b]) VG_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ctx->xfer_ev[b], 0));
        VG_TRY(vg_coset_lde(ctx, src, scs, h, c1 - c0, lde_shift_of(coset_shifts_or_null, (uint32_t)i), ext[b].as<uint32_t>(), H, true, m->bitrev_rows));
        if (overlap) {
            VG_CUDA(ctx, cudaEventRecord(ctx->xfer_ev[2], ctx->stream));
            VG_CUDA(ctx, cudaStreamWaitEvent(ctx->xfer_stream, ctx->xfer_ev[2], 0));
            VG_TRY(vg_exchange_cols_to_rows(ctx, ext[b].as<uint32_t>(), H, c0, c1, pd->ldes[i], ctx->xfer_stream));
            VG_CUDA(ctx, cudaEventRecord(ctx->xfer_ev[b], ctx->xfer_stream));
            used[b] = true;
        } else {
            VG_TRY(vg_exchange_cols_to_rows(ctx, ext[0].as<uint32_t>(), H, c0, c1, pd->ldes[i]));
        }
    }
    if (overlap) for (int b = 0; b < 2; b++) if (used[b]) VG_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ctx->xfer_ev[b], 0));
    return vg_comm_barrier(ctx);   // also orders the release of the column buffers (guard) behind every peer's stores
}

int32_t vgpu_commit_batches(vgpu_ctx* ctx, const vgpu_dmat* const* mats, uint32_t n, const uint32_t* coset_shifts_or_null,
                            uint32_t digest_out[8], vgpu_prover_data** out) {
    VG_TRY(vg_enter(ctx));
    if (ctx->merkle_hash == VGPU_MERKLE_POSEIDON16 && !ctx->challenger_set) VG_FAIL(ctx, "commit: the Poseidon-16 Merkle hash needs vgpu_set_challenger first");
    VgPd pd(new (std::nothrow) vgpu_prover_data());
    if (!pd) VG_FAIL(ctx, "out of host memory");
    pd->ctx = ctx;
    pd->ldes.assign(n, nullptr);
    std::vector<uint64_t> heights(n);
    std::vector<size_t> tall;
    for (uint32_t i = 0; i < n; i++) {
        if (!mats[i]) VG_FAIL(ctx, "commit: matrix %u is null", i);
        heights[i] = mats[i]->gh * 2;
        if (vg_trace_run(ctx, mats[i]->gh).split) tall.push_back(i);
        else if (mats[i]->dist != VG_FULL) VG_FAIL(ctx, "commit: matrix %u is a shard but too short to be split", i);
    }
    if (!tall.empty()) VG_TRY(extend_split(ctx, pd.get(), mats, tall, coset_shifts_or_null));
    // The other matrices one height group at a time, when the tree reaches that height; a matrix whose upload is still in
    // flight is waited for here, not earlier.  (Split proof: short matrices are extended, whole, by every rank.)
    auto extend_group = [&](const std::vector<size_t>& group) -> int32_t {
        for (size_t i : group) {
            if (pd->ldes[i]) continue;
            VG_TRY(vg_dmat_materialize(ctx, mats[i]));
            VG_TRY(vgpu_coset_lde_batch(ctx, mats[i], 1, lde_shift_of(coset_shifts_or_null, (uint32_t)i), 1, &pd->ldes[i]));
        }
        return 0;
    };
    VG_TRY(vg_merkle_build(ctx, pd.get(), heights, extend_group));
    if (digest_out) std::memcpy(digest_out, pd->root, 32);
    *out = pd.release();
    return 0;
}

int32_t vgpu_commit_batches_host(vgpu_ctx* ctx, const vgpu_matrix* mats, uint32_t n, int32_t repr, const uint32_t* coset_shifts_or_null,
                                 uint32_t digest_out[8], vgpu_prover_data** out) {
    std::vector<VgMat> dm(n);
    for (uint32_t i = 0; i < n; i++) {   // a split proof uploads each rank's rows only
        vgpu_dmat* m = nullptr;
        VG_TRY(vgpu_dmat_upload_rows(ctx, &mats[i], repr, &m));
        dm[i].reset(m);
    }
    return vgpu_commit_batches(ctx, vg_handles(dm).data(), n, coset_shifts_or_null, digest_out, out);
}

int32_t vgpu_prover_data_lde(const vgpu_prover_data* pd, uint32_t i, const vgpu_dmat** view) {
    if (i >= pd->ldes.size()) return -1;
    *view = pd->ldes[i];
    return 0;
}
void vgpu_prover_data_free(vgpu_prover_data* pd) {
    if (!pd) return;
    for (auto* m : pd->ldes) vgpu_dmat_free(m);
    delete pd;                                   // and with it the tree's digests
}

}  // extern "C"
