// Internal context / device-matrix definitions shared by the kernels' host wrappers.
#pragma once
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <memory>
#include <string>
#include <vector>
#include <map>
#include <type_traits>
#include <cuda_runtime.h>
#include "../../include/valida_b200.h"
#include "bb.cuh"

constexpr int VG_LOG_NMAX = 27;                    // BabyBear two-adicity: largest transform/LDE size
constexpr int VG_POW_LO_BITS = 12;                 // two-level power tables: base^e = lo[e & 4095] * hi[e >> 12]
constexpr uint32_t VG_POW_LO = 1u << VG_POW_LO_BITS;

struct PowTable {            // device tables of Montgomery words
    uint32_t* lo = nullptr;  // base^j, j < 4096
    uint32_t* hi = nullptr;  // scale * base^(4096 j), j < hi_len
    uint32_t hi_len = 0;
    uint32_t base = 0;       // the base itself (Montgomery), without the scale
};
// base^e (times the scale) from a PowTable's lo / hi tables, e < 4096 * hi_len
__device__ __forceinline__ uint32_t vg_pow_lookup(const uint32_t* lo, const uint32_t* hi, uint64_t e) {
    return bb::mul(__ldg(lo + (e & (VG_POW_LO - 1))), __ldg(hi + (e >> VG_POW_LO_BITS)));
}

// kernel classes for the optional per-launch CUDA-event timing (bench.py's roofline line)
enum KClass { KC_NTT = 0, KC_LEAF_HASH, KC_COMPRESS, KC_FRI_LEAF, KC_TRANSPOSE, KC_PERM, KC_QUOTIENT, KC_INVDEN, KC_BARY, KC_REDUCED_OPENING, KC_FRI_FOLD, KC_EXCHANGE, KC_COLLECTIVE, KC_OTHER, KC_CHECK, KC_TREE_PATH,
             KC_P16_LEAF, KC_P16_COMPRESS, KC_P16_FRI_LEAF, KC_P16_PATH,   // KC_P16_*: the Poseidon-16 Merkle kernels (merkle.cu)
             KC_DEVICE_IO, KC_COUNT };                                     // KC_DEVICE_IO: import / borrow check / export of caller device memory (staging.cu)
struct KTimer { cudaEvent_t a, b; int cls; double bytes; };

struct vgpu_ctx {
    int device = 0;
    cudaStream_t stream = nullptr;
    bool own_stream = false;
    std::string err;
    uint64_t launches = 0;
    int sm_count = 132;
    PowTable root_table;                                        // base = two_adic_generator(27)
    uint32_t* root3 = nullptr;                                   // 3 x 512 words: w^(i), w^(512 i), w^(2^18 i) — a 6 KB, L1-resident form of the same table
    std::map<std::pair<uint32_t, uint32_t>, PowTable> shift_tables;  // (shift, scale) canonical -> table
    // Poseidon challenger instance (host side; the transcript is sequential and tiny)
    uint32_t poseidon_rc[480];
    uint32_t poseidon_mds[256];
    bool challenger_set = false;
    bool poseidon_has_mds = false;
    void* challenger = nullptr;                                  // vgh::Challenger* (host/challenger.h)
    void* poseidon = nullptr;                                    // vgh::Poseidon16*
    uint32_t* d_poseidon = nullptr;                              // device copy of the round constants + MDS (pow.cu), dropped when they change
    int32_t merkle_hash = VGPU_MERKLE_KECCAK256;                 // the MMCS hash of the commits and Merkle checks that follow (vgpu_ctx_set_merkle_hash)
    std::vector<std::pair<const char*, float>> phases;          // last prove: per-phase milliseconds
    struct PhaseMark { const char* name; cudaEvent_t a, b; };
    std::vector<PhaseMark> phase_marks;                         // event pairs of the last prove (read by vgpu_last_prove_phases)
    std::vector<std::pair<const char*, float>> host_phases;     // host-side stretches of the last prove (wall clock)
    bool in_host_prove = false;
    bool debug_checks = false;                                  // vgpu_prove*: check_constraints on every chip before committing to a proof
    // size-keyed cache of device buffers: a proof repeats the same allocation sizes every step, so after the
    // first step no driver allocator call is made (single stream => reuse in enqueue order is safe)
    std::multimap<size_t, void*> free_bufs;
    std::map<void*, size_t> live_bufs;
    size_t cached_bytes = 0, live_bytes = 0, peak_bytes = 0;
    // multi-GPU (host/comm.cc): one rank per GPU.  Two transports with one interface: NCCL + CUDA IPC between processes
    // (torchrun ranks), or a thread per GPU inside one process (vgpu_comm_init_local: host barrier + direct peer pointers).
    void* nccl = nullptr;                                        // ncclComm_t
    void* local_group = nullptr;                                 // VgLocalGroup* (in-process ranks)
    int comm_rank = 0, comm_size = 1;
    bool sharding = false;                                       // ONE proof split across the ranks (row shards after one exchange)
    // symmetric heap: one allocation per rank, identical allocation sequence on every rank => identical offsets, so a
    // peer's copy of a buffer is peer_base[d] + (p - symm_base).  Kernels store / load through those pointers over NVLink.
    uint8_t* symm_base = nullptr; size_t symm_bytes = 0;
    std::vector<uint8_t*> peer_base;                             // [comm_size]; peer_base[comm_rank] == symm_base
    std::map<size_t, size_t> symm_free;                          // offset -> length of the free runs
    std::map<void*, size_t> symm_live;
    size_t symm_live_bytes = 0, symm_peak_bytes = 0;
    uint32_t* comm_scratch = nullptr;                            // small device buffer for barriers / handle exchange
    cudaEvent_t bar_ev[2] = {nullptr, nullptr}; uint32_t bar_slot = 0;   // in-process stream-ordered barrier
    struct CommStat { uint32_t calls = 0; double bytes = 0; };
    CommStat stat_barrier, stat_allgather, stat_exchange;        // per-proof collective counters (bench.py)
    cudaStream_t copy_stream = nullptr;                         // H2D copies of a pipelined vgpu_prove (staging.cu)
    void* stager = nullptr;                                     // VgStager*: host threads staging pageable traces through pinned chunks
    cudaStream_t xfer_stream = nullptr;                         // split proof: peer-store exchange of matrix i behind the LDE of matrix i+1
    cudaEvent_t xfer_ev[3] = {nullptr, nullptr, nullptr};       // [0], [1]: exchange out of buffer 0 / 1 done; [2]: LDE done
    bool ntt_attrs_set = false, bary_attrs_set = false;          // cudaFuncSetAttribute is per device: tracked per context, not per process
    bool ktiming = false;
    std::vector<KTimer> ktimers;
    std::vector<cudaEvent_t> event_pool;
};

// Distribution of a matrix over the ranks of a split proof.  FULL: every rank holds all of it (also the only kind on a lone
// GPU).  ROWS: this rank holds the contiguous run [row0, row0 + h) of the STORED row order (natural rows for traces,
// bit-reversed rows for committed LDEs / quotient chunks) of a gh x gw matrix (vg_dmat_alloc_run).
enum VgDist { VG_FULL = 0, VG_ROWS = 1 };
struct vgpu_dmat {
    vgpu_ctx* ctx = nullptr;
    uint32_t* d = nullptr;       // column-major: LOCAL element (r, c) at d[c * col_stride + r], Montgomery form
    uint64_t h = 0, w = 0, col_stride = 0;     // local extent
    uint64_t gh = 0, gw = 0, row0 = 0;         // logical extent and the first local row in it
    int dist = VG_FULL;
    bool symm = false;           // d lives in the symmetric heap
    bool owns = true;
    bool bitrev_rows = false;    // row r of the logical matrix is stored at reverse_bits(r) (quotient-chunk output order)
    // pipelined upload: the row-major image is (being) copied into pend_stage on the copy stream; the transpose into
    // `d` runs on the context's stream at first use (vg_dmat_materialize)
    uint32_t* pend_stage = nullptr;
    cudaEvent_t pend_ev = nullptr;
    int32_t pend_repr = 0;
    void* pend_job = nullptr;    // StageJob* when the source is pageable memory copied by the context's staging threads
};

#define VG_FAIL(ctx, ...) do { char _b[512]; snprintf(_b, sizeof _b, __VA_ARGS__); (ctx)->err = _b; return -1; } while (0)
#define VG_CUDA(ctx, expr) do { cudaError_t _e = (expr); if (_e != cudaSuccess) { VG_FAIL(ctx, "%s failed at %s:%d: %s", #expr, __FILE__, __LINE__, cudaGetErrorString(_e)); } } while (0)
#define VG_TRY(expr) do { int32_t _r = (expr); if (_r != 0) return _r; } while (0)
#define VG_LAUNCH_CHECK(ctx) do { (ctx)->launches++; cudaError_t _e = cudaGetLastError(); if (_e != cudaSuccess) { VG_FAIL(ctx, "kernel launch failed at %s:%d: %s", __FILE__, __LINE__, cudaGetErrorString(_e)); } } while (0)

// an event from ctx->event_pool (where its users return the ones they are done with), or a new one
inline cudaError_t vg_take_event(vgpu_ctx* ctx, cudaEvent_t* e) {
    if (ctx->event_pool.empty()) return cudaEventCreate(e);
    *e = ctx->event_pool.back();
    ctx->event_pool.pop_back();
    return cudaSuccess;
}

// RAII scope: when ctx->ktiming is on, brackets the launches inside it with a CUDA event pair on ctx->stream.
struct KScope {
    vgpu_ctx* ctx; bool on; size_t idx = 0;      // scopes nest (a collective inside a sweep): each closes ITS pair
    KScope(vgpu_ctx* c, int cls, double bytes) : ctx(c), on(c->ktiming) {
        if (!on) return;
        KTimer t; t.cls = cls; t.bytes = bytes;
        vg_take_event(c, &t.a);
        vg_take_event(c, &t.b);
        cudaEventRecord(t.a, c->stream);
        c->ktimers.push_back(t);
        idx = c->ktimers.size() - 1;
    }
    ~KScope() { if (on) cudaEventRecord(ctx->ktimers[idx].b, ctx->stream); }
};

int32_t vg_enter(vgpu_ctx* ctx);                          // make ctx->device current on the calling thread
int32_t vg_alloc(vgpu_ctx* ctx, void** p, size_t bytes);
void vg_free(vgpu_ctx* ctx, void* p);

// The owner of one vg_alloc block: the block goes back to the context's cache when the owner does (or at reset()), on every
// exit path, so a call that fails leaves nothing live.
struct VgBuf {
    vgpu_ctx* ctx = nullptr;
    void* p = nullptr;
    explicit VgBuf(vgpu_ctx* c = nullptr) : ctx(c) {}
    VgBuf(VgBuf&& o) noexcept : ctx(o.ctx), p(o.release()) {}
    VgBuf& operator=(VgBuf&& o) noexcept { if (this != &o) { reset(); ctx = o.ctx; p = o.release(); } return *this; }
    ~VgBuf() { reset(); }
    int32_t alloc(size_t bytes) { reset(); return vg_alloc(ctx, &p, bytes); }
    // count elements copied from the host on the context's stream; a pageable `host` may go once this returns (the runtime
    // stages such a copy before the call returns)
    template <class T> int32_t upload(const T* host, size_t count) {
        VG_TRY(alloc(std::max<size_t>(count, 1) * sizeof(T)));
        if (count) VG_CUDA(ctx, cudaMemcpyAsync(p, host, count * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
        return 0;
    }
    template <class T> T* as() const { return (T*)p; }
    explicit operator bool() const { return p != nullptr; }
    void reset() { vg_free(ctx, p); p = nullptr; }
    void* release() { void* q = p; p = nullptr; return q; }
};
// Owners of the handles the entry points hand out; an entry point passes its result on with release() once it has succeeded.
struct VgMatFree { void operator()(vgpu_dmat* m) const { vgpu_dmat_free(m); } };
struct VgPdFree { void operator()(vgpu_prover_data* p) const { vgpu_prover_data_free(p); } };
using VgMat = std::unique_ptr<vgpu_dmat, VgMatFree>;
using VgPd = std::unique_ptr<vgpu_prover_data, VgPdFree>;
// the handles of owned matrices, for the calls that take an array of them
inline std::vector<vgpu_dmat*> vg_handles(const std::vector<VgMat>& v) {
    std::vector<vgpu_dmat*> r;
    for (const VgMat& m : v) r.push_back(m.get());
    return r;
}
// pow.cu: the context's Poseidon-16 constants on the device (poseidon.cuh layout), uploaded on first use; an error before vgpu_set_challenger
int32_t vg_poseidon_consts(vgpu_ctx* ctx, uint32_t** out);
int32_t vg_get_shift_table(vgpu_ctx* ctx, uint32_t shift_canonical, uint32_t scale_canonical, uint64_t max_exp, const PowTable** out);

inline bool vg_sharded(const vgpu_ctx* ctx) { return ctx->sharding && ctx->comm_size > 1; }
// Which rows each rank of a split proof holds.  Every rank must reach the same answer at every allocation, upload, sweep and query
// answer (or the proof hangs at a barrier or comes out wrong), so this is the one place that decides it.
// The rule, for N = nranks ranks (1..16): with P = 2^ceil(log2 N), a split vector of n stored rows is cut into V = 8 P units of
// n / V rows, and rank r holds the contiguous units [floor(r V / N), floor((r + 1) V / N)).  At a power of two N that is rows
// [r n / N, (r + 1) n / N); otherwise the runs differ by at most one unit (N = 3: 10 / 11 / 11 of 32 units).
constexpr int VG_MAX_RANKS = 16;
inline uint64_t vg_units(uint64_t nranks) { uint64_t p = 1; while (p < nranks) p <<= 1; return 8 * p; }
// first unit of `rank` (rank == nranks: V)
inline uint64_t vg_unit_begin(uint64_t nranks, uint64_t rank) { return rank * vg_units(nranks) / nranks; }
// A run of stored rows: this rank holds [begin, begin + count) of them; split = they are cut into one run of units per rank.
struct VgRun { uint64_t begin, count; bool split; };
// rank d's run of a split vector of n rows begins at row vg_run_bound(n, N, d) (d = N: n); exact whenever the split rules below
// split n (V divides n, or n is a layer whose run boundaries fall on whole nodes)
inline uint64_t vg_run_bound(uint64_t n, uint64_t nranks, uint64_t rank) { return vg_unit_begin(nranks, rank) * n / vg_units(nranks); }
// At a power-of-two nranks the units of a rank are rows [rank n / nranks, (rank + 1) n / nranks): the even split, computed as such.
inline VgRun vg_run_even(uint64_t n, uint64_t nranks, uint64_t rank, bool split) {
    return split ? VgRun{rank * (n / nranks), n / nranks, true} : VgRun{0, n, false};
}
inline VgRun vg_run(uint64_t n, uint64_t nranks, uint64_t rank, bool split) {
    if (!split || !(nranks & (nranks - 1))) return vg_run_even(n, nranks, rank, split);
    const uint64_t b = vg_run_bound(n, nranks, rank);
    return VgRun{b, vg_run_bound(n, nranks, rank + 1) - b, true};
}
// the longest run of any rank: what a symmetric-heap shard is sized for on every rank (the heap's offsets must match)
inline uint64_t vg_run_max(uint64_t n, uint64_t nranks) {
    uint64_t m = 0;
    for (uint64_t d = 0; d < nranks; d++) m = std::max(m, vg_run_bound(n, nranks, d + 1) - vg_run_bound(n, nranks, d));
    return m;
}
// A matrix / vector of `n` stored rows is cut into runs when n >= 4096 P (a unit keeps >= 512 rows, so a rank's run is whole
// 256-leaf sub-trees and whole FRI leaf pairs); shorter ones are replicated (every rank computes and holds all of them).  Stored
// heights are powers of two, and for those n >= 4096 N is the same test (4096 P is the least power of two >= 4096 N).
inline bool vg_split_rows_n(uint64_t n, int nranks) { return nranks > 1 && n >= (uint64_t)nranks * 4096; }
inline bool vg_split_rows(const vgpu_ctx* ctx, uint64_t n) { return vg_sharded(ctx) && n >= (uint64_t)ctx->comm_size * 4096; }
inline VgRun vg_row_run(const vgpu_ctx* ctx, uint64_t n) { return vg_run(n, ctx->comm_size, ctx->comm_rank, vg_split_rows(ctx, n)); }
// A trace of h rows is split when its LDE of 2h rows is: its rank r holds the natural rows of its units of h.
inline VgRun vg_trace_run(const vgpu_ctx* ctx, uint64_t h) { return vg_run(h, ctx->comm_size, ctx->comm_rank, vg_split_rows(ctx, 2 * h)); }
// A Merkle tree layer of `len` nodes is cut into runs while every rank's run is a whole number of nodes (merkle.h): down to the layer
// of N nodes (the sub-roots) at a power of two N, down to the layer of V nodes otherwise.
inline bool vg_layer_split(uint64_t len, int nranks) {
    if (nranks <= 1) return false;
    for (int d = 1; d < nranks; d++) if (vg_unit_begin(nranks, d) * len % vg_units(nranks)) return false;
    return true;
}
inline VgRun vg_layer_run(uint64_t len, int nranks, int rank) { return vg_run(len, nranks, rank, vg_layer_split(len, nranks)); }
// The first row of this rank's run in m (null for no matrix): a row shard starts there, a whole matrix is entered at run.begin.
inline const uint32_t* vg_run_rows(const vgpu_dmat* m, const VgRun& run) { return m ? m->d + (m->dist == VG_ROWS ? 0 : run.begin) : nullptr; }
// A query answer is summed over the ranks, so of data every rank holds only rank 0 reports its words.
inline bool vg_reports_replicated(const vgpu_ctx* ctx) { return ctx->comm_rank == 0 || !vg_sharded(ctx); }
// Whether this rank sweeps a trace of h rows in a machine-wide report (*run: its rows): its run if the trace is split, else rank 0 only.
inline bool vg_reports_trace(const vgpu_ctx* ctx, uint64_t h, VgRun* run) { *run = vg_trace_run(ctx, h); return run->split || vg_reports_replicated(ctx); }
// m's word at stored row `row`, column col, when this rank reports it (holds the row in its shard, or is rank 0 of a whole m); else null
inline const uint32_t* vg_reported_word(const vgpu_ctx* ctx, const vgpu_dmat* m, uint64_t row, uint64_t col) {
    const bool mine = m->dist == VG_ROWS ? (row >= m->row0 && row < m->row0 + m->h) : vg_reports_replicated(ctx);
    return mine ? m->d + col * m->col_stride + (row - m->row0) : nullptr;
}
// The part of a gh x gw matrix this rank holds: its run of stored rows when `split` (VG_ROWS), else all of it (VG_FULL).
// symm: taken from the symmetric heap (peers store into it and read it); such a shard has the column stride vg_run_max on every rank,
// so that every rank's allocation, and a column's place in it, is the same.
int32_t vg_dmat_alloc_run(vgpu_ctx* ctx, uint64_t gh, uint64_t gw, bool split, bool symm, VgMat* out);
inline int32_t vg_dmat_alloc(vgpu_ctx* ctx, uint64_t h, uint64_t w, VgMat* out) { return vg_dmat_alloc_run(ctx, h, w, false, false, out); }

// host/comm.cc — every rank calls these in the same order with the same sizes
// buf holds comm_size consecutive blocks of `words_per_rank` u32; this rank's block is already filled
int32_t vg_comm_allgather_inplace(vgpu_ctx* ctx, uint32_t* buf, uint64_t words_per_rank);
// buf holds all n rows (`words` u32 each, row i at buf + i * words) of a vector split by the rule above (vg_run over n); this rank's
// run is already filled.  Afterwards every row is.  Equal runs (a power of two N) are one vg_comm_allgather_inplace.
int32_t vg_comm_allgather_runs(vgpu_ctx* ctx, uint32_t* buf, uint64_t n, uint64_t words);
// stream-ordered barrier: everything enqueued before it on ANY rank's stream completes before anything enqueued after it
// on any rank's stream starts (peer stores become visible, peer buffers may be reused)
int32_t vg_comm_barrier(vgpu_ctx* ctx);
int32_t vg_comm_group_begin(vgpu_ctx* ctx);   // NCCL group around several all-gathers (no-ops for in-process ranks)
int32_t vg_comm_group_end(vgpu_ctx* ctx);
void vg_comm_free(vgpu_ctx* ctx);
// symmetric heap (collective: same calls, same sizes, same order on every rank)
int32_t vg_symm_reserve(vgpu_ctx* ctx, size_t extra_bytes);     // make room for `extra_bytes` more (grows the heap when nothing is live)
int32_t vg_symm_alloc(vgpu_ctx* ctx, void** p, size_t bytes);
void vg_symm_free(vgpu_ctx* ctx, void* p);
inline size_t vg_symm_round(size_t bytes) { return (bytes + 1023) & ~(size_t)1023; }
template <class T> inline T* vg_peer_ptr(const vgpu_ctx* ctx, T* mine, int peer) {
    return reinterpret_cast<T*>(ctx->peer_base[peer] + (reinterpret_cast<uint8_t*>(const_cast<typename std::remove_const<T>::type*>(mine)) - ctx->symm_base));
}
// exchange.cu — the two transposing exchanges of a split commit, as kernels storing through peer pointers
int32_t vg_exchange_rows_to_cols(vgpu_ctx* ctx, const vgpu_dmat* rows, uint32_t* cols_symm, const uint32_t* col_begin);
int32_t vg_exchange_cols_to_rows(vgpu_ctx* ctx, const uint32_t* lde_cols, uint64_t H, uint64_t c0, uint64_t c1, vgpu_dmat* shard, cudaStream_t on = nullptr);
size_t vg_commit_symm_need(const vgpu_ctx* ctx, const std::vector<std::pair<uint64_t, uint64_t>>& dims_all);

// ntt.cu
int32_t vg_ntt_nat2nat(vgpu_ctx* ctx, const uint32_t* src, uint64_t src_cs, uint32_t* dst, uint64_t dst_cs, int log_n, uint64_t w,
                       bool inverse, const PowTable* coset_or_null, uint32_t* tmp, uint64_t tmp_cs);
int32_t vg_coset_lde(vgpu_ctx* ctx, const uint32_t* src, uint64_t src_cs, uint64_t h, uint64_t w, uint32_t shift_canonical,
                     uint32_t* dst, uint64_t dst_cs, bool bit_reversed, bool src_bitrev = false, uint32_t log_blowup = 1);
// staging.cu
int32_t vg_upload_begin(vgpu_ctx* ctx, const uint32_t* host, uint64_t h, uint64_t w, int32_t repr, vgpu_dmat* dst);   // async copy only
int32_t vg_stager_start(vgpu_ctx* ctx);                       // after the last vg_upload_begin of a proof
int32_t vg_stager_finish(vgpu_ctx* ctx);                      // before the caller's buffers may change again
void vg_stager_free(vgpu_ctx* ctx);
int32_t vg_dmat_materialize(vgpu_ctx* ctx, const vgpu_dmat* m);                                                       // no-op unless an upload is pending
int32_t vg_upload_rowmajor(vgpu_ctx* ctx, const uint32_t* host, uint64_t h, uint64_t w, int32_t repr, vgpu_dmat* dst);
int32_t vg_download_rowmajor(vgpu_ctx* ctx, const vgpu_dmat* src, int32_t repr, uint32_t* host);
int32_t vg_import_strided(vgpu_ctx* ctx, const uint32_t* src, uint64_t h, uint64_t w, uint64_t rs, uint64_t cs, int32_t repr, vgpu_dmat* dst_or_null,
                          unsigned long long* bad_key);                                                                    // synchronises
int32_t vg_export_strided(vgpu_ctx* ctx, const vgpu_dmat* src, int32_t repr, uint32_t* dst, uint64_t rs, uint64_t cs);       // no host sync
