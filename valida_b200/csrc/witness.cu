// Witness generation on the device — SURVEY.md §8(f)1: Chip::generate_trace of the chips whose traces grow with the run
// (cpu, memory incl. the (addr, clk) sort, add, sub, lt, bitwise), straight into column-major Montgomery HBM.  The interpreter
// (Machine::run) stays on the host — it is a serial loop — and hands over its LOGS (host/vmlog.h: 24 bytes per cycle, 16 per
// memory operation, 12-16 per ALU operation: about an eighth of the bytes of the traces they expand to), so the 2 GB host row
// fill, the 2 GB upload and the transposes disappear.
//   * one thread per trace row: the row functions of chip_rows.cuh (the ones the host builder calls) assemble the row in
//     registers / local memory, and the kernel writes it column by column (coalesced) in Montgomery form;
//   * memory chip: stable LSD radix sort of the log by address on the device (8-bit digits, digits that are the same for every
//     address are skipped; the log is in clock order, so a stable sort on the address IS the reference's (addr, clk) order);
//   * column 27 of the CPU and lt rows: the inverse by Fermat per row (the host builder uses a table for the CPU: same values);
//   * split proof: a rank builds only ITS rows of the tall chips (the sort is repeated on every rank: 9 M keys).
// The short chips (program, mul floor, range, static data, the empty ones) are built on the host (vg_short_chip_traces, a few KB)
// and uploaded.  Parity: every trace equals the host builder's word for word (tests/test_gpu_witness.py; digests in
// tests/golden/trace_hashes.json).
// The host side builds one chip per call (VgWitnessBuilder, witness.h): vgpu_witness_device builds them all, vgpu_diff_witness one at a
// time, comparing each before it builds the next.
#include "ctx.h"
#include "chip_rows.cuh"
#include "witness.h"
#include <algorithm>
#include <memory>

struct vgpu_vmlog;
extern "C" const VgVmLogs* vg_vmlog_view(const vgpu_vmlog* l);

namespace {

__device__ __forceinline__ uint32_t mont(uint32_t raw) { return bb::to_monty(raw); }

struct RowRange { uint64_t row0, rows; uint32_t* out; uint64_t cs; };      // this launch fills rows [row0, row0 + rows) into out[c * cs + (row - row0)]

__global__ void __launch_bounds__(128) cpu_rows_kernel(const VgCpuRec* __restrict__ cpu, const VgMemOp* __restrict__ mem, const int32_t* __restrict__ prog,
                                                      uint64_t n, uint64_t n_mem, RowRange rr) {
    const uint64_t li = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (li >= rr.rows) return;
    const uint64_t i = rr.row0 + li;
    uint32_t row[CPU_COLS], dinv_m = 0;
    if (i < n) {
        const VgCpuRec r = cpu[i];
        const uint64_t k1 = i + 1 < n ? (uint64_t)cpu[i + 1].mem0 : n_mem;
        const uint32_t d = cpu_row(row, i, r, prog + 6 * (size_t)r.instr, mem + r.mem0, k1 - r.mem0);
        if (d) dinv_m = bb::inv(mont(d));
    } else {
        cpu_pad_row(row, i, cpu[n - 1]);
    }
#pragma unroll
    for (int c = 0; c < CPU_COLS; c++) rr.out[(uint64_t)c * rr.cs + li] = c == 27 ? dinv_m : mont(row[c]);
}

__global__ void __launch_bounds__(256) mem_rows_kernel(const VgMemOp* __restrict__ mem, const uint32_t* __restrict__ order /* sorted position -> log index, or null */,
                                                      uint64_t n, const uint32_t* __restrict__ st_addr, const uint32_t* __restrict__ st_val, uint64_t n0, RowRange rr) {
    const uint64_t li = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (li >= rr.rows) return;
    const uint64_t i = rr.row0 + li;
    uint32_t row[MEM_COLS] = {};
    if (i < n0) mem_row(row, i, {0u, st_addr[i], st_val[i], 1u}, true);
    else if (i < n0 + n) mem_row(row, i, mem[order ? order[i - n0] : i - n0], false);
#pragma unroll
    for (int c = 0; c < MEM_COLS; c++) rr.out[(uint64_t)c * rr.cs + li] = mont(row[c]);
}

__global__ void __launch_bounds__(256) addsub_rows_kernel(const VgAluRec* __restrict__ ops, uint64_t n, int is_add, RowRange rr) {
    const uint64_t li = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (li >= rr.rows) return;
    const uint64_t i = rr.row0 + li;
    uint32_t row[ADDSUB_COLS] = {};
    if (i < n) addsub_row(row, ops[i], is_add);
#pragma unroll
    for (int c = 0; c < ADDSUB_COLS; c++) rr.out[(uint64_t)c * rr.cs + li] = mont(row[c]);
}

__global__ void __launch_bounds__(128) lt_rows_kernel(const VgAluOpRec* __restrict__ ops, uint64_t n, RowRange rr) {
    const uint64_t li = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (li >= rr.rows) return;
    const uint64_t i = rr.row0 + li;
    uint32_t row[LT_COLS] = {}, inv_m = 0;
    if (i < n) {
        if (const uint32_t d = lt_row(row, ops[i])) inv_m = bb::inv(mont(d));
    }
#pragma unroll
    for (int c = 0; c < LT_COLS; c++) rr.out[(uint64_t)c * rr.cs + li] = c == 27 ? inv_m : mont(row[c]);
}

__global__ void __launch_bounds__(128) bitwise_rows_kernel(const VgAluOpRec* __restrict__ ops, uint64_t n, RowRange rr) {
    const uint64_t li = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (li >= rr.rows) return;
    const uint64_t i = rr.row0 + li;
    const bool real = i < n;
    uint32_t row[BITWISE_COLS];
    bitwise_row(row, real ? ops[i] : VgAluOpRec{});     // unconditional: each word can then be computed next to its store
#pragma unroll
    for (int c = 0; c < BITWISE_COLS; c++) rr.out[(uint64_t)c * rr.cs + li] = real ? mont(row[c]) : 0u;
}

// ---- stable LSD radix sort of the memory log by address: (key, log index) pairs, 8-bit digits -----------------------------------
constexpr int SORT_TILE = 4096, SORT_THREADS = 256, SORT_ROUNDS = SORT_TILE / SORT_THREADS;
__global__ void addr_bits_kernel(const VgMemOp* __restrict__ mem, uint64_t n, uint32_t* __restrict__ or_and /* [or, and] */) {
    uint32_t o = 0, a = 0xffffffffu;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) { const uint32_t k = mem[i].addr; o |= k; a &= k; }
    for (int s = 16; s > 0; s >>= 1) { o |= __shfl_xor_sync(0xffffffffu, o, s); a &= __shfl_xor_sync(0xffffffffu, a, s); }
    if ((threadIdx.x & 31) == 0) { atomicOr(or_and, o); atomicAnd(or_and + 1, a); }
}
__global__ void sort_init_kernel(const VgMemOp* __restrict__ mem, uint64_t n, uint32_t* __restrict__ keys, uint32_t* __restrict__ idx) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { keys[i] = mem[i].addr; idx[i] = (uint32_t)i; }
}
// hist[d * nblocks + block] = number of keys of the block's tile with digit d
__global__ void __launch_bounds__(SORT_THREADS) sort_hist_kernel(const uint32_t* __restrict__ keys, uint64_t n, int shift, uint32_t* __restrict__ hist, uint32_t nblocks) {
    __shared__ uint32_t h[256];
    h[threadIdx.x] = 0;
    __syncthreads();
    const uint64_t base = (uint64_t)blockIdx.x * SORT_TILE;
    for (int r = 0; r < SORT_ROUNDS; r++) {
        const uint64_t i = base + (uint64_t)r * SORT_THREADS + threadIdx.x;
        if (i < n) atomicAdd(&h[(keys[i] >> shift) & 255], 1u);
    }
    __syncthreads();
    hist[(uint64_t)threadIdx.x * nblocks + blockIdx.x] = h[threadIdx.x];
}
// exclusive scan of `n` counters by one block (n = 256 * nblocks: ~0.6 M for a 9 M-entry log)
__global__ void __launch_bounds__(1024) scan_u32_kernel(uint32_t* __restrict__ data, uint64_t n) {
    __shared__ uint32_t wsum[32];
    __shared__ uint32_t carry_s;
    if (threadIdx.x == 0) carry_s = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    for (uint64_t base = 0; base < n; base += 1024) {
        const uint64_t i = base + threadIdx.x;
        const uint32_t x = i < n ? data[i] : 0;
        uint32_t v = x;
        for (int o = 1; o < 32; o <<= 1) { const uint32_t u = __shfl_up_sync(0xffffffffu, v, o); if (lane >= o) v += u; }
        if (lane == 31) wsum[wid] = v;
        __syncthreads();
        if (wid == 0) {
            uint32_t w = wsum[lane];
            for (int o = 1; o < 32; o <<= 1) { const uint32_t u = __shfl_up_sync(0xffffffffu, w, o); if (lane >= o) w += u; }
            wsum[lane] = w;
        }
        __syncthreads();
        const uint32_t incl = v + carry_s + (wid > 0 ? wsum[wid - 1] : 0);
        if (i < n) data[i] = incl - x;
        __syncthreads();
        if (threadIdx.x == 1023) carry_s = incl;
        __syncthreads();
    }
}
// stable scatter: within a tile keys are taken in order, 256 at a time; equal digits inside a warp are ranked by lane
__global__ void __launch_bounds__(SORT_THREADS) sort_scatter_kernel(const uint32_t* __restrict__ keys, const uint32_t* __restrict__ idx, uint64_t n, int shift,
                                                                   const uint32_t* __restrict__ offs, uint32_t nblocks, uint32_t* __restrict__ keys_out, uint32_t* __restrict__ idx_out) {
    __shared__ uint32_t running[256];                       // next output slot of every digit for this tile
    __shared__ uint32_t whist[SORT_THREADS / 32][256];      // per-round, per-warp digit counts
    running[threadIdx.x] = offs[(uint64_t)threadIdx.x * nblocks + blockIdx.x];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint64_t base = (uint64_t)blockIdx.x * SORT_TILE;
    for (int r = 0; r < SORT_ROUNDS; r++) {
        for (int w = 0; w < SORT_THREADS / 32; w++) whist[w][threadIdx.x] = 0;
        __syncthreads();
        const uint64_t i = base + (uint64_t)r * SORT_THREADS + threadIdx.x;
        const bool live = i < n;
        const uint32_t key = live ? keys[i] : 0, d = live ? (key >> shift) & 255 : 256 + (uint32_t)lane;   // dead lanes match nobody
        const uint32_t peers = __match_any_sync(0xffffffffu, d);
        const uint32_t rank = __popc(peers & ((1u << lane) - 1));
        if (live && rank == 0) whist[wid][d] = __popc(peers);
        __syncthreads();
        if (live) {
            uint32_t pos = running[d] + rank;
            for (int w = 0; w < wid; w++) pos += whist[w][d];
            keys_out[pos] = key; idx_out[pos] = idx[i];
        }
        __syncthreads();
        { uint32_t t = 0; for (int w = 0; w < SORT_THREADS / 32; w++) t += whist[w][threadIdx.x]; running[threadIdx.x] += t; }
        __syncthreads();
    }
}

// sorted position -> log index; null result = the log is already in address order (every address identical)
int32_t sort_log_by_addr(vgpu_ctx* ctx, const VgMemOp* d_mem, uint64_t n, VgBuf& out_idx) {
    if (n < 2) return 0;
    VgBuf bits(ctx), k0(ctx), k1(ctx), i0(ctx), i1(ctx), hist(ctx);
    VG_TRY(bits.alloc(8));
    const uint32_t init[2] = {0u, 0xffffffffu};
    VG_CUDA(ctx, cudaMemcpyAsync(bits.p, init, 8, cudaMemcpyHostToDevice, ctx->stream));
    addr_bits_kernel<<<2 * ctx->sm_count, 256, 0, ctx->stream>>>(d_mem, n, bits.as<uint32_t>());
    VG_LAUNCH_CHECK(ctx);
    uint32_t oa[2];
    VG_CUDA(ctx, cudaMemcpyAsync(oa, bits.p, 8, cudaMemcpyDeviceToHost, ctx->stream));
    VG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    const uint32_t varying = oa[0] ^ oa[1];
    if (!varying) return 0;
    const uint32_t nblocks = (uint32_t)((n + SORT_TILE - 1) / SORT_TILE);
    VG_TRY(k0.alloc(n * 4)); VG_TRY(k1.alloc(n * 4));
    VG_TRY(i0.alloc(n * 4)); VG_TRY(i1.alloc(n * 4));
    VG_TRY(hist.alloc((size_t)256 * nblocks * 4));
    sort_init_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(d_mem, n, k0.as<uint32_t>(), i0.as<uint32_t>());
    VG_LAUNCH_CHECK(ctx);
    uint32_t *ka = k0.as<uint32_t>(), *kb = k1.as<uint32_t>(), *ia = i0.as<uint32_t>(), *ib = i1.as<uint32_t>();
    for (int shift = 0; shift < 32; shift += 8) {
        if (((varying >> shift) & 255) == 0) continue;
        sort_hist_kernel<<<nblocks, SORT_THREADS, 0, ctx->stream>>>(ka, n, shift, hist.as<uint32_t>(), nblocks);
        VG_LAUNCH_CHECK(ctx);
        scan_u32_kernel<<<1, 1024, 0, ctx->stream>>>(hist.as<uint32_t>(), (uint64_t)256 * nblocks);
        VG_LAUNCH_CHECK(ctx);
        sort_scatter_kernel<<<nblocks, SORT_THREADS, 0, ctx->stream>>>(ka, ia, n, shift, hist.as<uint32_t>(), nblocks, kb, ib);
        VG_LAUNCH_CHECK(ctx);
        std::swap(ka, kb); std::swap(ia, ib);
    }
    // hand the buffer holding the final order to the caller
    out_idx = std::move(ia == i0.as<uint32_t>() ? i0 : i1);
    return 0;
}

}  // namespace

struct VgWitnessBuilder::Impl {
    vgpu_ctx* ctx;
    const VgVmLogs& L;
    VgBuf d_prog, d_cpu, d_mem, d_adds, d_subs, d_lts, d_bits, d_sa, d_sv;
    std::unique_ptr<vgpu_traces, void (*)(vgpu_traces*)> st{nullptr, vgpu_traces_free};
    Impl(vgpu_ctx* c, const VgVmLogs& l)
        : ctx(c), L(l), d_prog(c), d_cpu(c), d_mem(c), d_adds(c), d_subs(c), d_lts(c), d_bits(c), d_sa(c), d_sv(c) {}
    // a tall chip's trace: whole, or this rank's run of rows (split proof)
    int32_t alloc_rows(uint64_t h, uint64_t w, VgMat* out, RowRange* rr) {
        VG_TRY(vg_dmat_alloc_run(ctx, h, w, vg_trace_run(ctx, h).split, false, out));
        rr->row0 = (*out)->row0; rr->rows = (*out)->h; rr->out = (*out)->d; rr->cs = (*out)->col_stride;
        return 0;
    }
    int32_t upload(const vgpu_matrix* hm, VgMat* out) {
        vgpu_dmat* m = nullptr;
        VG_TRY(vgpu_dmat_upload(ctx, hm, VGPU_REPR_CANONICAL, &m));
        out->reset(m);
        return 0;
    }
};

VgWitnessBuilder::VgWitnessBuilder(vgpu_ctx* ctx, const VgVmLogs& L) : impl_(new Impl(ctx, L)) {}
VgWitnessBuilder::~VgWitnessBuilder() = default;

int32_t VgWitnessBuilder::start() {
    Impl& w = *impl_;
    const VgVmLogs& L = w.L;
    VG_TRY(w.d_prog.upload(L.program, 6 * L.n_instr));
    VG_TRY(w.d_cpu.upload(L.cpu, L.n_cpu));
    VG_TRY(w.d_mem.upload(L.mem, L.n_mem));
    VG_TRY(w.d_adds.upload(L.adds, L.n_adds));
    VG_TRY(w.d_subs.upload(L.subs, L.n_subs));
    VG_TRY(w.d_lts.upload(L.lts, L.n_lts));
    VG_TRY(w.d_bits.upload(L.bits, L.n_bits));
    VG_TRY(w.d_sa.upload(L.static_addr, L.n_static));
    VG_TRY(w.d_sv.upload(L.static_value, L.n_static));
    w.st.reset(vg_short_chip_traces(L));
    return 0;
}

uint64_t VgWitnessBuilder::height(int c) const {
    const VgVmLogs& L = impl_->L;
    switch (c) {
        case 0: return next_pow2(L.n_cpu);
        case 2: return next_pow2(L.n_static + L.n_mem);
        case 3: return next_pow2(L.n_adds);
        case 4: return next_pow2(L.n_subs);
        case 8: return next_pow2(L.n_lts);
        case 10: return next_pow2(L.n_bits);
        default: return vgpu_traces_main(impl_->st.get(), (uint32_t)c)->height;
    }
}

int32_t VgWitnessBuilder::main(int c, VgMat* out) {
    Impl& w = *impl_;
    vgpu_ctx* ctx = w.ctx;
    const VgVmLogs& L = w.L;
    RowRange rr{};
    switch (c) {
        case 0:
            VG_TRY(w.alloc_rows(height(0), 51, out, &rr));
            cpu_rows_kernel<<<(unsigned)((rr.rows + 127) / 128), 128, 0, ctx->stream>>>(w.d_cpu.as<VgCpuRec>(), w.d_mem.as<VgMemOp>(), w.d_prog.as<int32_t>(), L.n_cpu, L.n_mem, rr);
            VG_LAUNCH_CHECK(ctx);
            return 0;
        case 2: {   // sort by address (stable), then the rows
            VgBuf d_order(ctx);
            VG_TRY(sort_log_by_addr(ctx, w.d_mem.as<VgMemOp>(), L.n_mem, d_order));
            VG_TRY(w.alloc_rows(height(2), 14, out, &rr));
            mem_rows_kernel<<<(unsigned)((rr.rows + 255) / 256), 256, 0, ctx->stream>>>(w.d_mem.as<VgMemOp>(), d_order.as<uint32_t>(), L.n_mem, w.d_sa.as<uint32_t>(), w.d_sv.as<uint32_t>(), L.n_static, rr);
            VG_LAUNCH_CHECK(ctx);
            return 0;
        }
        case 3: case 4: {
            const int which = c - 3;
            VG_TRY(w.alloc_rows(height(c), 16, out, &rr));
            addsub_rows_kernel<<<(unsigned)((rr.rows + 255) / 256), 256, 0, ctx->stream>>>(which ? w.d_subs.as<VgAluRec>() : w.d_adds.as<VgAluRec>(), which ? L.n_subs : L.n_adds, which == 0, rr);
            VG_LAUNCH_CHECK(ctx);
            return 0;
        }
        case 8:
            VG_TRY(w.alloc_rows(height(8), 45, out, &rr));
            lt_rows_kernel<<<(unsigned)((rr.rows + 127) / 128), 128, 0, ctx->stream>>>(w.d_lts.as<VgAluOpRec>(), L.n_lts, rr);
            VG_LAUNCH_CHECK(ctx);
            return 0;
        case 10:
            VG_TRY(w.alloc_rows(height(10), 79, out, &rr));
            bitwise_rows_kernel<<<(unsigned)((rr.rows + 127) / 128), 128, 0, ctx->stream>>>(w.d_bits.as<VgAluOpRec>(), L.n_bits, rr);
            VG_LAUNCH_CHECK(ctx);
            return 0;
        default:    // the short chips: built on the host by start() and uploaded whole
            return w.upload(vgpu_traces_main(w.st.get(), (uint32_t)c), out);
    }
}

int32_t VgWitnessBuilder::prep(int which, VgMat* out) {
    return impl_->upload(vgpu_traces_preprocessed(impl_->st.get(), (uint32_t)which), out);
}

extern "C" {

// Chip::generate_trace x14 from the interpreter's logs, on the device: main_out[14] / prep_out[2] receive device matrices (column-major
// Montgomery; this rank's row shard for a chip tall enough to be split — vgpu_dmat_upload_rows' rule), ready for vgpu_prove_device.
int32_t vgpu_witness_device(vgpu_ctx* ctx, const vgpu_vmlog* log, vgpu_dmat* main_out[VGPU_NUM_CHIPS], vgpu_dmat* prep_out[2]) {
    if (!ctx || !log || !main_out || !prep_out) return -1;
    VG_TRY(vg_enter(ctx));
    const VgVmLogs& L = *vg_vmlog_view(log);
    for (int i = 0; i < VGPU_NUM_CHIPS; i++) main_out[i] = nullptr;
    prep_out[0] = prep_out[1] = nullptr;
    if (!L.n_cpu) VG_FAIL(ctx, "witness: the run has no cycles");
    VgMat main[VGPU_NUM_CHIPS], prep[2];                   // handed out only once every trace is built
    VgWitnessBuilder wb(ctx, L);
    VG_TRY(wb.start());
    for (int c : {0, 2, 3, 4, 8, 10}) VG_TRY(wb.main(c, &main[c]));     // the tall chips, built from the logs on the device
    for (int c = 0; c < VGPU_NUM_CHIPS; c++)
        if (!main[c]) VG_TRY(wb.main(c, &main[c]));
    for (int w = 0; w < 2; w++) VG_TRY(wb.prep(w, &prep[w]));
    VG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));      // the logs are the caller's (pageable) memory: they may go once this returns
    for (int i = 0; i < VGPU_NUM_CHIPS; i++) main_out[i] = main[i].release();
    for (int i = 0; i < 2; i++) prep_out[i] = prep[i].release();
    return 0;
}

}  // extern "C"
