// Witness generation on the device — SURVEY.md §8(f)1: Chip::generate_trace of the chips whose traces grow with the run
// (cpu/src/lib.rs:79-97,163-373; memory/src/lib.rs:143-194 incl. the (addr, clk) sort; alu_u32/src/{add,sub,lt,bitwise}/mod.rs
// op_to_row), straight into column-major Montgomery HBM.  The interpreter (Machine::run) stays on the host — it is a serial
// loop — and hands over its LOGS (host/vmlog.h: 24 bytes per cycle, 16 per memory operation, 12-16 per ALU operation: about an
// eighth of the bytes of the traces they expand to), so the 2 GB host row fill, the 2 GB upload and the transposes disappear.
//   * one thread per trace row; a row is assembled in registers / local memory and written column by column (coalesced);
//   * memory chip: stable LSD radix sort of the log by address on the device (8-bit digits, digits that are the same for every
//     address are skipped; the log is in clock order, so a stable sort on the address IS the reference's (addr, clk) order);
//   * CPU chip: diff_inv = 1 / sum_k (b_k - c_k)^2 by Fermat per row (the host builder uses a table: same values);
//   * split proof: a rank builds only ITS rows of the tall chips (the sort is repeated on every rank: 9 M keys).
// The short chips (program, mul floor, range, static data, the empty ones) are built on the host (a few KB) and uploaded.
// Parity: every trace equals the host builder's word for word (tests/test_gpu_witness.py; digests in tests/golden/trace_hashes.json).
#include "ctx.h"
#include "host/vmlog.h"
#include <algorithm>
#include <memory>

struct vgpu_vmlog;
extern "C" const VgVmLogs* vg_vmlog_view(const vgpu_vmlog* l);

namespace {

constexpr uint32_t OP_STOP = 8, OP_LT32 = 104, OP_AND32 = 107, OP_OR32 = 108, OP_LTE32 = 115, OP_SLT32 = 117;

__device__ __forceinline__ uint32_t mont(uint32_t raw) { return bb::to_monty(raw); }           // any u32 -> (raw mod p) in Montgomery form
__device__ __forceinline__ uint32_t from_i32(int32_t x) { return x < 0 ? (bb::P - (uint32_t)(-(int64_t)x) % bb::P) % bb::P : (uint32_t)x % bb::P; }
__device__ __forceinline__ void word_be(uint32_t v, uint32_t* out) { out[0] = v >> 24; out[1] = (v >> 16) & 0xff; out[2] = (v >> 8) & 0xff; out[3] = v & 0xff; }

struct RowRange { uint64_t row0, rows; uint32_t* out; uint64_t cs; };      // this launch fills rows [row0, row0 + rows) into out[c * cs + (row - row0)]

// ---- CPU chip (51 columns; cpu/src/columns.rs:8-37) -------------------------------------------------------------------------
__global__ void __launch_bounds__(128) cpu_rows_kernel(const VgCpuRec* __restrict__ cpu, const VgMemOp* __restrict__ mem, const int32_t* __restrict__ prog,
                                                      uint64_t n, uint64_t n_mem, RowRange rr) {
    const uint64_t li = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (li >= rr.rows) return;
    const uint64_t i = rr.row0 + li;
    uint32_t row[51];
#pragma unroll
    for (int c = 0; c < 51; c++) row[c] = 0;
    uint32_t dinv_m = 0;
    if (i < n) {
        const VgCpuRec r = cpu[i];
        const int32_t* w = prog + 6 * (size_t)r.instr;
        row[0] = (uint32_t)i; row[1] = r.pc; row[2] = r.fp; row[3] = (uint32_t)w[0];
        for (int k = 0; k < 5; k++) row[4 + k] = from_i32(w[1 + k]);
        bool left_imm = false;
        switch (r.kind) {
            case VG_K_STORE32: row[16] = 1; break;
            case VG_K_LOAD32: row[13] = 1; break;
            case VG_K_JAL: row[20] = 1; break;
            case VG_K_JALV: row[21] = 1; break;
            case VG_K_BEQ: row[18] = 1; break;
            case VG_K_BNE: row[19] = 1; break;
            case VG_K_IMM32: row[22] = 1; break;
            case VG_K_BUS: row[9] = 1; break;
            case VG_K_STOP: row[24] = 1; break;
            case VG_K_LOADFP: row[25] = 1; break;
            case VG_K_BUS_LEFT_IMM: row[9] = 1; break;
        }
        if (r.has_imm && r.kind == VG_K_BUS_LEFT_IMM) {   // set_left_imm_value (cpu/src/lib.rs:364-371)
            row[12] = 1; left_imm = true;
            word_be(r.imm, &row[32]);
            row[5] = r.imm % bb::P;
        } else if (r.has_imm) {                             // set_imm_value (cpu/src/lib.rs:355-362)
            row[11] = 1;
            word_be(r.imm, &row[39]);
            row[6] = r.imm % bb::P;
        }
        row[30] = 1; row[37] = 1;
        const uint64_t k0 = r.mem0, k1 = i + 1 < n ? (uint64_t)cpu[i + 1].mem0 : n_mem;
        bool first_read = true;
        for (uint64_t k = k0; k < k1; k++) {
            const VgMemOp m = mem[k];
            uint32_t ch;
            if (m.is_write) ch = 43;
            else if (first_read && !left_imm) { ch = 29; first_read = false; }
            else ch = 36;
            row[ch] = 1; row[ch + 2] = m.addr; word_be(m.value, &row[ch + 3]);
        }
        uint32_t dsum = 0;
        for (int k = 0; k < 4; k++) { const int32_t dd = (int32_t)row[32 + k] - (int32_t)row[39 + k]; dsum += (uint32_t)(dd * dd); }
        row[26] = dsum;                                      // <= 4 * 255^2 < p
        if (dsum) { dinv_m = bb::inv(mont(dsum)); row[28] = 1; }
    } else {                                                 // pad_to_power_of_two (cpu/src/lib.rs:318-353): STOP rows
        const VgCpuRec last = cpu[n - 1];
        row[1] = last.pc; row[2] = last.fp; row[0] = (uint32_t)(n - 1) + (uint32_t)(i - n) + 1;
        row[24] = 1; row[3] = OP_STOP;
        row[30] = 1; row[37] = 1;
    }
#pragma unroll
    for (int c = 0; c < 51; c++) rr.out[(uint64_t)c * rr.cs + li] = c == 27 ? dinv_m : mont(row[c]);
}

// ---- memory chip (14 columns; memory/src/columns.rs:8-39) -------------------------------------------------------------------
__global__ void __launch_bounds__(256) mem_rows_kernel(const VgMemOp* __restrict__ mem, const uint32_t* __restrict__ order /* sorted position -> log index, or null */,
                                                      uint64_t n, const uint32_t* __restrict__ st_addr, const uint32_t* __restrict__ st_val, uint64_t n0, RowRange rr) {
    const uint64_t li = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (li >= rr.rows) return;
    const uint64_t i = rr.row0 + li;
    uint32_t row[14];
#pragma unroll
    for (int c = 0; c < 14; c++) row[c] = 0;
    if (i < n0) {                                            // the static cells open the trace (memory/src/lib.rs:163-169)
        row[0] = st_addr[i]; word_be(st_val[i], &row[1]);
        row[6] = 1; row[8] = 1; row[12] = (uint32_t)i;
    } else if (i < n0 + n) {
        const uint64_t j = i - n0;
        const VgMemOp m = mem[order ? order[j] : j];
        row[0] = m.addr; word_be(m.value, &row[1]);
        row[5] = m.clk;
        row[7] = m.is_write ? 0 : 1; row[8] = m.is_write ? 1 : 0;
        row[12] = (uint32_t)i;
    }
#pragma unroll
    for (int c = 0; c < 14; c++) rr.out[(uint64_t)c * rr.cs + li] = mont(row[c]);
}

// ---- add / sub (16 columns; alu_u32/src/add/mod.rs:38-129, sub/mod.rs:103-111) ----------------------------------------------
__global__ void __launch_bounds__(256) addsub_rows_kernel(const VgAluRec* __restrict__ ops, uint64_t n, int is_add, RowRange rr) {
    const uint64_t li = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (li >= rr.rows) return;
    const uint64_t i = rr.row0 + li;
    uint32_t row[16];
#pragma unroll
    for (int c = 0; c < 16; c++) row[c] = 0;
    if (i < n) {
        const VgAluRec o = ops[i];
        uint32_t a[4], b[4], c[4];
        word_be(o.a, a); word_be(o.b, b); word_be(o.c, c);
#pragma unroll
        for (int k = 0; k < 4; k++) { row[k] = b[k]; row[4 + k] = c[k]; row[11 + k] = a[k]; }
        if (is_add) {
            const uint32_t c1 = (b[3] + c[3] > 255), c2 = (b[2] + c[2] + c1 > 255), c3 = (b[1] + c[1] + c2 > 255);
            row[8] = c1; row[9] = c2; row[10] = c3;
        } else {   // exactly as the reference: no borrow propagation into the comparison
            row[8] = (b[3] < c[3]); row[9] = (b[2] < c[2]); row[10] = (b[1] < c[1]);
        }
        row[15] = 1;
    }
#pragma unroll
    for (int c = 0; c < 16; c++) rr.out[(uint64_t)c * rr.cs + li] = mont(row[c]);
}

// ---- lt family (45 columns; alu_u32/src/lt/mod.rs:86-160) -------------------------------------------------------------------
__global__ void __launch_bounds__(128) lt_rows_kernel(const VgAluOpRec* __restrict__ ops, uint64_t n, RowRange rr) {
    const uint64_t li = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (li >= rr.rows) return;
    const uint64_t i = rr.row0 + li;
    uint32_t row[45];
#pragma unroll
    for (int c = 0; c < 45; c++) row[c] = 0;
    uint32_t inv_m = 0;
    if (i < n) {
        const VgAluOpRec o = ops[i];
        uint32_t a[4], b[4], c[4];
        word_be(o.a, a); word_be(o.b, b); word_be(o.c, c);
#pragma unroll
        for (int k = 0; k < 4; k++) { row[k] = b[k]; row[4 + k] = c[k]; }
        row[21] = a[3];
        const bool is_signed = o.opcode == OP_SLT32 || o.opcode == OP_SLT32 + 1;
        row[o.opcode == OP_LT32 ? 23 : o.opcode == OP_LTE32 ? 24 : o.opcode == OP_SLT32 ? 25 : 26] = 1;
        for (int k = 0; k < 4; k++) {
            if (b[k] != c[k]) {
                const uint32_t z = 256u + b[k] - c[k];
                for (int bit = 0; bit < 9; bit++) row[12 + bit] = (z >> bit) & 1;
                row[8 + k] = 1;
                const uint32_t diff = (b[k] + bb::P - c[k]) % bb::P;
                inv_m = bb::inv(mont(diff));
                break;
            }
        }
        for (int bit = 0; bit < 8; bit++) { row[28 + bit] = (b[0] >> bit) & 1; row[36 + bit] = (c[0] >> bit) & 1; }
        row[44] = (is_signed && row[35] != row[43]) ? 1 : 0;
        row[22] = 1;
    }
#pragma unroll
    for (int c = 0; c < 45; c++) rr.out[(uint64_t)c * rr.cs + li] = c == 27 ? inv_m : mont(row[c]);
}

// ---- and / or / xor (79 columns; alu_u32/src/bitwise/mod.rs:84-131) -----------------------------------------------------------
__global__ void __launch_bounds__(128) bitwise_rows_kernel(const VgAluOpRec* __restrict__ ops, uint64_t n, RowRange rr) {
    const uint64_t li = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (li >= rr.rows) return;
    const uint64_t i = rr.row0 + li;
    const bool real = i < n;
    VgAluOpRec o{0, 0, 0, 0};
    if (real) o = ops[i];
    uint32_t a[4], b[4], c[4];
    word_be(o.a, a); word_be(o.b, b); word_be(o.c, c);
    auto put = [&](int col, uint32_t v) { rr.out[(uint64_t)col * rr.cs + li] = real ? mont(v) : 0u; };
#pragma unroll
    for (int k = 0; k < 4; k++) { put(k, b[k]); put(4 + k, c[k]); put(72 + k, a[k]); }
#pragma unroll
    for (int k = 0; k < 4; k++)
#pragma unroll
        for (int bit = 0; bit < 8; bit++) { put(8 + 8 * k + bit, (b[k] >> bit) & 1); put(40 + 8 * k + bit, (c[k] >> bit) & 1); }
    put(76, o.opcode == OP_AND32); put(77, o.opcode == OP_OR32); put(78, real && o.opcode != OP_AND32 && o.opcode != OP_OR32);
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

uint64_t next_pow2(uint64_t n) { uint64_t p = 1; while (p < n) p <<= 1; return p; }

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
    // a tall chip's trace: whole, or this rank's run of rows (split proof)
    auto alloc_rows = [&](uint64_t h, uint64_t w, VgMat* out, RowRange* rr) -> int32_t {
        VG_TRY(vg_dmat_alloc_run(ctx, h, w, vg_trace_run(ctx, h).split, false, out));
        rr->row0 = (*out)->row0; rr->rows = (*out)->h; rr->out = (*out)->d; rr->cs = (*out)->col_stride;
        return 0;
    };
    auto small = [&](const std::vector<uint32_t>& rows, uint64_t h, uint64_t w, VgMat* out) -> int32_t {   // host-built short chip
        vgpu_matrix hm{rows.data(), h, w};
        vgpu_dmat* m = nullptr;
        VG_TRY(vgpu_dmat_upload(ctx, &hm, VGPU_REPR_CANONICAL, &m));
        out->reset(m);
        return 0;
    };
    VgBuf d_prog(ctx), d_cpu(ctx), d_mem(ctx), d_adds(ctx), d_subs(ctx), d_lts(ctx), d_bits(ctx), d_sa(ctx), d_sv(ctx), d_order(ctx);
    VG_TRY(d_prog.upload(L.program, 6 * L.n_instr));
    VG_TRY(d_cpu.upload(L.cpu, L.n_cpu));
    VG_TRY(d_mem.upload(L.mem, L.n_mem));
    VG_TRY(d_adds.upload(L.adds, L.n_adds));
    VG_TRY(d_subs.upload(L.subs, L.n_subs));
    VG_TRY(d_lts.upload(L.lts, L.n_lts));
    VG_TRY(d_bits.upload(L.bits, L.n_bits));
    VG_TRY(d_sa.upload(L.static_addr, L.n_static));
    VG_TRY(d_sv.upload(L.static_value, L.n_static));
    RowRange rr{};
    {   // 0 cpu
        const uint64_t h = next_pow2(L.n_cpu);
        VG_TRY(alloc_rows(h, 51, &main[0], &rr));
        cpu_rows_kernel<<<(unsigned)((rr.rows + 127) / 128), 128, 0, ctx->stream>>>(d_cpu.as<VgCpuRec>(), d_mem.as<VgMemOp>(), d_prog.as<int32_t>(), L.n_cpu, L.n_mem, rr);
        VG_LAUNCH_CHECK(ctx);
    }
    {   // 2 memory: sort by address (stable), then the rows
        VG_TRY(sort_log_by_addr(ctx, d_mem.as<VgMemOp>(), L.n_mem, d_order));
        const uint64_t h = next_pow2(L.n_static + L.n_mem);
        VG_TRY(alloc_rows(h, 14, &main[2], &rr));
        mem_rows_kernel<<<(unsigned)((rr.rows + 255) / 256), 256, 0, ctx->stream>>>(d_mem.as<VgMemOp>(), d_order.as<uint32_t>(), L.n_mem, d_sa.as<uint32_t>(), d_sv.as<uint32_t>(), L.n_static, rr);
        VG_LAUNCH_CHECK(ctx);
    }
    for (int which = 0; which < 2; which++) {   // 3 add, 4 sub
        const uint64_t n = which ? L.n_subs : L.n_adds, h = next_pow2(n);
        VG_TRY(alloc_rows(h, 16, &main[3 + which], &rr));
        addsub_rows_kernel<<<(unsigned)((rr.rows + 255) / 256), 256, 0, ctx->stream>>>(which ? d_subs.as<VgAluRec>() : d_adds.as<VgAluRec>(), n, which == 0, rr);
        VG_LAUNCH_CHECK(ctx);
    }
    {   // 8 lt
        const uint64_t h = next_pow2(L.n_lts);
        VG_TRY(alloc_rows(h, 45, &main[8], &rr));
        lt_rows_kernel<<<(unsigned)((rr.rows + 127) / 128), 128, 0, ctx->stream>>>(d_lts.as<VgAluOpRec>(), L.n_lts, rr);
        VG_LAUNCH_CHECK(ctx);
    }
    {   // 10 bitwise
        const uint64_t h = next_pow2(L.n_bits);
        VG_TRY(alloc_rows(h, 79, &main[10], &rr));
        bitwise_rows_kernel<<<(unsigned)((rr.rows + 127) / 128), 128, 0, ctx->stream>>>(d_bits.as<VgAluOpRec>(), L.n_bits, rr);
        VG_LAUNCH_CHECK(ctx);
    }
    // ---- the short chips, on the host ----
    {   // 1 program: 1 main column (execution counts) + 7 preprocessed (program/src/lib.rs:38-81, program/src/stark.rs:22-40)
        const uint64_t h = next_pow2(L.n_instr);
        std::vector<uint32_t> counts(h, 0), prep_rows(h * 7, 0);
        for (size_t i = 0; i < L.n_instr; i++) counts[i] = L.prog_counts[i];
        for (uint64_t i = 0; i < h; i++) {
            prep_rows[i * 7] = (uint32_t)i;
            if (i < L.n_instr) {
                prep_rows[i * 7 + 1] = (uint32_t)L.program[6 * i];
                for (int k = 0; k < 5; k++) { const int32_t x = L.program[6 * i + 1 + k]; prep_rows[i * 7 + 2 + k] = x < 0 ? (bb::P - (uint32_t)(-(int64_t)x) % bb::P) % bb::P : (uint32_t)x % bb::P; }
            }
        }
        VG_TRY(small(counts, h, 1, &main[1]));
        VG_TRY(small(prep_rows, h, 7, &prep[0]));
    }
    {   // 5 mul: 2^10 counter rows (alu_u32/src/mul/mod.rs:38-64)
        std::vector<uint32_t> m(1024 * 18, 0);
        for (uint32_t i = 0; i < 1024; i++) m[i * 18 + 17] = i + 1;
        VG_TRY(small(m, 1024, 18, &main[5]));
    }
    {   // the chips without rows in the provable instruction subset: one zero row each
        const int ids[5] = {6, 7, 9, 11, 13}; const uint64_t ws[5] = {14, 28, 14, 7, 6};
        for (int k = 0; k < 5; k++) {
            if (ids[k] == 13 && L.n_static) continue;
            std::vector<uint32_t> z(ws[k], 0);
            VG_TRY(small(z, 1, ws[k], &main[ids[k]]));
        }
    }
    if (L.n_static) {   // 13 static data: (addr, value[4], is_real), ascending address (static_data/src/lib.rs:60-96)
        const uint64_t h = next_pow2(L.n_static);
        std::vector<uint32_t> s(h * 6, 0);
        for (size_t i = 0; i < L.n_static; i++) {
            uint32_t* row = &s[i * 6];
            const uint32_t v = L.static_value[i];
            row[0] = L.static_addr[i]; row[1] = v >> 24; row[2] = (v >> 16) & 0xff; row[3] = (v >> 8) & 0xff; row[4] = v & 0xff; row[5] = 1;
        }
        VG_TRY(small(s, h, 6, &main[13]));
    }
    {   // 12 range: (multiplicity, counter) + preprocessed counter (range/src/lib.rs:32-72)
        std::vector<uint32_t> r(512), p(256);
        for (uint32_t i = 0; i < 256; i++) { r[2 * i] = L.range_count[i]; r[2 * i + 1] = i; p[i] = i; }
        VG_TRY(small(r, 256, 2, &main[12]));
        VG_TRY(small(p, 256, 1, &prep[1]));
    }
    VG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));      // the logs are the caller's (pageable) memory: they may go once this returns
    for (int i = 0; i < VGPU_NUM_CHIPS; i++) main_out[i] = main[i].release();
    for (int i = 0; i < 2; i++) prep_out[i] = prep[i].release();
    return 0;
}

}  // extern "C"
