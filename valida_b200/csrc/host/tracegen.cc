// Host witness generation for BasicMachine: a small Valida VM for the instruction subset the
// reference's proving tests exercise (imm32, add32/sub32 with and without immediates, lt32/lte32/
// slt32/sle32 incl. left immediates, jal, jalv, beq, bne, load32, store32, loadfp, stop) and the Chip::generate_trace of every chip.
// This is the INPUT side of the proving path (SURVEY.md §8a "Chip::generate_trace x14 — kept on
// host, input to the GPU path"); it follows
//   run loop + STOP padding        basic/src/lib.rs:127-145, 1063-1188
//   instruction semantics          cpu/src/lib.rs:437-923, alu_u32/src/add/mod.rs:138-169, sub/mod.rs:126-166
//   CPU rows                       cpu/src/lib.rs:79-97, 163-373
//   memory rows                    memory/src/lib.rs:85-136, 143-194, 237-263
//   add/sub rows                   alu_u32/src/add/mod.rs:38-129, alu_u32/src/sub/mod.rs
//   mul floor (2^10 counter rows)  alu_u32/src/mul/mod.rs:38-64
//   range / program rows           range/src/lib.rs:32-72, program/src/lib.rs:38-81, program/src/stark.rs:22-40
//   static data                    static_data/src/lib.rs:26-79 (chip rows), memory/src/lib.rs:132-135, 163-169, 265-283
//                                  (write_static, the static rows that open the memory trace); basic/src/lib.rs:131
// Output: 14 row-major matrices of canonical BabyBear words in chip order
// (cpu, program, mem, add, sub, mul, div, shift, lt, com, bitwise, output, range, static_data)
// plus the two preprocessed traces.
#include <cstdint>
#include <cstring>
#include <cstdlib>
#include <vector>
#include <algorithm>
#include <string>
#include <memory>
#include <new>
#include <exception>
#include <cstdio>
#include <omp.h>
#include "../../../include/valida_b200.h"
#include "vmlog.h"

namespace {

constexpr uint32_t P = 2013265921u;
inline uint32_t fmul(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) % P); }
inline uint32_t fpow(uint32_t a, uint32_t e) { uint32_t r = 1; while (e) { if (e & 1) r = fmul(r, a); a = fmul(a, a); e >>= 1; } return r; }
inline uint32_t from_i32(int32_t x) { return x < 0 ? (P - (uint32_t)(-(int64_t)x) % P) % P : (uint32_t)x % P; }
inline size_t next_pow2(size_t n) { size_t p = 1; while (p < n) p <<= 1; return p; }

enum : uint32_t { OP_LOAD32 = 1, OP_STORE32 = 2, OP_JAL = 3, OP_JALV = 4, OP_BEQ = 5, OP_BNE = 6, OP_IMM32 = 7, OP_STOP = 8, OP_LOADFP = 10,
                  OP_ADD32 = 100, OP_SUB32 = 101, OP_LT32 = 104, OP_AND32 = 107, OP_OR32 = 108, OP_XOR32 = 109, OP_LTE32 = 115, OP_SLT32 = 117, OP_SLE32 = 118 };
using CpuOp = uint8_t;
enum : uint8_t { K_STORE32 = VG_K_STORE32, K_LOAD32 = VG_K_LOAD32, K_JAL = VG_K_JAL, K_JALV = VG_K_JALV, K_BEQ = VG_K_BEQ, K_BNE = VG_K_BNE, K_IMM32 = VG_K_IMM32,
                 K_BUS = VG_K_BUS, K_STOP = VG_K_STOP, K_LOADFP = VG_K_LOADFP, K_BUS_LEFT_IMM = VG_K_BUS_LEFT_IMM };

// log records: the layouts of host/vmlog.h (the device witness builder reads the same arrays)
using MemOp = VgMemOp;
using CpuRec = VgCpuRec;
using AluRec = VgAluRec;
using LtRec = VgAluOpRec;
using BitRec = VgAluOpRec;

// Append-only log of trivially copyable records.  Growth goes through realloc(), which glibc serves with mremap() for large
// blocks — no copy of the 150 MB memory log at every doubling (std::vector growth cost 0.2-0.3 s of a 0.5 s run loop).
template <class T> struct PodVec {
    T* p = nullptr; size_t n = 0, cap = 0;
    PodVec() = default;
    PodVec(const PodVec&) = delete; PodVec& operator=(const PodVec&) = delete;
    ~PodVec() { std::free(p); }
    void push_back(const T& v) {
        if (n == cap) {
            const size_t nc = cap ? 2 * cap : 4096;
            T* q = (T*)std::realloc(p, nc * sizeof(T));
            if (!q) throw std::bad_alloc();
            p = q; cap = nc;
        }
        p[n++] = v;
    }
    size_t size() const { return n; }
    bool empty() const { return n == 0; }
    const T* data() const { return p; }
    const T& operator[](size_t i) const { return p[i]; }
    const T* begin() const { return p; }
    const T* end() const { return p + n; }
};

// Memory cells of the VM: open addressing, linear probing, power-of-two table (the interpreter touches it two or three
// times per cycle; std::unordered_map made that the slowest part of the run loop).
struct CellMap {
    std::vector<uint32_t> keys, vals;
    std::vector<uint8_t> used;
    size_t count = 0, mask = 0;
    CellMap() { rehash(1 << 12); }
    static size_t slot_of(uint32_t k, size_t mask) { return (size_t)((k * 0x9E3779B1u) >> 7) & mask; }
    void rehash(size_t cap) {
        std::vector<uint32_t> ok(std::move(keys)), ov(std::move(vals));
        std::vector<uint8_t> ou(std::move(used));
        keys.assign(cap, 0); vals.assign(cap, 0); used.assign(cap, 0); mask = cap - 1; count = 0;
        for (size_t i = 0; i < ou.size(); i++) if (ou[i]) set(ok[i], ov[i]);
    }
    bool get(uint32_t k, uint32_t* v) const {
        for (size_t i = slot_of(k, mask);; i = (i + 1) & mask) {
            if (!used[i]) return false;
            if (keys[i] == k) { *v = vals[i]; return true; }
        }
    }
    void set(uint32_t k, uint32_t v) {
        if (2 * (count + 1) > mask + 1) rehash(2 * (mask + 1));
        for (size_t i = slot_of(k, mask);; i = (i + 1) & mask) {
            if (!used[i]) { used[i] = 1; keys[i] = k; vals[i] = v; count++; return; }
            if (keys[i] == k) { vals[i] = v; return; }
        }
    }
};

// Trace storage: zero-filled by all host threads (a 2^24 x 14 matrix is 0.9 GB; a single-threaded std::vector::assign
// spends longer faulting its pages in than the row loop spends filling them).
struct Buf {
    uint32_t* p = nullptr; size_t n = 0;
    Buf() = default;
    Buf(const Buf&) = delete; Buf& operator=(const Buf&) = delete;
    ~Buf() { std::free(p); }
    uint32_t* alloc(size_t count) {                      // uninitialised
        std::free(p);
        n = count;
        p = (uint32_t*)std::malloc((count ? count : 1) * sizeof(uint32_t));
        if (!p) { n = 0; throw std::bad_alloc(); }         // caught at the C boundary (vgpu_machine_run_static)
        return p;
    }
    void clear_range(size_t begin, size_t end) {         // words [begin, end), all host threads
        if (end <= begin) return;
        const size_t count = end - begin;
        const long chunks = (long)((count + (1 << 18) - 1) >> 18);
#pragma omp parallel for schedule(static)
        for (long c = 0; c < chunks; c++) {
            const size_t b = begin + ((size_t)c << 18), e = std::min(end, b + ((size_t)1 << 18));
            std::memset(p + b, 0, (e - b) * sizeof(uint32_t));
        }
    }
    uint32_t* zeros(size_t count) { alloc(count); clear_range(0, count); return p; }
    uint32_t* data() { return p; }
    uint32_t& operator[](size_t i) { return p[i]; }
};

struct Vm {
    const int32_t* prog; size_t n_instr;
    uint32_t pc = 0, fp = 0, clock = 0;
    CellMap cells;
    std::vector<std::pair<uint32_t, uint32_t>> static_cells;   // (addr, value), ascending addr (the reference keeps a BTreeMap)
    PodVec<MemOp> mem_ops;
    PodVec<CpuRec> cpu;
    PodVec<AluRec> adds, subs;
    PodVec<LtRec> lts;
    PodVec<BitRec> bits;
    std::vector<uint32_t> prog_counts;
    uint32_t range_count[256] = {0};
    std::string err;

    bool read(uint32_t addr, uint32_t& v) {
        if (!cells.get(addr, &v)) { err = "memory chip: read before write at " + std::to_string(addr) + " (pc=" + std::to_string(pc) + ")"; return false; }
        mem_ops.push_back({clock, addr, v, 0u});
        return true;
    }
    void write(uint32_t addr, uint32_t v) { mem_ops.push_back({clock, addr, v, 1u}); cells.set(addr, v); }
    void range_check(uint32_t w) { for (int i = 0; i < 4; i++) range_count[(w >> (8 * i)) & 0xff]++; }
    size_t cycle_mem0 = 0;      // first memory operation of the cycle being executed
    void push(CpuOp kind, uint32_t instr_pc, uint32_t pc_before, uint32_t fp_before, bool has_imm = false, uint32_t imm = 0) {
        cpu.push_back({pc_before, fp_before, instr_pc, imm, (uint32_t)cycle_mem0, kind, (uint8_t)(has_imm ? 1 : 0), {0, 0}});
        cycle_mem0 = mem_ops.size();
        clock++;
    }
    // returns 1 when STOP executed, 0 otherwise, -1 on error
    int step() {
        if (pc >= n_instr) { err = "pc out of range"; return -1; }
        const int32_t* w = prog + 6 * (size_t)pc;
        uint32_t opcode = (uint32_t)w[0];
        int32_t a = w[1], b = w[2], c = w[3], d = w[4], e = w[5];
        uint32_t pc0 = pc, fp0 = fp;
        auto at = [&](int32_t off) { return (uint32_t)((int32_t)fp0 + off); };
        switch (opcode) {
            case OP_IMM32: {
                uint32_t v = ((uint32_t)(uint8_t)b << 24) | ((uint32_t)(uint8_t)c << 16) | ((uint32_t)(uint8_t)d << 8) | (uint32_t)(uint8_t)e;
                write(at(a), v); pc++; push(K_IMM32, pc0, pc0, fp0); break; }
            case OP_ADD32: case OP_SUB32: {
                uint32_t bv, cv; bool imm = (e == 1);
                if (!read(at(b), bv)) return -1;
                if (imm) cv = (uint32_t)c; else if (!read(at(c), cv)) return -1;
                uint32_t av = opcode == OP_ADD32 ? bv + cv : bv - cv;
                write(at(a), av);
                (opcode == OP_ADD32 ? adds : subs).push_back({av, bv, cv});
                pc++; push(K_BUS, pc0, pc0, fp0, imm, cv);
                range_check(av); break; }
            case OP_AND32: case OP_OR32: case OP_XOR32: {
                // alu_u32/src/bitwise/mod.rs:150-262: read b, read c or take it as the immediate, no range check
                uint32_t bv, cv; bool imm = (e == 1);
                if (!read(at(b), bv)) return -1;
                if (imm) cv = (uint32_t)c; else if (!read(at(c), cv)) return -1;
                uint32_t av = opcode == OP_AND32 ? (bv & cv) : opcode == OP_OR32 ? (bv | cv) : (bv ^ cv);
                write(at(a), av);
                bits.push_back({av, bv, cv, opcode});
                pc++; push(K_BUS, pc0, pc0, fp0, imm, cv); break; }
            case OP_LT32: case OP_LTE32: case OP_SLT32: case OP_SLE32: {
                // alu_u32/src/lt/mod.rs:162-205 (execute_with_closure): d == 1 -> left operand is the immediate b;
                // e == 1 -> right operand is the immediate c (and `imm` then holds c, as in the reference)
                uint32_t s1, s2; bool limm = (d == 1), rimm = (e == 1);
                uint32_t immv = 0; bool has_imm = false;
                if (limm) { s1 = (uint32_t)b; immv = s1; has_imm = true; } else if (!read(at(b), s1)) return -1;
                if (rimm) { s2 = (uint32_t)c; immv = s2; has_imm = true; } else if (!read(at(c), s2)) return -1;
                bool r;
                if (opcode == OP_LT32) r = s1 < s2; else if (opcode == OP_LTE32) r = s1 <= s2;
                else if (opcode == OP_SLT32) r = (int32_t)s1 < (int32_t)s2; else r = (int32_t)s1 <= (int32_t)s2;
                write(at(a), r ? 1u : 0u);
                lts.push_back({r ? 1u : 0u, s1, s2, opcode});
                pc++; push(limm ? K_BUS_LEFT_IMM : K_BUS, pc0, pc0, fp0, has_imm, immv); break; }
            case OP_JAL: {
                write(at(a), 24u * (pc0 + 1)); pc = (uint32_t)b / 24u; fp = at(c); push(K_JAL, pc0, pc0, fp0); break; }
            case OP_JALV: {
                write(at(a), 24u * (pc0 + 1));
                uint32_t t, off;
                if (!read(at(b), t)) return -1;
                pc = t / 24u;
                if (!read(at(c), off)) return -1;
                fp = (uint32_t)((int32_t)fp0 + (int32_t)off);
                push(K_JALV, pc0, pc0, fp0); break; }
            case OP_BEQ: case OP_BNE: {
                uint32_t v1, v2; bool imm = (e == 1);
                if (!read(at(b), v1)) return -1;
                if (imm) v2 = (uint32_t)c; else if (!read(at(c), v2)) return -1;
                bool take = (opcode == OP_BEQ) ? (v1 == v2) : (v1 != v2);
                pc = take ? (uint32_t)a / 24u : pc0 + 1;
                push(opcode == OP_BEQ ? K_BEQ : K_BNE, pc0, pc0, fp0, imm, v2); break; }
            case OP_LOADFP: { write(at(a), at(b)); pc++; push(K_LOADFP, pc0, pc0, fp0); break; }
            case OP_LOAD32: {
                uint32_t p, cell;
                if (!read(at(c), p)) return -1;
                if (!read(p, cell)) return -1;
                write(at(a), cell); pc++; push(K_LOAD32, pc0, pc0, fp0); break; }
            case OP_STORE32: {
                uint32_t waddr, cell;
                if (!read(at(b), waddr)) return -1;
                if (!read(at(c), cell)) return -1;
                write(waddr, cell); pc++; push(K_STORE32, pc0, pc0, fp0); break; }
            case OP_STOP: { push(K_STOP, pc0, pc0, fp0); break; }
            default: err = "unsupported opcode " + std::to_string(opcode) + " at pc " + std::to_string(pc0); return -1;
        }
        prog_counts[pc0]++;
        return opcode == OP_STOP ? 1 : 0;
    }
};

struct Traces {
    vgpu_matrix main[14];
    vgpu_matrix prep[2];
    Buf store[16];
    uint32_t clock = 0, n_mem_ops = 0, n_add_ops = 0, n_sub_ops = 0;
    CellMap cells;
};

inline void word_be(uint32_t v, uint32_t* out) { out[0] = v >> 24; out[1] = (v >> 16) & 0xff; out[2] = (v >> 8) & 0xff; out[3] = v & 0xff; }

void build_cpu(const Vm& vm, Traces& t) {
    constexpr size_t W = 51;
    size_t n = vm.cpu.size(), h = next_pow2(n);
    Buf& v = t.store[0];
    v.zeros(h * W);
    // the memory operations of a cycle are contiguous in vm.mem_ops: [cpu[i].mem0, cpu[i + 1].mem0)
    auto first_of = [&](size_t i) { return i < n ? (size_t)vm.cpu[i].mem0 : vm.mem_ops.size(); };
    std::vector<uint32_t> diff(n, 0);
#pragma omp parallel for schedule(static)
    for (long i = 0; i < (long)n; i++) {
        const CpuRec& r = vm.cpu[i];
        uint32_t* row = &v[(size_t)i * W];
        const int32_t* w = vm.prog + 6 * (size_t)r.instr;
        row[0] = (uint32_t)i; row[1] = r.pc; row[2] = r.fp % P;      // from_canonical_u32 (cpu/src/lib.rs:171-172) reduces mod p
        row[3] = (uint32_t)w[0];
        for (int k = 0; k < 5; k++) row[4 + k] = from_i32(w[1 + k]);
        bool left_imm = false;
        switch (r.kind) {
            case K_STORE32: row[16] = 1; break;
            case K_LOAD32: row[13] = 1; break;
            case K_JAL: row[20] = 1; break;
            case K_JALV: row[21] = 1; break;
            case K_BEQ: row[18] = 1; break;
            case K_BNE: row[19] = 1; break;
            case K_IMM32: row[22] = 1; break;
            case K_BUS: row[9] = 1; break;
            case K_STOP: row[24] = 1; break;
            case K_LOADFP: row[25] = 1; break;
            case K_BUS_LEFT_IMM: row[9] = 1; break;
        }
        if (r.has_imm && r.kind == K_BUS_LEFT_IMM) {  // set_left_imm_value (cpu/src/lib.rs:364-371)
            row[12] = 1; left_imm = true;
            word_be(r.imm, &row[29 + 3]);
            row[5] = r.imm % P;
        } else if (r.has_imm) {  // set_imm_value (cpu/src/lib.rs:355-362)
            row[11] = 1;
            word_be(r.imm, &row[36 + 3]);
            row[6] = r.imm % P;
        }
        row[29 + 1] = 1; row[36 + 1] = 1; row[43 + 1] = 0;
        bool first_read = true;
        for (size_t k = first_of(i), ke = first_of(i + 1); k < ke; k++) {
            const MemOp& m = vm.mem_ops[k];
            uint32_t ch;
            if (m.is_write) ch = 43;
            else if (first_read && !left_imm) { ch = 29; first_read = false; }
            else ch = 36;
            row[ch] = 1; row[ch + 2] = m.addr % P; word_be(m.value, &row[ch + 3]);     // cpu/src/lib.rs:263-276
        }
        uint64_t dsum = 0;
        for (int k = 0; k < 4; k++) { int64_t dd = (int64_t)row[32 + k] - (int64_t)row[39 + k]; dsum += (uint64_t)(dd * dd); }
        diff[i] = (uint32_t)(dsum % P);
    }
    // diff_inv through a table over the possible values (diff <= 4*255^2): mark, invert the marked entries, fill
    {
        constexpr uint32_t DMAX = 4 * 255 * 255;
        std::vector<uint32_t> invs(DMAX + 1, 0);
        std::vector<uint8_t> seen(DMAX + 1, 0);
#pragma omp parallel for schedule(static)
        for (long i = 0; i < (long)n; i++) if (diff[i]) seen[diff[i]] = 1;     // benign race: every writer stores 1
#pragma omp parallel for schedule(dynamic, 1024)
        for (long d = 1; d <= (long)DMAX; d++) if (seen[d]) invs[d] = fpow((uint32_t)d, P - 2);
#pragma omp parallel for schedule(static)
        for (long i = 0; i < (long)n; i++) {
            uint32_t* row = &v[(size_t)i * W];
            row[26] = diff[i];
            if (diff[i]) { row[27] = invs[diff[i]]; row[28] = 1; }
        }
    }
    // pad_to_power_of_two (cpu/src/lib.rs:318-353)
    if (n) {
        const uint32_t* last = &v[(n - 1) * W];
        uint32_t pc = last[1], fp = last[2], clk = last[0];        // fp already reduced
#pragma omp parallel for schedule(static)
        for (long i = (long)n; i < (long)h; i++) {
            uint32_t* row = &v[(size_t)i * W];
            row[1] = pc; row[2] = fp; row[0] = clk + (uint32_t)(i - n) + 1;
            row[24] = 1; row[3] = OP_STOP;
            row[29 + 1] = 1; row[36 + 1] = 1;
        }
    }
    t.main[0] = {v.data(), h, W};
}

// Stable sort of the memory log by address (memory/src/lib.rs:158 sorts by (addr, clk); the log is already in clk order, so a
// STABLE sort on the address alone gives the same order).  LSD radix, 11 bits per pass, passes whose digit is the same for
// every key are skipped; per-thread histograms over contiguous chunks keep each pass stable.
// Returns the sorted log (a fresh array, or `in` itself when no pass was needed); `hold` owns whatever was allocated.
const MemOp* sort_by_addr(const PodVec<MemOp>& in, std::unique_ptr<MemOp[]> hold[2]) {
    const size_t n = in.size();
    if (n < 2) return in.data();
    uint32_t all_or = 0, all_and = 0xffffffffu;
#pragma omp parallel for schedule(static) reduction(|: all_or) reduction(&: all_and)
    for (long i = 0; i < (long)n; i++) { all_or |= in[i].addr; all_and &= in[i].addr; }
    const uint32_t varying = all_or ^ all_and;
    constexpr int BITS = 11, BUCKETS = 1 << BITS;
    const int T = std::max(1, omp_get_max_threads());
    std::vector<size_t> hist((size_t)T * BUCKETS);
    const MemOp* src = in.data();
    int next = 0;
    for (int shift = 0; shift < 32; shift += BITS) {
        if (((varying >> shift) & (BUCKETS - 1)) == 0) continue;
        if (!hold[next]) hold[next].reset(new MemOp[n]);       // default-initialised: no serial zero fill of 16 n bytes
        MemOp* dst = hold[next].get();
        std::fill(hist.begin(), hist.end(), 0);
#pragma omp parallel num_threads(T)
        {
            const int tid = omp_get_thread_num(), nt = omp_get_num_threads();
            const size_t b = n * (size_t)tid / nt, e = n * (size_t)(tid + 1) / nt;
            size_t* h = &hist[(size_t)tid * BUCKETS];
            for (size_t i = b; i < e; i++) h[(src[i].addr >> shift) & (BUCKETS - 1)]++;
#pragma omp barrier
#pragma omp single
            {
                size_t run = 0;
                for (int d = 0; d < BUCKETS; d++)
                    for (int k = 0; k < nt; k++) { size_t c = hist[(size_t)k * BUCKETS + d]; hist[(size_t)k * BUCKETS + d] = run; run += c; }
            }
            for (size_t i = b; i < e; i++) dst[h[(src[i].addr >> shift) & (BUCKETS - 1)]++] = src[i];
        }
        src = dst;
        next ^= 1;
    }
    return src;
}

void build_mem(const Vm& vm, Traces& t) {
    constexpr size_t W = 14;
    std::unique_ptr<MemOp[]> hold[2];
    const MemOp* ops = sort_by_addr(vm.mem_ops, hold);
    // the static cells open the trace (memory/src/lib.rs:163-169): is_static_initial = 1, clk = 0, is_write = 1, counter = n
    const size_t n0 = vm.static_cells.size();
    size_t n = vm.mem_ops.size(), h = next_pow2(n0 + n);
    Buf& v = t.store[2];
    v.alloc(h * W);
    for (size_t i = 0; i < n0; i++) {
        uint32_t* row = &v[i * W];
        std::memset(row, 0, W * sizeof(uint32_t));
        row[0] = vm.static_cells[i].first % P; word_be(vm.static_cells[i].second, &row[1]);     // memory/src/lib.rs:276
        row[6] = 1; row[8] = 1; row[12] = (uint32_t)i;
    }
    // every word of the n operation rows is written here and the padding rows are cleared below: no zero fill of the
    // whole 0.9 GB matrix first
#pragma omp parallel for schedule(static)
    for (long i = 0; i < (long)n; i++) {
        uint32_t* row = &v[(n0 + (size_t)i) * W];
        row[0] = ops[i].addr % P; word_be(ops[i].value, &row[1]);      // sorted by the u32 address, stored reduced (memory/src/lib.rs:247-262)
        row[5] = ops[i].clk; row[6] = 0;
        row[7] = ops[i].is_write ? 0 : 1; row[8] = ops[i].is_write ? 1 : 0;
        row[9] = 0; row[10] = 0; row[11] = 0;
        row[12] = (uint32_t)(n0 + (size_t)i); row[13] = 0;
    }
    v.clear_range((n0 + n) * W, h * W);
    t.main[2] = {v.data(), h, W};
}

void build_addsub(const PodVec<AluRec>& ops, bool is_add, Buf& v, vgpu_matrix& out) {
    constexpr size_t W = 16;
    size_t n = ops.size(), h = next_pow2(n);
    v.zeros(h * W);
#pragma omp parallel for schedule(static)
    for (long i = 0; i < (long)n; i++) {
        uint32_t* row = &v[(size_t)i * W];
        uint32_t a[4], b[4], c[4];
        word_be(ops[i].a, a); word_be(ops[i].b, b); word_be(ops[i].c, c);
        std::memcpy(row + 0, b, 16); std::memcpy(row + 4, c, 16); std::memcpy(row + 11, a, 16);
        if (is_add) {
            uint32_t c1 = (b[3] + c[3] > 255), c2 = (b[2] + c[2] + c1 > 255), c3 = (b[1] + c[1] + c2 > 255);
            row[8] = c1; row[9] = c2; row[10] = c3;
        } else {  // alu_u32/src/sub/mod.rs op_to_row
            // exactly as the reference (no borrow propagation into the comparison): sub/mod.rs:103-111
            uint32_t b1 = (b[3] < c[3]), b2 = (b[2] < c[2]), b3 = (b[1] < c[1]);
            row[8] = b1; row[9] = b2; row[10] = b3;
        }
        row[15] = 1;
    }
    out = {v.data(), h, W};
}

// Lt32Chip::op_to_row / set_cols (alu_u32/src/lt/mod.rs:86-160)
void build_lt(const PodVec<LtRec>& ops, Buf& v, vgpu_matrix& out) {
    constexpr size_t W = 45;
    size_t n = ops.size(), h = next_pow2(n);
    v.zeros(h * W);
#pragma omp parallel for schedule(static)
    for (long i = 0; i < (long)n; i++) {
        uint32_t* row = &v[(size_t)i * W];
        uint32_t a[4], b[4], c[4];
        word_be(ops[i].a, a); word_be(ops[i].b, b); word_be(ops[i].c, c);
        std::memcpy(row + 0, b, 16); std::memcpy(row + 4, c, 16);
        row[21] = a[3];
        bool is_signed = ops[i].opcode == OP_SLT32 || ops[i].opcode == OP_SLE32;
        row[ops[i].opcode == OP_LT32 ? 23 : ops[i].opcode == OP_LTE32 ? 24 : ops[i].opcode == OP_SLT32 ? 25 : 26] = 1;
        for (int k = 0; k < 4; k++) {
            if (b[k] != c[k]) {
                uint32_t z = 256u + b[k] - c[k];
                for (int bit = 0; bit < 9; bit++) row[12 + bit] = (z >> bit) & 1;
                row[8 + k] = 1;
                uint32_t diff = (b[k] + P - c[k]) % P;
                row[27] = fpow(diff, P - 2);
                break;
            }
        }
        for (int bit = 0; bit < 8; bit++) { row[28 + bit] = (b[0] >> bit) & 1; row[36 + bit] = (c[0] >> bit) & 1; }
        row[44] = (is_signed && row[28 + 7] != row[36 + 7]) ? 1 : 0;
        row[22] = 1;
    }
    out = {v.data(), h, W};
}

// Bitwise32Chip::op_to_row / set_cols (alu_u32/src/bitwise/mod.rs:84-131): input_1 0..3, input_2 4..7,
// bits_1[byte][bit] 8 + 8*byte + bit, bits_2 40 + ..., output 72..75, is_and 76, is_or 77, is_xor 78
void build_bitwise(const PodVec<BitRec>& ops, Buf& v, vgpu_matrix& out) {
    constexpr size_t W = 79;
    size_t n = ops.size(), h = next_pow2(n);
    v.zeros(h * W);
#pragma omp parallel for schedule(static)
    for (long i = 0; i < (long)n; i++) {
        uint32_t* row = &v[(size_t)i * W];
        uint32_t a[4], b[4], c[4];
        word_be(ops[i].a, a); word_be(ops[i].b, b); word_be(ops[i].c, c);
        std::memcpy(row + 0, b, 16); std::memcpy(row + 4, c, 16); std::memcpy(row + 72, a, 16);
        for (int k = 0; k < 4; k++)
            for (int bit = 0; bit < 8; bit++) { row[8 + 8 * k + bit] = (b[k] >> bit) & 1; row[40 + 8 * k + bit] = (c[k] >> bit) & 1; }
        row[ops[i].opcode == OP_AND32 ? 76 : ops[i].opcode == OP_OR32 ? 77 : 78] = 1;
    }
    out = {v.data(), h, W};
}

void zero_chip(Buf& v, vgpu_matrix& out, size_t w) { v.zeros(w); out = {v.data(), 1, w}; }

}  // namespace

struct vgpu_traces { Traces t; };

extern "C" {

// Machine::run: the interpreter loop; what it leaves behind is the input of every Chip::generate_trace
static int vm_run_impl(const int32_t* program_words, uint64_t n_instr, uint32_t initial_pc, uint32_t initial_fp, uint64_t max_cycles,
                       const uint32_t* static_addrs, const uint32_t* static_values, uint64_t n_static, Vm& vm, char* err, uint64_t err_len) {
    vm.prog = program_words; vm.n_instr = n_instr; vm.pc = initial_pc; vm.fp = initial_fp;
    vm.prog_counts.assign(n_instr, 0);
    {   // MachineWithStaticDataChip::initialize_memory (static_data/src/lib.rs:26-30): cells are preloaded, nothing is logged
        std::vector<std::pair<uint32_t, uint32_t>> sc;
        for (uint64_t i = 0; i < n_static; i++) sc.push_back({static_addrs[i], static_values[i]});
        std::stable_sort(sc.begin(), sc.end(), [](const std::pair<uint32_t, uint32_t>& x, const std::pair<uint32_t, uint32_t>& y) { return x.first < y.first; });
        for (auto& c : sc) {            // a repeated address keeps the LAST value, as BTreeMap::insert does
            if (!vm.static_cells.empty() && vm.static_cells.back().first == c.first) vm.static_cells.back().second = c.second;
            else vm.static_cells.push_back(c);
        }
        for (auto& c : vm.static_cells) vm.cells.set(c.first, c.second);
    }
    int rc = 0;
    while ((rc = vm.step()) == 0) {
        if (vm.clock >= max_cycles) { vm.err = "cycle limit reached"; rc = -1; break; }
    }
    if (rc < 0) { if (err && err_len) { std::strncpy(err, vm.err.c_str(), err_len - 1); err[err_len - 1] = 0; } return -1; }
    // STOP padding reads the program word at the final pc (basic/src/lib.rs:140-144)
    size_t padded = next_pow2(vm.clock);
    vm.prog_counts[vm.pc] += (uint32_t)(padded - vm.clock);
    return 0;
}

// Chip::generate_trace x14 on the host
static vgpu_traces* build_traces_host(Vm& vm) {
    const int32_t* program_words = vm.prog;
    const uint64_t n_instr = vm.n_instr;
    std::unique_ptr<vgpu_traces> tr(new vgpu_traces());      // released to the caller at the end; freed if an allocation below throws
    Traces& t = tr->t;
    t.clock = vm.clock; t.n_mem_ops = (uint32_t)vm.mem_ops.size(); t.n_add_ops = (uint32_t)vm.adds.size(); t.n_sub_ops = (uint32_t)vm.subs.size();
    build_cpu(vm, t);
    build_mem(vm, t);
    {  // program: 1 main column (counts) + 7 preprocessed
        size_t h = next_pow2(n_instr);
        t.store[1].zeros(h);
        for (size_t i = 0; i < n_instr; i++) t.store[1][i] = vm.prog_counts[i];
        t.main[1] = {t.store[1].data(), h, 1};
        t.store[14].zeros(h * 7);
        for (size_t i = 0; i < h; i++) {
            uint32_t* row = &t.store[14][i * 7];
            row[0] = (uint32_t)i;
            // every row of the program, executed or not: InstructionWord::flatten takes the opcode from_canonical_u32 (machine/src/program.rs:44)
            if (i < n_instr) { row[1] = (uint32_t)program_words[6 * i] % P; for (int k = 0; k < 5; k++) row[2 + k] = from_i32(program_words[6 * i + 1 + k]); }
        }
        t.prep[0] = {t.store[14].data(), h, 7};
    }
    build_addsub(vm.adds, true, t.store[3], t.main[3]);
    build_addsub(vm.subs, false, t.store[4], t.main[4]);
    {  // mul: 2^10 counter rows
        t.store[5].zeros(1024 * 18);
        for (size_t i = 0; i < 1024; i++) t.store[5][i * 18 + 17] = (uint32_t)i + 1;
        t.main[5] = {t.store[5].data(), 1024, 18};
    }
    zero_chip(t.store[6], t.main[6], 14);   // div
    zero_chip(t.store[7], t.main[7], 28);   // shift
    build_lt(vm.lts, t.store[8], t.main[8]);   // lt
    zero_chip(t.store[9], t.main[9], 14);   // com
    build_bitwise(vm.bits, t.store[10], t.main[10]);   // bitwise
    zero_chip(t.store[11], t.main[11], 7);  // output
    {  // range: (mult, counter) + preprocessed counter
        t.store[12].zeros(256 * 2); t.store[15].zeros(256);
        for (uint32_t i = 0; i < 256; i++) { t.store[12][i * 2] = vm.range_count[i]; t.store[12][i * 2 + 1] = i; t.store[15][i] = i; }
        t.main[12] = {t.store[12].data(), 256, 2};
        t.prep[1] = {t.store[15].data(), 256, 1};
    }
    {   // static_data: (addr, value[4], is_real) per cell in address order, padded to a power of two (one zero row when empty)
        const size_t n0 = vm.static_cells.size(), h = next_pow2(n0 ? n0 : 1);
        t.store[13].zeros(h * 6);
        for (size_t i = 0; i < n0; i++) {
            uint32_t* row = &t.store[13][i * 6];
            row[0] = vm.static_cells[i].first % P; word_be(vm.static_cells[i].second, &row[1]); row[5] = 1;    // static_data/src/lib.rs:67
        }
        t.main[13] = {t.store[13].data(), h, 6};
    }
    t.cells = vm.cells;
    return tr.release();
}

static int machine_run_impl(const int32_t* program_words, uint64_t n_instr, uint32_t initial_pc, uint32_t initial_fp, uint64_t max_cycles,
                            const uint32_t* static_addrs, const uint32_t* static_values, uint64_t n_static,
                            vgpu_traces** out, char* err, uint64_t err_len) {
    Vm vm;
    if (vm_run_impl(program_words, n_instr, initial_pc, initial_fp, max_cycles, static_addrs, static_values, n_static, vm, err, err_len) != 0) return -1;
    *out = build_traces_host(vm);
    return 0;
}

// ---- the interpreter's logs as an object: Machine::run without the row fill (the device builds the rows, witness.cu) ----
}  // extern "C"
struct vgpu_vmlog { Vm vm; std::vector<int32_t> program; std::vector<uint32_t> st_addr, st_val; VgVmLogs view; };
extern "C" {

int32_t vgpu_vm_run(const int32_t* program_words, uint64_t n_instr, uint32_t initial_pc, uint32_t initial_fp, uint64_t max_cycles,
                    const uint32_t* static_addrs, const uint32_t* static_values, uint64_t n_static, vgpu_vmlog** out, char* err, uint64_t err_len) {
    try {
        std::unique_ptr<vgpu_vmlog> L(new vgpu_vmlog());
        L->program.assign(program_words, program_words + 6 * n_instr);
        if (vm_run_impl(L->program.data(), n_instr, initial_pc, initial_fp, max_cycles, static_addrs, static_values, n_static, L->vm, err, err_len) != 0) return -1;
        Vm& vm = L->vm;
        for (auto& c : vm.static_cells) { L->st_addr.push_back(c.first); L->st_val.push_back(c.second); }
        VgVmLogs& v = L->view;
        v.program = L->program.data(); v.n_instr = n_instr;
        v.cpu = vm.cpu.data(); v.n_cpu = vm.cpu.size();
        v.mem = vm.mem_ops.data(); v.n_mem = vm.mem_ops.size();
        v.adds = vm.adds.data(); v.n_adds = vm.adds.size();
        v.subs = vm.subs.data(); v.n_subs = vm.subs.size();
        v.lts = vm.lts.data(); v.n_lts = vm.lts.size();
        v.bits = vm.bits.data(); v.n_bits = vm.bits.size();
        v.prog_counts = vm.prog_counts.data(); v.range_count = vm.range_count;
        v.static_addr = L->st_addr.data(); v.static_value = L->st_val.data(); v.n_static = L->st_addr.size();
        *out = L.release();
        return 0;
    } catch (const std::exception& e) {
        if (err && err_len) { std::snprintf(err, err_len, "interpreter run failed: %s", e.what()); }
        return -1;
    }
}
const VgVmLogs* vg_vmlog_view(const vgpu_vmlog* l) { return &l->view; }
void vgpu_vmlog_stats(const vgpu_vmlog* l, uint32_t* clock, uint32_t* mem_ops, uint32_t* add_ops) {
    *clock = l->vm.clock; *mem_ops = (uint32_t)l->vm.mem_ops.size(); *add_ops = (uint32_t)l->vm.adds.size();
}
// Chip::generate_trace x14 on the host from the same logs (the reference witness the device builder is compared with)
int32_t vgpu_vmlog_traces(vgpu_vmlog* l, vgpu_traces** out, char* err, uint64_t err_len) {
    try { *out = build_traces_host(l->vm); return 0; }
    catch (const std::exception& e) { if (err && err_len) std::snprintf(err, err_len, "host witness generation failed: %s", e.what()); return -1; }
}
void vgpu_vmlog_free(vgpu_vmlog* l) { delete l; }


int vgpu_machine_run_static(const int32_t* program_words, uint64_t n_instr, uint32_t initial_pc, uint32_t initial_fp, uint64_t max_cycles,
                          const uint32_t* static_addrs, const uint32_t* static_values, uint64_t n_static,
                          vgpu_traces** out, char* err, uint64_t err_len) {
    try {   // no exception crosses the C boundary: host allocation failures (traces are gigabytes) come back as an error string
        return machine_run_impl(program_words, n_instr, initial_pc, initial_fp, max_cycles, static_addrs, static_values, n_static, out, err, err_len);
    } catch (const std::exception& e) {
        if (err && err_len) { std::snprintf(err, err_len, "host witness generation failed: %s", e.what()); }
        return -1;
    }
}

int vgpu_machine_run(const int32_t* program_words, uint64_t n_instr, uint32_t initial_pc, uint32_t initial_fp, uint64_t max_cycles,
                   vgpu_traces** out, char* err, uint64_t err_len) {
    return vgpu_machine_run_static(program_words, n_instr, initial_pc, initial_fp, max_cycles, nullptr, nullptr, 0, out, err, err_len);
}

const vgpu_matrix* vgpu_traces_main(const vgpu_traces* t, uint32_t chip) { return chip < 14 ? &t->t.main[chip] : nullptr; }
const vgpu_matrix* vgpu_traces_preprocessed(const vgpu_traces* t, uint32_t which) { return which < 2 ? &t->t.prep[which] : nullptr; }
void vgpu_traces_stats(const vgpu_traces* t, uint32_t* clock, uint32_t* mem_ops, uint32_t* add_ops) {
    *clock = t->t.clock; *mem_ops = t->t.n_mem_ops; *add_ops = t->t.n_add_ops;
}
int vgpu_traces_mem_cell(const vgpu_traces* t, uint32_t addr, uint32_t* value) {
    return t->t.cells.get(addr, value) ? 0 : -1;
}
void vgpu_traces_free(vgpu_traces* t) { delete t; }

// fib_program of basic/tests/test_prover.rs:35-188 with `imm32 -8(fp)` carrying n (big-endian bytes).
uint64_t vgpu_fib_program(uint32_t n, int32_t* out_words /* 25*6 */) {
    const int32_t B = 24;
    const int32_t bb0 = 8 * B, bb0_1 = 13 * B, bb0_2 = 15 * B, bb0_3 = 19 * B, bb0_4 = 21 * B;
    const int32_t prog[25][6] = {
        {OP_IMM32, -4, 0, 0, 0, 0},
        {OP_IMM32, -8, (int32_t)(n >> 24), (int32_t)((n >> 16) & 0xff), (int32_t)((n >> 8) & 0xff), (int32_t)(n & 0xff)},
        {OP_ADD32, -16, -8, 0, 0, 1},
        {OP_IMM32, -20, 0, 0, 0, 28},
        {OP_JAL, -28, bb0, -28, 0, 0},
        {OP_ADD32, -12, -24, 0, 0, 1},
        {OP_ADD32, 4, -12, 0, 0, 1},
        {OP_STOP, 0, 0, 0, 0, 0},
        {OP_ADD32, -4, 12, 0, 0, 1},
        {OP_IMM32, -8, 0, 0, 0, 0},
        {OP_IMM32, -12, 0, 0, 0, 1},
        {OP_IMM32, -16, 0, 0, 0, 0},
        {OP_BEQ, bb0_1, 0, 0, 0, 0},
        {OP_BNE, bb0_2, -16, -4, 0, 0},
        {OP_BEQ, bb0_4, 0, 0, 0, 0},
        {OP_ADD32, -20, -8, -12, 0, 0},
        {OP_ADD32, -8, -12, 0, 0, 1},
        {OP_ADD32, -12, -20, 0, 0, 1},
        {OP_BEQ, bb0_3, 0, 0, 0, 0},
        {OP_ADD32, -16, -16, 1, 0, 1},
        {OP_BEQ, bb0_1, 0, 0, 0, 0},
        {OP_ADD32, 4, -8, 0, 0, 1},
        {OP_JALV, -4, 0, 8, 0, 0},
    };
    (void)bb0_3;
    std::memcpy(out_words, prog, sizeof(int32_t) * 23 * 6);
    return 23;
}

}  // extern "C"
