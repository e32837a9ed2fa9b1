// Host witness generation for BasicMachine: a small Valida VM for the instruction subset the
// reference's proving tests exercise (imm32, add32/sub32 with and without immediates, lt32/lte32/
// slt32/sle32 incl. left immediates, jal, jalv, beq, bne, load32, store32, loadfp, stop) and the Chip::generate_trace of every chip.
// This is the INPUT side of the proving path (SURVEY.md §8a "Chip::generate_trace x14 — kept on
// host, input to the GPU path"); it follows
//   run loop + STOP padding        basic/src/lib.rs:127-145, 1063-1188
//   instruction semantics          cpu/src/lib.rs:437-923, alu_u32/src/add/mod.rs:138-169, sub/mod.rs:126-166
//   mul floor (2^10 counter rows)  alu_u32/src/mul/mod.rs:38-64
//   range / program rows           range/src/lib.rs:32-72, program/src/lib.rs:38-81, program/src/stark.rs:22-40
//   static data                    static_data/src/lib.rs:26-79 (chip rows), memory/src/lib.rs:132-135, 163-169, 265-283
//                                  (write_static, the static rows that open the memory trace); basic/src/lib.rs:131
// The builders read the interpreter's logs through VgVmLogs (vmlog.h), the view the device builder (witness.cu) reads too.  The
// rows of the tall chips (cpu, memory, add, sub, lt, bitwise) come from the row functions of chip_rows.cuh, which the device
// builder calls as well; the short chips come from vg_short_chip_traces, whose matrices the device builder uploads.
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
#include "../chip_rows.cuh"

namespace {

using bb::P;
inline uint32_t fmul(uint32_t a, uint32_t b) { return (uint32_t)(((uint64_t)a * b) % P); }
inline uint32_t fpow(uint32_t a, uint32_t e) { uint32_t r = 1; while (e) { if (e & 1) r = fmul(r, a); a = fmul(a, a); e >>= 1; } return r; }

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
    std::vector<uint32_t> static_addr, static_value;           // ascending addr (the reference keeps a BTreeMap)
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
    // the logs of the run as the view both witness builders read
    VgVmLogs logs() const {
        VgVmLogs v;
        v.program = prog; v.n_instr = n_instr;
        v.cpu = cpu.data(); v.n_cpu = cpu.size();
        v.mem = mem_ops.data(); v.n_mem = mem_ops.size();
        v.adds = adds.data(); v.n_adds = adds.size();
        v.subs = subs.data(); v.n_subs = subs.size();
        v.lts = lts.data(); v.n_lts = lts.size();
        v.bits = bits.data(); v.n_bits = bits.size();
        v.prog_counts = prog_counts.data(); v.range_count = range_count;
        v.static_addr = static_addr.data(); v.static_value = static_value.data(); v.n_static = static_addr.size();
        return v;
    }
};

struct Traces {
    vgpu_matrix main[14];
    vgpu_matrix prep[2];
    Buf store[16];
    uint32_t clock = 0, n_mem_ops = 0, n_add_ops = 0, n_sub_ops = 0;
    CellMap cells;
};

void build_cpu(const VgVmLogs& L, Traces& t) {
    constexpr size_t W = CPU_COLS;
    const size_t n = L.n_cpu, h = next_pow2(n);       // n >= 1: a run ends with STOP
    Buf& v = t.store[0];
    v.alloc(h * W);                                   // every row is written below: the n cycles, then the STOP padding
    std::vector<uint32_t> diff(n);
#pragma omp parallel for schedule(static)
    for (long i = 0; i < (long)n; i++) {
        const CpuRec& r = L.cpu[i];
        // the memory operations of a cycle are contiguous in the log: [cpu[i].mem0, cpu[i + 1].mem0)
        const size_t k1 = (size_t)i + 1 < n ? L.cpu[i + 1].mem0 : L.n_mem;
        diff[i] = cpu_row(&v[(size_t)i * W], i, r, L.program + 6 * (size_t)r.instr, L.mem + r.mem0, k1 - r.mem0);
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
        for (long i = 0; i < (long)n; i++) if (diff[i]) v[(size_t)i * W + 27] = invs[diff[i]];
    }
#pragma omp parallel for schedule(static)
    for (long i = (long)n; i < (long)h; i++) cpu_pad_row(&v[(size_t)i * W], i, L.cpu[n - 1]);
    t.main[0] = {v.data(), h, W};
}

// Stable sort of the memory log by address (memory/src/lib.rs:158 sorts by (addr, clk); the log is already in clk order, so a
// STABLE sort on the address alone gives the same order).  LSD radix, 11 bits per pass, passes whose digit is the same for
// every key are skipped; per-thread histograms over contiguous chunks keep each pass stable.
// Returns the sorted log (a fresh array, or `in` itself when no pass was needed); `hold` owns whatever was allocated.
const MemOp* sort_by_addr(const MemOp* in, size_t n, std::unique_ptr<MemOp[]> hold[2]) {
    if (n < 2) return in;
    uint32_t all_or = 0, all_and = 0xffffffffu;
#pragma omp parallel for schedule(static) reduction(|: all_or) reduction(&: all_and)
    for (long i = 0; i < (long)n; i++) { all_or |= in[i].addr; all_and &= in[i].addr; }
    const uint32_t varying = all_or ^ all_and;
    constexpr int BITS = 11, BUCKETS = 1 << BITS;
    const int T = std::max(1, omp_get_max_threads());
    std::vector<size_t> hist((size_t)T * BUCKETS);
    const MemOp* src = in;
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

// The n x W rows fill(row, i) writes, zero rows up to a power of two: every word of the n rows is written by the row function and
// only the padding is cleared (no zero fill of a 0.9 GB matrix first)
template <class Fill> void build_rows(size_t n, size_t W, Buf& v, vgpu_matrix& out, Fill fill) {
    const size_t h = next_pow2(n);
    v.alloc(h * W);
#pragma omp parallel for schedule(static)
    for (long i = 0; i < (long)n; i++) fill(&v[(size_t)i * W], (size_t)i);
    v.clear_range(n * W, h * W);
    out = {v.data(), h, W};
}

void build_mem(const VgVmLogs& L, Traces& t) {
    std::unique_ptr<MemOp[]> hold[2];
    const MemOp* ops = sort_by_addr(L.mem, L.n_mem, hold);
    const size_t n0 = L.n_static;                     // the static cells open the trace
    build_rows(n0 + L.n_mem, MEM_COLS, t.store[2], t.main[2], [&](uint32_t* row, size_t i) {
        if (i < n0) mem_row(row, i, {0u, L.static_addr[i], L.static_value[i], 1u}, true);
        else mem_row(row, i, ops[i - n0], false);
    });
}

}  // namespace

struct vgpu_traces { Traces t; };

// The short chips: a zero-filled h-row trace of chip `id` in store[id], preprocessed trace `which` in store[14 + which]; widths
// from the machine's chip table
vgpu_traces* vg_short_chip_traces(const VgVmLogs& L) {
    std::unique_ptr<vgpu_traces> tr(new vgpu_traces());      // freed if an allocation below throws
    Traces& t = tr->t;
    const auto chip = [&](uint32_t id, size_t h) {
        const size_t w = vgpu_basic_machine_chip(id)->width;
        t.main[id] = {t.store[id].zeros(h * w), h, w};
        return t.store[id].data();
    };
    const auto prep = [&](int which, uint32_t id, size_t h) {
        const size_t w = vgpu_basic_machine_chip(id)->preprocessed_width;
        t.prep[which] = {t.store[14 + which].zeros(h * w), h, w};
        return t.store[14 + which].data();
    };
    {   // program: 1 main column (execution counts) + 7 preprocessed
        const size_t h = next_pow2(L.n_instr);
        uint32_t* counts = chip(1, h);
        uint32_t* pre = prep(0, 1, h);
        for (size_t i = 0; i < h; i++) {
            uint32_t* row = &pre[i * 7];
            row[0] = (uint32_t)i;
            // every row of the program, executed or not: InstructionWord::flatten takes the opcode from_canonical_u32 (machine/src/program.rs:44)
            if (i < L.n_instr) {
                counts[i] = L.prog_counts[i];
                row[1] = (uint32_t)L.program[6 * i] % P;
                for (int k = 0; k < 5; k++) row[2 + k] = from_i32(L.program[6 * i + 1 + k]);
            }
        }
    }
    {   // mul: 2^10 counter rows
        uint32_t* m = chip(5, 1024);
        for (uint32_t i = 0; i < 1024; i++) m[i * 18 + 17] = i + 1;
    }
    for (uint32_t id : {6u, 7u, 9u, 11u}) chip(id, 1);      // div, shift, com, output: no rows in the provable instruction subset
    {   // range: (multiplicity, counter) + preprocessed counter
        uint32_t* r = chip(12, 256);
        uint32_t* c = prep(1, 12, 256);
        for (uint32_t i = 0; i < 256; i++) { r[2 * i] = L.range_count[i]; r[2 * i + 1] = i; c[i] = i; }
    }
    {   // static_data: (addr, value[4], is_real) per cell in address order, padded to a power of two (one zero row when empty)
        uint32_t* s = chip(13, next_pow2(L.n_static ? L.n_static : 1));
        for (size_t i = 0; i < L.n_static; i++) {
            uint32_t* row = &s[i * 6];
            row[0] = L.static_addr[i] % P; word_be(L.static_value[i], &row[1]); row[5] = 1;    // static_data/src/lib.rs:67
        }
    }
    return tr.release();
}

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
            if (!vm.static_addr.empty() && vm.static_addr.back() == c.first) vm.static_value.back() = c.second;
            else { vm.static_addr.push_back(c.first); vm.static_value.push_back(c.second); }
        }
        for (size_t i = 0; i < vm.static_addr.size(); i++) vm.cells.set(vm.static_addr[i], vm.static_value[i]);
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

// Chip::generate_trace x14 on the host from the interpreter's logs; `cells` is the memory the run left (vgpu_traces_mem_cell)
static vgpu_traces* build_traces_host(const VgVmLogs& L, const CellMap& cells) {
    std::unique_ptr<vgpu_traces> tr(vg_short_chip_traces(L));      // released to the caller at the end; freed if an allocation below throws
    Traces& t = tr->t;
    t.clock = (uint32_t)L.n_cpu; t.n_mem_ops = (uint32_t)L.n_mem; t.n_add_ops = (uint32_t)L.n_adds; t.n_sub_ops = (uint32_t)L.n_subs;
    build_cpu(L, t);
    build_mem(L, t);
    build_rows(L.n_adds, ADDSUB_COLS, t.store[3], t.main[3], [&](uint32_t* row, size_t i) { addsub_row(row, L.adds[i], true); });
    build_rows(L.n_subs, ADDSUB_COLS, t.store[4], t.main[4], [&](uint32_t* row, size_t i) { addsub_row(row, L.subs[i], false); });
    build_rows(L.n_lts, LT_COLS, t.store[8], t.main[8], [&](uint32_t* row, size_t i) {
        if (const uint32_t d = lt_row(row, L.lts[i])) row[27] = fpow(d, P - 2);
    });
    build_rows(L.n_bits, BITWISE_COLS, t.store[10], t.main[10], [&](uint32_t* row, size_t i) { bitwise_row(row, L.bits[i]); });
    t.cells = cells;
    return tr.release();
}

static int machine_run_impl(const int32_t* program_words, uint64_t n_instr, uint32_t initial_pc, uint32_t initial_fp, uint64_t max_cycles,
                            const uint32_t* static_addrs, const uint32_t* static_values, uint64_t n_static,
                            vgpu_traces** out, char* err, uint64_t err_len) {
    Vm vm;
    if (vm_run_impl(program_words, n_instr, initial_pc, initial_fp, max_cycles, static_addrs, static_values, n_static, vm, err, err_len) != 0) return -1;
    *out = build_traces_host(vm.logs(), vm.cells);
    return 0;
}

// ---- the interpreter's logs as an object: Machine::run without the row fill (the device builds the rows, witness.cu) ----
}  // extern "C"
struct vgpu_vmlog { Vm vm; std::vector<int32_t> program; VgVmLogs view; };
extern "C" {

int32_t vgpu_vm_run(const int32_t* program_words, uint64_t n_instr, uint32_t initial_pc, uint32_t initial_fp, uint64_t max_cycles,
                    const uint32_t* static_addrs, const uint32_t* static_values, uint64_t n_static, vgpu_vmlog** out, char* err, uint64_t err_len) {
    try {
        std::unique_ptr<vgpu_vmlog> L(new vgpu_vmlog());
        L->program.assign(program_words, program_words + 6 * n_instr);
        if (vm_run_impl(L->program.data(), n_instr, initial_pc, initial_fp, max_cycles, static_addrs, static_values, n_static, L->vm, err, err_len) != 0) return -1;
        L->view = L->vm.logs();
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
    try { *out = build_traces_host(l->view, l->vm.cells); return 0; }
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
