// One row of Chip::generate_trace for each chip whose trace grows with the run, from the interpreter's logs (host/vmlog.h).
// Both witness builders call these: host/tracegen.cc (row-major, OpenMP) and witness.cu (one thread per row, column-major
// Montgomery), so the trace layout is written down once.  Each function writes every word of its row, canonical (< p).
// The CPU and lt rows leave column 27 at 0 and return the field element whose inverse belongs there (0 = none): each builder
// inverts it in its own representation.
#pragma once
#include "bb.cuh"
#include "host/vmlog.h"

constexpr int CPU_COLS = 51, MEM_COLS = 14, ADDSUB_COLS = 16, LT_COLS = 45, BITWISE_COLS = 79;

BB_HD uint32_t from_i32(int32_t x) { return x < 0 ? (bb::P - (uint32_t)(-(int64_t)x) % bb::P) % bb::P : (uint32_t)x % bb::P; }
BB_HD void word_be(uint32_t v, uint32_t* out) { out[0] = v >> 24; out[1] = (v >> 16) & 0xff; out[2] = (v >> 8) & 0xff; out[3] = v & 0xff; }
BB_HD uint64_t next_pow2(uint64_t n) { uint64_t p = 1; while (p < n) p <<= 1; return p; }

// ---- CPU chip (cpu/src/columns.rs:8-37; cpu/src/lib.rs:163-373) ---------------------------------------------------------------
// cycle i: its record, its instruction's six program words, and its memory operations mem[0, n_mem) in execution order
BB_HD uint32_t cpu_row(uint32_t row[CPU_COLS], uint64_t i, const VgCpuRec& r, const int32_t* w, const VgMemOp* mem, uint64_t n_mem) {
#pragma unroll
    for (int c = 0; c < CPU_COLS; c++) row[c] = 0;
    row[0] = (uint32_t)i; row[1] = r.pc; row[2] = r.fp % bb::P;      // from_canonical_u32 (cpu/src/lib.rs:171-172) reduces mod p
    row[3] = (uint32_t)w[0];
    for (int k = 0; k < 5; k++) row[4 + k] = from_i32(w[1 + k]);
    switch (r.kind) {
        case VG_K_STORE32: row[16] = 1; break;
        case VG_K_LOAD32: row[13] = 1; break;
        case VG_K_JAL: row[20] = 1; break;
        case VG_K_JALV: row[21] = 1; break;
        case VG_K_BEQ: row[18] = 1; break;
        case VG_K_BNE: row[19] = 1; break;
        case VG_K_IMM32: row[22] = 1; break;
        case VG_K_BUS: case VG_K_BUS_LEFT_IMM: row[9] = 1; break;
        case VG_K_STOP: row[24] = 1; break;
        case VG_K_LOADFP: row[25] = 1; break;
    }
    const bool left_imm = r.has_imm && r.kind == VG_K_BUS_LEFT_IMM;
    if (left_imm) {                                 // set_left_imm_value (cpu/src/lib.rs:364-371)
        row[12] = 1;
        word_be(r.imm, &row[29 + 3]);
        row[5] = r.imm % bb::P;
    } else if (r.has_imm) {                         // set_imm_value (cpu/src/lib.rs:355-362)
        row[11] = 1;
        word_be(r.imm, &row[36 + 3]);
        row[6] = r.imm % bb::P;
    }
    row[29 + 1] = 1; row[36 + 1] = 1;
    bool first_read = true;
    for (uint64_t k = 0; k < n_mem; k++) {          // channels: first read 29 (36 after a left immediate), second read 36, write 43
        const VgMemOp m = mem[k];
        uint32_t ch;
        if (m.is_write) ch = 43;
        else if (first_read && !left_imm) { ch = 29; first_read = false; }
        else ch = 36;
        row[ch] = 1; row[ch + 2] = m.addr % bb::P; word_be(m.value, &row[ch + 3]);     // cpu/src/lib.rs:263-276
    }
    uint32_t dsum = 0;                              // diff = sum_k (read_1_k - read_2_k)^2 <= 4 * 255^2 < p
    for (int k = 0; k < 4; k++) { const int32_t dd = (int32_t)row[32 + k] - (int32_t)row[39 + k]; dsum += (uint32_t)(dd * dd); }
    row[26] = dsum; row[28] = dsum != 0;
    return dsum;
}

// pad_to_power_of_two (cpu/src/lib.rs:318-353): row i >= n repeats STOP at the last cycle's pc and fp
BB_HD void cpu_pad_row(uint32_t row[CPU_COLS], uint64_t i, const VgCpuRec& last) {
#pragma unroll
    for (int c = 0; c < CPU_COLS; c++) row[c] = 0;
    row[0] = (uint32_t)i; row[1] = last.pc; row[2] = last.fp % bb::P; row[3] = OP_STOP;
    row[24] = 1; row[29 + 1] = 1; row[36 + 1] = 1;
}

// ---- memory chip (memory/src/columns.rs:8-39) ----------------------------------------------------------------------------------
// row i: a static cell opening the trace ({0, addr, value, 1}, memory/src/lib.rs:163-169, 276) or an operation of the log sorted
// by address (memory/src/lib.rs:247-262); the address is stored reduced
BB_HD void mem_row(uint32_t row[MEM_COLS], uint64_t i, const VgMemOp& m, bool is_static) {
#pragma unroll
    for (int c = 0; c < MEM_COLS; c++) row[c] = 0;
    row[0] = m.addr % bb::P; word_be(m.value, &row[1]);
    row[5] = m.clk; row[6] = is_static;
    row[7] = m.is_write ? 0 : 1; row[8] = m.is_write ? 1 : 0;
    row[12] = (uint32_t)i;
}

// ---- add / sub (alu_u32/src/add/mod.rs:38-129, alu_u32/src/sub/mod.rs:103-111) --------------------------------------------------
BB_HD void addsub_row(uint32_t row[ADDSUB_COLS], const VgAluRec& o, bool is_add) {
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

// ---- lt family (Lt32Chip::op_to_row / set_cols, alu_u32/src/lt/mod.rs:86-160) ----------------------------------------------------
BB_HD uint32_t lt_row(uint32_t row[LT_COLS], const VgAluOpRec& o) {
#pragma unroll
    for (int c = 0; c < LT_COLS; c++) row[c] = 0;
    uint32_t a[4], b[4], c[4];
    word_be(o.a, a); word_be(o.b, b); word_be(o.c, c);
#pragma unroll
    for (int k = 0; k < 4; k++) { row[k] = b[k]; row[4 + k] = c[k]; }
    row[21] = a[3];
    const bool is_signed = o.opcode == OP_SLT32 || o.opcode == OP_SLE32;
    row[o.opcode == OP_LT32 ? 23 : o.opcode == OP_LTE32 ? 24 : o.opcode == OP_SLT32 ? 25 : 26] = 1;
    uint32_t diff = 0;
    for (int k = 0; k < 4; k++) {                   // the first differing byte
        if (b[k] != c[k]) {
            const uint32_t z = 256u + b[k] - c[k];
            for (int bit = 0; bit < 9; bit++) row[12 + bit] = (z >> bit) & 1;
            row[8 + k] = 1;
            diff = (b[k] + bb::P - c[k]) % bb::P;
            break;
        }
    }
    for (int bit = 0; bit < 8; bit++) { row[28 + bit] = (b[0] >> bit) & 1; row[36 + bit] = (c[0] >> bit) & 1; }
    row[44] = (is_signed && row[28 + 7] != row[36 + 7]) ? 1 : 0;
    row[22] = 1;
    return diff;
}

// ---- and / or / xor (Bitwise32Chip::op_to_row / set_cols, alu_u32/src/bitwise/mod.rs:84-131) ------------------------------------
// input_1 0..3, input_2 4..7, bits_1[byte][bit] 8 + 8*byte + bit, bits_2 40 + ..., output 72..75, is_and 76, is_or 77, is_xor 78
BB_HD void bitwise_row(uint32_t row[BITWISE_COLS], const VgAluOpRec& o) {
    uint32_t a[4], b[4], c[4];
    word_be(o.a, a); word_be(o.b, b); word_be(o.c, c);
#pragma unroll
    for (int k = 0; k < 4; k++) {
        row[k] = b[k]; row[4 + k] = c[k]; row[72 + k] = a[k];
#pragma unroll
        for (int bit = 0; bit < 8; bit++) { row[8 + 8 * k + bit] = (b[k] >> bit) & 1; row[40 + 8 * k + bit] = (c[k] >> bit) & 1; }
    }
    row[76] = o.opcode == OP_AND32; row[77] = o.opcode == OP_OR32; row[78] = o.opcode != OP_AND32 && o.opcode != OP_OR32;
}
