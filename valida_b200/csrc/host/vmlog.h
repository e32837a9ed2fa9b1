// The interpreter's logs — what Machine::run leaves behind for Chip::generate_trace (cpu/src/lib.rs:79-97, memory/src/lib.rs:143-194,
// alu_u32/src/*/mod.rs generate_trace): plain arrays that both witness builders read, the host one (host/tracegen.cc) and the
// device one (witness.cu).  Both fill the rows of the tall chips with the row functions of chip_rows.cuh and take the short chips
// from vg_short_chip_traces.
#pragma once
#include <cstddef>
#include <cstdint>

// opcodes of the instruction subset the interpreter runs
enum : uint32_t { OP_LOAD32 = 1, OP_STORE32 = 2, OP_JAL = 3, OP_JALV = 4, OP_BEQ = 5, OP_BNE = 6, OP_IMM32 = 7, OP_STOP = 8, OP_LOADFP = 10,
                  OP_ADD32 = 100, OP_SUB32 = 101, OP_LT32 = 104, OP_AND32 = 107, OP_OR32 = 108, OP_XOR32 = 109, OP_LTE32 = 115, OP_SLT32 = 117, OP_SLE32 = 118 };

enum : uint8_t { VG_K_STORE32, VG_K_LOAD32, VG_K_JAL, VG_K_JALV, VG_K_BEQ, VG_K_BNE, VG_K_IMM32, VG_K_BUS, VG_K_STOP, VG_K_LOADFP, VG_K_BUS_LEFT_IMM };

struct VgMemOp { uint32_t clk, addr, value, is_write; };                       // in execution (clock) order
struct VgCpuRec { uint32_t pc, fp, instr, imm, mem0; uint8_t kind, has_imm, pad[2]; };   // mem0: first memory operation of the cycle
struct VgAluRec { uint32_t a, b, c; };                                        // a = b op c
struct VgAluOpRec { uint32_t a, b, c, opcode; };

struct VgVmLogs {
    const int32_t* program; size_t n_instr;                                   // n_instr x 6 words
    const VgCpuRec* cpu; size_t n_cpu;
    const VgMemOp* mem; size_t n_mem;
    const VgAluRec* adds; size_t n_adds;
    const VgAluRec* subs; size_t n_subs;
    const VgAluOpRec* lts; size_t n_lts;
    const VgAluOpRec* bits; size_t n_bits;
    const uint32_t* prog_counts;                                              // n_instr executions per instruction (STOP padding included)
    const uint32_t* range_count;                                              // 256
    const uint32_t* static_addr; const uint32_t* static_value; size_t n_static;   // ascending address
};

// The traces of the short chips (program and its preprocessed trace, mul, div, shift, com, output, range and its preprocessed
// trace, static data), row-major canonical, a few KB; the tall chips' matrices are left empty.  Throws std::bad_alloc.
struct vgpu_traces;
vgpu_traces* vg_short_chip_traces(const VgVmLogs& L);
