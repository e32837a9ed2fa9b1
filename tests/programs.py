"""Synthetic multi-chip programs shared by the CPU and GPU tests (SURVEY 8(d) config 5: a loop mixing add, sub,
lt/lte/slt/sle, and/or/xor on a linear-congruential value stream; mul/div/shift are excluded there because the
reference's range-bus accounting does not balance for them, and eq/ne because the reference's Com32Chip::op_to_row
fills only the opcode flags — alu_u32/src/com/mod.rs:84-100 — so its bus receive can never match the CPU's send)."""
import numpy as np

B = 24
LOAD32, STORE32, JAL, JALV, BEQ, BNE, IMM32, STOP, LOADFP, ADD32, SUB32 = 1, 2, 3, 4, 5, 6, 7, 8, 10, 100, 101
LT32, LTE32, SLT32, SLE32 = 104, 115, 117, 118


def _ins(op, a=0, b=0, c=0, d=0, e=0):
    return [op, a, b, c, d, e]


def _word(v):                      # big-endian bytes, the operand order of imm32
    v &= 0xFFFFFFFF
    return ((v >> 24) & 255, (v >> 16) & 255, (v >> 8) & 255, v & 255)


def mixed_program(iters):
    """cpu + mem + add + lt + range + program: add / lt / lte / slt / sle (incl. left immediates), bne back-edge."""
    return np.array([
        [7, -4, 0, 0, 0, 0],                                  # i = 0
        [7, -8, 0x12, 0x34, 0x56, 0x78],                      # x = seed
        [100, -8, -8, 1013904223, 0, 1],                      # x += c            (add32 imm)
        [100, -12, -8, -4, 0, 0],                             # y = x + i         (add32)
        [104, -16, -12, -8, 0, 0],                            # y < x             (lt32)
        [117, -20, -8, -12, 0, 0],                            # x <s y            (slt32)
        [115, -24, 77, -8, 1, 0],                             # 77 <= x           (lte32, left immediate)
        [118, -28, -12, 1000, 0, 1],                          # y <=s 1000        (sle32, right immediate)
        [100, -4, -4, 1, 0, 1],                               # i += 1
        [6, 2 * B, -4, iters, 0, 1],                          # bne loop, i, iters
        [8, 0, 0, 0, 0, 0],
    ], dtype=np.int32)


def config5_program(iters):
    """cpu + mem + add + sub + lt + bitwise + range + program.  x <- x*1664525 + 1013904223 is replaced by an
    add/xor/and/or mix (no mul); every ALU flavour appears with a memory operand and with an immediate.
    The sub operands are shaped so that no byte borrows (minuend bytes >= 0x80 > subtrahend bytes): the reference's
    Sub32Chip::op_to_row derives each borrow from the operand bytes alone (alu_u32/src/sub/mod.rs:103-111) and its AIR
    has no top-byte borrow (sub/stark.rs:42-45), so a subtraction that borrows is unprovable in the reference too."""
    return np.array([
        [7, -4, 0, 0, 0, 0],                                  # i = 0
        [7, -8, 0x9e, 0x37, 0x79, 0xb9],                      # x = seed
        [7, -32, 0x0f, 0xf0, 0x55, 0xaa],                     # m = mask
        [100, -8, -8, 1013904223, 0, 1],                      # x += c                       (add32 imm)     <- loop
        [109, -12, -8, -32, 0, 0],                            # y = x ^ m                    (xor32)
        [107, -16, -12, 0x7f7f7f7f, 0, 1],                    # t = y & 0x7f7f7f7f           (and32 imm)
        [108, -20, -8, -0x7f7f7f80, 0, 1],                    # s = x | 0x80808080           (or32 imm)
        [101, -24, -20, -16, 0, 0],                           # d = s - t                    (sub32)
        [101, -28, -20, 12345, 0, 1],                         # e = s - 12345                (sub32 imm)
        [109, -8, -8, -28, 0, 0],                             # x ^= e                       (xor32)
        [104, -36, -24, -8, 0, 0],                            # d < x                        (lt32)
        [118, -40, -28, -12, 0, 0],                           # e <=s y                      (sle32)
        [117, -44, 5, -28, 1, 0],                             # 5 <s e                       (slt32 left imm)
        [115, -48, -20, 4096, 0, 1],                          # s <= 4096                    (lte32 imm)
        [107, -32, -32, -12, 0, 0],                           # m &= y                       (and32)
        [108, -32, -32, 0x01010101, 0, 1],                    # m |= 0x01010101              (or32 imm)
        [100, -4, -4, 1, 0, 1],                               # i += 1
        [6, 3 * B, -4, iters, 0, 1],                          # bne loop, i, iters
        [8, 0, 0, 0, 0, 0],
    ], dtype=np.int32)


def static_data_program():
    """prove_static_data of the reference (basic/tests/test_static_data.rs:30-55): loops forever unless the static value is loaded.
        _start: imm32 0(fp), 0, 0, 0, 0x10 ; load32 -4(fp), 0(fp) ; bnei _start, -4(fp), 0x25 ; stop
    with static cells 0x10 = Word([0,0,0,0x25]), 0x14 = Word([0,0,0,0x32]) (test_static_data.rs:59-60)."""
    prog = np.array([
        [7, 0, 0, 0, 0, 0x10],
        [1, -4, 0, 0, 0, 0],
        [6, 0, -4, 0x25, 0, 1],
        [8, 0, 0, 0, 0, 0],
    ], dtype=np.int32)
    return prog, {0x10: 0x25, 0x14: 0x32}


def loads_stores_edge_program():
    """Every instruction of the restated subset that the Fibonacci program does not reach: load32 / store32 through pointers,
    loadfp, sub32 with and without an immediate (incl. a NEGATIVE immediate: operand c is replaced by the reduced bytes of
    c as u32, cpu/src/lib.rs:364-371), bne on an immediate, a backwards jal with a frame change and back with jalv.
    Ends with [fp-36] = 254, pc 13, fp 0x1000; two sub32 and one add32 operations."""
    return np.array([
        _ins(IMM32, -4, 0, 0, 1, 44),            # [fp-4] = 300
        _ins(IMM32, -8, 0, 0, 0, 7),             # [fp-8] = 7
        _ins(LOADFP, -12, -8),                   # [fp-12] = fp-8  (a pointer)
        _ins(LOAD32, -16, 0, -12),               # [fp-16] = [[fp-12]] = 7
        _ins(SUB32, -20, -4, -8),                # 300 - 7 = 293
        _ins(SUB32, -24, -20, 38, 0, 1),         # 293 - 38 = 255 : borrow pattern in the low byte
        _ins(ADD32, -28, -24, -1, 0, 1),         # 255 + 0xFFFFFFFF = 254 (wraps): immediate operand -1
        _ins(LOADFP, -32, -36),                  # pointer to fp-36
        _ins(STORE32, 0, -32, -28),              # [[fp-32]] = [fp-28] -> [fp-36] = 254
        _ins(BNE, 12 * 24, -36, 254, 0, 1),      # equal: falls through
        _ins(BEQ, 12 * 24, -36, -28),            # equal: taken, skips the next instruction
        _ins(IMM32, -4, 9, 9, 9, 9),             # skipped
        _ins(JAL, -40, 14 * 24, -64),            # call: return address at [fp-40], fp -= 64, to pc 14
        _ins(STOP),
        _ins(IMM32, 4, 0, 0, 0, 64),             # callee: [fp+4] = 64 (the frame offset back)
        _ins(JALV, -4, 24, 4),                   # back to [fp+24] = [old fp-40] = 13*24, fp += [fp+4] = 64
    ], dtype=np.int32)


def lt_edge_operands_program():
    """Equal operands (no differing byte: flags, bits and diff_inv stay zero), operands that differ in the TOP byte only, sign
    boundaries, both immediates at once (the recorded immediate is the right one, written through the LEFT-immediate path).
    Ends with [fp-100] = 1 and [fp-104] = 1."""
    vals = [0, 1, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFF, 0x01000000, 0x00FFFFFF]
    prog = []
    for i, v in enumerate(vals):
        prog.append(_ins(IMM32, -4 * (i + 1), *_word(v)))
    k = 0
    for i in range(len(vals)):
        for j in range(len(vals)):
            op = (LT32, LTE32, SLT32, SLE32)[(i + j) % 4]
            prog.append(_ins(op, -64 - 4 * (k % 8), -4 * (i + 1), -4 * (j + 1)))
            k += 1
    prog.append(_ins(SLT32, -100, -5, -4, 1, 0))            # left immediate -5 against [fp-4] = 0
    prog.append(_ins(LTE32, -104, 7, 7, 1, 1))              # both immediates
    prog.append(_ins(STOP))
    return np.array(prog, dtype=np.int32)


def single_address_program(reps):
    """Every memory operation at ONE address: fp-4 holds a pointer to itself, then `reps` times store32 and load32 through it
    (each reads the pointer and the value and writes the value back, all at fp-4).  Straight-line: a loop counter would be a
    second address."""
    prog = [_ins(LOADFP, -4, -4)]                           # [fp-4] = fp-4
    for _ in range(reps):
        prog.append(_ins(STORE32, 0, -4, -4))               # [[fp-4]] = [fp-4]
        prog.append(_ins(LOAD32, -4, 0, -4))                # [fp-4] = [[fp-4]]
    prog.append(_ins(STOP))
    return np.array(prog, dtype=np.int32)
