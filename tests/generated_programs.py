"""Seeded generator of terminating programs for witness parity tests: every run writes a cell before it reads it, so the host
interpreter, the plain restatement (tracegen_restated.py) and both witness builders can run them.  They need not be provable.

generated_program(seed, regime, cycles) is a loop whose body mixes imm32 (random and edge words), add/sub (negative and >= p
immediates, borrows), the lt family (left and double immediates, equal operands, a first difference at each byte), and/or/xor,
loadfp, beq/bne forward skips, jal/jalv pairs with a frame change, and store32/load32 through a pointer recomputed every
iteration from an add/xor/and/or stream, as config5_program does.  Frame slots are absolute addresses (fp is only the base of
the operand offsets), so the address set of the whole memory log follows the regime:

    a  every byte varies, addresses at or above p and near 2^32 included (odd pointers, the frame on even addresses)
    b  only the top byte varies: the device sort skips digit passes 0-2, the host sort its passes 0-1
    c  only bits 7-8 vary: both in the host's first 11-bit digit, across the device's 8-bit digits 0 and 1
    d  a few dozen pointer addresses revisited every iteration: equal keys in every tile of the sort
    e  every pointer address distinct (an odd walk with an even step)

counted_program() is straight-line with exact operation counts, for the padding and row-run edges.  with_dead_rows() appends rows
that never run, with opcode words at and above p."""
import numpy as np

from programs import ADD32, BEQ, BNE, IMM32, JAL, JALV, LOAD32, LOADFP, LT32, LTE32, SLE32, SLT32, STOP, STORE32, SUB32

AND32, OR32, XOR32 = 107, 108, 109
P = 2013265921
B = 24
M32 = 0xFFFFFFFF
EDGE_WORDS = [0, 1, 0x7F, 0x80, 0xFF, 0x100, 0xFFFF, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFF, 0xFFFFFFFE, P - 1, P, P + 1,
              0x78000000, 0x77FFFFFF, 0x00FFFFFF, 0x01000000, 0xFF000000, 0x80808080, 0x7F7F7F7F]
REGIMES = "abcde"


def _i32(v):                       # a u32 as the int32 operand word that carries it
    v &= M32
    return v - (1 << 32) if v >> 31 else v


def _bytes(v):
    v &= M32
    return [(v >> 24) & 255, (v >> 16) & 255, (v >> 8) & 255, v & 255]


class _Asm:
    def __init__(self, rng, fp):
        self.rng, self.fp, self.code, self.callees = rng, fp, [], []

    def off(self, addr, fp=None):  # operand that addresses the cell `addr` from frame pointer fp
        return _i32(addr - (self.fp if fp is None else fp))

    def emit(self, op, a=0, b=0, c=0, d=0, e=0):
        self.code.append([op, a, b, c, d, e])

    def word(self):
        r = self.rng
        return int(r.choice(EDGE_WORDS)) if r.random() < 0.4 else int(r.integers(0, 1 << 32))

    def imm(self):                 # an immediate operand: small, negative, >= p as a u32, or any int32
        r = self.rng
        k = r.integers(0, 4)
        return [int(r.integers(-300, 300)), _i32(self.word()), -int(r.integers(1, 1 << 31)), int(r.integers(0, 1 << 31))][k]

    def imm32(self, dst, v):
        self.emit(IMM32, self.off(dst), *_bytes(v))

    def alu(self, dst, srcs, one_op=False):
        """One random ALU operation writing dst from the cells srcs (one_op: the forms with one memory read only)."""
        r, o = self.rng, self.off
        x, y = (int(s) for s in r.choice(srcs, 2))
        kind = int(r.integers(0, 4))
        if kind == 0:                                                  # add / sub, register or immediate
            op = ADD32 if r.random() < 0.5 else SUB32
            if one_op or r.random() < 0.5:
                self.emit(op, o(dst), o(x), self.imm(), 0, 1)
            else:
                self.emit(op, o(dst), o(x), o(y))
        elif kind == 1:                                                # and / or / xor
            op = int(r.choice([AND32, OR32, XOR32]))
            if one_op or r.random() < 0.5:
                self.emit(op, o(dst), o(x), self.imm(), 0, 1)
            else:
                self.emit(op, o(dst), o(x), o(y))
        else:                                                          # the lt family
            op = int(r.choice([LT32, LTE32, SLT32, SLE32]))
            form = int(r.integers(0, 6 if not one_op else 3))
            if form == 0:
                self.emit(op, o(dst), o(x), self.imm(), 0, 1)          # right immediate
            elif form == 1:
                self.emit(op, o(dst), self.imm(), o(x), 1, 0)          # left immediate
            elif form == 2:
                a = self.imm()
                self.emit(op, o(dst), a, a if r.random() < 0.3 else self.imm(), 1, 1)   # both immediates
            elif form == 3:
                self.emit(op, o(dst), o(x), o(x))                      # equal operands
            elif form == 4:                                            # first difference at byte k (big-endian order)
                k, bit = int(r.integers(0, 4)), int(r.integers(0, 8))
                self.emit(XOR32, o(dst), o(x), _i32(1 << (8 * (3 - k) + bit)), 0, 1)
                self.emit(op, o(dst), o(dst), o(x)) if r.random() < 0.5 else self.emit(op, o(dst), o(x), o(dst))
            else:
                self.emit(op, o(dst), o(x), o(y))

    def call(self, ret, s1, s2, dist):
        """jal to a callee after STOP with the frame moved by dist, and back by jalv: the callee writes the way back into s1
        (imm32) and jalv writes s2; ret, s1 and s2 are distinct cells."""
        here = len(self.code)
        fp2 = (self.fp + dist) & M32
        body = [[IMM32, self.off(s1, fp2), *_bytes(-dist)],
                [JALV, self.off(s2, fp2), self.off(ret, fp2), self.off(s1, fp2), 0, 0]]
        self.callees.append((here, body))
        self.emit(JAL, self.off(ret), 0, _i32(dist))                   # target patched in program()

    def program(self):
        code = [list(x) for x in self.code] + [[STOP, 0, 0, 0, 0, 0]]
        for at, body in self.callees:
            code[at][2] = B * len(code)
            code += body
        return np.array(code, dtype=np.int32)


def _regime_layout(regime, rng):
    """(frame cells: counter, stream, pointer, scratch...; the (op, immediate) steps that make the pointer from the stream cell,
    None for the walk of regime e)."""
    if regime == "a":
        base = int(rng.choice([0x1000, 0x77FFFF00, 0x78000000, 0xFFFFF000, int(rng.integers(0, 1 << 30)) * 4]))
        cells = [(base + 4 * k) & M32 for k in range(12)]
        return cells, [(OR32, 1)]                                      # odd: never a frame cell
    if regime == "b":
        top, low = int(rng.choice([0x00, 0xC0])), int(rng.integers(0, 1 << 24))
        cells = [((top + k) << 24 | low) & M32 for k in range(12)]
        return cells, [(AND32, 0x3F000000), (ADD32, (top + 0x80) << 24 & M32), (OR32, low)]    # top bytes disjoint from the frame
    if regime == "c":
        base = int(rng.choice([0x00012000, 0xF0000000, 0x78000000, int(rng.integers(0, 1 << 23)) << 9]))
        cells = [base, base | 0x80, base | 0x100, base | 0x180]       # counter, stream, pointer, scratch
        return cells, [(AND32, 0x100), (OR32, base | 0x80)]           # the stream cell or the scratch cell
    if regime == "d":
        base = int(rng.choice([0x1000, 0xFFFFF000, int(rng.integers(0, 1 << 30)) * 4]))
        far = int(rng.choice([0x9E370001, 0x78000001, 0x00400001]))
        cells = [(base + 4 * k) & M32 for k in range(12)]
        return cells, [(AND32, 0x7C), (OR32, far)]                    # 32 odd addresses
    if regime == "e":
        base = int(rng.choice([0x1000, 0xFFFFF000, int(rng.integers(0, 1 << 30)) * 4]))
        cells = [(base + 4 * k) & M32 for k in range(13)]             # the last one walks
        return cells, None
    raise ValueError(regime)


def generated_program(seed, regime, cycles, fp=None, edge_pointers=True):
    """A loop of about `cycles` cycles in address regime `regime` (a-e); fp defaults to a seeded choice.  Returns the program."""
    rng = np.random.default_rng([seed, ord(regime)])
    cells, ptr = _regime_layout(regime, rng)
    if fp is None:
        fp = int(rng.choice([0x1000, 0x78000000, 0x80000000, 0xFFFFF000, int(rng.integers(0, 1 << 32))]))
    asm = _Asm(rng, fp)
    cnt, x, p, scratch = cells[0], cells[1], cells[2], cells[3:]
    if regime == "e":
        walk, scratch = scratch[-1], scratch[:-1]
    # the counter, the pointer and the stream it is made from are never a destination (regime c has no other cell to spare for the
    # stream: its pointer takes one of two values whatever the stream holds)
    writable = scratch + ([x] if regime == "c" else [])
    readable = writable if regime == "c" else writable + [x]
    asm.imm32(cnt, 0)
    for c in cells[1:]:
        asm.imm32(c, asm.word())
    if regime == "e":
        asm.imm32(walk, int(rng.integers(0, 1 << 31)) * 2 + 1)
    if regime == "a" and edge_pointers:                                # pointers at and around p and near 2^32, written then read
        for e in (0xFFFFFFFF, 0xFFFFFFFD, P, P + 2, P - 2, 0x80000001, 0x7FFFFFFF):
            asm.imm32(p, e)
            asm.emit(STORE32, 0, asm.off(p), asm.off(x))
            asm.emit(LOAD32, asm.off(scratch[0]), 0, asm.off(p))
    loop = len(asm.code)
    body0 = len(asm.code)

    def random_ops(k):
        for _ in range(k):
            u = rng.random()
            dst = int(rng.choice(writable))
            if u < 0.08:
                asm.imm32(dst, asm.word())
            elif u < 0.14:
                asm.emit(LOADFP, asm.off(dst), int(rng.choice([0, -4, 1 << 20, -(1 << 31), int(rng.integers(-(1 << 31), 1 << 31))])))
            elif u < 0.22:                                             # beq / bne skipping the next operation
                op = BEQ if rng.random() < 0.5 else BNE
                y = int(rng.choice(readable))
                if rng.random() < 0.5:
                    asm.emit(op, B * (len(asm.code) + 2), asm.off(y), asm.imm(), 0, 1)
                else:
                    asm.emit(op, B * (len(asm.code) + 2), asm.off(y), asm.off(int(rng.choice(readable))))
                asm.alu(dst, readable)
            elif u < 0.26:
                if regime == "c":
                    ret, s1, s2 = scratch[0], p, x                     # the pointer cell is recomputed before its next use
                else:
                    ret, s1, s2 = (int(v) for v in rng.choice(scratch, 3, replace=False))
                asm.call(ret, s1, s2, int(rng.choice([-64, 1 << 24, 0x80000000 - fp, int(rng.integers(-(1 << 31), 1 << 31))])))
            else:
                asm.alu(dst, readable)

    asm.emit(ADD32, asm.off(x), asm.off(x), 1013904223, 0, 1)            # the stream
    asm.emit(XOR32, asm.off(x), asm.off(x), asm.off(cnt))
    random_ops(10)
    if regime == "e":
        asm.emit(ADD32, asm.off(walk), asm.off(walk), _i32(0x9E3779BA), 0, 1)
        asm.emit(XOR32, asm.off(p), asm.off(walk), 0x5A5A5A5A, 0, 1)
    else:
        op, v = ptr[0]
        asm.emit(op, asm.off(p), asm.off(x), _i32(v), 0, 1)
        for op, v in ptr[1:]:
            asm.emit(op, asm.off(p), asm.off(p), _i32(v), 0, 1)
    src = int(rng.choice(readable))
    asm.emit(STORE32, 0, asm.off(p), asm.off(src))
    asm.emit(LOAD32, asm.off(scratch[0]), 0, asm.off(p))
    random_ops(6)
    body = len(asm.code) - body0 + 2 + 2 * len(asm.callees)
    iters = max(1, (cycles - loop) // body)
    asm.emit(ADD32, asm.off(cnt), asm.off(cnt), 1, 0, 1)
    asm.emit(BNE, B * loop, asm.off(cnt), iters, 0, 1)
    # stop in another frame, at or above p: the STOP padding rows carry the last fp, which is not the first
    end = int(rng.choice([0x80000000, 0xFFFFF000, P + 4]))
    asm.emit(JAL, asm.off(scratch[0]), B * (len(asm.code) + 1), _i32((end if end != fp else 0xFFFFFFF0) - fp))
    return asm.program(), fp


def counted_program(seed, adds=0, subs=0, lts=0, bits=0, cycles=None, mem=None, n_static=0, fp=0x1000):
    """Straight-line: exactly `adds`, `subs`, `lts`, `bits` ALU operations with random operands, then imm32 fill so that the run
    takes exactly `cycles` cycles (STOP included) or makes exactly `mem` memory operations; `n_static` static cells on both sides
    of p, a few of them loaded.  Returns (program, static data, fp)."""
    rng = np.random.default_rng(seed)
    asm = _Asm(rng, fp)
    cells = [(fp - 4 * (k + 1)) & M32 for k in range(8)]
    srcs, dst = cells[:6], cells[6:]
    n_mem = 0
    for c in srcs:
        asm.imm32(c, asm.word())
        n_mem += 1
    static = {}
    if n_static:
        addrs = rng.choice(1 << 31, n_static, replace=False).astype(np.int64) * 2 + 1          # odd: never a frame cell
        static = {int(a): int(rng.integers(0, 1 << 32)) for a in addrs}
        for a in sorted(static)[:: max(1, n_static // 8)]:
            asm.imm32(dst[1], a)
            asm.emit(LOAD32, asm.off(dst[0]), 0, asm.off(dst[1]))
            n_mem += 4
    for op, n in ((ADD32, adds), (SUB32, subs), (LT32, lts), (AND32, bits)):
        for _ in range(n):
            o = asm.off
            x, y = (int(s) for s in rng.choice(srcs, 2))
            if op in (ADD32, SUB32):
                asm.emit(op, o(dst[0]), o(x), asm.imm(), 0, 1)
            elif op == LT32:
                v = int(rng.choice([LT32, LTE32, SLT32, SLE32]))
                asm.emit(v, o(dst[0]), o(x), asm.imm(), 0, 1) if rng.random() < 0.5 else asm.emit(v, o(dst[0]), asm.imm(), o(x), 1, 0)
            else:
                asm.emit(int(rng.choice([AND32, OR32, XOR32])), o(dst[0]), o(x), asm.imm(), 0, 1)
            n_mem += 2
    ran = len(asm.code)
    if cycles is not None:
        fill = cycles - 1 - ran
    else:
        fill = mem - n_mem
    assert fill >= 0, "the counts do not fit"
    for i in range(fill):
        asm.imm32(srcs[i % 6], asm.word())
    return asm.program(), static, fp


def with_dead_rows(program, seed=0):
    """The program followed by rows no run reaches (after its STOP and callees), whose opcode words are p, p + 1, 2^32 - 1 and
    random: the program chip still holds them, so they must be reduced like every other word."""
    rng = np.random.default_rng(seed)
    dead = [[_i32(op), *(int(v) for v in rng.integers(-(1 << 31), 1 << 31, 5))] for op in (P, P + 1, M32, int(rng.integers(P, 1 << 32)), 0x7FFFFFFF)]
    return np.concatenate([np.asarray(program, dtype=np.int32), np.array(dead, dtype=np.int32)])
