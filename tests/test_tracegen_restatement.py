"""A second reading, in plain Python and written from the Rust text, of the INPUT side of the proving path: `Machine::run`
(basic/src/lib.rs:127-145, 1063-1188) and `Chip::generate_trace` of the chips a Fibonacci-class program reaches —

    instruction semantics     cpu/src/lib.rs:440-872 (load32, store32, jal, jalv, beq, bne, imm32, stop, loadfp),
                              alu_u32/src/add/mod.rs:138-169, alu_u32/src/sub/mod.rs:126-166
    CPU rows                  cpu/src/lib.rs:79-97 (generate_trace), 163-236 (op_to_row), 244-284 (memory channels),
                              286-321 (word diffs), 323-362 (STOP padding), 364-381 (immediates); columns cpu/src/columns.rs:8-75
    memory rows               memory/src/lib.rs:143-194, 237-263; columns memory/src/columns.rs:8-41
    add / sub rows            alu_u32/src/add/mod.rs:38-129, alu_u32/src/sub/mod.rs:90-117
    lt family                 alu_u32/src/lt/mod.rs:87-165 (rows), 167-216 (operands incl. LEFT immediates), 232-309; Word ordering machine/src/core.rs:321-330
    and / or / xor            alu_u32/src/bitwise/mod.rs:84-131 (rows), 140-254
    mul floor                 alu_u32/src/mul/mod.rs:38-64 (2^10 counter rows)
    static data               static_data/src/lib.rs:26-33 (initialize_memory), 59-79 (rows); memory/src/lib.rs:132-135, 163-169, 265-283
    range / program           range/src/lib.rs:32-72, range/src/stark.rs:22-25, program/src/lib.rs:38-48, 73-80, program/src/stark.rs:22-40

— compared WORD FOR WORD with the product's host witness generator (valida_b200/csrc/host/tracegen.cc via vgpu_machine_run).
The trace digests of tests/golden/trace_hashes.json pin the generator against itself; this file is the independent text
(data structures of its own: a dict of cells, per-clock operation lists, Python's stable sort), like test_perm_trace_restatement.py
and test_quotient_restatement.py are for the LogUp and quotient code.  No GPU."""
import numpy as np
import pytest

from programs import loads_stores_edge_program, lt_edge_operands_program, single_address_program

P = 2013265921
LOAD32, STORE32, JAL, JALV, BEQ, BNE, IMM32, STOP, LOADFP, ADD32, SUB32 = 1, 2, 3, 4, 5, 6, 7, 8, 10, 100, 101
LT32, AND32, OR32, XOR32, LTE32, SLT32, SLE32 = 104, 107, 108, 109, 115, 117, 118
BYTES_PER_INSTR = 24
M32 = 0xFFFFFFFF


def word(v):                       # From<u32> for Word<u8>: big-endian bytes (machine/src/core.rs:99-107)
    v &= M32
    return ((v >> 24) & 255, (v >> 16) & 255, (v >> 8) & 255, v & 255)


def u32(w):                        # Into<u32> (core.rs:83-91)
    return (w[0] << 24) | (w[1] << 16) | (w[2] << 8) | w[3]


def felt_i32(x):                   # Operands::from_i32_slice (machine/src/program.rs:157-164): -abs for negatives
    return (P - (-x) % P) % P if x < 0 else x % P


def next_pow2(n):                  # usize::next_power_of_two: 0 -> 1
    p = 1
    while p < n:
        p *= 2
    return p


class Vm:
    """BasicMachine as the reference's prove_program sets it up (basic/tests/test_prover.rs:403-411): fp = 0x1000, the initial
    register state saved by hand, then run()."""

    def __init__(self, program, fp=0x1000, static_data=None):
        self.program = [(int(r[0]), [int(x) for x in r[1:6]]) for r in program]
        self.counts = [0] * len(self.program)
        self.pc, self.fp, self.clock = 0, fp, 0
        self.registers = [(self.pc, self.fp)]           # save_register_state()
        self.ops, self.instrs = [], []
        self.static = {a: word(v) for a, v in sorted((static_data or {}).items())}     # BTreeMap<u32, Word<u8>>
        self.cells = dict(self.static)                   # initialize_memory -> write_static: no operation is logged
        self.mem_ops = {}                                # clk -> [(kind, addr, word)], BTreeMap<u32, Vec<Operation>>
        self.adds, self.subs, self.lts, self.bits = [], [], [], []
        self.range_count = {}

    # memory chip (memory/src/lib.rs:85-130)
    def read(self, addr):
        addr &= M32
        if addr not in self.cells:
            raise RuntimeError("read before write: %d" % addr)
        v = self.cells[addr]
        self.mem_ops.setdefault(self.clock, []).append(("R", addr, v))
        return v

    def write(self, addr, w):
        addr &= M32
        self.mem_ops.setdefault(self.clock, []).append(("W", addr, w))
        self.cells[addr] = w

    def push_op(self, kind, imm, opcode, operands):     # cpu/src/lib.rs:907-922
        self.ops.append((kind, imm))
        self.instrs.append((opcode, operands))
        self.registers.append((self.pc, self.fp))
        self.clock += 1

    def range_check(self, w):                           # range/src/lib.rs:62-70
        for b in w:
            self.range_count[b] = self.range_count.get(b, 0) + 1

    def step(self):
        pc = self.pc
        opcode, o = self.program[pc]
        a, b, c, d, e = o
        fp = self.fp
        if opcode == LOAD32:
            addr2 = u32(self.read(fp + c))
            cell = self.read(addr2)
            self.write(fp + a, cell)
            self.pc += 1
            self.push_op("load", None, opcode, o)
        elif opcode == STORE32:
            waddr = u32(self.read(fp + b))
            cell = self.read(fp + c)
            self.write(waddr, cell)
            self.pc += 1
            self.push_op("store", None, opcode, o)
        elif opcode == JAL:
            self.write(fp + a, word(BYTES_PER_INSTR * (pc + 1)))
            self.pc = (b & M32) // BYTES_PER_INSTR
            self.fp = (fp + c) & M32
            self.push_op("jal", None, opcode, o)
        elif opcode == JALV:
            self.write(fp + a, word(BYTES_PER_INSTR * (pc + 1)))
            self.pc = u32(self.read(fp + b)) // BYTES_PER_INSTR
            off = u32(self.read(fp + c))                # read with the OLD fp (state.cpu().fp is still unchanged)
            self.fp = (fp + off) & M32                  # cell as i32, two's complement add
            self.push_op("jalv", None, opcode, o)
        elif opcode in (BEQ, BNE):
            imm = None
            c1 = self.read(fp + b)
            if e == 1:
                c2 = imm = word(c)
            else:
                c2 = self.read(fp + c)
            taken = (c1 == c2) if opcode == BEQ else (c1 != c2)
            self.pc = (a & M32) // BYTES_PER_INSTR if taken else pc + 1
            self.push_op("beq" if opcode == BEQ else "bne", imm, opcode, o)
        elif opcode == IMM32:
            self.write(fp + a, (b & 255, c & 255, d & 255, e & 255))
            self.pc += 1
            self.push_op("imm32", None, opcode, o)
        elif opcode == STOP:
            self.push_op("stop", None, opcode, o)
        elif opcode == LOADFP:
            self.write(fp + a, word(fp + b))
            self.pc += 1
            self.push_op("loadfp", None, opcode, o)
        elif opcode in (ADD32, SUB32):
            imm = None
            bw = self.read(fp + b)
            if e == 1:
                cw = imm = word(c)
            else:
                cw = self.read(fp + c)
            aw = word(u32(bw) + u32(cw)) if opcode == ADD32 else word(u32(bw) - u32(cw))
            self.write(fp + a, aw)
            (self.adds if opcode == ADD32 else self.subs).append((aw, bw, cw))
            self.pc += 1                                # push_bus_op
            self.push_op("bus", imm, opcode, o)
            self.range_check(aw)
        elif opcode in (LT32, LTE32, SLT32, SLE32):       # Lt32Chip::execute_with_closure
            imm = None
            if d == 1:
                src1 = imm = word(b)
            else:
                src1 = self.read(fp + b)
            if e == 1:
                src2 = imm = word(c)                    # with both flags set the LATER immediate is the one recorded
            else:
                src2 = self.read(fp + c)
            if opcode in (LT32, LTE32):                 # Ord for Word<u8>: lexicographic on the big-endian bytes
                x, y = src1, src2
            else:                                       # Into<i32>: two's complement
                x, y = u32(src1) - ((u32(src1) >> 31) << 32), u32(src2) - ((u32(src2) >> 31) << 32)
            res = (x < y) if opcode in (LT32, SLT32) else (x <= y)
            dst = word(1 if res else 0)
            self.write(fp + a, dst)
            self.pc += 1
            self.push_op("bus_left" if d == 1 else "bus", imm, opcode, o)
            self.lts.append((opcode, dst, src1, src2))
        elif opcode in (AND32, OR32, XOR32):
            imm = None
            bw = self.read(fp + b)
            if e == 1:
                cw = imm = word(c)
            else:
                cw = self.read(fp + c)
            f = {AND32: lambda x, y: x & y, OR32: lambda x, y: x | y, XOR32: lambda x, y: x ^ y}[opcode]
            aw = tuple(f(x, y) for x, y in zip(bw, cw))
            self.write(fp + a, aw)
            self.bits.append((opcode, aw, bw, cw))
            self.pc += 1
            self.push_op("bus", imm, opcode, o)
        else:
            raise RuntimeError("opcode %d is outside this restatement" % opcode)
        self.counts[pc] += 1                            # read_word(pc) AFTER the execution, with the pc that was fetched
        return opcode == STOP

    def run(self):
        while not self.step():
            pass
        n = next_pow2(self.clock) - self.clock          # "Record padded STOP instructions" (basic/src/lib.rs:140-144)
        self.counts[self.pc] += n
        return self


# ---- column maps (cpu/src/columns.rs, memory/src/columns.rs) ------------------------------------------------------------------
CLK, PC, FP, OPCODE, OPERANDS = 0, 1, 2, 3, 4
FLAGS = {name: 9 + i for i, name in enumerate(
    ["bus_op", "bus_op_with_mem", "imm_op", "left_imm_op", "load", "load_u8", "load_s8", "store", "store_u8", "beq", "bne", "jal", "jalv",
     "imm32", "advice", "stop", "loadfp"])}
DIFF, DIFF_INV, NOT_EQUAL = 26, 27, 28
CH = [29, 36, 43]                  # used, is_read, addr, value[4]
NUM_CPU_COLS = 51


def cpu_trace(vm):
    rows = []
    for clk, (kind, imm) in enumerate(vm.ops):
        r = [0] * NUM_CPU_COLS
        r[PC], r[FP] = vm.registers[clk]
        r[CLK] = clk
        opcode, operands = vm.instrs[clk]
        r[OPCODE] = opcode
        for i, x in enumerate(operands):
            r[OPERANDS + i] = felt_i32(x)
        r[FLAGS["bus_op" if kind in ("bus", "bus_left") else kind]] = 1
        if kind in ("beq", "bne", "bus") and imm is not None:         # set_imm_value
            r[FLAGS["imm_op"]] = 1
            for i in range(4):
                r[CH[1] + 3 + i] = imm[i]
            r[OPERANDS + 2] = u32(imm) % P                            # Word::reduce of the immediate's bytes
        if kind == "bus_left" and imm is not None:                    # set_left_imm_value
            r[FLAGS["left_imm_op"]] = 1
            for i in range(4):
                r[CH[0] + 3 + i] = imm[i]
            r[OPERANDS + 1] = u32(imm) % P
        r[CH[0] + 1] = r[CH[1] + 1] = 1                               # is_read of the two read channels
        first_read = r[FLAGS["left_imm_op"]] == 0                     # a left-immediate op's only read takes the SECOND channel
        for op, addr, val in vm.mem_ops.get(clk, []):
            ch = 2
            if op == "R":
                ch = 0 if first_read else 1
                first_read = False
            r[CH[ch]] = 1
            r[CH[ch] + 2] = addr % P
            for i in range(4):
                r[CH[ch] + 3 + i] = val[i]
        rows.append(r)
    for r in rows:                                                    # compute_word_diffs
        d = sum((r[CH[0] + 3 + i] - r[CH[1] + 3 + i]) ** 2 for i in range(4)) % P
        r[DIFF] = d
        r[DIFF_INV] = pow(d, P - 2, P) if d else 0
        r[NOT_EQUAL] = 1 if d else 0
    last = rows[-1]
    for n in range(next_pow2(len(rows)) - len(rows)):                 # pad_to_power_of_two: STOP rows
        r = [0] * NUM_CPU_COLS
        r[PC], r[FP], r[CLK] = last[PC], last[FP], (last[CLK] + n + 1) % P
        r[FLAGS["stop"]] = 1
        r[OPCODE] = STOP
        r[CH[0] + 1] = r[CH[1] + 1] = 1
        rows.append(r)
    return np.array(rows, dtype=np.uint64).astype(np.uint32)


def mem_trace(vm):
    ops = [(clk, op) for clk in sorted(vm.mem_ops) for op in vm.mem_ops[clk]]
    ops.sort(key=lambda t: (t[1][1], t[0]))                           # sort_by_key((addr, clk)): stable
    rows = []
    for n, (addr, val) in enumerate(vm.static.items()):                # static_data_to_row: these rows OPEN the trace
        r = [0] * 14
        r[0], r[1:5], r[6], r[8], r[12] = addr % P, val, 1, 1, n
        rows.append(r)
    n0 = len(rows)
    for n, (clk, (kind, addr, val)) in enumerate(ops):
        r = [0] * 14
        r[0] = addr % P
        r[1:5] = val
        r[5] = clk
        r[7 if kind == "R" else 8] = 1
        r[12] = n0 + n                                                 # counter
        rows.append(r)
    rows += [[0] * 14] * (next_pow2(len(rows)) - len(rows))
    return np.array(rows, dtype=np.uint32)


def alu_trace(ops, is_add):
    rows = []
    for a, b, c in ops:
        r = [0] * 16
        r[0:4], r[4:8], r[11:15], r[15] = b, c, a, 1
        if is_add:                                                     # carries (add/mod.rs:110-124)
            c1 = 1 if b[3] + c[3] > 255 else 0
            c2 = 1 if b[2] + c[2] + c1 > 255 else 0
            c3 = 1 if b[1] + c[1] + c2 > 255 else 0
            r[8:11] = [c1, c2, c3]
        else:                                                          # borrows as the reference writes them (sub/mod.rs:103-111)
            r[8:11] = [int(b[3] < c[3]), int(b[2] < c[2]), int(b[1] < c[1])]
        rows.append(r)
    rows += [[0] * 16] * (next_pow2(len(rows)) - len(rows))
    return np.array(rows, dtype=np.uint32)


def lt_trace(ops):
    rows = []
    for opcode, a, b, c in ops:
        r = [0] * 45
        r[{LT32: 23, LTE32: 24, SLT32: 25, SLE32: 26}[opcode]] = 1
        r[0:4], r[4:8], r[21] = b, c, a[3]
        n = next((i for i in range(4) if b[i] != c[i]), None)
        if n is not None:
            z = 256 + b[n] - c[n]
            for i in range(9):
                r[12 + i] = (z >> i) & 1
            r[8 + n] = 1
            r[27] = pow((b[n] - c[n]) % P, P - 2, P)
        for i in range(8):
            r[28 + i] = (b[0] >> i) & 1
            r[36 + i] = (c[0] >> i) & 1
        r[44] = int(opcode in (SLT32, SLE32) and r[28 + 7] != r[36 + 7])
        r[22] = 1
        rows.append(r)
    rows += [[0] * 45] * (next_pow2(len(rows)) - len(rows))
    return np.array(rows, dtype=np.uint64).astype(np.uint32)


def bitwise_trace(ops):
    rows = []
    for opcode, a, b, c in ops:
        r = [0] * 79
        r[0:4], r[4:8], r[72:76] = b, c, a
        for i in range(4):
            for j in range(8):
                r[8 + 8 * i + j] = (b[i] >> j) & 1
                r[40 + 8 * i + j] = (c[i] >> j) & 1
        r[{AND32: 76, OR32: 77, XOR32: 78}[opcode]] = 1
        rows.append(r)
    rows += [[0] * 79] * (next_pow2(len(rows)) - len(rows))
    return np.array(rows, dtype=np.uint32)


def all_traces(vm):
    main = {0: cpu_trace(vm), 2: mem_trace(vm), 3: alu_trace(vm.adds, True), 4: alu_trace(vm.subs, False), 8: lt_trace(vm.lts), 10: bitwise_trace(vm.bits)}
    counts = vm.counts + [0] * (next_pow2(len(vm.counts)) - len(vm.counts))
    main[1] = np.array(counts, dtype=np.uint32).reshape(-1, 1)
    mul = np.zeros((1024, 18), dtype=np.uint32)
    mul[:, 17] = np.arange(1, 1025)
    main[5] = mul
    rng = np.zeros((256, 2), dtype=np.uint32)
    for v, cnt in vm.range_count.items():
        rng[v, 0] = cnt
    rng[:, 1] = np.arange(256)
    main[12] = rng
    for chip, w in ((6, 14), (7, 28), (9, 14), (11, 7)):              # no operation: one zero row
        main[chip] = np.zeros((1, w), dtype=np.uint32)
    sd = [[a % P, *v, 1] for a, v in vm.static.items()]
    sd += [[0] * 6] * (next_pow2(len(sd)) - len(sd))
    main[13] = np.array(sd, dtype=np.uint32)
    prog = np.zeros((next_pow2(len(vm.program)), 7), dtype=np.uint32)
    prog[:, 0] = np.arange(prog.shape[0])
    for n, (opcode, operands) in enumerate(vm.program):
        prog[n, 1] = opcode
        prog[n, 2:7] = [felt_i32(x) for x in operands]
    return [main[i] for i in range(14)], [prog, np.arange(256, dtype=np.uint32).reshape(-1, 1)]


def check(program, fp=0x1000, static_data=None):
    import valida_b200 as vb

    got = vb.run_program(program, initial_fp=fp, static_data=static_data)
    vm = Vm(program, fp, static_data).run()
    main, prep = all_traces(vm)
    names = "cpu program mem add sub mul div shift lt com bitwise output range static_data".split()
    for i, (a, b) in enumerate(zip(got.main, main)):
        assert a.shape == b.shape, (names[i], a.shape, b.shape)
        if not np.array_equal(a, b):
            bad = np.argwhere(a != b)[0]
            raise AssertionError("%s trace differs first at row %d column %d: generator %d, restatement %d" % (names[i], bad[0], bad[1], a[tuple(bad)], b[tuple(bad)]))
    for a, b in zip(got.preprocessed, prep):
        assert np.array_equal(a, b)
    return vm, got


@pytest.mark.parametrize("n", [0, 1, 3, 25, 582, 2339, 9359])       # 9359: 2^16 CPU rows, 2^18 memory rows — the sizes at which the generator uses all threads
def test_fibonacci_traces_word_for_word(built, n):
    import valida_b200 as vb

    vm, got = check(vb.fib_program(n))
    if n == 25:                                                        # the reference test's own figures (basic/tests/test_prover.rs:479-486)
        assert (vm.clock, sum(len(v) for v in vm.mem_ops.values()), len(vm.adds)) == (192, 401, 105)
        assert vm.cells[(0x1000 + 4) & M32] == (0, 1, 37, 17)          # Word([0, 1, 37, 17]) = fib(25) = 75025


def _ins(op, a=0, b=0, c=0, d=0, e=0):
    return [op, a, b, c, d, e]


def test_loads_stores_loadfp_sub_and_signed_immediates(built):
    # every instruction of the restated subset that the Fibonacci program does not reach (tests/programs.py; the device witness
    # and the GPU proof are checked on the same program in test_gpu_witness.py / test_gpu_prove.py)
    vm, got = check(loads_stores_edge_program())
    assert vm.cells[(0x1000 - 36) & M32] == word(254) and vm.pc == 13 and vm.fp == 0x1000
    assert len(vm.subs) == 2 and len(vm.adds) == 1


def test_degenerate_memory_logs(built):
    # a lone STOP (no memory operation at all) and a log whose every operation is at one address
    vm, got = check(np.array([_ins(STOP)], dtype=np.int32))
    assert vm.clock == 1 and not vm.mem_ops
    vm, got = check(single_address_program(5))
    assert {addr for ops in vm.mem_ops.values() for _, addr, _ in ops} == {(0x1000 - 4) & M32}


def test_the_references_other_test_programs_and_the_multi_chip_mixes(built):
    # basic/tests/test_prover.rs:490-625 (left immediates, signed inequalities, loadfp) as recorded in tests/golden/programs.json,
    # and the synthetic programs of tests/programs.py (add, sub, lt family incl. left immediates, and / or / xor, bne back-edge)
    import json
    import os

    from programs import config5_program, mixed_program

    golden = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "programs.json")))
    for name in ("left_imm_ops_program", "signed_inequality_program", "loadfp_program"):
        vm, _ = check(np.array(golden[name]["program"], dtype=np.int32))
        for addr, value in golden[name]["expected_cells"]:                 # the reference tests' own assertions on mem().cells
            assert u32(vm.cells[addr & M32]) == value & M32, (name, hex(addr))
    vm, _ = check(mixed_program(37))
    assert len(vm.lts) == 4 * 37 and len(vm.adds) == 3 * 37
    vm, _ = check(config5_program(40))
    assert len(vm.bits) == 6 * 40 and len(vm.subs) == 2 * 40 and len(vm.lts) == 4 * 40
    big = ((1 << 16) - 8) // 15                                                # 2^16 CPU rows: every chip's multi-threaded row fill
    vm, _ = check(config5_program(big))
    assert vm.clock == 3 + 15 * big + 1 and len(vm.bits) == 6 * big


def test_lt_family_edge_operands(built):
    # equal operands (no differing byte: flags, bits and diff_inv stay zero), operands that differ in the TOP byte only, sign
    # boundaries, both immediates at once (the recorded immediate is the right one, written through the LEFT-immediate path)
    vm, _ = check(lt_edge_operands_program())
    assert u32(vm.cells[(0x1000 - 100) & M32]) == 1 and u32(vm.cells[(0x1000 - 104) & M32]) == 1


def test_static_data_program(built):
    # prove_static_data (basic/tests/test_static_data.rs:30-113): two static cells, one of them loaded through a pointer
    from programs import static_data_program

    prog, cells = static_data_program()
    vm, got = check(prog, static_data=cells)
    assert vm.clock == 4 and u32(vm.cells[(0x1000 - 4) & M32]) == 0x25
    # more cells than a power of two, out of address order on the way in, one of them overwritten by the program later
    prog2 = np.array([_ins(IMM32, 0, 0, 0, 0, 0x20), _ins(LOAD32, -4, 0, 0), _ins(ADD32, -8, -4, 5, 0, 1), _ins(LOADFP, -12, -8),
                      _ins(IMM32, -16, 0, 0, 0, 0x18), _ins(STORE32, 0, -16, -8), _ins(STOP)], dtype=np.int32)
    vm, got = check(prog2, static_data={0x20: 1000, 0x10: 7, 0x18: 9})
    assert u32(vm.cells[0x18]) == 1005 and got.main[13].shape == (4, 6) and got.main[2][:3, 6].tolist() == [1, 1, 1]
