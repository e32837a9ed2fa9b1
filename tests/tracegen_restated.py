"""The plain-Python restatement of `Machine::run` and `Chip::generate_trace` that the host and device witness builders are compared
with (test_tracegen_restatement.py, test_generated_traces.py, test_gpu_witness_generated.py).  Written from the Rust text:

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

Its data structures are its own (a dict of cells, per-clock operation lists, Python's stable sort).  Every u32 the run produces that
becomes a field element (fp, addresses) goes through from_canonical_u32, which reduces mod p."""
import numpy as np

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
        r[FP] %= P                                                    # from_canonical_u32(fp) (cpu/src/lib.rs:172)
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
        prog[n, 1] = (opcode & M32) % P                               # from_canonical_u32 (machine/src/program.rs:44), rows never run included
        prog[n, 2:7] = [felt_i32(x) for x in operands]
    return [main[i] for i in range(14)], [prog, np.arange(256, dtype=np.uint32).reshape(-1, 1)]


CHIPS = "cpu program mem add sub mul div shift lt com bitwise output range static_data".split()


def assert_traces_equal(main_a, prep_a, main_b, prep_b, name_a="a", name_b="b"):
    """Every chip's trace and both preprocessed traces equal in shape and word for word; a failure names the first differing word."""
    for what, xs, ys in (("", main_a, main_b), ("preprocessed ", prep_a, prep_b)):
        assert len(xs) == len(ys)
        for i, (a, b) in enumerate(zip(xs, ys)):
            name = what + (CHIPS[i] if not what else ("program", "range")[i])
            assert a.shape == b.shape, "%s trace: %s %s, %s %s" % (name, name_a, a.shape, name_b, b.shape)
            if not np.array_equal(a, b):
                bad = tuple(np.argwhere(a != b)[0])
                raise AssertionError("%s trace differs first at row %d column %d: %s %d, %s %d"
                                     % (name, bad[0], bad[1], name_a, a[bad], name_b, b[bad]))


def assert_canonical(mats, what):
    """Every word below p: the traces are documented as canonical field elements."""
    for i, m in enumerate(mats):
        if m.size and int(m.max()) >= P:
            bad = tuple(np.argwhere(m >= P)[0])
            raise AssertionError("%s matrix %d: word %d at row %d column %d is not below p" % (what, i, int(m[bad]), bad[0], bad[1]))
