"""The device witness (vgpu_witness_device, csrc/witness.cu) against the host builder and the plain restatement on seeded generated
programs (generated_programs.py): every chip and both preprocessed traces word for word.

- Generated programs in every address regime, and with rows that never run whose opcode words are at or above p, with operands that reach lt_rows_kernel's first-differing-byte search, the CPU
  chip's per-row Fermat diff_inv and the immediate paths.
- Tall memory-log sorts in every regime: about 2^16 operations against the restatement (16 tiles of 4096 keys, so the one-block
  scan of 256 * tiles counters loops 4 times), then 2^20 and 2^22 against the host builder (1024 tiles, 262 144 counters).
- Padding extremes: each tall chip with exactly 2^k and 2^k + 1 real rows, the ALU chips also with 0 and 1 operations.
- Split runs at 2, 4 and 8 thread ranks on one GPU: every rank's rows of every chip equal the host rows, with the real/padding
  boundary inside a run and on a run boundary, a static-cell prefix longer than a run, and program and static-data chips tall
  enough to be split (they are built on the host and arrive whole).
- Proofs of a config5-shaped program with static data and of Fibonacci at fp 0x80000000 from the device witness, on one GPU and
  split over 2 ranks: vgpu_prove's bytes on the host traces, the oracle's bytes, accepted by the oracle's verifier."""
import numpy as np
import pytest

from generated_programs import REGIMES, counted_program, generated_program, with_dead_rows
from programs import config5_program
from tracegen_restated import Vm, all_traces, assert_canonical, assert_traces_equal

pytestmark = pytest.mark.gpu
TILE = 4096                        # SORT_TILE of csrc/witness.cu


def _device(ctx, log):
    dm, dp = log.witness_device(ctx)
    return [m.download() for m in dm], [m.download() for m in dp]


def _check(ctx, prog, fp, static_data=None, restate=True):
    """device == host (== restatement); returns the log and the host traces."""
    import valida_b200 as vb

    log = vb.run_program_log(prog, initial_fp=fp, static_data=static_data)
    host = log.traces()
    assert_canonical(host.main + host.preprocessed, "host")
    if restate:
        assert_traces_equal(host.main, host.preprocessed, *all_traces(Vm(prog, fp, static_data).run()), "host", "restatement")
    assert_traces_equal(*_device(ctx, log), host.main, host.preprocessed, "device", "host")
    return log, host


def _sized(regime, seed, n_mem):
    """A generated program of the regime whose memory log has at least n_mem operations (and not many more)."""
    import valida_b200 as vb

    prog, fp = generated_program(seed, regime, 4096)
    per_cycle = vb.run_program_log(prog, initial_fp=fp).mem_ops / 4096
    prog, fp = generated_program(seed, regime, int(n_mem / per_cycle * 1.02) + 64)
    return prog, fp


@pytest.mark.parametrize("regime", REGIMES)
def test_generated_programs(ctx, regime):
    for seed in (11, 12, 13):
        _check(ctx, *generated_program(seed, regime, 3000))


def test_rows_that_never_run_with_opcodes_at_or_above_p(ctx):
    # the program chip is built on the host and uploaded: its opcode words p, 2^32 - 1, ... arrive reduced, as the host builds them
    for regime in "ac":
        prog, fp = generated_program(6, regime, 800)
        _check(ctx, with_dead_rows(prog, 1), fp)


@pytest.mark.parametrize("regime", REGIMES)
def test_tall_sort_against_the_restatement(ctx, regime):
    prog, fp = _sized(regime, 21, 1 << 16)
    log, _ = _check(ctx, prog, fp)
    assert 16 * TILE <= log.mem_ops < 17 * TILE


@pytest.mark.parametrize("log_n", [20, 22])
@pytest.mark.parametrize("regime", REGIMES)
def test_tall_sort_against_the_host(ctx, regime, log_n):
    prog, fp = _sized(regime, 31 + log_n, 1 << log_n)
    log, _ = _check(ctx, prog, fp, restate=False)
    assert (1 << log_n) <= log.mem_ops < (1 << log_n) + (1 << (log_n - 4))
    assert (log.mem_ops + TILE - 1) // TILE >= (1 << log_n) // TILE


PADDING = [("cpu", dict(cycles=1 << 12)), ("cpu", dict(cycles=(1 << 12) + 1)),
           ("mem", dict(mem=(1 << 12) - 9, n_static=9)), ("mem", dict(mem=(1 << 12) + 1 - 9, n_static=9)),
           ("mem", dict(mem=1 << 12)), ("mem", dict(mem=(1 << 12) + 1))]
for _chip in ("adds", "subs", "lts", "bits"):
    PADDING += [(_chip, {_chip: n, "cycles": 3000}) for n in (0, 1, 1 << 10, (1 << 10) + 1)]


@pytest.mark.parametrize("case", range(len(PADDING)))
def test_padding_extremes(ctx, case):
    chip, kw = PADDING[case]
    prog, static, fp = counted_program(100 + case, **kw)
    log, host = _check(ctx, prog, fp, static)
    if chip == "cpu":
        i, n = 0, log.clock
        assert n == kw["cycles"]
    elif chip == "mem":
        i, n = 2, log.mem_ops + len(static)
        assert n == kw["mem"] + kw.get("n_static", 0)
    else:                                                              # real rows: add / sub is_real, lt is_real, bitwise flags
        i = {"adds": 3, "subs": 4, "lts": 8, "bits": 10}[chip]
        n = int(host.main[i][:, {3: [15], 4: [15], 8: [22], 10: [76, 77, 78]}[i]].sum())
        assert n == kw[chip]
    assert host.main[i].shape[0] == max(1, 1 << (n - 1).bit_length()) if n else host.main[i].shape[0] == 1


def _split_program(n):
    """Counts that put each ALU chip's real/padding boundary inside a run or on a run boundary of n ranks, the CPU chip's on a run
    boundary (its last row for 2 ranks), a program chip of more than 2048 * n rows and a static prefix longer than a run."""
    h = 2048 * n                                                       # the smallest split height
    counts = dict(adds=h - h // n if n > 2 else h, subs=h // 2 + h // (2 * n) + 1, lts=h // 2 + 1, bits=h - 1)
    hc = 4 * h
    cycles = hc - hc // n if n > 2 else hc
    prog, static, fp = counted_program(200 + n, cycles=cycles, n_static=1, **counts)
    import valida_b200 as vb

    m = vb.run_program_log(prog, initial_fp=fp, static_data=static).mem_ops + 64
    hm = 1 << (4 * m - 1).bit_length()
    n_static = hm // 2 + hm // 8                                       # > hm / n, and n_static + m <= hm
    return counted_program(200 + n, cycles=cycles, n_static=n_static, **counts), counts, cycles


@pytest.mark.parametrize("n", [2, 4, 8])
def test_split_witness_rows(ctx, n):
    import torch
    import valida_b200 as vb

    (prog, static, fp), counts, cycles = _split_program(n)
    log = vb.run_program_log(prog, initial_fp=fp, static_data=static)
    host = log.traces()
    mats = host.main + host.preprocessed
    assert log.clock == cycles and len(prog) > 2048 * n and len(static) > 2048 * n
    assert len(static) > host.main[2].shape[0] // n and len(static) + log.mem_ops <= host.main[2].shape[0]
    k = torch.cuda.device_count()
    ctxs = [vb.Context(i % k) for i in range(n)]
    try:
        vb.comm_init_local(ctxs)

        def rank(r, c):
            dm, dp = log.witness_device(c)
            split = 0
            for i, (m, a) in enumerate(zip(dm + dp, mats)):
                r0, rows = m.local_rows()
                assert m.shape == a.shape
                if i in (0, 2, 3, 4, 8, 10):                           # built on the device: this rank's run of rows
                    assert (r0, rows) == c.local_rows(a.shape[0]) and rows == a.shape[0] // n, (i, r0, rows)
                    split += 1
                got = m.download()[r0:r0 + rows]
                if not np.array_equal(got, a[r0:r0 + rows]):
                    bad = np.argwhere(got != a[r0:r0 + rows])[0]
                    raise AssertionError("rank %d matrix %d: row %d column %d: device %d, host %d"
                                         % (r, i, r0 + bad[0], bad[1], got[tuple(bad)], a[r0 + bad[0], bad[1]]))
            return split

        assert vb.run_ranks(rank, ctxs) == [6] * n
    finally:
        for c in ctxs:
            c.close()


def _config5_static():
    """config5_program with four static cells, two of them loaded after the loop (provable: static addresses below p)."""
    p = config5_program(300)[:-1].tolist()
    p += [[7, -52, 0, 0, 0, 0x10], [1, -56, 0, -52, 0, 0], [7, -60, 0, 0, 0, 0x1c], [1, -64, 0, -60, 0, 0], [8, 0, 0, 0, 0, 0]]
    return np.array(p, dtype=np.int32), {0x10: 5, 0x14: 0xFFFFFFFF, 0x18: 0x78000001, 0x1c: 0x80000000}, 0x1000


@pytest.mark.parametrize("which", ["config5_static", "fib_fp_0x80000000"])
def test_proofs_from_the_device_witness(ctx, oracle, which):
    import torch
    import valida_b200 as vb

    prog, static, fp = _config5_static() if which == "config5_static" else (vb.fib_program(582), None, 0x80000000)
    log, host = _check(ctx, prog, fp, static)
    cfg = vb.StarkConfig(ctx, oracle.rc480)
    ref = vb.prove_machine(cfg, host)
    assert ref == oracle.prove(host.main, host.preprocessed, debug_checks=False).cbor()
    assert oracle.verify(ref, host.preprocessed) == 0
    dm, dp = log.witness_device(ctx)
    assert vb.prove_machine(cfg, host, device_resident=(dm, dp)) == ref
    k = torch.cuda.device_count()
    ctxs = [vb.Context(i % k) for i in range(2)]
    try:
        vb.comm_init_local(ctxs)
        cfgs = [vb.StarkConfig(c, oracle.rc480) for c in ctxs]
        assert vb.run_ranks(lambda r, c: vb.prove_machine(cfgs[r], host, device_resident=log.witness_device(c)), ctxs) == [ref, ref]
    finally:
        for c in ctxs:
            c.close()
