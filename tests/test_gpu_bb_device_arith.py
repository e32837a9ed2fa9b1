"""The product's BabyBear / ext5 arithmetic (valida_b200/csrc/bb.cuh) as the kernels compile it — the __CUDA_ARCH__ branches:
__umulhi in mul and monty_reduce64, __brev, the lazy 64-bit accumulators Lazy5 / madw / lazy_fold and the device e5_mul built on
them — checked against plain Python integers.  The device twin of test_bb_host_arith.py: tests/c/bb_device_check.cu reads the
same line protocol as tests/c/bb_host_check.cc.

Lazy5 is driven to its bound: a limb folded from 2^64 - 1 (just under 2^60 + 2^32) with four pending products of (p-1)^2 is
1.737e19 against 2^64 = 1.845e19, and a fifth product would wrap.  The quotient, the permutation traces, the barycentric sums and
the reduced openings all rely on that bound; random field elements never get near it."""
import os
import random
import subprocess

import pytest

from test_bb_host_arith import P, R, RINV, e5_mul_canon, mont, unmont

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
R1 = 0x0FFFFFFE                     # Montgomery one, the multiplier of lazy_fold's high word
M64 = (1 << 64) - 1


def compile_twin(out):
    subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "-I",
                    os.path.join(ROOT, "valida_b200", "csrc"), os.path.join(ROOT, "tests", "c", "bb_device_check.cu"), "-o", out],
                   check=True)
    return out


def test_device_twin_compiles_for_sm_90a(tmp_path):
    assert os.path.getsize(compile_twin(str(tmp_path / "bb_device_check"))) > 0


@pytest.fixture(scope="module")
def exe(built, tmp_path_factory):
    return compile_twin(str(tmp_path_factory.mktemp("bbd") / "bb_device_check"))


def run(exe, lines):
    r = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True)
    out = [[int(x) for x in ln.split()] for ln in r.stdout.splitlines()]
    assert len(out) == len(lines)
    return out


def lazy_fold(t):
    return (t >> 32) * R1 + (t & 0xFFFFFFFF)


def lazy_expected(t, nbase, next_, v):
    """Lazy5 preset to lazy_fold(t) on every limb, nbase x fma_base((v,)*5, v), next_ x fma_ext(x, x, 2x): value() = sum / 2^32."""
    v2 = (2 * v) % P
    out = []
    for k in range(5):
        s = lazy_fold(t) + nbase * v * v + next_ * ((k + 1) * v * v + (4 - k) * v * v2)
        out.append(s * RINV % P)
    return out


@pytest.mark.gpu
def test_base_field_on_device(exe):
    rng = random.Random(20261015)
    edge = [0, 1, 2, P - 1, P - 2, (P - 1) // 2, R, 0x78000000, 0x7FFFFFFF % P]
    vals = edge + [rng.randrange(P) for _ in range(200)]
    lines, want = [], []
    for _ in range(400):
        a, b = rng.choice(vals), rng.choice(vals)
        lines.append("mul %d %d" % (mont(a), mont(b))); want.append(mont(a * b % P))
        lines.append("add %d %d" % (mont(a), mont(b))); want.append(mont((a + b) % P))
        lines.append("sub %d %d" % (mont(a), mont(b))); want.append(mont((a - b) % P))
    for a in vals:
        lines.append("neg %d" % mont(a)); want.append(mont(-a % P))
        lines.append("to_monty %d" % a); want.append(mont(a))
        lines.append("from_monty %d" % mont(a)); want.append(a)
        if a:
            lines.append("inv %d" % mont(a)); want.append(mont(pow(a, P - 2, P)))
        e = rng.randrange(1 << 40)
        lines.append("pow %d %d" % (mont(a), e)); want.append(mont(pow(a, e, P)))
    # the Montgomery product takes ANY 32-bit left factor (the NTT feeds it unreduced differences A - B + p), up to 2^32 - 1
    for a in [(1 << 32) - 1, 1 << 31, P, 2 * P - 1] + [rng.randrange(1 << 32) for _ in range(300)]:
        for b in (P - 1, 1, rng.randrange(P)):
            lines.append("mul %d %d" % (a, b)); want.append(a * b * RINV % P)
    # 64-bit lazy sums: any t < 2^64, including a high word >= 2p (two conditional subtractions)
    for t in [0, 1, M64, 1 << 63, (2 * P) << 32, ((2 * P) << 32) - 1, (P << 32) | 0xFFFFFFFF, 4 * (P - 1) ** 2 + (1 << 60),
              lazy_fold(M64) + 4 * (P - 1) ** 2] + [rng.randrange(1 << 64) for _ in range(300)]:
        lines.append("reduce64 %d" % t); want.append(t * RINV % P)
    got = run(exe, lines)
    assert [g[0] for g in got] == want


@pytest.mark.gpu
def test_bit_reversal_and_generators_on_device(exe):
    rng = random.Random(8)
    lines, want = [], []
    for bits in range(0, 28):
        for x in ([0, (1 << bits) - 1, 1, 1 << (bits - 1)] if bits else [0]) + [rng.randrange(1 << bits) if bits else 0 for _ in range(8)]:
            lines.append("revbits %d %d" % (x, bits))
            want.append(int(format(x, "0%db" % bits)[::-1], 2) if bits else 0)
    assert [g[0] for g in run(exe, lines)] == want
    gens = [unmont(g[0]) for g in run(exe, ["gen %d" % b for b in range(0, 28)])]
    assert gens == [pow(0x1A427A41, 1 << (27 - b), P) for b in range(28)]


@pytest.mark.gpu
def test_lazy5_at_its_bound(exe):
    assert lazy_fold(M64) + 4 * (P - 1) ** 2 < 1 << 64 <= lazy_fold(M64) + 5 * (P - 1) ** 2     # the bound is tight
    assert 5 * (P - 1) ** 2 >= 1 << 64                                                              # five products wrap even from 0
    rng = random.Random(3)
    cases = []
    for nbase in (0, 1, 3, 4):
        for nxt in range(0, 14):                 # the fold lands on every step of fma_ext's five-round loop
            cases.append((M64, nbase, nxt, P - 1))
            cases.append((0, nbase, nxt, P - 1))
    for _ in range(60):
        cases.append((rng.choice([M64, rng.randrange(1 << 64)]), rng.randrange(5), rng.randrange(14), rng.choice([P - 1, P - 2, rng.randrange(P)])))
    got = run(exe, ["lazy %d %d %d %d" % c for c in cases])
    for c, g in zip(cases, got):
        assert g == lazy_expected(*c), c


@pytest.mark.gpu
def test_ext5_on_device(exe):
    rng = random.Random(6)

    def rnd():
        return [rng.randrange(P) for _ in range(5)]
    specials = [[0] * 5, [1, 0, 0, 0, 0], [0, 1, 0, 0, 0], [P - 1] * 5, [0, 0, 0, 0, 1], [P - 1, 0, 0, 0, 0], [0, 0, 0, 0, P - 1]]
    elems = specials + [rnd() for _ in range(80)]
    lines, want = [], []
    for a in specials:                           # every pair of specials, then random pairs
        for b in specials:
            lines.append("e5mul %s %s" % (" ".join(str(mont(x)) for x in a), " ".join(str(mont(x)) for x in b)))
            want.append([mont(x) for x in e5_mul_canon(a, b)])
    for _ in range(300):
        a, b = rng.choice(elems), rng.choice(elems)
        am, bm = " ".join(str(mont(x)) for x in a), " ".join(str(mont(x)) for x in b)
        lines.append("e5mul %s %s" % (am, bm)); want.append([mont(x) for x in e5_mul_canon(a, b)])
        lines.append("e5add %s %s" % (am, bm)); want.append([mont((x + y) % P) for x, y in zip(a, b)])
        lines.append("e5sub %s %s" % (am, bm)); want.append([mont((x - y) % P) for x, y in zip(a, b)])
    # raw words p - 1 in every limb: the largest products the device e5_mul accumulates
    lines.append("e5mul %s %s" % (" ".join([str(P - 1)] * 5), " ".join([str(P - 1)] * 5)))
    want.append([x * RINV % P for x in e5_mul_canon([P - 1] * 5, [P - 1] * 5)])
    assert run(exe, lines) == want
    # inverses: base-field elements (c1..c4 = 0), elements with c0 = 0, random ones; a * a^-1 = 1 and the base-field inverse exact
    base = [[x, 0, 0, 0, 0] for x in (1, 2, P - 1, 7, rng.randrange(1, P))]
    c0zero = [[0] + rnd()[1:] for _ in range(6)] + [[0, 1, 0, 0, 0], [0, 0, 0, 0, 1], [0, P - 1, P - 1, P - 1, P - 1]]
    nz = base + c0zero + [rnd() for _ in range(10)]
    inv = run(exe, ["e5inv " + " ".join(str(mont(x)) for x in a) for a in nz])
    for a, g in zip(nz, inv):
        assert e5_mul_canon(a, [unmont(x) for x in g]) == [1, 0, 0, 0, 0], a
    for a, g in zip(base, inv):
        assert [unmont(x) for x in g] == [pow(a[0], P - 2, P), 0, 0, 0, 0]
