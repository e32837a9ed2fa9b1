"""The product's BabyBear / ext5 arithmetic (valida_b200/csrc/bb.cuh) instantiated on the host and checked against plain Python
integers: Montgomery form R = 2^32, X^5 = 2, Frobenius inverse, bit reversal, two-adic generators.  The same text is what every
kernel compiles; its __CUDA_ARCH__ branches — __umulhi, __brev, the lazy 64-bit accumulators Lazy5 — are checked the same way,
on the device and at their bounds, by test_gpu_bb_device_arith.py.  The host instantiation is what the verifier and the
transcript run."""
import os
import random
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
P = 2013265921
R = (1 << 32) % P
RINV = pow(R, P - 2, P)


def mont(x):
    return x * R % P


def unmont(x):
    return x * RINV % P


def e5_mul_canon(a, b):
    out = [0] * 9
    for i in range(5):
        for j in range(5):
            out[i + j] += a[i] * b[j]
    return [(out[k] + 2 * (out[k + 5] if k + 5 < 9 else 0)) % P for k in range(5)]


def e5_pow_canon(a, e):
    r = [1, 0, 0, 0, 0]
    while e:
        if e & 1:
            r = e5_mul_canon(r, a)
        a = e5_mul_canon(a, a)
        e >>= 1
    return r


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("bb") / "bb_host_check")
    cuda_inc = "/usr/local/cuda/include"
    subprocess.run(["g++", "-O1", "-std=c++17", "-I", os.path.join(ROOT, "valida_b200", "csrc"), "-I", cuda_inc,
                    os.path.join(ROOT, "tests", "c", "bb_host_check.cc"), "-o", out], check=True)
    return out


def run(exe, lines):
    r = subprocess.run([exe], input="\n".join(lines) + "\n", capture_output=True, text=True, check=True)
    return [ln.split() for ln in r.stdout.splitlines()]


def test_base_field(exe):
    rng = random.Random(20260924)
    edge = [0, 1, 2, P - 1, P - 2, (P - 1) // 2, R, 0x78000000, 0x7FFFFFFF % P]
    vals = edge + [rng.randrange(P) for _ in range(300)]
    lines, want = [], []
    for _ in range(600):
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
    # the Montgomery product takes ANY 32-bit left factor (the NTT feeds it unreduced differences A - B + p)
    for _ in range(300):
        a, b = rng.randrange(1 << 32), rng.randrange(P)
        lines.append("mul %d %d" % (a, b)); want.append(a * b * RINV % P)
    # 64-bit lazy sums: any t < 2^64
    for t in [0, 1, (1 << 64) - 1, (1 << 63), 4 * (P - 1) ** 2 + (1 << 60)] + [rng.randrange(1 << 64) for _ in range(300)]:
        lines.append("reduce64 %d" % t); want.append(t * RINV % P)
    got = run(exe, lines)
    assert [int(g[0]) for g in got] == want


def test_bit_reversal_and_generators(exe):
    rng = random.Random(7)
    lines, want = [], []
    for bits in range(0, 28):
        for _ in range(8):
            x = rng.randrange(1 << bits) if bits else 0
            lines.append("revbits %d %d" % (x, bits))
            want.append(int(format(x, "0%db" % bits)[::-1], 2) if bits else 0)
    got = run(exe, lines)
    assert [int(g[0]) for g in got] == want
    gens = [unmont(int(g[0])) for g in run(exe, ["gen %d" % b for b in range(0, 28)])]
    assert gens[0] == 1 and gens[1] == P - 1 and gens[27] == 0x1A427A41
    for b in range(1, 28):
        assert pow(gens[b], 1 << b, P) == 1 and pow(gens[b], 1 << (b - 1), P) == P - 1      # exact order 2^b
        assert gens[b - 1] == gens[b] * gens[b] % P


def test_ext5(exe):
    rng = random.Random(5)
    def rnd():
        return [rng.randrange(P) for _ in range(5)]
    specials = [[0] * 5, [1, 0, 0, 0, 0], [0, 1, 0, 0, 0], [P - 1] * 5, [0, 0, 0, 0, 1]]
    elems = specials + [rnd() for _ in range(120)]
    lines, want = [], []
    for _ in range(400):
        a, b = rng.choice(elems), rng.choice(elems)
        am, bm = " ".join(str(mont(x)) for x in a), " ".join(str(mont(x)) for x in b)
        lines.append("e5mul %s %s" % (am, bm)); want.append([mont(x) for x in e5_mul_canon(a, b)])
        lines.append("e5add %s %s" % (am, bm)); want.append([mont((x + y) % P) for x, y in zip(a, b)])
        lines.append("e5sub %s %s" % (am, bm)); want.append([mont((x - y) % P) for x, y in zip(a, b)])
    got = run(exe, lines)
    assert [[int(x) for x in g] for g in got] == want
    # inverse and Frobenius: a * a^-1 = 1, frob(a) = a^p
    nz = [e for e in elems if any(e)][:40]
    inv = run(exe, ["e5inv " + " ".join(str(mont(x)) for x in a) for a in nz])
    for a, g in zip(nz, inv):
        assert e5_mul_canon(a, [unmont(int(x)) for x in g]) == [1, 0, 0, 0, 0]
    fr = run(exe, ["e5frob " + " ".join(str(mont(x)) for x in a) for a in nz[:6]])
    for a, g in zip(nz[:6], fr):
        assert [unmont(int(x)) for x in g] == e5_pow_canon(a, P)
