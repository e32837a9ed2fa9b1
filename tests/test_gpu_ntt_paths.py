"""Every NTT pass shape the prover can run, compared word for word with an exact reference.

`csrc/ntt.cu` splits each transform into one or two passes and runs each pass through one of several load and store
branches, chosen on the host from the height alone.  The first half of this module restates that host dispatch in plain
Python (the model) and checks, without a GPU, that the grid of GPU cases below reaches every (sub-transform length,
load branch, store branch, pre-multiplier, post-multiplier) that any entry point can reach up to 2^27 rows.  The GPU tests
then run that grid against:
  * the defining sums (exact integer arithmetic) up to 2^10 rows;
  * the oracle's dft / coset_lde up to ORACLE_MAX_LOG;
  * above that, identities that need multiplications only: the DFT of a geometric column, and the coset LDE with a
    shift inside the 2n-th roots of unity, whose bit-reversed rows are the input rotated.
Every GPU case also checks that the call launches exactly the passes the model predicts.
"""
import os
import re
from collections import namedtuple

import numpy as np
import pytest

P = 2013265921
G27 = 0x1A427A41                       # two-adic generator of order 2^27
HERE = os.path.dirname(os.path.abspath(__file__))
NTT_CU = os.path.join(HERE, "..", "valida_b200", "csrc", "ntt.cu")
CTX_H = os.path.join(HERE, "..", "valida_b200", "csrc", "ctx.h")

# ---- the host dispatch of ntt.cu, restated ----------------------------------------------------------------------------
LOG_ROW_MAX, LOG_COL_MAX, LOG_TILE_ELEMS, LOG_NMAX = 14, 12, 14, 27
GRID_Y = 65535

Pass = namedtuple("Pass", "log_len groups src_rs src_gs dst_rs dst_gs src_bitrev natural pre post")


def _pass(log_len, groups, src_rs, src_gs, dst_rs, dst_gs, src_bitrev=0, natural=0, pre=0, post=0):
    return Pass(log_len, groups, src_rs, src_gs, dst_rs, dst_gs, src_bitrev, natural, pre, post)


def split_col_row(log_n):
    if log_n <= LOG_ROW_MAX:
        return 0, log_n
    lc = max(min(log_n - LOG_ROW_MAX, LOG_COL_MAX), 4)
    return lc, log_n - lc


def choose_tile(log_len, groups):
    t = 1 << min(max(LOG_TILE_ELEMS - log_len, 0), 6)
    while t > groups:
        t >>= 1
    return max(t, 1)


def pass_threads(log_len, tile):
    return max(32, min(512, ((1 << log_len) * tile) // 16))


def nat2nat(log_n, inverse, coset):
    n = 1 << log_n
    last = 2 if coset else 3 if inverse else 0
    if log_n <= LOG_ROW_MAX:
        return [_pass(log_n, 1, 1, n, 1, n, natural=1, post=last)]
    l1 = (log_n + 1) // 2
    l2 = log_n - l1
    n1, n2 = 1 << l1, 1 << l2
    return [_pass(l1, n2, n2, 1, 1, n1, natural=1, post=1), _pass(l2, n1, n1, 1, n1, 1, natural=1, post=last)]


def intt_nat2bitrev_scaled(log_n):
    n = 1 << log_n
    lc, lr = split_col_row(log_n)
    if lc == 0:
        return [_pass(log_n, 1, 1, n, 1, n, post=2)]
    n1, n2 = 1 << lc, 1 << lr
    return [_pass(lc, n2, n2, 1, n2, 1, post=1), _pass(lr, n1, 1, n2, 1, n2, post=2)]


def ntt_bitrev2bitrev(log_n, odd, tab):
    n = 1 << log_n
    lc, lr = split_col_row(log_n)
    if lc == 0:
        return [_pass(log_n, 1, 1, n, 1, n, src_bitrev=1, pre=odd, post=2 if tab else 0)]
    n1, n2 = 1 << lc, 1 << lr
    return [_pass(lr, n1, 1, n2, 1, n2, src_bitrev=1, pre=odd, post=1),
            _pass(lc, n2, n2, 1, 1, n1, src_bitrev=1, post=2 if tab else 0)]


def branches(p):
    """(LOG_LEN, load branch, store branch, pre mode, post mode) of one pass, as ntt_pass_kernel chooses them."""
    L = p.log_len
    T = choose_tile(L, p.groups)
    nt = pass_threads(L, T)
    std = 8 <= L <= 14 and T == 1 << (14 - L) and nt == 512
    load = None
    if std and L >= 9 and p.pre and p.src_bitrev and p.src_rs == 1 and p.src_gs != 1:
        load = "load_rows_odd_std"
    elif std and not p.pre:
        if L <= 12 and p.src_gs == 1:
            load = "load_strided_std/" + ("bitrev" if p.src_bitrev else "natural")
        elif L >= 9 and p.src_rs == 1 and p.src_gs != 1:
            load = "load_rows_std/" + ("bitrev" if p.src_bitrev else "natural")
    if load is None:
        if p.pre and p.src_bitrev and p.src_gs != 1 and (1 << L) >= 4 * nt:
            load = "load_odd_running"
        else:
            load = "load_element/" + ("strided" if p.src_gs == 1 else "rows")
    store, order = None, "natural" if p.natural else "raw"
    if std:
        if L <= 12 and p.dst_gs == 1:
            store = "store_strided_std/" + order
        elif p.dst_rs == 1 and p.dst_gs != 1:
            if L >= 9:
                store = "store_rows_std/" + order
            elif p.post in (0, 3):
                store = "store_short_rows_std/" + order
    if store is None:
        strided = p.dst_gs == 1
        log_nt, log_t = nt.bit_length() - 1, T.bit_length() - 1
        fast = (nt >= T and log_nt - log_t <= L) if strided else (1 << L) >= nt
        store = ("store_running/" if fast and p.post in (1, 2) else "store_element/") + ("strided" if strided else "rows")
    return (L, load, store, p.pre, p.post)


# entry points: vgpu_ntt_batch (dft / idft), the bit-reversed LDE of the commit path, the same from a quotient-chunk
# matrix (rows stored bit-reversed), and the natural-order LDE with blowup 2^1 .. 2^4
ENTRIES = ("dft", "idft", "lde", "lde_bitrev_rows", "lde_nat1", "lde_nat2", "lde_nat3", "lde_nat4")


def max_log_h(entry):
    if entry in ("dft", "idft"):
        return LOG_NMAX
    if entry.startswith("lde_nat"):
        return min(LOG_ROW_MAX + LOG_COL_MAX, LOG_NMAX - int(entry[-1]))
    return LOG_ROW_MAX + LOG_COL_MAX


def entry_passes(entry, log_h):
    """The passes of one call on one batch of columns, and how many other kernels the batch launches."""
    if entry == "dft":
        return nat2nat(log_h, False, False), 0
    if entry == "idft":
        return nat2nat(log_h, True, False), 0
    if log_h == 0:
        return [], 1                                                     # repeat_row_kernel
    if entry == "lde":
        first = intt_nat2bitrev_scaled(log_h)
    elif entry == "lde_bitrev_rows":
        first = ntt_bitrev2bitrev(log_h, 0, True)
    else:
        return nat2nat(log_h, True, True) + nat2nat(log_h + int(entry[-1]), False, False), 1   # + zero_pad_kernel
    return first + ntt_bitrev2bitrev(log_h, 0, False) + ntt_bitrev2bitrev(log_h, 1, False), 0


def model_launches(entry, log_h, w):
    ps, extra = entry_passes(entry, log_h)
    if entry in ("dft", "idft"):
        batches = [w]
    elif log_h == 0:
        return 1
    else:                                                                # vg_coset_lde's column batches
        b = min(max((2 << 30) // (8 << log_h), 1), w)
        batches = [min(b, w - c0) for c0 in range(0, w, b)]
    return sum(len(ps) * -(-wc // GRID_Y) + extra for wc in batches)


def reachable(cases):
    return {branches(p) for entry, log_h in cases for p in entry_passes(entry, log_h)[0]}


ALL_CASES = [(e, lh) for e in ENTRIES for lh in range(max_log_h(e) + 1)]

# branch variants and the multiplier modes each accepts; the ones no entry reaches at any height
LOAD_MODES = {"load_strided_std/natural": (0,), "load_strided_std/bitrev": (0,), "load_rows_std/natural": (0,), "load_rows_std/bitrev": (0,),
              "load_rows_odd_std": (1,), "load_odd_running": (1,), "load_element/rows": (0, 1), "load_element/strided": (0, 1)}
STORE_MODES = {"store_strided_std/natural": (0, 1, 2, 3), "store_strided_std/raw": (0, 1, 2, 3),
               "store_rows_std/natural": (0, 1, 2, 3), "store_rows_std/raw": (0, 1, 2, 3),
               "store_short_rows_std/natural": (0, 3), "store_short_rows_std/raw": (0, 3),
               "store_running/rows": (1, 2), "store_running/strided": (1, 2),
               "store_element/rows": (0, 1, 2, 3), "store_element/strided": (0, 1, 2, 3)}
UNREACHABLE = {
    # pre-multiplied (odd-coset) loads of strided sub-transforms: the odd coset's pre-multiplier is on its row pass only
    ("load_element/strided", 1),
    # natural-order output of length-2^8 row passes only exists with the twiddle post-multiplier (nat2nat's 2^15 and 2^16
    # column passes), which the short-row store refuses
    ("store_short_rows_std/natural", 0), ("store_short_rows_std/natural", 3),
    # post mode 3 (the 1/n of an idft) is on natural-order passes only
    ("store_short_rows_std/raw", 3), ("store_rows_std/raw", 3), ("store_strided_std/raw", 3),
    # a raw-order strided store is the iNTT's column pass, always with twiddles
    ("store_strided_std/raw", 0), ("store_strided_std/raw", 2),
    # a natural-order strided store is the last pass of nat2nat: never twiddled
    ("store_strided_std/natural", 1),
    # row-type running stores: only the single-pass coset transforms (table, mode 2); twiddled row passes have L >= 11
    ("store_running/rows", 1),
    # the per-element strided store with twiddles: every strided twiddled pass is fast enough for the running product
    ("store_element/strided", 1), ("store_element/strided", 2),
}


def test_model_constants_match_the_source():
    src = open(NTT_CU).read()
    for name, v in (("LOG_ROW_MAX", LOG_ROW_MAX), ("LOG_COL_MAX", LOG_COL_MAX), ("LOG_TILE_ELEMS", LOG_TILE_ELEMS)):
        assert re.search(r"constexpr int %s = (\d+);" % name, src).group(1) == str(v), name
    assert re.search(r"constexpr int VG_LOG_NMAX = (\d+);", open(CTX_H).read()).group(1) == str(LOG_NMAX)
    assert "getenv" not in src, "the NTT pass shapes depend on the height alone"


def test_every_std_helper_and_generic_branch_is_in_the_model():
    src = open(NTT_CU).read()
    helpers = set(re.findall(r"__device__ __forceinline__ void (\w+_std)\(", src))
    assert len(helpers) == 6, helpers
    modelled = {b.split("/")[0] for b in list(LOAD_MODES) + list(STORE_MODES)}
    assert helpers <= modelled, helpers - modelled
    assert {b.split("/")[0] for b in list(LOAD_MODES) + list(STORE_MODES) if "_std" in b} == helpers
    R = reachable(ALL_CASES)
    assert {b for _, ld, st, _, _ in R for b in (ld, st)} <= set(LOAD_MODES) | set(STORE_MODES)
    reached = {(ld, pre) for _, ld, _, pre, _ in R} | {(st, post) for _, _, st, _, post in R}
    declared = {(b, m) for b, ms in list(LOAD_MODES.items()) + list(STORE_MODES.items()) for m in ms}
    assert reached <= declared
    assert declared - reached == UNREACHABLE


def test_gpu_grid_reaches_every_modelled_pass():
    want = reachable(ALL_CASES)
    got = reachable(GRID_CASES)
    # not run: the quotient-chunk LDE's column pass with the shift table at 2^25 and 2^26 (L = 2^11, 2^12); the same
    # helpers run there without the table in the commit LDE, and with the table at L = 2^9 and 2^10
    assert want - got == {(11, "load_strided_std/bitrev", "store_rows_std/raw", 0, 2), (12, "load_strided_std/bitrev", "store_rows_std/raw", 0, 2)}
    # the pass of each benchmark-scale LDE the issue of record names: column passes of the 2^24 .. 2^26 commits, the
    # 2^22 quotient-chunk LDE's generic table store, the odd-coset running-product loader at 2^17
    assert (10, "load_strided_std/natural", "store_strided_std/raw", 0, 1) in reachable([("lde", 24)])
    assert (12, "load_strided_std/natural", "store_strided_std/raw", 0, 1) in reachable([("lde", 26)])
    assert (8, "load_strided_std/bitrev", "store_element/rows", 0, 2) in reachable([("lde_bitrev_rows", 22)])
    assert (13, "load_rows_odd_std", "store_rows_std/raw", 1, 1) in reachable([("lde", 17)])
    assert (13, "load_element/strided", "store_running/strided", 0, 2) in reachable([("lde_nat1", 26)])


def test_model_launch_counts_of_host_loops():
    assert model_launches("dft", 4, 65537) == 2 and model_launches("dft", 20, 65537) == 4
    assert model_launches("lde", 20, 257) == 2 * 6 and model_launches("lde", 24, 17) == 2 * 6 and model_launches("lde", 24, 16) == 6
    assert model_launches("lde", 0, 65537) == 1 and model_launches("lde_nat3", 4, 2) == 3


# ---- exact references ---------------------------------------------------------------------------------------------------
def omega(log_n):
    return pow(G27, 1 << (LOG_NMAX - log_n), P)


def inv(a):
    return pow(a, P - 2, P)


def powers(base, n):
    """base^k for k < n (uint64), from two short tables: no reference transform involved."""
    lg = max(n - 1, 1).bit_length()
    m = 1 << ((lg + 1) // 2)
    lo, a = [], 1
    for _ in range(m):
        lo.append(a)
        a = a * base % P
    hi, b = [], 1
    for _ in range(-(-n // m)):
        hi.append(b)
        b = b * a % P
    out = np.array(hi, dtype=np.uint64)[:, None] * np.array(lo, dtype=np.uint64)[None, :] % np.uint64(P)
    return out.reshape(-1)[:n]


_REV8 = np.array([int(format(i, "08b")[::-1], 2) for i in range(256)], dtype=np.uint32)


def bitrev_perm(log_n):
    if log_n == 0:
        return np.zeros(1, dtype=np.int64)
    r = np.arange(1 << log_n, dtype=np.uint32)
    v = (_REV8[r & 255] << 24) | (_REV8[(r >> 8) & 255] << 16) | (_REV8[(r >> 16) & 255] << 8) | _REV8[r >> 24]
    return (v >> (32 - log_n)).astype(np.int64)


def eval_sum(coeffs, root, N):
    """out[m] = sum_K coeffs[K] * root^(mK) for m < N (root of order dividing N), in exact integer arithmetic: the
    matrix products run on 16-bit halves of the coefficients, so no partial sum reaches 2^64 (at most 2^10 terms)."""
    n = coeffs.shape[0]
    assert n <= 1 << 11
    pw = powers(root, N)
    W = pw[(np.arange(N, dtype=np.int64)[:, None] * np.arange(n, dtype=np.int64)[None, :]) % N]
    c = coeffs.astype(np.uint64)
    Pu = np.uint64(P)
    lo = (W @ (c & np.uint64(0xFFFF))) % Pu
    hi = (W @ (c >> np.uint64(16))) % Pu
    return ((lo + (hi << np.uint64(16)) % Pu) % Pu).astype(np.uint32)


def exact_dft(x, inverse=False):
    log_n = x.shape[0].bit_length() - 1
    if not inverse:
        return eval_sum(x, omega(log_n), x.shape[0])
    y = eval_sum(x, inv(omega(log_n)), x.shape[0]).astype(np.uint64)
    return (y * np.uint64(inv(x.shape[0])) % np.uint64(P)).astype(np.uint32)


def exact_lde(x, added_bits, shift, bitrev):
    """Coefficients from the inverse sum, scaled by shift^K, evaluated at the 2^added_bits * n-th roots of unity."""
    n = x.shape[0]
    log_n = n.bit_length() - 1
    c = exact_dft(x, inverse=True).astype(np.uint64) * powers(shift, n)[:, None] % np.uint64(P)
    out = eval_sum(c.astype(np.uint32), omega(log_n + added_bits), n << added_bits)
    return out[bitrev_perm(log_n + added_bits)] if bitrev else out


def geometric_columns(rng, log_n, w):
    """x_j = c * r^j, one (c, r) per column."""
    n = 1 << log_n
    cs = [int(v) for v in rng.integers(1, P, w)]
    rs = [int(v) for v in rng.integers(2, P, w)]
    x = np.empty((n, w), dtype=np.uint32)
    for j in range(w):
        x[:, j] = powers(rs[j], n) * np.uint64(cs[j]) % np.uint64(P)
    return x, cs, rs


def check_geometric(out, cs, rs, log_n, inverse):
    """dft of c * r^j: X_k (1 - r w^k) = c (1 - r^n).  idft of c * r^k: y_j (1 - r w^-j) = c (1 - r^n) / n.  Every output
    word is checked (except the k with r w^k = 1, which no random r hits)."""
    n = 1 << log_n
    root = inv(omega(log_n)) if inverse else omega(log_n)
    wk = powers(root, n)
    Pu = np.uint64(P)
    for j, (c, r) in enumerate(zip(cs, rs)):
        rhs = c * (1 - pow(r, n, P)) % P
        if inverse:
            rhs = rhs * inv(n) % P
        f = (np.uint64(P + 1) - wk * np.uint64(r) % Pu) % Pu
        lhs = out[:, j].astype(np.uint64) * f % Pu
        bad = np.flatnonzero(lhs != np.uint64(rhs))
        assert bad.size == 0, (j, bad[:8], bad.size)


def check_lde_root_shift(lde, x, log_n, added_bits, u, bitrev):
    """LDE with shift w_H^u (H = n << added_bits): natural output m is x[(m + u) / 2^added_bits] when 2^added_bits divides
    m + u.  In the bit-reversed order of a blowup-2 LDE those are the first n storage rows (u even) or the last n (u odd)."""
    n, B = 1 << log_n, 1 << added_bits
    rows = (-u) % B + B * np.arange(n, dtype=np.int64)
    src = ((rows + u) // B) % n
    if bitrev:                      # storage row r < n holds natural 2 bitrev(r), row n + r holds 2 bitrev(r) + 1
        assert added_bits == 1
        rows = np.arange(n, dtype=np.int64) + (n if u % 2 else 0)
        src = (2 * bitrev_perm(log_n) + u % 2 + u) // 2 % n
    got = lde[rows]
    want = x[src]
    bad = np.flatnonzero((got != want).any(axis=1))
    assert bad.size == 0, (u, rows[bad[:8]], bad.size)


ORACLE_MAX_LOG = 24                    # the oracle's 2^24-row LDE of one column takes about a second on one host core set
SUM_MAX_LOG = 10
GENERIC_SHIFT = 1234567                # a second shift outside every two-adic subgroup


def root_shifts(rng, log_n, added_bits):
    """Two shifts w_H^u: u a multiple of 2^added_bits (s = w_n^t, t != 0) and u odd."""
    B, n = 1 << added_bits, 1 << log_n
    t = int(rng.integers(1, n)) if n > 1 else 0
    u_odd = int(rng.integers(0, n * B // 2)) * 2 + 1
    return [t * B, u_odd]


def free_all(ctx, *mats):
    for m in mats:
        if m is not None:
            m.free()
    ctx.release_cached()


def counted(ctx, fn):
    n0 = ctx.launch_count
    out = fn()
    return out, ctx.launch_count - n0


# ---- the GPU grid ---------------------------------------------------------------------------------------------------------
def _dft_cases():
    out = []
    for lh in range(LOG_NMAX + 1):
        if lh <= SUM_MAX_LOG:
            out += [(lh, 1, "sum"), (lh, 3, "sum")]
        elif lh < 20:
            out += [(lh, 1, "oracle"), (lh, 3, "oracle")]
        elif lh <= ORACLE_MAX_LOG:
            out.append((lh, 3, "oracle"))
        else:
            out.append((lh, 4, "geometric"))
    return out


def _lde_cases():
    out = []
    for lh in range(LOG_ROW_MAX + LOG_COL_MAX + 1):
        if lh <= ORACLE_MAX_LOG:
            ref = "sum" if lh <= SUM_MAX_LOG else "oracle"
            out.append((lh, 3, 31, ref))
            if lh <= 20:
                out.append((lh, 1, GENERIC_SHIFT, ref))
        if lh >= 16:
            out.append((lh, 2, None, "root"))
    return out


def _nat_cases():
    out = []
    for lh in range(LOG_ROW_MAX + LOG_COL_MAX + 1):
        b = min(1 + lh % 4, LOG_NMAX - lh)
        ref = "sum" if lh <= 8 else "oracle" if lh + b <= 25 else "root"
        out.append((lh, b, ref))
    return out


DFT_CASES = _dft_cases()
LDE_CASES = _lde_cases()
BITREV_ROWS_LOGS = list(range(ORACLE_MAX_LOG + 1))   # 2^25 and 2^26 need 3.5 and 7 GB of random LDE-shaped input
NAT_CASES = _nat_cases()
HOST_LOOP_LOGS = (0, 1, 4)
GRID_CASES = ([(e, lh) for lh, _, _ in DFT_CASES for e in ("dft", "idft")] + [("lde", lh) for lh, _, _, _ in LDE_CASES]
              + [("lde_bitrev_rows", lh) for lh in BITREV_ROWS_LOGS] + [("lde_nat%d" % b, lh) for lh, b, _ in NAT_CASES])


@pytest.mark.gpu
@pytest.mark.parametrize("log_h,w,ref", DFT_CASES)
def test_dft_and_idft_exact(ctx, oracle, log_h, w, ref):
    """Forward and inverse transforms, each compared with a reference directly (not only by round trip)."""
    import valida_b200 as vb

    rng = np.random.default_rng(1000 + 10 * log_h + w)
    dft = vb.Radix2Dft(ctx)
    if ref == "geometric":
        x, cs, rs = geometric_columns(rng, log_h, w)
    else:
        x = rng.integers(0, P, (1 << log_h, w), dtype=np.uint32)
    for inverse in (False, True):
        d = ctx.upload(x)
        (dft.idft_batch if inverse else dft.dft_batch)(d)
        got = d.download()
        if ref == "geometric":
            check_geometric(got, cs, rs, log_h, inverse)
        else:
            want = exact_dft(x, inverse) if ref == "sum" else oracle.dft(x, inverse=inverse)
            assert np.array_equal(got, want)
        del got
        # the round trip, counting the launches of the warmed call
        _, n = counted(ctx, lambda: (dft.dft_batch if inverse else dft.idft_batch)(d))
        assert n == model_launches("idft" if not inverse else "dft", log_h, w)
        assert np.array_equal(d.download(), x)
        free_all(ctx, d)


@pytest.mark.gpu
@pytest.mark.parametrize("log_h,w,shift,ref", LDE_CASES)
def test_bitrev_coset_lde_exact(ctx, oracle, log_h, w, shift, ref):
    """The committed (bit-reversed) LDE, against the defining sums, the oracle, or a shift inside the 2n-th roots of unity."""
    import valida_b200 as vb

    rng = np.random.default_rng(2000 + 10 * log_h + w)
    x = rng.integers(0, P, (1 << log_h, w), dtype=np.uint32)
    d = ctx.upload(x)
    dft = vb.Radix2Dft(ctx)
    shifts = root_shifts(rng, log_h, 1) if ref == "root" else [shift]
    for s in shifts:
        sc = pow(omega(log_h + 1), s, P) if ref == "root" else s
        lde = dft.coset_lde_batch(d, 1, sc, bit_reversed=True)
        got = lde.download()
        lde.free()
        if ref == "root":
            check_lde_root_shift(got, x, log_h, 1, s, True)
        else:
            assert np.array_equal(got, exact_lde(x, 1, sc, True) if ref == "sum" else oracle.coset_lde(x, 1, sc, True))
        del got
        lde, n = counted(ctx, lambda: dft.coset_lde_batch(d, 1, sc, bit_reversed=True))
        assert n == model_launches("lde", log_h, w)
        lde.free()
    free_all(ctx, d)


def _quotient_chunks(ctx, oracle, log_degree, seed):
    """A quotient-chunk matrix (rows stored bit-reversed) of the program chip over random LDE-shaped inputs: only its
    layout matters here, its values are whatever the quotient makes of them."""
    import valida_b200 as vb

    chip = 1
    rng = np.random.default_rng(seed)
    h2 = 2 << log_degree
    mats = [ctx.upload(rng.integers(0, P, (h2, k), dtype=np.uint32))
            for k in (oracle.chip_prep_width(chip), oracle.chip_width(chip), oracle.chip_perm_width(chip))]
    ch, alpha, cs = (rng.integers(0, P, k, dtype=np.uint32) for k in (15, 5, 5))
    q = vb.quotient(ctx, chip, log_degree, mats[0], mats[1], mats[2], cs, ch, alpha)
    for m in mats:
        m.free()
    return q


@pytest.mark.gpu
@pytest.mark.parametrize("log_h", BITREV_ROWS_LOGS)
def test_lde_of_bitrev_rows_exact(ctx, oracle, log_h):
    """The quotient-chunk commit: the LDE of a matrix whose rows are stored bit-reversed (its inverse transform takes
    bit-reversed evaluations), against the oracle on the downloaded (natural-order) rows and with root-of-unity shifts."""
    import valida_b200 as vb

    rng = np.random.default_rng(3000 + log_h)
    q = _quotient_chunks(ctx, oracle, log_h, 3000 + log_h)
    x = q.download()
    assert len(np.unique(x)) > x.size // 2, "the quotient of random traces is not random-looking"
    w = x.shape[1]
    dft = vb.Radix2Dft(ctx)
    shifts = [(31, False)] if log_h <= ORACLE_MAX_LOG else []
    if log_h >= 1:
        shifts += [(u, True) for u in root_shifts(rng, log_h, 1)]
    for s, root in shifts:
        sc = pow(omega(log_h + 1), s, P) if root else s
        lde = dft.coset_lde_batch(q, 1, sc, bit_reversed=True)
        got = lde.download()
        lde.free()
        if root:
            check_lde_root_shift(got, x, log_h, 1, s, True)
        else:
            assert np.array_equal(got, oracle.coset_lde(x, 1, sc, True))
        del got
        lde, n = counted(ctx, lambda: dft.coset_lde_batch(q, 1, sc, bit_reversed=True))
        assert n == model_launches("lde_bitrev_rows", log_h, w)
        lde.free()
    free_all(ctx, q)


@pytest.mark.gpu
@pytest.mark.parametrize("log_h,added_bits,ref", NAT_CASES)
def test_natural_coset_lde_exact(ctx, oracle, log_h, added_bits, ref):
    """The natural-order LDE (coset iNTT with the shift table on its last pass, zero padding, forward transform) at every
    height, blowups 2 to 16; 2^23 rows with blowup 16 is an output of 2^27, and 2^26 with blowup 2 is the only caller
    of the strided running-product store with a host-computed table step."""
    import valida_b200 as vb

    rng = np.random.default_rng(4000 + log_h)
    w = 2
    x = rng.integers(0, P, (1 << log_h, w), dtype=np.uint32)
    d = ctx.upload(x)
    dft = vb.Radix2Dft(ctx)
    shifts = root_shifts(rng, log_h, added_bits) if ref == "root" else [31]
    for s in shifts:
        sc = pow(omega(log_h + added_bits), s, P) if ref == "root" else s
        lde = dft.coset_lde_batch(d, added_bits, sc)
        got = lde.download()
        lde.free()
        if ref == "root":
            check_lde_root_shift(got, x, log_h, added_bits, s, False)
        else:
            assert np.array_equal(got, exact_lde(x, added_bits, sc, False) if ref == "sum" else oracle.coset_lde(x, added_bits, sc, False))
        del got
        lde, n = counted(ctx, lambda: dft.coset_lde_batch(d, added_bits, sc))
        assert n == model_launches("lde_nat%d" % added_bits, log_h, w)
        lde.free()
    free_all(ctx, d)


@pytest.mark.gpu
@pytest.mark.parametrize("log_h", HOST_LOOP_LOGS)
def test_more_than_65535_columns(ctx, log_h):
    """65537 columns: launch_pass splits grid.y into chunks of 65535 columns (at one row the LDE is repeat_row_kernel)."""
    import valida_b200 as vb

    w = 65537
    rng = np.random.default_rng(5000 + log_h)
    x = rng.integers(0, P, (1 << log_h, w), dtype=np.uint32)
    dft = vb.Radix2Dft(ctx)
    for entry in ("dft", "idft"):
        d = ctx.upload(x)
        getattr(dft, entry + "_batch")(d)
        assert np.array_equal(d.download(), exact_dft(x, entry == "idft")), entry
        _, n = counted(ctx, lambda: getattr(dft, entry + "_batch")(d))
        assert n == model_launches(entry, log_h, w)
        d.free()
    d = ctx.upload(x)
    for entry, bits, br in (("lde", 1, True), ("lde_nat2", 2, False)):
        lde = dft.coset_lde_batch(d, bits, 31, bit_reversed=br)
        assert np.array_equal(lde.download(), exact_lde(x, bits, 31, br)), entry
        lde.free()
        lde, n = counted(ctx, lambda: dft.coset_lde_batch(d, bits, 31, bit_reversed=br))
        assert n == model_launches(entry, log_h, w)
        lde.free()
    free_all(ctx, d)


@pytest.mark.gpu
@pytest.mark.parametrize("log_h,w", [(20, 257), (24, 17)])
def test_bitrev_lde_column_batches(ctx, log_h, w):
    """vg_coset_lde transforms 2^28 / h columns at a time: 257 columns of 2^20 and 17 of 2^24 take two batches.  Both halves
    of every column are checked through the two root-of-unity shifts."""
    import valida_b200 as vb

    rng = np.random.default_rng(6000 + log_h)
    x = rng.integers(0, P, (1 << log_h, w), dtype=np.uint32)
    d = ctx.upload(x)
    dft = vb.Radix2Dft(ctx)
    for u in root_shifts(rng, log_h, 1):
        sc = pow(omega(log_h + 1), u, P)
        lde = dft.coset_lde_batch(d, 1, sc, bit_reversed=True)
        check_lde_root_shift(lde.download(), x, log_h, 1, u, True)
        lde.free()
        lde, n = counted(ctx, lambda: dft.coset_lde_batch(d, 1, sc, bit_reversed=True))
        assert n == model_launches("lde", log_h, w) == 12
        lde.free()
    free_all(ctx, d)


@pytest.mark.gpu
def test_lde_height_limits(ctx):
    import valida_b200 as vb

    dft = vb.Radix2Dft(ctx)
    d = ctx.upload(np.ones((1 << 27, 1), dtype=np.uint32))
    with pytest.raises(vb.VgpuError, match="heights above 2\\^26 are not built"):
        dft.coset_lde_batch(d, 1, 31, bit_reversed=True)
    with pytest.raises(vb.VgpuError, match="heights above 2\\^26 are not built"):
        dft.coset_lde_batch(d, 1, 31)
    d.free()
    d = ctx.upload(np.ones((1 << 24, 1), dtype=np.uint32))
    with pytest.raises(vb.VgpuError, match="LDE height 2\\^28 exceeds BabyBear two-adicity"):
        dft.coset_lde_batch(d, 4, 31)
    free_all(ctx, d)
