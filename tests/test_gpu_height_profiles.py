"""Whole proofs over many chip-height profiles (tests/height_profiles.py), byte for byte against the oracle, through every host
input route and both word representations the C ABI takes.

The stage kernels are compared with the oracle elsewhere; what these tests reach is the prover around them, which depends on the
profile: reduced openings counted per height, FRI folds that add the next height's openings only where it exists, query leaves
shifted per round, equal heights in the mixed-height trees, split or whole chips in a split proof.  Each profile is proven

  * from random traces: vgpu_prove with canonical and with Montgomery words (as the Rust caller passes them) and vgpu_prove_device
    after upload, each equal to the oracle's bytes; vgpu_verify with canonical and Montgomery preprocessed words gives the oracle's
    verdict;
  * from honest witnesses, which both verifiers accept, and from the same witnesses with one chip's trace replaced by random rows;
  * at 2^17 rows from pageable, pinned and registered host memory, twice on one context;
  * split over 2, 3 and 4 thread ranks on one GPU, through the host entry in Montgomery words and the device entry;
  * with Poseidon-16 Merkle trees.

A proof that differs names the first differing field (height_profiles.first_difference), and so its stage."""
import mmap
import types

import numpy as np
import pytest

from height_profiles import (ALL_PROFILES, HONEST, NUM_CHIPS, PROFILES, ROUTE_PROFILE, first_difference, log_heights, random_traces,
                             to_monty, with_chip_replaced)
from test_gpu_verify import expected

pytestmark = pytest.mark.gpu
SPLIT_PROFILES = ["staircase", "reverse_staircase", "twin_tallest", "one_tall", "program_tallest", "range_tallest"]
POSEIDON_PROFILES = ["one_row", "staircase", "program_tallest"]


def _traces(main, prep):
    return types.SimpleNamespace(main=main, preprocessed=prep)


def _monty(main, prep):
    return [to_monty(m) for m in main], [to_monty(m) for m in prep]


def _verdict(vb, cfg, proof, prep, repr):
    try:
        vb.verify_machine(cfg, proof, prep, repr=repr)
        return 0
    except vb.VerificationError as e:
        return e.verdict


def _differences(got, want):
    """{entry: first differing field} of the proofs in `got` that are not `want`."""
    return {k: first_difference(p, want) for k, p in got.items() if p != want}


@pytest.fixture(scope="module")
def cfg(ctx, oracle):
    import valida_b200 as vb

    return vb.StarkConfig(ctx, oracle.rc480)


# ---- random traces on every profile ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(ALL_PROFILES))
def test_random_traces_every_entry_equals_oracle(ctx, cfg, oracle, name):
    import valida_b200 as vb

    main, prep = random_traces(ALL_PROFILES[name], 1)
    want = oracle.prove(main, prep, debug_checks=False).cbor()
    mmain, mprep = _monty(main, prep)
    got = {"host canonical": vb.prove_machine(cfg, _traces(main, prep)),
           "host montgomery": vb.prove_machine(cfg, _traces(mmain, mprep), repr=vb.REPR_MONTY_R32)}
    dm = [ctx.upload(m) for m in main + prep]
    try:
        got["device"] = vb.prove_machine(cfg, None, device_resident=(dm[:NUM_CHIPS], dm[NUM_CHIPS:]))
    finally:
        for m in dm:
            m.free()
        ctx.release_cached()
    assert _differences(got, want) == {}
    code = oracle.verify(want, prep)
    assert code != 0                                       # random rows satisfy no chip's constraints
    assert _verdict(vb, cfg, want, prep, vb.REPR_CANONICAL) == expected(code)
    assert _verdict(vb, cfg, want, mprep, vb.REPR_MONTY_R32) == expected(code)


# ---- honest witnesses, and one chip replaced ------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(HONEST))
def test_honest_witness_profiles(cfg, oracle, name):
    import valida_b200 as vb

    t = HONEST[name](vb)
    main, prep = list(t.main), list(t.preprocessed)
    want = oracle.prove(main, prep, debug_checks=False).cbor()
    assert oracle.verify(want, prep) == 0, log_heights(main)
    mmain, mprep = _monty(main, prep)
    got = {"host canonical": vb.prove_machine(cfg, _traces(main, prep)),
           "host montgomery": vb.prove_machine(cfg, _traces(mmain, mprep), repr=vb.REPR_MONTY_R32)}
    assert _differences(got, want) == {}
    assert _verdict(vb, cfg, want, prep, vb.REPR_CANONICAL) == 0
    assert _verdict(vb, cfg, want, mprep, vb.REPR_MONTY_R32) == 0
    bad = []
    for chip in range(NUM_CHIPS):
        alt = with_chip_replaced(main, chip)
        ref = oracle.prove(alt, prep, debug_checks=False).cbor()
        proof = vb.prove_machine(cfg, _traces(alt, prep))
        if proof != ref:
            bad.append((chip, "bytes", first_difference(proof, ref)))
        code = oracle.verify(ref, prep)
        v = _verdict(vb, cfg, ref, prep, vb.REPR_CANONICAL)
        if v != expected(code):
            bad.append((chip, "verdict", code, v))
    assert bad == []


# ---- host input routes at a tall profile ----------------------------------------------------------------------------------
def _pinned(ms):
    import torch

    out = []
    for m in ms:
        t = torch.empty(m.shape, dtype=torch.int32, pin_memory=True)
        t.numpy().view(np.uint32)[...] = m
        out.append(t)
    return out


def _own_pages(ms):
    """Copies of the matrices, each in an anonymous mapping of its own: registering one never overlaps another's registration."""
    out = []
    for m in ms:
        a = np.frombuffer(mmap.mmap(-1, m.nbytes), dtype=np.uint32).reshape(m.shape)
        a[...] = m
        out.append(a)
    return out


def test_host_input_routes_at_a_tall_profile(ctx, cfg, oracle):
    """CPU, add and memory at 2^17 rows: 25.5 MiB (two staging chunks, the last partial), exactly 8 MiB (staged) and 7 MiB (one
    direct copy).  Pageable numpy arrays, torch pinned tensors and registered arrays, in both representations, twice on one
    context so that staging state left over from one call would show: twelve proofs, all the oracle's bytes."""
    import valida_b200 as vb

    main, prep = random_traces(ROUTE_PROFILE, 5)
    assert log_heights(main)[:4] == [17, 6, 17, 17]
    want = oracle.prove(main, prep, debug_checks=False).cbor()
    words = {vb.REPR_CANONICAL: main + prep, vb.REPR_MONTY_R32: [to_monty(m) for m in main + prep]}
    pinned = {r: _pinned(ms) for r, ms in words.items()}
    registered = {r: _own_pages(ms) for r, ms in words.items()}
    done = []
    try:
        for ms in registered.values():
            for a in ms:
                ctx.host_register(a)
                done.append(a)
        got = {}
        for rnd in range(2):
            for r, ms in words.items():
                for route, mats in (("pageable", ms), ("pinned", [t.numpy().view(np.uint32) for t in pinned[r]]),
                                    ("registered", registered[r])):
                    got[(rnd, route, r)] = vb.prove_machine(cfg, _traces(mats[:NUM_CHIPS], mats[NUM_CHIPS:]), repr=r)
    finally:
        for a in done:
            ctx.host_unregister(a)
        ctx.release_cached()
    assert len(got) == 12
    assert _differences(got, want) == {}


# ---- split proofs ---------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def split_cases(oracle):
    out = {}
    for name in SPLIT_PROFILES:
        main, prep = random_traces(PROFILES[name], 2)
        out[name] = (main, prep, oracle.prove(main, prep, debug_checks=False).cbor())
    return out


@pytest.mark.parametrize("nranks", [2, 3, 4])
def test_split_proofs_equal_single_gpu(oracle, split_cases, nranks):
    """Each profile has chips tall enough to be split into row runs and chips every rank holds whole (local_rows says which)."""
    import valida_b200 as vb
    from test_gpu_split_any import _close, _ranks

    ctxs = _ranks(nranks)
    bad = {}
    try:
        cfgs = [vb.StarkConfig(c, oracle.rc480) for c in ctxs]
        for name in SPLIT_PROFILES:
            main, prep, want = split_cases[name]
            split = [c for c in range(NUM_CHIPS) if ctxs[0].local_rows(main[c].shape[0])[1] < main[c].shape[0]]
            assert 0 < len(split) < NUM_CHIPS, (name, split)
            mmain, mprep = _monty(main, prep)

            def host(r, c):
                return vb.prove_machine(cfgs[r], _traces(mmain, mprep), repr=vb.REPR_MONTY_R32)

            def device(r, c):
                dm = [c.upload_rows(m) for m in main + prep]
                try:
                    return vb.prove_machine(cfgs[r], None, device_resident=(dm[:NUM_CHIPS], dm[NUM_CHIPS:]))
                finally:
                    for m in dm:
                        m.free()

            for entry, fn in (("host montgomery", host), ("device", device)):
                for r, p in enumerate(vb.run_ranks(fn, ctxs)):
                    if p != want:
                        bad[(name, entry, r)] = first_difference(p, want)
    finally:
        _close(ctxs)
    assert bad == {}


# ---- Poseidon-16 ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", POSEIDON_PROFILES)
def test_poseidon_profiles_equal_oracle(built, oracle, name):
    import valida_b200 as vb
    from poseidon_mmcs import PoseidonOracle

    mmcs = PoseidonOracle()
    main, prep = random_traces(PROFILES[name], 3)
    want = mmcs.prove(main, prep, debug_checks=False).cbor()
    ctx = vb.Context(0)
    try:
        cfg = vb.StarkConfig(ctx, oracle.rc480)
        ctx.set_merkle_hash(vb.MERKLE_POSEIDON16)
        mmain, mprep = _monty(main, prep)
        got = {"host canonical": vb.prove_machine(cfg, _traces(main, prep)),
               "host montgomery": vb.prove_machine(cfg, _traces(mmain, mprep), repr=vb.REPR_MONTY_R32)}
        assert _differences(got, want) == {}
        code = mmcs.verify(want, prep)
        assert code != 0
        assert _verdict(vb, cfg, want, mprep, vb.REPR_MONTY_R32) == expected(code)
    finally:
        ctx.close()
