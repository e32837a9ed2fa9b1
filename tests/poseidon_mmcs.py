"""The oracle with Poseidon-16 Merkle trees (tests/c/poseidon_mmcs_oracle.cc) — TEST INFRASTRUCTURE ONLY.

The library is the oracle's own entry points compiled over a Poseidon-16 MMCS; it is built on first use into the temporary
directory (keyed by its sources, so a changed oracle is rebuilt) and driven through the methods of oracle_binding.Oracle, which
therefore commit, open, prove and verify with Poseidon-16 trees here."""
import ctypes as C
import glob
import hashlib
import os
import subprocess
import tempfile

import numpy as np

from oracle_binding import ROOT, Oracle, _p, u32p

SRC = os.path.join(ROOT, "tests", "c", "poseidon_mmcs_oracle.cc")


def library():
    h = hashlib.sha256()
    for f in [SRC] + sorted(glob.glob(os.path.join(ROOT, "oracle", "*.h")) + glob.glob(os.path.join(ROOT, "oracle", "*.inc")) + glob.glob(os.path.join(ROOT, "oracle", "*.cc"))):
        h.update(open(f, "rb").read())
    out = os.path.join(tempfile.gettempdir(), "valida_b200_poseidon_oracle_%s_%d.so" % (h.hexdigest()[:16], os.getuid()))
    if not os.path.exists(out):
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"     # as oracle/Makefile: the compiler with OpenMP
        tmp = out + ".%d.tmp" % os.getpid()
        subprocess.run([cxx, "-O3", "-march=native", "-std=c++17", "-fPIC", "-fopenmp", "-Wall", "-Wno-unused-function", "-Wno-sign-compare",
                        "-shared", "-o", tmp, SRC], check=True)
        os.replace(tmp, out)
    return out


class PoseidonOracle(Oracle):
    """oracle_binding.Oracle over the Poseidon-16 MMCS.  The trees hash with the permutation of the round constants `rc` of each
    call (the challenger's), or of the default constants for the calls without one."""

    def __init__(self):
        self.L = L = C.CDLL(library())
        for name, res in (("orc_prove", C.c_void_p), ("orc_proof_cbor", C.c_uint64), ("orc_proof_perm_trace", C.c_uint64),
                          ("orc_proof_quotient_chunks", C.c_uint64), ("orc_proof_constraint_failure", C.c_int64), ("orc_proof_opened", C.c_uint64),
                          ("orc_merkle_open", C.c_uint32), ("orc_two_adic_generator", C.c_uint32), ("orc_mul", C.c_uint32), ("orc_inv", C.c_uint32),
                          ("orc_chip_perm_width", C.c_uint32), ("orc_chip_width", C.c_uint32), ("orc_chip_prep_width", C.c_uint32)):
            getattr(L, name).restype = res
        rc = (C.c_uint32 * 480)()
        L.orc_default_round_constants(rc)
        self.rc480 = np.array(list(rc), dtype=np.uint32)

    def _mmcs(self, rc):
        self.L.orc_mmcs_set_round_constants(_p(np.ascontiguousarray(self.rc480 if rc is None else rc, dtype=np.uint32)))

    def merkle_root(self, mats, rc=None):
        self._mmcs(rc)
        return super().merkle_root(mats)

    def commit_batches(self, mats, coset_shifts=None, want_ldes=False, rc=None):
        self._mmcs(rc)
        return super().commit_batches(mats, coset_shifts, want_ldes)

    def prove(self, main, preps, rc=None, debug_checks=True):
        self._mmcs(rc)
        return super().prove(main, preps, rc, debug_checks)

    def verify(self, proof_bytes, preps, rc=None):
        self._mmcs(rc)
        return super().verify(proof_bytes, preps, rc)

    def open(self, rounds, points, observe, shifts=None, rc=None, sample_ext_first=False):
        self._mmcs(rc)
        return super().open(rounds, points, observe, shifts, rc, sample_ext_first)

    def merkle_open(self, mats, index, rc=None):
        """(opened rows in the caller's order, sibling digests leaf level first) of leaf `index` of the tree over the matrices as given."""
        self._mmcs(rc)
        mats = [np.ascontiguousarray(m, dtype=np.uint32) for m in mats]
        n = len(mats)
        ptrs = (u32p * n)(*[_p(m) for m in mats])
        hs = (C.c_uint64 * n)(*[m.shape[0] for m in mats])
        ws = (C.c_uint64 * n)(*[m.shape[1] for m in mats])
        rows = np.zeros(sum(m.shape[1] for m in mats), dtype=np.uint32)
        path = np.zeros((64, 8), dtype=np.uint32)
        k = self.L.orc_merkle_open(n, ptrs, hs, ws, C.c_uint64(index), _p(rows), _p(path))
        out, at = [], 0
        for m in mats:
            out.append(rows[at:at + m.shape[1]].copy())
            at += m.shape[1]
        return out, path[:k].copy()
