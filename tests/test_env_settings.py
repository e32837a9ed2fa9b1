"""The library reads the environment in one place only (CPU test over the sources): host/comm.cc, for the three operational
settings of split proofs: the symmetric heap's size and floor and a collective's timeout.  Kernel variants and tuning values
are constants in the code, so every run of the library executes the same kernels."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "valida_b200", "csrc")
ALLOWED = {os.path.join("host", "comm.cc"): {"VGPU_SYMM_HEAP_MB", "VGPU_SYMM_HEAP_MIN_MB", "VGPU_COMM_TIMEOUT_S"}}


def _sources():
    for d, _, files in os.walk(CSRC):
        for f in files:
            p = os.path.join(d, f)
            yield os.path.relpath(p, CSRC), open(p, encoding="utf-8").read()


def test_getenv_only_reads_the_operational_settings():
    seen = {}
    for rel, src in _sources():
        calls = src.count("getenv")
        names = re.findall(r'getenv\("(\w+)"\)', src)
        if calls:
            assert rel in ALLOWED, (rel, names)
            assert len(names) == calls, (rel, "getenv with a name that is not a string literal")
            seen[rel] = set(names)
    assert seen == ALLOWED, seen
