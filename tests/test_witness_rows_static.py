"""Where the trace layout is written, read from the sources (CPU): the rows of the tall chips are defined once, by the row functions
of csrc/chip_rows.cuh, and both witness builders call them — the host one (csrc/host/tracegen.cc) and the device one
(csrc/witness.cu) — so a change to a chip's columns is made in one place."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "valida_b200", "csrc")
HEADER = "chip_rows.cuh"
BUILDERS = ("host/tracegen.cc", "witness.cu")

ROW_FUNCTIONS = ("cpu_row", "cpu_pad_row", "mem_row", "addsub_row", "lt_row", "bitwise_row")
HELPERS = ("from_i32", "word_be", "next_pow2")

# text of the row bodies the header replaced: none of it may come back into a builder
GONE = ("256u + b[k] - c[k]", "word_be(r.imm", "OP_SLT32 + 1", "{14, 28, 14, 7, 6}")


def _code(text):
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    text = re.sub(r'"(?:\\.|[^"\\])*"', '""', text)
    return re.sub(r"//[^\n]*", "", text)


def _sources():
    for d, _, files in os.walk(CSRC):
        for f in sorted(files):
            if f.endswith((".h", ".cuh", ".cu", ".cc", ".inc")):
                with open(os.path.join(d, f)) as fh:
                    yield os.path.relpath(os.path.join(d, f), CSRC), _code(fh.read())


def _definitions(code, name):
    return re.findall(r"\b(?:void|u?int(?:32|64)_t|size_t)\s+%s\s*\([^;{]*\)\s*\{" % name, code)


def _calls(code, name):
    return [m for m in re.finditer(r"\b%s\s*\(" % name, code)
            if not re.search(r"\b(?:void|u?int(?:32|64)_t|size_t)\s+$", code[code.rfind("\n", 0, m.start()) + 1:m.start()])]


def test_row_functions_are_defined_once_and_called_by_both_builders():
    sources = dict(_sources())
    for name in ROW_FUNCTIONS + HELPERS:
        defined_in = [f for f, code in sources.items() if _definitions(code, name)]
        assert defined_in == [HEADER], (name, defined_in)
    for name in ROW_FUNCTIONS:
        for f in BUILDERS:
            assert _calls(sources[f], name), "%s does not call %s" % (f, name)


def test_builders_hold_no_row_body_of_their_own():
    sources = dict(_sources())
    for f in BUILDERS:
        for text in GONE:
            assert text not in sources[f], (f, text)
        assert not re.search(r"\bOP_STOP\s*=", sources[f]), f        # the opcodes live in host/vmlog.h
