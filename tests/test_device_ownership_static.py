"""Who frees device memory, read from the sources (CPU): every scratch block, matrix and prover data a call allocates is held by one
of the owner types of csrc/ctx.h (VgBuf, VgMat, VgPd), so a call that fails part-way leaves nothing live in the context.  The raw
allocator and the free functions are called only where they are defined, inside those owners, and at the sites listed below, which
keep memory beyond the call that allocates it."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "valida_b200", "csrc")

CALLS = ("vg_alloc", "vg_free", "vgpu_dmat_free", "vgpu_prover_data_free")

# (file, call) -> why the call is not made through an owner
ALLOWED = {
    # the owner types and their deleters
    ("ctx.h", "vg_alloc(ctx, &p, bytes)"): "VgBuf::alloc",
    ("ctx.h", "vg_free(ctx, p)"): "VgBuf::reset",
    ("ctx.h", "vgpu_dmat_free(m)"): "the deleter of VgMat",
    ("ctx.h", "vgpu_prover_data_free(p)"): "the deleter of VgPd",
    # a matrix's own storage: allocated with the handle, released with it or once its last reader is enqueued
    ("api.cu", "vg_alloc(ctx, (void**)&m->d, bytes)"): "vg_dmat_alloc_run: the columns of a new matrix",
    ("api.cu", "vg_free(m->ctx, m->pend_stage)"): "vgpu_dmat_free: the staging block of an upload that was never consumed",
    ("api.cu", "vg_free(m->ctx, m->d)"): "vgpu_dmat_free: the columns of an owned matrix",
    ("api.cu", "vgpu_dmat_free(m)"): "vgpu_prover_data_free: the LDEs a prover data owns",
    ("staging.cu", "vg_alloc(ctx, (void**)&dst->pend_stage, h * w * 4)"): "vg_upload_begin: the staging block lives until the matrix's first use",
    ("staging.cu", "vg_free(ctx, m->pend_stage)"): "vg_dmat_materialize: the staging block goes once the transpose is enqueued",
    ("prover.cc", "vg_free(ctx, m->d)"): "prove_device: the main traces vgpu_prove copied go once the permutation traces are built",
    # tables that live as long as the context
    ("api.cu", "vg_alloc(ctx, (void**)&ctx->root3, t.size() * 4)"): "vgpu_ctx_create: the three-level root table",
    ("api.cu", "vg_free(ctx, it->second.lo)"): "vg_get_shift_table: a shift table replaced by a longer one",
    ("api.cu", "vg_free(ctx, it->second.hi)"): "vg_get_shift_table: a shift table replaced by a longer one",
    ("api.cu", "vg_free(ctx, ctx->root_table.lo)"): "vgpu_ctx_destroy",
    ("api.cu", "vg_free(ctx, ctx->root_table.hi)"): "vgpu_ctx_destroy",
    ("api.cu", "vg_free(ctx, kv.second.lo)"): "vgpu_ctx_destroy: the shift tables",
    ("api.cu", "vg_free(ctx, kv.second.hi)"): "vgpu_ctx_destroy: the shift tables",
    ("pow.cu", "vg_alloc(ctx, (void**)&ctx->d_poseidon, (c.size() + 16 + 1) * 4)"): "vg_poseidon_consts: the context's Poseidon-16 constants",
    ("challenger.cc", "vg_free(ctx, ctx->d_poseidon)"): "vgpu_set_challenger: constants that no longer hold",
}

GONE = ("PdGuard", "BufGuard", "MatGuard", "ExtGuard", "DevBuf", "OpenScratch", "vg_tree_free", "struct Free", "struct Undo", "new KScope")


def _sources():
    for d, _, files in os.walk(CSRC):
        for f in sorted(files):
            if f.endswith((".h", ".cuh", ".cu", ".cc", ".inc")):
                with open(os.path.join(d, f)) as fh:
                    yield f, fh.read()


def _code(text):
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    text = re.sub(r'"(?:\\.|[^"\\])*"', '""', text)
    return re.sub(r"//[^\n]*", "", text)


def _calls(code):
    """(call text) of every call of CALLS that is not a declaration or definition of the function itself"""
    for m in re.finditer(r"\b(%s)\(" % "|".join(CALLS), code):
        line_start = code.rfind("\n", 0, m.start()) + 1
        if re.match(r"\s*(?:int32_t|void)\s+$", code[line_start:m.start()]):
            continue
        depth, i = 0, m.end() - 1
        while True:
            depth += {"(": 1, ")": -1}.get(code[i], 0)
            if depth == 0:
                break
            i += 1
        yield re.sub(r"\s+", " ", code[m.start():i + 1])


def test_the_hand_written_guards_are_gone():
    for f, text in _sources():
        for name in GONE:
            assert name not in text, (f, name)


def test_device_memory_is_freed_only_by_its_owners():
    found = set()
    for f, text in _sources():
        for call in _calls(_code(text)):
            assert (f, call) in ALLOWED, "%s: %s is called outside the owner types (VgBuf, VgMat, VgPd)" % (f, call)
            found.add((f, call))
    assert found == set(ALLOWED), sorted(set(ALLOWED) - found)
