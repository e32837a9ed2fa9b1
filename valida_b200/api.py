"""ctypes binding of libvalida_b200.so, shaped after the reference's Rust interfaces.

Reference interfaces mirrored (names and argument meaning kept):
  * p3_dft::TwoAdicSubgroupDft: dft_batch / idft_batch / coset_lde_batch        -> Radix2Dft
  * UnivariatePcsWithLde (machine/src/config.rs:17-22): commit_batches,
    commit_shifted_batches, get_ldes, coset_shift, log_blowup                    -> TwoAdicFriPcs
  * Machine::run / Chip::generate_trace (machine/src/machine.rs:13-30)          -> run_program / MachineTraces
Errors: the reference panics (derive/src/lib.rs:319,364,396); here every non-zero status raises
VgpuError carrying vgpu_last_error().
"""
import collections
import ctypes as C
import os
import weakref

import numpy as np

BABYBEAR_P = 2013265921
REPR_CANONICAL, REPR_MONTY_R32 = 0, 1
NUM_CHIPS = 14
MERKLE_KECCAK256, MERKLE_POSEIDON16 = 0, 1     # vgpu_ctx_set_merkle_hash

_HERE = os.path.dirname(os.path.abspath(__file__))
lib_path = os.path.join(_HERE, "libvalida_b200.so")


class VgpuError(RuntimeError):
    pass


class _Matrix(C.Structure):
    _fields_ = [("data", C.POINTER(C.c_uint32)), ("height", C.c_uint64), ("width", C.c_uint64)]


class _DevMatrix(C.Structure):
    """vgpu_dev_matrix: a strided view of device memory (strides in elements)."""
    _fields_ = [("data", C.c_void_p), ("height", C.c_uint64), ("width", C.c_uint64), ("row_stride", C.c_uint64), ("col_stride", C.c_uint64)]


class _CheckReport(C.Structure):
    """vgpu_check_report: one chip's verdict of vgpu_check_witness."""
    _fields_ = [("first_row", C.c_int64), ("first_constraint", C.c_uint32), ("failing_rows", C.c_uint64), ("cumulative_sum", C.c_uint32 * 5)]


class _PairCol(C.Structure):
    _fields_ = [("constant", C.c_uint32), ("n_terms", C.c_uint32), ("terms", C.c_uint32 * 12)]


class _Interaction(C.Structure):
    _fields_ = [("n_fields", C.c_uint32), ("fields", _PairCol * 14), ("count", _PairCol), ("bus", C.c_uint32), ("is_send", C.c_uint32)]


class _ChipDesc(C.Structure):
    """vgpu_chip_desc (the fields constraint_label reads)."""
    _fields_ = [("chip_id", C.c_uint32), ("width", C.c_uint32), ("preprocessed_width", C.c_uint32), ("n_interactions", C.c_uint32),
                ("interactions", _Interaction * 5)]


# vgpu_check_failure: one (row, constraint) on which a chip's check does not vanish, and the constraint's canonical value there
CHECK_FAILURE_DTYPE = np.dtype([("row", "<i8"), ("constraint", "<u4"), ("value", "<u4", (5,))])
# vgpu_bus_event / vgpu_bus_imbalance (include/valida_b200.h)
BUS_EVENT_DTYPE = np.dtype([("chip", "<u4"), ("interaction", "<u4"), ("row", "<i8"), ("multiplicity", "<u4"), ("is_send", "<u4")])
BUS_IMBALANCE_DTYPE = np.dtype([("bus", "<u4"), ("fields", "<u4", (14,)), ("net", "<u4"), ("first_event", "<u8"), ("n_events", "<u8")], align=True)
# vgpu_bus_link (include/valida_b200.h): one item's tuple, its own count, and the events that carry its tuple
BUS_LINK_DTYPE = np.dtype([("bus", "<u4"), ("fields", "<u4", (14,)), ("multiplicity", "<u4"), ("sends", "<u4"), ("receives", "<u4"),
                           ("n_events", "<u8"), ("first_event", "<u8")], align=True)
# BasicMachine's chips and buses (basic/src/lib.rs:151-166, 1190-1212), by id
CHIP_NAMES = ("cpu", "program", "memory", "add", "sub", "mul", "div", "shift", "lt", "com", "bitwise", "output", "range", "static_data")
BUS_NAMES = ("general", "program", "memory", "range")
# vgpu_cell (include/valida_b200.h): which trace, the row itself (0) or the next row (1), the column
TRACE_MAIN, TRACE_PREPROCESSED, TRACE_PERMUTATION = 0, 1, 2
CELL_DTYPE = np.dtype([("trace", "<u4"), ("next", "<u4"), ("column", "<u4")])
CELL_ABSENT = 0xFFFFFFFF      # vgpu_explain_failures' word for a permutation cell when no permutation trace was passed
# vgpu_cell_diff / vgpu_diff_summary (include/valida_b200.h)
CELL_DIFF_DTYPE = np.dtype([("chip", "<u4"), ("trace", "<u4"), ("column", "<u4"), ("row", "<i8"), ("have", "<u4"), ("want", "<u4")], align=True)
DIFF_SUMMARY_DTYPE = np.dtype([("height_have", "<u8"), ("height_want", "<u8"), ("cells", "<u8"), ("first_row", "<i8")])
# vgpu_free_cell (include/valida_b200.h): one main-trace cell no check pins
FREE_CELL_DTYPE = np.dtype([("row", "<i8"), ("column", "<u4")], align=True)
# vgpu_cell_alternative (include/valida_b200.h): one cell the constraints would accept at other values
CELL_ALTERNATIVE_DTYPE = np.dtype([("row", "<i8"), ("column", "<u4"), ("value", "<u4"), ("n_values", "<u4"), ("values", "<u4", 3),
                                   ("bus", "<u4"), ("reserved", "<u4")], align=True)


def _load():
    if not os.path.exists(lib_path):
        raise VgpuError(
            "libvalida_b200.so is missing (%s): build it with `python -m valida_b200.build` — there is no CPU fallback" % lib_path
        )
    L = C.CDLL(lib_path)
    vp, u32p, u64 = C.c_void_p, C.POINTER(C.c_uint32), C.c_uint64
    sig = {
        "vgpu_ctx_create": (C.c_int32, [C.c_int32, vp, C.POINTER(vp)]),
        "vgpu_ctx_destroy": (None, [vp]),
        "vgpu_last_error": (C.c_char_p, [vp]),
        "vgpu_ctx_synchronize": (C.c_int32, [vp]),
        "vgpu_ctx_wait_event": (C.c_int32, [vp, vp]),
        "vgpu_ctx_record_event": (C.c_int32, [vp, vp]),
        "vgpu_ctx_launch_count": (u64, [vp]),
        "vgpu_ctx_release_cached": (C.c_int32, [vp]),
        "vgpu_ctx_memory_stats": (C.c_int32, [vp, C.POINTER(u64), C.c_int32]),
        "vgpu_ctx_set_kernel_timing": (C.c_int32, [vp, C.c_int32]),
        "vgpu_ctx_kernel_stats": (C.c_uint32, [vp, C.POINTER(C.c_char_p), u32p, C.POINTER(C.c_float), C.POINTER(C.c_double), C.c_uint32]),
        "vgpu_host_register": (C.c_int32, [vp, vp, u64]),
        "vgpu_host_unregister": (C.c_int32, [vp, vp]),
        "vgpu_dmat_upload": (C.c_int32, [vp, C.POINTER(_Matrix), C.c_int32, C.POINTER(vp)]),
        "vgpu_dmat_upload_rows": (C.c_int32, [vp, C.POINTER(_Matrix), C.c_int32, C.POINTER(vp)]),
        "vgpu_dmat_local_rows": (C.c_int32, [vp, C.POINTER(u64), C.POINTER(u64)]),
        "vgpu_dmat_download": (C.c_int32, [vp, vp, C.c_int32, u32p]),
        "vgpu_dmat_import": (C.c_int32, [vp, C.POINTER(_DevMatrix), C.c_int32, C.POINTER(vp)]),
        "vgpu_dmat_import_rows": (C.c_int32, [vp, C.POINTER(_DevMatrix), C.c_int32, C.POINTER(vp)]),
        "vgpu_dmat_borrow": (C.c_int32, [vp, vp, u64, u64, u64, C.POINTER(vp)]),
        "vgpu_dmat_export": (C.c_int32, [vp, vp, C.c_int32, C.POINTER(_DevMatrix)]),
        "vgpu_ctx_local_rows": (C.c_int32, [vp, u64, C.POINTER(u64), C.POINTER(u64)]),
        "vgpu_dmat_import_local": (C.c_int32, [vp, C.POINTER(_DevMatrix), u64, C.c_int32, C.POINTER(vp)]),
        "vgpu_dmat_borrow_local": (C.c_int32, [vp, vp, u64, u64, u64, C.POINTER(vp)]),
        "vgpu_dmat_export_local": (C.c_int32, [vp, vp, C.c_int32, C.POINTER(_DevMatrix)]),
        "vgpu_dmat_dims": (C.c_int32, [vp, C.POINTER(u64), C.POINTER(u64)]),
        "vgpu_dmat_free": (None, [vp]),
        "vgpu_ntt_batch": (C.c_int32, [vp, vp, C.c_int32]),
        "vgpu_coset_lde_batch": (C.c_int32, [vp, vp, C.c_uint32, C.c_uint32, C.c_int32, C.POINTER(vp)]),
        "vgpu_ntt_batch_host": (C.c_int32, [vp, u32p, u64, u64, C.c_int32, C.c_int32]),
        "vgpu_commit_batches": (C.c_int32, [vp, C.POINTER(vp), C.c_uint32, u32p, u32p, C.POINTER(vp)]),
        "vgpu_commit_batches_host": (C.c_int32, [vp, C.POINTER(_Matrix), C.c_uint32, C.c_int32, u32p, u32p, C.POINTER(vp)]),
        "vgpu_prover_data_lde": (C.c_int32, [vp, C.c_uint32, C.POINTER(vp)]),
        "vgpu_prover_data_free": (None, [vp]),
        "vgpu_basic_machine_chip": (vp, [C.c_uint32]),
        "vgpu_perm_trace": (C.c_int32, [vp, vp, vp, vp, u32p, C.POINTER(vp), u32p]),
        "vgpu_quotient": (C.c_int32, [vp, vp, C.c_uint32, vp, vp, vp, u32p, u32p, u32p, C.POINTER(vp)]),
        "vgpu_check_constraints": (C.c_int32, [vp, vp, vp, vp, vp, u32p, C.POINTER(C.c_int64), u32p, C.POINTER(u64)]),
        "vgpu_check_constraints_local": (C.c_int32, [vp, vp, vp, vp, vp, u32p, C.POINTER(C.c_int64), u32p, C.POINTER(u64)]),
        "vgpu_chip_constraint_count": (C.c_int32, [vp, u32p, u32p]),
        "vgpu_check_failures": (C.c_int32, [vp, vp, vp, vp, vp, u32p, u64, vp, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64)]),
        "vgpu_chip_column_name": (C.c_char_p, [vp, C.c_int32, C.c_uint32]),
        "vgpu_chip_constraint_cells": (C.c_int32, [vp, C.c_uint32, C.POINTER(C.c_char_p), vp, C.c_uint32, u32p]),
        "vgpu_explain_failures": (C.c_int32, [vp, vp, vp, vp, vp, vp, u64, C.POINTER(u64), u32p, u64, C.POINTER(u64)]),
        "vgpu_check_witness": (C.c_int32, [vp, C.POINTER(vp), C.POINTER(vp), u32p, C.POINTER(_CheckReport), C.POINTER(C.c_int32)]),
        "vgpu_check_buses": (C.c_int32, [vp, C.POINTER(vp), C.POINTER(vp), u32p, u64, vp, C.POINTER(u64), vp, C.POINTER(u64), C.POINTER(u64)]),
        "vgpu_bus_links": (C.c_int32, [vp, C.POINTER(vp), C.POINTER(vp), vp, u64, vp, u64, vp, C.POINTER(u64), C.POINTER(u64)]),
        "vgpu_ctx_set_debug_checks": (C.c_int32, [vp, C.c_int32]),
        "vgpu_set_challenger": (C.c_int32, [vp, u32p, u32p]),
        "vgpu_ctx_set_merkle_hash": (C.c_int32, [vp, C.c_int32]),
        "vgpu_challenger_reset": (C.c_int32, [vp]),
        "vgpu_challenger_observe": (C.c_int32, [vp, u32p, C.c_uint32]),
        "vgpu_challenger_sample_ext": (C.c_int32, [vp, u32p]),
        "vgpu_comm_unique_id": (C.c_int32, [C.c_char_p]),
        "vgpu_comm_init": (C.c_int32, [vp, C.c_int32, C.c_int32, C.c_char_p]),
        "vgpu_comm_init_local": (C.c_int32, [C.POINTER(vp), C.c_int32]),
        "vgpu_comm_stats": (None, [vp, u32p, C.POINTER(C.c_double), C.c_int32]),
        "vgpu_comm_set_sharding": (C.c_int32, [vp, C.c_int32]),
        "vgpu_shard_range": (None, [u64, C.c_int32, C.c_int32, C.POINTER(u64), C.POINTER(u64)]),
        "vgpu_split_column_plan": (None, [C.c_int32, C.c_uint32, C.POINTER(u64), C.POINTER(u64), u32p]),
        "vgpu_tree_share": (None, [u64, C.c_int32, C.c_int32, C.POINTER(u64), C.POINTER(u64), C.POINTER(C.c_int32)]),
        "vgpu_row_share": (None, [u64, C.c_int32, C.c_int32, C.POINTER(u64), C.POINTER(u64), C.POINTER(C.c_int32)]),
        "vgpu_open": (C.c_int32, [vp, C.POINTER(vp), C.c_uint32, u32p, u32p, C.POINTER(C.POINTER(C.c_uint8)), C.POINTER(u64)]),
        "vgpu_verify": (C.c_int32, [vp, C.c_char_p, u64, C.POINTER(_Matrix), C.c_int32, C.POINTER(C.c_int32)]),
        "vgpu_prove": (C.c_int32, [vp, C.POINTER(_Matrix), C.POINTER(_Matrix), C.c_int32, C.POINTER(C.POINTER(C.c_uint8)), C.POINTER(u64)]),
        "vgpu_prove_device": (C.c_int32, [vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(C.POINTER(C.c_uint8)), C.POINTER(u64)]),
        "vgpu_free_bytes": (None, [C.POINTER(C.c_uint8)]),
        "vgpu_last_prove_phases": (C.c_uint32, [vp, C.POINTER(C.c_char_p), C.POINTER(C.c_float), C.c_uint32]),
        "vgpu_machine_run": (C.c_int32, [C.POINTER(C.c_int32), u64, C.c_uint32, C.c_uint32, u64, C.POINTER(vp), C.c_char_p, u64]),
        "vgpu_machine_run_static": (C.c_int32, [C.POINTER(C.c_int32), u64, C.c_uint32, C.c_uint32, u64, u32p, u32p, u64, C.POINTER(vp), C.c_char_p, u64]),
        "vgpu_traces_main": (C.POINTER(_Matrix), [vp, C.c_uint32]),
        "vgpu_traces_preprocessed": (C.POINTER(_Matrix), [vp, C.c_uint32]),
        "vgpu_traces_stats": (None, [vp, u32p, u32p, u32p]),
        "vgpu_traces_mem_cell": (C.c_int32, [vp, C.c_uint32, u32p]),
        "vgpu_traces_free": (None, [vp]),
        "vgpu_fib_program": (u64, [C.c_uint32, C.POINTER(C.c_int32)]),
        "vgpu_vm_run": (C.c_int32, [C.POINTER(C.c_int32), u64, C.c_uint32, C.c_uint32, u64, u32p, u32p, u64, C.POINTER(vp), C.c_char_p, u64]),
        "vgpu_vmlog_stats": (None, [vp, u32p, u32p, u32p]),
        "vgpu_vmlog_traces": (C.c_int32, [vp, C.POINTER(vp), C.c_char_p, u64]),
        "vgpu_witness_device": (C.c_int32, [vp, vp, C.POINTER(vp), C.POINTER(vp)]),
        "vgpu_witness_column_count": (u64, []),
        "vgpu_diff_witness": (C.c_int32, [vp, vp, C.POINTER(vp), C.POINTER(vp), u64, vp, C.POINTER(u64), C.POINTER(u64), vp, C.POINTER(u64)]),
        "vgpu_vmlog_free": (None, [vp]),
        "vgpu_free_cells": (C.c_int32, [vp, vp, vp, vp, u64, vp, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64)]),
        "vgpu_cell_alternatives": (C.c_int32, [vp, vp, vp, vp, u64, vp, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64), C.POINTER(u64)]),
    }
    for name, (res, args) in sig.items():
        f = getattr(L, name)
        f.restype, f.argtypes = res, args
    return L


_lib = None


def lib():
    global _lib
    if _lib is None:
        _lib = _load()
    return _lib


def _as_u32(a):
    a = np.ascontiguousarray(a, dtype=np.uint32)
    return a


def _mat(a):
    return _Matrix(a.ctypes.data_as(C.POINTER(C.c_uint32)), a.shape[0], a.shape[1])


class Context:
    """One context per device/stream (single-threaded)."""

    def __init__(self, device=0, stream=None):
        self.device = device
        self._children = weakref.WeakSet()      # handles that point into this context: released before the context goes
        self._h = C.c_void_p()
        rc = lib().vgpu_ctx_create(device, C.c_void_p(stream) if stream else None, C.byref(self._h))
        if rc != 0:
            msg = lib().vgpu_last_error(self._h).decode() if self._h else "context allocation failed"
            if self._h:
                lib().vgpu_ctx_destroy(self._h)
                self._h = None
            raise VgpuError(msg)

    def check(self, rc):
        if rc != 0:
            raise VgpuError(lib().vgpu_last_error(self._h).decode())

    def synchronize(self):
        self.check(lib().vgpu_ctx_synchronize(self._h))

    def release_cached(self):
        """Free the device buffers kept for reuse by later calls (e.g. after a proof that filled most of the GPU)."""
        self.check(lib().vgpu_ctx_release_cached(self._h))

    def memory_stats(self, reset=False):
        """Device memory of this context in bytes: {"live", "peak" (of live, since creation or the last reset), "cached" (freed
        buffers kept for reuse; release_cached() empties it), "symm_peak" (symmetric heap of a split proof)}.  reset=True restarts
        both peaks from the current live bytes."""
        out = (C.c_uint64 * 4)()
        self.check(lib().vgpu_ctx_memory_stats(self._h, out, 1 if reset else 0))
        return dict(zip(("live", "peak", "cached", "symm_peak"), (int(v) for v in out)))

    @property
    def launch_count(self):
        return int(lib().vgpu_ctx_launch_count(self._h))

    def set_kernel_timing(self, on):
        lib().vgpu_ctx_set_kernel_timing(self._h, 1 if on else 0)

    def set_debug_checks(self, on):
        """Debug mode of prove_machine (the reference's debug builds): check_constraints on every chip and the cumulative sums
        before committing to a proof; a bad witness raises VgpuError naming each failing chip, row and constraint."""
        self.check(lib().vgpu_ctx_set_debug_checks(self._h, 1 if on else 0))

    def set_merkle_hash(self, hash):
        """The Merkle tree hash of the commits, openings, proofs and verifications that follow on this context:
        MERKLE_KECCAK256 (the default) or MERKLE_POSEIDON16 (PaddingFreeSponge / TruncatedPermutation over the challenger's
        Poseidon-16, which StarkConfig must have set first).  Proof bytes keep their format; a proof verifies only under the
        hash it was made with.  Every rank of a split proof makes the same call."""
        self.check(lib().vgpu_ctx_set_merkle_hash(self._h, int(hash)))

    def kernel_stats(self):
        """[(kernel class, launches, total ms, algorithmic bytes)] since the last call (synchronises)."""
        names = (C.c_char_p * 32)(); ln = (C.c_uint32 * 32)(); ms = (C.c_float * 32)(); by = (C.c_double * 32)()
        n = lib().vgpu_ctx_kernel_stats(self._h, names, ln, ms, by, 32)
        return [(names[i].decode(), int(ln[i]), float(ms[i]), float(by[i])) for i in range(n)]

    # ---- multi-GPU: one rank per GPU (include/valida_b200.h, "multi-GPU") ----
    def comm_init(self, rank, world_size, unique_id):
        """Join the NCCL communicator named by unique_id (comm_unique_id() of rank 0, distributed by the caller)."""
        self.check(lib().vgpu_comm_init(self._h, world_size, rank, bytes(unique_id)))
        self.rank, self.world_size = rank, world_size

    def comm_init_from_torch(self):
        """Convenience for torchrun ranks: rank 0 creates the id, torch.distributed carries it to the others."""
        import torch.distributed as dist

        ids = [comm_unique_id() if dist.get_rank() == 0 else None]
        dist.broadcast_object_list(ids, src=0)
        self.comm_init(dist.get_rank(), dist.get_world_size(), ids[0])

    def set_sharding(self, on):
        """False: this rank works alone (independent replicas); True: ONE proof is split across the ranks."""
        self.check(lib().vgpu_comm_set_sharding(self._h, 1 if on else 0))

    def comm_stats(self, reset=True):
        """Collectives since the last reset: {name: (calls, bytes sent to peers)} for barriers, all-gathers, peer-store exchanges."""
        calls = (C.c_uint32 * 3)(); by = (C.c_double * 3)()
        lib().vgpu_comm_stats(self._h, calls, by, 1 if reset else 0)
        return {n: (int(calls[i]), float(by[i])) for i, n in enumerate(("barrier", "allgather", "exchange"))}

    def upload_rows(self, row_major, repr=REPR_CANONICAL):
        """Split proof: of a trace tall enough to be split, keep this rank's run of rows only (otherwise like upload)."""
        a = _as_u32(row_major)
        m = _mat(a)
        out = C.c_void_p()
        self.check(lib().vgpu_dmat_upload_rows(self._h, C.byref(m), repr, C.byref(out)))
        return DeviceMatrix(self, out)

    # ---- caller device memory: torch tensors in, torch tensors out (include/valida_b200.h, vgpu_dmat_import / _borrow / _export) ----
    def _wait_for_torch(self, device):
        """The context's stream waits for torch's current stream on `device` (what it enqueued so far wrote the tensor)."""
        import torch

        ev = torch.cuda.Event()
        ev.record(torch.cuda.current_stream(device))
        self.check(lib().vgpu_ctx_wait_event(self._h, C.c_void_p(ev.cuda_event)))

    def _torch_waits(self, device):
        """torch's current stream on `device` waits for what the context's stream has enqueued so far."""
        import torch

        stream = torch.cuda.current_stream(device)
        ev = torch.cuda.Event()
        ev.record(stream)                       # creates the event on the device; the context's stream records it again
        self.check(lib().vgpu_ctx_record_event(self._h, C.c_void_p(ev.cuda_event)))
        stream.wait_event(ev)

    def _import_tensor(self, fn, what, t, repr):
        v = _tensor_view(self, t, what)
        self._wait_for_torch(t.device)
        out = C.c_void_p()
        self.check(fn(self._h, C.byref(v), repr, C.byref(out)))
        return DeviceMatrix(self, out)

    def import_tensor(self, t, repr=REPR_CANONICAL):
        """A 2-D CUDA tensor (torch.int32 or torch.uint32 bits, any non-negative strides, on this context's device) -> a
        library-owned DeviceMatrix, equal to upload() of the same words.  Ordered after torch's current stream; every word must be
        below p (VgpuError names the first that is not).  The tensor may change once this returns."""
        return self._import_tensor(lib().vgpu_dmat_import, "import_tensor", t, repr)

    def import_tensor_rows(self, t, repr=REPR_CANONICAL):
        """Split proof: import_tensor of this rank's run of rows of a trace tall enough to be split (every rank passes the whole
        tensor on its own device); otherwise like import_tensor."""
        return self._import_tensor(lib().vgpu_dmat_import_rows, "import_tensor_rows", t, repr)

    def _borrow_tensor(self, what, t, call):
        v = _tensor_view(self, t, what)
        if v.row_stride != 1:
            raise ValueError("%s: the tensor is not column-major (stride(0) = %d, must be 1)" % (what, v.row_stride))
        self._wait_for_torch(t.device)
        out = C.c_void_p()
        self.check(call(v, out))
        m = DeviceMatrix(self, out)
        m._tensor = t
        return m

    def borrow_tensor(self, t):
        """Zero-copy: a column-major tensor of Montgomery words (stride(0) == 1, stride(1) >= shape(0)) becomes a DeviceMatrix read in
        place.  Its words are checked once (below p); it is never written, and the DeviceMatrix keeps a reference to it.  Leave it
        unchanged while the DeviceMatrix is alive."""
        return self._borrow_tensor("borrow_tensor", t,
                                   lambda v, out: lib().vgpu_dmat_borrow(self._h, v.data, v.height, v.width, v.col_stride, C.byref(out)))

    # ---- row shards in caller device memory: each rank holds only its own rows (include/valida_b200.h, vgpu_dmat_*_local) ----
    def local_rows(self, height):
        """(row0, rows): the rows of a matrix of logical height `height` that this rank holds, and so must supply to
        import_tensor_local / borrow_tensor_local: its run of a trace tall enough to be split, otherwise (0, height)."""
        r0, n = C.c_uint64(), C.c_uint64()
        self.check(lib().vgpu_ctx_local_rows(self._h, height, C.byref(r0), C.byref(n)))
        return int(r0.value), int(n.value)

    def import_tensor_local(self, t, height, repr=REPR_CANONICAL):
        """import_tensor of this rank's rows only: `t` has local_rows(height)[1] rows (any strides), local row i being row row0 + i of
        the matrix.  Equal to import_tensor_rows of the whole tensor; a word not below p is named by its row in the whole matrix."""
        return self._import_tensor(lambda h, v, r, out: lib().vgpu_dmat_import_local(h, v, height, r, out), "import_tensor_local", t, repr)

    def borrow_tensor_local(self, t, height):
        """borrow_tensor of this rank's rows only: a column-major Montgomery tensor of local_rows(height)[1] rows (stride(0) == 1,
        stride(1) >= its rows, 4-byte alignment).  Read in place and never written; the DeviceMatrix keeps a reference to it."""
        def call(v, out):
            row0, rows = self.local_rows(height)
            if v.height != rows:
                raise ValueError("borrow_tensor_local: the tensor has %d rows, but of a matrix of height %d this rank holds rows = %d "
                                 "starting at row0 = %d" % (v.height, height, rows, row0))
            return lib().vgpu_dmat_borrow_local(self._h, v.data, height, v.width, v.col_stride, C.byref(out))

        return self._borrow_tensor("borrow_tensor_local", t, call)

    def host_register(self, array):
        """Page-lock a numpy array the caller will prove from repeatedly (its uploads then overlap the commits)."""
        self.check(lib().vgpu_host_register(self._h, C.c_void_p(array.ctypes.data), array.nbytes))

    def host_unregister(self, array):
        self.check(lib().vgpu_host_unregister(self._h, C.c_void_p(array.ctypes.data)))

    def upload(self, row_major, repr=REPR_CANONICAL):
        """RowMajorMatrix<Val> (numpy h x w uint32) -> DeviceMatrix."""
        a = _as_u32(row_major)
        if a.ndim != 2:
            raise ValueError("expected a 2-D row-major matrix")
        m = _mat(a)
        out = C.c_void_p()
        self.check(lib().vgpu_dmat_upload(self._h, C.byref(m), repr, C.byref(out)))
        return DeviceMatrix(self, out)

    def close(self):
        """Destroys the context.  Device matrices / prover data created from it are released first (their handles would dangle)."""
        if getattr(self, "_h", None):
            for child in list(getattr(self, "_children", ())):
                try:
                    child.free()
                except Exception:
                    pass
            lib().vgpu_ctx_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _tensor_view(ctx, t, what):
    """_DevMatrix of a 2-D CUDA tensor of 32-bit words on the context's device.  Strides of a dimension of size 1 are never used to
    address an element; they are normalised so that a column (h x 1) and a row (1 x w) read as column-major views."""
    import torch

    if not isinstance(t, torch.Tensor):
        raise TypeError("%s: expected a torch.Tensor, got %s" % (what, type(t).__name__))
    if t.device.type != "cuda":
        raise ValueError("%s: the tensor is on %s; a CUDA tensor on cuda:%d is needed" % (what, t.device, ctx.device))
    if t.device.index != ctx.device:
        raise ValueError("%s: the tensor is on %s, the context on cuda:%d" % (what, t.device, ctx.device))
    if t.dtype not in (torch.int32, torch.uint32):
        raise TypeError("%s: dtype %s; torch.int32 or torch.uint32 words are needed" % (what, t.dtype))
    if t.dim() != 2:
        raise ValueError("%s: a 2-D tensor is needed, got %d dimensions" % (what, t.dim()))
    (h, w), (rs, cs) = t.shape, t.stride()
    if rs < 0 or cs < 0:
        raise ValueError("%s: negative strides %s" % (what, t.stride()))
    if h <= 1:
        rs = 1
    if w <= 1:
        cs = max(cs, h)
    return _DevMatrix(t.data_ptr(), h, w, rs, cs)


class DeviceMatrix:
    def __init__(self, ctx, handle, owned=True):
        self.ctx, self._h, self._owned = ctx, handle, owned
        self._tensor = None                      # borrow_tensor: the caller's tensor the matrix reads in place
        ctx._children.add(self)

    @property
    def shape(self):
        h, w = C.c_uint64(), C.c_uint64()
        lib().vgpu_dmat_dims(self._h, C.byref(h), C.byref(w))
        return int(h.value), int(w.value)

    def local_rows(self):
        """(first row, rows) held on this rank — the whole matrix unless it is a row shard of a split proof."""
        r0, n = C.c_uint64(), C.c_uint64()
        lib().vgpu_dmat_local_rows(self._h, C.byref(r0), C.byref(n))
        return int(r0.value), int(n.value)

    def download(self, repr=REPR_CANONICAL, out=None):
        """The matrix as an (h, w) numpy uint32 array in natural row order, `repr` words.  Of a row shard only the rows this rank holds
        are written, at their natural rows (those of a bit-reversed shard, such as a split quotient's chunks, are scattered); the other
        rows are left as they were in `out`, or uninitialised without it."""
        h, w = self.shape
        if out is None:
            out = np.empty((h, w), dtype=np.uint32)
        elif out.shape != (h, w) or out.dtype != np.uint32 or not out.flags.c_contiguous:
            raise ValueError("download: out must be a C-contiguous (%d, %d) uint32 array" % (h, w))
        self.ctx.check(lib().vgpu_dmat_download(self.ctx._h, self._h, repr, out.ctypes.data_as(C.POINTER(C.c_uint32))))
        return out

    def to_tensor(self, repr=REPR_CANONICAL, out=None):
        """The matrix as a (h, w) torch.int32 CUDA tensor on the context's device (natural row order, `repr` words), or written into
        `out` (int32 or uint32, any strides).  Enqueued on the context's stream; torch's current stream waits for it.  Of a row shard
        only this rank's rows are written."""
        import torch

        h, w = self.shape
        dev = torch.device("cuda", self.ctx.device)
        if out is None:
            out = torch.empty((h, w), dtype=torch.int32, device=dev)
        v = _tensor_view(self.ctx, out, "to_tensor")
        if (v.height, v.width) != (h, w):
            raise ValueError("to_tensor: out has shape %s, the matrix is %d x %d" % (tuple(out.shape), h, w))
        self.ctx._wait_for_torch(dev)            # out may have been allocated or last used on torch's stream
        self.ctx.check(lib().vgpu_dmat_export(self.ctx._h, self._h, repr, C.byref(v)))
        self.ctx._torch_waits(dev)
        return out

    def local_to_tensor(self, repr=REPR_CANONICAL, out=None):
        """The rows held on this rank (local_rows()) as a (rows, w) torch.int32 CUDA tensor, local row i at row i, or written into
        `out` (int32 or uint32, any strides); of a whole matrix the same as to_tensor.  Ordered as to_tensor."""
        import torch

        _, rows = self.local_rows()
        w = self.shape[1]
        dev = torch.device("cuda", self.ctx.device)
        if out is None:
            out = torch.empty((rows, w), dtype=torch.int32, device=dev)
        v = _tensor_view(self.ctx, out, "local_to_tensor")
        self.ctx._wait_for_torch(dev)
        self.ctx.check(lib().vgpu_dmat_export_local(self.ctx._h, self._h, repr, C.byref(v)))
        self.ctx._torch_waits(dev)
        return out

    def free(self):
        if self._h and self._owned and self.ctx._h:
            lib().vgpu_dmat_free(self._h)
            if self._tensor is not None:         # torch may reuse the tensor's memory only after the context's reads of it
                self.ctx._torch_waits(self._tensor.device)
        self._h = None
        self._tensor = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class Radix2Dft:
    """p3_dft::TwoAdicSubgroupDft over device matrices (Radix2DitParallel / Radix2Bowers give the same values)."""

    def __init__(self, ctx):
        self.ctx = ctx

    def dft_batch(self, m):
        self.ctx.check(lib().vgpu_ntt_batch(self.ctx._h, m._h, 0))
        return m

    def idft_batch(self, m):
        self.ctx.check(lib().vgpu_ntt_batch(self.ctx._h, m._h, 1))
        return m

    def coset_lde_batch(self, m, added_bits, shift, bit_reversed=False):
        out = C.c_void_p()
        self.ctx.check(lib().vgpu_coset_lde_batch(self.ctx._h, m._h, added_bits, shift, 1 if bit_reversed else 0, C.byref(out)))
        return DeviceMatrix(self.ctx, out)


class ProverData:
    def __init__(self, ctx, handle, n):
        self.ctx, self._h, self.n = ctx, handle, n
        ctx._children.add(self)

    def free(self):
        if self._h and self.ctx._h:
            lib().vgpu_prover_data_free(self._h)
        self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class TwoAdicFriPcs:
    """UnivariatePcsWithLde surface used by Machine::prove (machine/src/config.rs:17-22)."""

    GENERATOR = 31

    def __init__(self, ctx, log_blowup=1, num_queries=40, proof_of_work_bits=8):
        if log_blowup != 1:
            raise VgpuError("the commit path is built for log_blowup = 1 (FriConfig of basic/src/bin/valida.rs:385-390); Radix2Dft.coset_lde_batch takes 1..4")
        self.ctx, self._log_blowup = ctx, log_blowup
        self.num_queries, self.proof_of_work_bits = num_queries, proof_of_work_bits

    def coset_shift(self):
        return self.GENERATOR

    def log_blowup(self):
        return self._log_blowup

    def commit_batches(self, polynomials):
        return self.commit_shifted_batches(polynomials, None)

    def commit_shifted_batches(self, polynomials, coset_shifts):
        n = len(polynomials)
        digest = (C.c_uint32 * 8)()
        out = C.c_void_p()
        shifts = None
        if coset_shifts is not None:
            shifts = (C.c_uint32 * n)(*[int(s) for s in coset_shifts])
        if n and isinstance(polynomials[0], DeviceMatrix):
            arr = (C.c_void_p * n)(*[m._h for m in polynomials])
            self.ctx.check(lib().vgpu_commit_batches(self.ctx._h, arr, n, shifts, digest, C.byref(out)))
        else:
            keep = [_as_u32(p) for p in polynomials]
            arr = (_Matrix * n)(*[_mat(a) for a in keep])
            self.ctx.check(lib().vgpu_commit_batches_host(self.ctx._h, arr, n, REPR_CANONICAL, shifts, digest, C.byref(out)))
        return np.array(list(digest), dtype=np.uint32), ProverData(self.ctx, out, n)

    def open_multi_batches(self, rounds, challenger=None):
        """rounds: [(ProverData, [[point, ...] per matrix])], points as 5 canonical words.  Uses the context's
        challenger (StarkConfig.challenger()).  Returns the CBOR bytes of (opened_values, proof)."""
        handles = (C.c_void_p * len(rounds))(*[pd._h for pd, _ in rounds])
        npts = np.array([len(p) for _, pts in rounds for p in pts], dtype=np.uint32)
        flat = np.array([w for _, pts in rounds for p in pts for z in p for w in z], dtype=np.uint32)
        out = C.POINTER(C.c_uint8)()
        n = C.c_uint64()
        self.ctx.check(lib().vgpu_open(self.ctx._h, handles, len(rounds), npts.ctypes.data_as(C.POINTER(C.c_uint32)),
                                       flat.ctypes.data_as(C.POINTER(C.c_uint32)), C.byref(out), C.byref(n)))
        data = C.string_at(out, n.value)
        lib().vgpu_free_bytes(out)
        return data

    def get_ldes(self, prover_data):
        """Committed LDEs (rows stored bit-reversed), borrowed views."""
        out = []
        for i in range(prover_data.n):
            v = C.c_void_p()
            self.ctx.check(lib().vgpu_prover_data_lde(prover_data._h, i, C.byref(v)))
            out.append(DeviceMatrix(self.ctx, v, owned=False))
        return out


def _u32arr(a, n):
    a = np.ascontiguousarray(a, dtype=np.uint32).reshape(-1)
    assert a.size == n
    return (C.c_uint32 * n)(*[int(x) for x in a])


def _h(m):
    """The handle of an optional DeviceMatrix argument."""
    return m._h if m is not None else None


def _witness_handles(main, prep):
    """The handle arrays of a machine witness: 14 main and 2 preprocessed DeviceMatrix traces."""
    return (C.c_void_p * NUM_CHIPS)(*[m._h for m in main]), (C.c_void_p * 2)(*[m._h for m in prep])


def generate_permutation_trace(ctx, chip_id, main, prep, random_elements):
    """machine/src/chip.rs:121 — returns (flattened perm trace DeviceMatrix, cumulative_sum[5])."""
    chip = lib().vgpu_basic_machine_chip(chip_id)
    out = C.c_void_p()
    cs = (C.c_uint32 * 5)()
    ctx.check(lib().vgpu_perm_trace(ctx._h, chip, main._h, _h(prep), _u32arr(random_elements, 15), C.byref(out), cs))
    return DeviceMatrix(ctx, out), np.array(list(cs), dtype=np.uint32)


def quotient(ctx, chip_id, log_degree, prep_lde, main_lde, perm_lde, cumulative_sum, perm_challenges, alpha):
    """machine/src/quotient.rs:18 — returns the h x 10 quotient-chunk DeviceMatrix."""
    chip = lib().vgpu_basic_machine_chip(chip_id)
    out = C.c_void_p()
    ctx.check(lib().vgpu_quotient(ctx._h, chip, log_degree, _h(prep_lde), main_lde._h, perm_lde._h,
                                  _u32arr(cumulative_sum, 5), _u32arr(perm_challenges, 15), _u32arr(alpha, 5), C.byref(out)))
    return DeviceMatrix(ctx, out)


def _check_chip(fn, ctx, chip_id, main, prep, perm, perm_challenges):
    row, con, n = C.c_int64(), C.c_uint32(), C.c_uint64()
    ctx.check(fn(ctx._h, lib().vgpu_basic_machine_chip(chip_id), main._h, _h(prep), perm._h, _u32arr(perm_challenges, 15),
                 C.byref(row), C.byref(con), C.byref(n)))
    return int(row.value), int(con.value), int(n.value)


def check_constraints(ctx, chip_id, main, prep, perm, perm_challenges):
    """machine/src/check_constraints.rs:14-84 on whole device traces (perm: the flattened permutation trace) — returns
    (first failing row or -1, index in eval order of its first failing constraint, number of rows with a failure)."""
    return _check_chip(lib().vgpu_check_constraints, ctx, chip_id, main, prep, perm, perm_challenges)


def check_constraints_local(ctx, chip_id, main, prep, perm, perm_challenges):
    """check_constraints on a split context: every rank calls it with its own matrices (its row shards of the tall traces, or whole
    matrices) and gets what check_constraints returns for the whole traces on one GPU.  On a context that does not split proofs it is
    check_constraints."""
    return _check_chip(lib().vgpu_check_constraints_local, ctx, chip_id, main, prep, perm, perm_challenges)


def constraint_count(chip_id):
    """(assertions of the chip's Air::eval, all its constraints: those, one per interaction, and the three LogUp constraints)."""
    air, total = C.c_uint32(), C.c_uint32()
    if lib().vgpu_chip_constraint_count(lib().vgpu_basic_machine_chip(chip_id), C.byref(air), C.byref(total)) != 0:
        raise VgpuError("constraint_count: unknown chip id %r" % (chip_id,))
    return int(air.value), int(total.value)


def constraint_label(chip_id, index):
    """What constraint `index` (eval order, as check_constraints and check_failures number them) of a chip is, from the chip
    description: "Air::eval assertion i", "interaction m (bus b, send|receive)", "LogUp transition", "LogUp first row" or
    "LogUp last row"."""
    air, total = constraint_count(chip_id)
    if not 0 <= index < total:
        raise VgpuError("constraint_label: chip %d has %d constraints, not %r" % (chip_id, total, index))
    if index < air:
        return "Air::eval assertion %d" % index
    desc = C.cast(lib().vgpu_basic_machine_chip(chip_id), C.POINTER(_ChipDesc)).contents
    m = index - air
    if m < desc.n_interactions:
        it = desc.interactions[m]
        return "interaction %d (bus %d, %s)" % (m, it.bus, "send" if it.is_send else "receive")
    return ("LogUp transition", "LogUp first row", "LogUp last row")[m - desc.n_interactions]


def check_failures(ctx, chip_id, main, prep, perm, perm_challenges, cap=1 << 16):
    """Every (row, constraint) on which check_constraints' constraints do not vanish, not only the first.  Takes what
    check_constraints_local takes (whole matrices, or on a split context this rank's row shards; collective there, with the same
    result on every rank).  Returns (failures, total, rows_per_constraint): the first min(cap, total) failures in ascending (row,
    constraint) order as a CHECK_FAILURE_DTYPE array (value: the constraint's canonical value, limbs 1..4 zero for a base-field
    constraint), the number of failures, and per constraint the number of rows on which it fails."""
    chip = lib().vgpu_basic_machine_chip(chip_id)
    _, total_constraints = constraint_count(chip_id)
    out = np.zeros(int(cap), dtype=CHECK_FAILURE_DTYPE)
    per = np.zeros(total_constraints, dtype=np.uint64)
    n, total = C.c_uint64(), C.c_uint64()
    ctx.check(lib().vgpu_check_failures(ctx._h, chip, main._h, _h(prep), perm._h, _u32arr(perm_challenges, 15),
                                        int(cap), out.ctypes.data_as(C.c_void_p) if cap else None, C.byref(n), C.byref(total),
                                        per.ctypes.data_as(C.POINTER(C.c_uint64))))
    return out[:n.value].copy(), int(total.value), per


def column_name(chip_id, trace, column):
    """The name of a column of the chip's main, preprocessed or flattened permutation trace (TRACE_MAIN / TRACE_PREPROCESSED /
    TRACE_PERMUTATION), after the reference's column structs, e.g. "mem_channels[1].value[2]"; permutation column 5m + l is
    "interactions[m].reciprocal[l]", or "running_sum[l]" for m = k.  None when the column is out of range."""
    name = lib().vgpu_chip_column_name(lib().vgpu_basic_machine_chip(chip_id), int(trace), int(column))
    return name.decode() if name is not None else None


Cell = collections.namedtuple("Cell", "trace next column name")
CellValue = collections.namedtuple("CellValue", "trace next column name value")
Explanation = collections.namedtuple("Explanation", "row constraint label cells")


def _constraint_cells(chip, chip_id, index):
    label, n = C.c_char_p(), C.c_uint32()
    if lib().vgpu_chip_constraint_cells(chip, int(index), C.byref(label), None, 0, C.byref(n)) != 0:
        raise VgpuError("constraint_cells: chip %r has no constraint %r" % (chip_id, index))
    cells = np.zeros(n.value, dtype=CELL_DTYPE)
    lib().vgpu_chip_constraint_cells(chip, int(index), C.byref(label), cells.ctypes.data_as(C.c_void_p), n.value, C.byref(n))
    return label.value.decode(), cells


def constraint_cells(chip_id, index):
    """What constraint `index` of a chip (eval order, as check_constraints and check_failures number it) reads, from the same AIR text
    the kernels evaluate: (label, [Cell(trace, next, column, name)]) in ascending (trace, next, column) order.  An Air::eval
    assertion's label names the block of the reference's eval it transcribes (e.g. "CpuChip::eval_pc"); the others are worded as
    constraint_label words them."""
    _, total = constraint_count(chip_id)
    if not 0 <= index < total:
        raise VgpuError("constraint_cells: chip %d has %d constraints, not %r" % (chip_id, total, index))
    label, cells = _constraint_cells(lib().vgpu_basic_machine_chip(chip_id), chip_id, index)
    return label, [Cell(int(c["trace"]), bool(c["next"]), int(c["column"]), column_name(chip_id, c["trace"], c["column"])) for c in cells]


def explain_failures(ctx, chip_id, main, prep, perm, items):
    """For each (row, constraint) item, the constraint's label and the values of the cells it reads on that row (a next-row cell at
    row (row + 1) mod h): one Explanation(row, constraint, label, cells=[CellValue(trace, next, column, name, value)]) per item,
    values canonical.  items: check_failures' array (its values are ignored) or a list of (row, constraint) pairs; a bus event of
    check_buses is (row, air_constraints + interaction).  perm None: permutation cells have value None.  Takes what check_failures
    takes (whole matrices, or on a split context this rank's row shards; collective there, every rank passing the same items and
    getting the same answer)."""
    chip = lib().vgpu_basic_machine_chip(chip_id)
    if isinstance(items, np.ndarray) and items.dtype == CHECK_FAILURE_DTYPE:
        arr = np.ascontiguousarray(items)
    else:
        pairs = list(items)
        arr = np.zeros(len(pairs), dtype=CHECK_FAILURE_DTYPE)
        for i, (row, con) in enumerate(pairs):
            arr[i]["row"], arr[i]["constraint"] = row, con
    n = len(arr)
    first = np.zeros(n + 1, dtype=np.uint64)
    # the catalogue sizes the output exactly (an out-of-range item is left for the call to refuse, naming it)
    _, total = constraint_count(chip_id)
    cat = {}
    for c in set(int(x) for x in arr["constraint"]):
        if 0 <= c < total:
            cat[c] = _constraint_cells(chip, chip_id, c)
    cap = sum(len(cat[int(c)][1]) for c in arr["constraint"] if int(c) in cat)
    values = np.zeros(max(cap, 1), dtype=np.uint32)
    nv = C.c_uint64()
    ctx.check(lib().vgpu_explain_failures(ctx._h, chip, main._h, _h(prep), _h(perm), arr.ctypes.data_as(C.c_void_p) if n else None, n,
                                          first.ctypes.data_as(C.POINTER(C.c_uint64)), values.ctypes.data_as(C.POINTER(C.c_uint32)), cap,
                                          C.byref(nv)))
    out = []
    for i in range(n):
        c = int(arr[i]["constraint"])
        label, cells = cat[c]
        vals = values[int(first[i]):int(first[i + 1])]
        out.append(Explanation(int(arr[i]["row"]), c, label,
                               [CellValue(int(x["trace"]), bool(x["next"]), int(x["column"]), column_name(chip_id, x["trace"], x["column"]),
                                          None if int(v) == CELL_ABSENT else int(v)) for x, v in zip(cells, vals)]))
    return out


def check_witness(ctx, main, prep, challenges):
    """check_constraints of the 14 chips and check_cumulative_sums over a machine witness (the reference's debug-build check), without
    a proof: main / prep are the 14 + 2 DeviceMatrix traces (whole, or this rank's row shards on a split context, where every rank
    calls it).  Returns ([(first row or -1, constraint, failing rows, cumulative sum [5]) per chip], sums_cancel)."""
    rep = (_CheckReport * NUM_CHIPS)()
    cancel = C.c_int32()
    ctx.check(lib().vgpu_check_witness(ctx._h, *_witness_handles(main, prep), _u32arr(challenges, 15), rep, C.byref(cancel)))
    return ([(int(r.first_row), int(r.first_constraint), int(r.failing_rows), np.array(list(r.cumulative_sum), dtype=np.uint32)) for r in rep],
            bool(cancel.value))


BusEvent = collections.namedtuple("BusEvent", "chip chip_name interaction row multiplicity send")
BusImbalance = collections.namedtuple("BusImbalance", "bus bus_name fields net events")
BusCheck = collections.namedtuple("BusCheck", "tuples complete unexamined")


def check_buses(ctx, main, prep, challenges, cap=1 << 16):
    """Every bus tuple the witness leaves unbalanced (sends minus receives not 0 mod p), with every event that sends or receives it.
    Takes what check_witness takes (whole traces, or this rank's row shards on a split context, where every rank calls it and gets
    the same answer).  Returns BusCheck(tuples, complete, unexamined): tuples in ascending (bus, fields) order, each a
    BusImbalance(bus, bus_name, fields trimmed of trailing zeros, net as a signed integer in (-p/2, p/2], events), its events
    BusEvent(chip, chip_name, interaction, row, multiplicity, send) in ascending (chip, row, interaction) order.  cap bounds the events
    (and so the tuples) examined; complete is False when unexamined > 0 candidate groups did not fit, and every tuple listed is exact
    either way.  The list is empty exactly when the LogUp sums cancel."""
    cap = int(cap)
    tup = np.zeros(cap, dtype=BUS_IMBALANCE_DTYPE)
    ev = np.zeros(cap, dtype=BUS_EVENT_DTYPE)
    nt, ne, un = C.c_uint64(), C.c_uint64(), C.c_uint64()
    ctx.check(lib().vgpu_check_buses(ctx._h, *_witness_handles(main, prep), _u32arr(challenges, 15), cap, tup.ctypes.data_as(C.c_void_p) if cap else None,
                                     C.byref(nt), ev.ctypes.data_as(C.c_void_p) if cap else None, C.byref(ne), C.byref(un)))
    out = []
    for t in tup[:nt.value]:
        fields = [int(x) for x in t["fields"]]
        while fields and fields[-1] == 0:
            fields.pop()
        net = int(t["net"])
        e0 = int(t["first_event"])
        events = [BusEvent(int(e["chip"]), CHIP_NAMES[int(e["chip"])], int(e["interaction"]), int(e["row"]), int(e["multiplicity"]), bool(e["is_send"]))
                  for e in ev[e0:e0 + int(t["n_events"])]]
        out.append(BusImbalance(int(t["bus"]), BUS_NAMES[int(t["bus"])] if t["bus"] < len(BUS_NAMES) else "bus %d" % t["bus"], fields,
                                net - BABYBEAR_P if net > BABYBEAR_P // 2 else net, events))
    return BusCheck(out, un.value == 0, int(un.value))


BusLink = collections.namedtuple("BusLink", "bus bus_name fields multiplicity sends receives n_events events")
BusLinks = collections.namedtuple("BusLinks", "links complete unlisted")
Cycles = collections.namedtuple("Cycles", "cycles complete")


def _bus_name(bus):
    return BUS_NAMES[bus] if bus < len(BUS_NAMES) else "bus %d" % bus


def bus_links(ctx, main, prep, items, cap=1 << 16):
    """Every event of the witness that carries each item's bus tuple, sends and receives alike: the CPU cycle whose general-bus send
    carries an ALU row's tuple, the memory row that receives a CPU channel's operation, the add and sub rows that send a range row's
    byte.  items: a BUS_EVENT_DTYPE array, check_buses' BusEvents or (chip, interaction, row) triples (multiplicity and direction are
    ignored, so an answer's events are items as they are).  Takes what check_buses takes (whole traces, or this rank's row shards on a
    split context, where every rank calls it with the same items and gets the same answer).  Returns BusLinks(links, complete,
    unlisted), one BusLink(bus, bus_name, fields trimmed of trailing zeros, multiplicity, sends, receives, n_events, events) per item:
    its tuple on its row, its own count (0: the item is no event), the summed send and receive multiplicities and the number of all
    events carrying the tuple (exact whatever cap is), and those events as BusEvents in ascending (chip, row, interaction) order, or
    None when its tuple was not listed.  Distinct tuples are listed in ascending (bus, fields) order while their events fit in cap;
    unlisted counts the others."""
    if isinstance(items, np.ndarray) and items.dtype == BUS_EVENT_DTYPE:
        arr = np.ascontiguousarray(items)
    else:
        triples = [(x.chip, x.interaction, x.row) if isinstance(x, BusEvent) else tuple(x) for x in items]
        arr = np.zeros(len(triples), dtype=BUS_EVENT_DTYPE)
        for i, (chip, m, row) in enumerate(triples):
            arr[i]["chip"], arr[i]["interaction"], arr[i]["row"] = chip, m, row
    n, cap = len(arr), int(cap)
    links = np.zeros(max(n, 1), dtype=BUS_LINK_DTYPE)
    ev = np.zeros(max(cap, 1), dtype=BUS_EVENT_DTYPE)
    ne, un = C.c_uint64(), C.c_uint64()
    ctx.check(lib().vgpu_bus_links(ctx._h, *_witness_handles(main, prep), arr.ctypes.data_as(C.c_void_p) if n else None, n,
                                   links.ctypes.data_as(C.c_void_p), cap, ev.ctypes.data_as(C.c_void_p) if cap else None,
                                   C.byref(ne), C.byref(un)))
    evs = [BusEvent(chip, CHIP_NAMES[chip], m, row, mult, bool(send)) for chip, m, row, mult, send in ev[:ne.value].tolist()]
    out = []
    for bus, fields, mult, sends, receives, k, e0 in links[:n].tolist():
        fields = fields.tolist()
        while fields and fields[-1] == 0:
            fields.pop()
        events = evs[e0:e0 + k] if e0 != 0xFFFFFFFFFFFFFFFF else None
        out.append(BusLink(bus, _bus_name(bus), fields, mult, sends, receives, k, events))
    return BusLinks(out, un.value == 0, int(un.value))


def _neighbours(ctx, main, prep, nodes, cap):
    """For each (chip, row) node, the nodes that carry an event of a tuple it carries an event of (itself left out), by one
    bus_links call over every interaction of every node; and whether every tuple was listed."""
    nodes = sorted(set(nodes))
    items = [(chip, m, row) for chip, row in nodes for m in range(_interaction_count(chip))]
    res = bus_links(ctx, main, prep, items, cap)
    out = {node: set() for node in nodes}
    for (chip, _, row), link in zip(items, res.links):
        if link.multiplicity and link.events is not None:
            out[(chip, row)].update((e.chip, e.row) for e in link.events)
    for node in nodes:
        out[node].discard(node)
    return out, res.complete


def _interaction_count(chip):
    return C.cast(lib().vgpu_basic_machine_chip(chip), C.POINTER(_ChipDesc)).contents.n_interactions


def cycles_of(ctx, main, prep, chip, rows, cap=1 << 16):
    """The cycles behind rows of one chip: in the graph whose nodes are (chip, row) and whose edges join two nodes that each carry an
    event of the same bus tuple, the CPU rows (cycles) at the least distance from the row, searching up to distance 2.  A CPU row is
    its own cycle; an ALU or memory row is at distance 1 from the cycles that send it its tuple; a range row reaches cycles through the
    add and sub rows that send it its byte.  Empty when no CPU row is that close: a static-initial memory row, a row without events,
    a row whose tuple no CPU row sends.  Two bus_links calls at most (so collective on a split context, as bus_links is).  Returns
    Cycles(cycles, complete): per row, its cycles ascending, and whether cap let every tuple consulted list its events."""
    rows = [int(r) for r in rows]
    if chip == 0:
        h = main[0].shape[0]
        bad = [r for r in rows if not 0 <= r < h]
        if bad:
            raise VgpuError("cycles_of: row %d is outside the CPU trace of height %d" % (bad[0], h))
        return Cycles([[r] for r in rows], True)
    near, complete = _neighbours(ctx, main, prep, [(chip, r) for r in rows], cap)
    far_nodes = {x for r in rows if not any(c == 0 for c, _ in near[(chip, r)]) for x in near[(chip, r)]}
    far, done = _neighbours(ctx, main, prep, far_nodes, cap) if far_nodes else ({}, True)
    cycles = []
    for r in rows:
        hit = sorted(x for c, x in near[(chip, r)] if c == 0)
        if not hit:
            hit = sorted({x for node in near[(chip, r)] for c, x in far[node] if c == 0})
        cycles.append(hit)
    return Cycles(cycles, complete and done)


CellDiff = collections.namedtuple("CellDiff", "chip chip_name trace column column_name row have want")
ChipDiff = collections.namedtuple("ChipDiff", "chip chip_name height_have height_want cells first_row")
WitnessDiff = collections.namedtuple("WitnessDiff", "cells total complete chips per_column")


def witness_column_count():
    """The length of diff_witness' per-column counts: the main columns of chips 0..13 in chip order, then the 7 program and the 1
    range preprocessed columns."""
    return int(lib().vgpu_witness_column_count())


def diff_witness(ctx, log, main, prep, cap=1 << 16):
    """Every cell of a witness (main / prep: the 14 + 2 DeviceMatrix traces, whole or this rank's row shards on a split context, where
    every rank calls it and gets the same answer) that differs from what Chip::generate_trace writes for the run `log` (a VmLog)
    records.  Returns WitnessDiff(cells, total, complete, chips, per_column):
      - cells: the first min(cap, total) CellDiff(chip, chip_name, trace, column, column_name, row, have, want) in ascending (chip,
        trace, row, column) order (trace TRACE_MAIN, or TRACE_PREPROCESSED for the program and range traces; have: the witness' word,
        want: generate_trace's, both canonical), so the first CPU entry is on the first cycle whose row differs;
      - total: the number of differing cells, complete: whether cells holds them all;
      - chips: one ChipDiff(chip, chip_name, height_have, height_want, cells, first_row) per chip (first_row -1: none).  A chip whose
        height differs from the run's is reported there and its cells are not compared;
      - per_column: the differing cells of each column (witness_column_count() entries).
    The expected witness is built on the GPU one chip at a time and compared there; nothing is downloaded but the result."""
    cap = int(cap)
    out = np.zeros(cap, dtype=CELL_DIFF_DTYPE)
    summ = np.zeros(NUM_CHIPS, dtype=DIFF_SUMMARY_DTYPE)
    per = np.zeros(witness_column_count(), dtype=np.uint64)
    n, total = C.c_uint64(), C.c_uint64()
    ctx.check(lib().vgpu_diff_witness(ctx._h, log._h, *_witness_handles(main, prep), cap, out.ctypes.data_as(C.c_void_p) if cap else None, C.byref(n), C.byref(total),
                                      summ.ctypes.data_as(C.c_void_p), per.ctypes.data_as(C.POINTER(C.c_uint64))))
    names = {}

    def name(chip, trace, column):
        key = (chip, trace, column)
        if key not in names:
            names[key] = column_name(chip, trace, column)
        return names[key]

    cells = [CellDiff(int(e["chip"]), CHIP_NAMES[int(e["chip"])], int(e["trace"]), int(e["column"]), name(int(e["chip"]), int(e["trace"]), int(e["column"])),
                      int(e["row"]), int(e["have"]), int(e["want"])) for e in out[:n.value]]
    chips = [ChipDiff(c, CHIP_NAMES[c], int(x["height_have"]), int(x["height_want"]), int(x["cells"]), int(x["first_row"])) for c, x in enumerate(summ)]
    return WitnessDiff(cells, int(total.value), n.value == total.value, chips, per)


FreeCell = collections.namedtuple("FreeCell", "row column column_name")
FreeCells = collections.namedtuple("FreeCells", "cells total complete per_column")


def free_cells(ctx, chip_id, main, prep, cap=1 << 16):
    """Every main-trace cell of one chip's witness that no check pins: no assertion of the chip's Air::eval changes with the cell (on
    its row, and on the row before as that row's next row), and no bus event does (no interaction's count reads its column, and on a
    row where an interaction's count is not 0 none of its fields does).  Changing one such cell of a witness that passes check_witness
    leaves it passing, so its proof still verifies: the cells are the chip's AIR gaps on this witness.  Takes what check_failures
    takes without perm and challenges (whole matrices, or on a split context this rank's row shards; collective there, with the same
    result on every rank).  Returns FreeCells(cells, total, complete, per_column): the first min(cap, total) FreeCell(row, column,
    column_name) in ascending (row, column) order, the number of free cells, whether cells holds them all, and per column name its
    number of free rows."""
    cap = int(cap)
    chip = lib().vgpu_basic_machine_chip(chip_id)
    if not chip:
        raise VgpuError("free_cells: unknown chip id %r" % (chip_id,))
    width = C.cast(chip, C.POINTER(_ChipDesc)).contents.width
    out = np.zeros(cap, dtype=FREE_CELL_DTYPE)
    per = np.zeros(width, dtype=np.uint64)
    n, total = C.c_uint64(), C.c_uint64()
    ctx.check(lib().vgpu_free_cells(ctx._h, chip, main._h, _h(prep), cap, out.ctypes.data_as(C.c_void_p) if cap else None, C.byref(n),
                                    C.byref(total), per.ctypes.data_as(C.POINTER(C.c_uint64))))
    names = [column_name(chip_id, TRACE_MAIN, c) for c in range(width)]
    cells = [FreeCell(int(e["row"]), int(e["column"]), names[int(e["column"])]) for e in out[:n.value]]
    return FreeCells(cells, int(total.value), n.value == total.value, {names[c]: int(per[c]) for c in range(width)})


CellAlternative = collections.namedtuple("CellAlternative", "row column column_name value values bus")
CellAlternatives = collections.namedtuple("CellAlternatives", "cells total bus_free complete per_column")


def cell_alternatives(ctx, chip_id, main, prep, cap=1 << 16):
    """Every main-trace cell of one chip's witness that the chip's Air::eval assertions would also accept at another value: S, the
    assertions whose value depends on the cell (on its row, and on the row before as that row's next row), is not empty and its
    polynomials in the cell share a root other than the cell's value.  Those roots are the cell's values.  bus: a bus event reads the
    cell (free_cells' rule).  Setting one such cell with bus False of a witness that passes check_witness to one of its values leaves
    the witness passing check_witness and check_buses, so its proof still verifies; on a witness with one wrong cell that an assertion
    reads, the right value is among that cell's values.  Takes what free_cells takes (collective on a split context, with the same
    result on every rank).  Returns CellAlternatives(cells, total, bus_free, complete, per_column): the first min(cap, total)
    CellAlternative(row, column, column_name, value, values, bus) in ascending (row, column) order (value and values canonical, values
    ascending), the number of listed cells and of those with bus False, whether cells holds them all, and per column name
    (listed, bus_free) rows."""
    cap = int(cap)
    chip = lib().vgpu_basic_machine_chip(chip_id)
    if not chip:
        raise VgpuError("cell_alternatives: unknown chip id %r" % (chip_id,))
    width = C.cast(chip, C.POINTER(_ChipDesc)).contents.width
    out = np.zeros(cap, dtype=CELL_ALTERNATIVE_DTYPE)
    per = np.zeros(2 * width, dtype=np.uint64)
    n, total, bus_free = C.c_uint64(), C.c_uint64(), C.c_uint64()
    ctx.check(lib().vgpu_cell_alternatives(ctx._h, chip, main._h, _h(prep), cap, out.ctypes.data_as(C.c_void_p) if cap else None,
                                           C.byref(n), C.byref(total), C.byref(bus_free), per.ctypes.data_as(C.POINTER(C.c_uint64))))
    names = [column_name(chip_id, TRACE_MAIN, c) for c in range(width)]
    cells = [CellAlternative(int(e["row"]), int(e["column"]), names[int(e["column"])], int(e["value"]),
                             tuple(int(v) for v in e["values"][:int(e["n_values"])]), bool(e["bus"])) for e in out[:n.value]]
    return CellAlternatives(cells, int(total.value), int(bus_free.value), n.value == total.value,
                            {names[c]: (int(per[c]), int(per[width + c])) for c in range(width)})


class StarkConfig:
    """StarkConfigImpl (machine/src/config.rs:33-76): the PCS plus the initial challenger.

    round_constants: the 480 Poseidon round constants the caller's RNG produced
    (Poseidon::new_from_rng(4, 22, mds, rng), basic/src/bin/valida.rs:364-365), canonical words.
    """

    def __init__(self, ctx, round_constants, mds=None):
        self.ctx = ctx
        self.pcs_ = TwoAdicFriPcs(ctx)
        rc = _u32arr(round_constants, 480)
        m = _u32arr(mds, 256) if mds is not None else None
        ctx.check(lib().vgpu_set_challenger(ctx._h, rc, m))

    def pcs(self):
        return self.pcs_


def prove_machine(config, traces, device_resident=None, repr=REPR_CANONICAL):
    """Machine::prove (machine/src/machine.rs:22-24): returns the CBOR bytes of MachineProof.

    traces: MachineTraces (host, row-major; every word in the representation `repr`: REPR_CANONICAL, or REPR_MONTY_R32 as the Rust
    caller passes BabyBear's own words).  device_resident: optional pair ([14 DeviceMatrix], [2 DeviceMatrix]) already uploaded
    (bench's HBM-resident timing); `repr` does not apply to it."""
    ctx = config.ctx
    out = C.POINTER(C.c_uint8)()
    n = C.c_uint64()
    if device_resident is not None:
        ctx.check(lib().vgpu_prove_device(ctx._h, *_witness_handles(*device_resident), C.byref(out), C.byref(n)))
    else:
        keep = [_as_u32(m) for m in traces.main] + [_as_u32(m) for m in traces.preprocessed]
        a = (_Matrix * NUM_CHIPS)(*[_mat(m) for m in keep[:NUM_CHIPS]])
        b = (_Matrix * 2)(*[_mat(m) for m in keep[NUM_CHIPS:]])
        ctx.check(lib().vgpu_prove(ctx._h, a, b, repr, C.byref(out), C.byref(n)))
    proof = C.string_at(out, n.value)
    lib().vgpu_free_bytes(out)
    return proof


COMM_ID_BYTES = 128


def comm_init_local(contexts):
    """One process, one worker THREAD per context (a Rust host with a thread per GPU): contexts[i] becomes rank i of a
    split proof.  Afterwards every rank's calls must come from its own thread — the collectives wait for all ranks.
    Several contexts may share a device (how the split-proof tests run on a one-GPU box)."""
    n = len(contexts)
    arr = (C.c_void_p * n)(*[c._h for c in contexts])
    rc = lib().vgpu_comm_init_local(arr, n)
    if rc != 0:
        raise VgpuError(lib().vgpu_last_error(contexts[0]._h).decode())
    for i, c in enumerate(contexts):
        c.rank, c.world_size = i, n


def run_ranks(fn, contexts):
    """Run fn(rank, ctx) on one thread per context and return the results in rank order (re-raises the first failure)."""
    import threading

    out, err = [None] * len(contexts), [None] * len(contexts)

    def work(i):
        try:
            out[i] = fn(i, contexts[i])
        except BaseException as e:   # noqa: BLE001
            err[i] = e

    th = [threading.Thread(target=work, args=(i,)) for i in range(len(contexts))]
    for t in th:
        t.start()
    for t in th:
        t.join()
    for e in err:
        if e is not None:
            raise e
    return out


def comm_unique_id():
    buf = C.create_string_buffer(COMM_ID_BYTES)
    if lib().vgpu_comm_unique_id(buf) != 0:
        raise VgpuError("NCCL is not available (libnccl.so.2 could not be loaded)")
    return buf.raw


def shard_range(total, world_size, rank):
    """Contiguous balanced split used for the column shares: (begin, end)."""
    b, e = C.c_uint64(), C.c_uint64()
    lib().vgpu_shard_range(total, world_size, rank, C.byref(b), C.byref(e))
    return int(b.value), int(e.value)


def split_column_plan(world_size, shapes):
    """Column ownership of one split commit: shapes = [(height, width), ...] -> per matrix the list of world_size + 1 first-column indices."""
    n = len(shapes)
    hs = (C.c_uint64 * n)(*[int(h) for h, _ in shapes])
    ws = (C.c_uint64 * n)(*[int(w) for _, w in shapes])
    out = (C.c_uint32 * (n * (world_size + 1)))()
    lib().vgpu_split_column_plan(world_size, n, hs, ws, out)
    return [[int(out[i * (world_size + 1) + r]) for r in range(world_size + 1)] for i in range(n)]


def tree_share(length, world_size, rank):
    """(begin, count, split) — the part of a tree layer a rank derives itself when commits are split (any world_size 1..16)."""
    b, c, sp = C.c_uint64(), C.c_uint64(), C.c_int32()
    lib().vgpu_tree_share(length, world_size, rank, C.byref(b), C.byref(c), C.byref(sp))
    return int(b.value), int(c.value), bool(sp.value)


def row_share(length, world_size, rank):
    """(begin, count, split) — the run of a matrix / vector of `length` stored rows a rank holds in a split proof of world_size
    (1..16) ranks: with P the next power of two >= world_size, a length >= 4096 P is cut into 8 P units and rank r holds units
    [r * 8P // world_size, (r + 1) * 8P // world_size); a shorter one is held whole by every rank (split False)."""
    b, c, sp = C.c_uint64(), C.c_uint64(), C.c_int32()
    lib().vgpu_row_share(length, world_size, rank, C.byref(b), C.byref(c), C.byref(sp))
    return int(b.value), int(c.value), bool(sp.value)


class VerificationError(Exception):
    """Machine::verify rejected the proof; .verdict is the VGPU_REJECT_* code of include/valida_b200.h."""

    NAMES = {-1: "malformed proof", -2: "shape mismatch", -3: "invalid proof-of-work witness", -4: "input Merkle opening",
             -5: "FRI Merkle opening", -6: "FRI final polynomial mismatch", -7: "non-zero cumulative sum"}

    def __init__(self, verdict):
        self.verdict = verdict
        what = self.NAMES.get(verdict) or ("out-of-domain evaluation mismatch on chip %d" % (-100 - verdict))
        super().__init__("proof rejected: %s (verdict %d)" % (what, verdict))


def verify_machine(config, proof, preprocessed, repr=REPR_CANONICAL):
    """Machine::verify (machine/src/machine.rs:26-31): raises VerificationError unless the proof is accepted.

    proof: CBOR bytes of MachineProof; preprocessed: the two preprocessed traces (program, range), row-major, words in the
    representation `repr` (REPR_CANONICAL or REPR_MONTY_R32)."""
    ctx = config.ctx
    keep = [_as_u32(m) for m in preprocessed]
    b = (_Matrix * 2)(*[_mat(m) for m in keep])
    verdict = C.c_int32(-1)
    ctx.check(lib().vgpu_verify(ctx._h, bytes(proof), len(proof), b, repr, C.byref(verdict)))
    if verdict.value != 0:
        raise VerificationError(verdict.value)


def last_prove_phases(ctx):
    names = (C.c_char_p * 32)()
    ms = (C.c_float * 32)()
    n = lib().vgpu_last_prove_phases(ctx._h, names, ms, 32)
    return [(names[i].decode(), float(ms[i])) for i in range(min(n, 32))]


class MachineTraces:
    """Host witness of one BasicMachine run: 14 main traces (chip order) + 2 preprocessed traces."""

    CHIPS = ["cpu", "program", "mem", "add", "sub", "mul", "div", "shift", "lt", "com", "bitwise", "output", "range", "static_data"]

    def __init__(self, handle):
        self._h = handle
        L = lib()
        self.main = []
        for i in range(NUM_CHIPS):
            m = L.vgpu_traces_main(handle, i).contents
            self.main.append(np.ctypeslib.as_array(m.data, shape=(m.height * m.width,)).reshape(m.height, m.width))
        self.preprocessed = []
        for i in range(2):
            m = L.vgpu_traces_preprocessed(handle, i).contents
            self.preprocessed.append(np.ctypeslib.as_array(m.data, shape=(m.height * m.width,)).reshape(m.height, m.width))
        c, mo, ao = C.c_uint32(), C.c_uint32(), C.c_uint32()
        L.vgpu_traces_stats(handle, C.byref(c), C.byref(mo), C.byref(ao))
        self.clock, self.mem_ops, self.add_ops = c.value, mo.value, ao.value

    def mem_cell(self, addr):
        v = C.c_uint32()
        if lib().vgpu_traces_mem_cell(self._h, addr, C.byref(v)) != 0:
            return None
        return v.value

    def free(self):
        if self._h:
            self.main, self.preprocessed = [], []
            lib().vgpu_traces_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


class VmLog:
    """Machine::run without the row fill: the interpreter's logs (one record per cycle / memory operation / ALU operation)."""

    def __init__(self, handle):
        self._h = handle
        c, mo, ao = C.c_uint32(), C.c_uint32(), C.c_uint32()
        lib().vgpu_vmlog_stats(handle, C.byref(c), C.byref(mo), C.byref(ao))
        self.clock, self.mem_ops, self.add_ops = c.value, mo.value, ao.value

    def traces(self):
        """Chip::generate_trace x14 on the host from these logs."""
        h = C.c_void_p()
        err = C.create_string_buffer(512)
        if lib().vgpu_vmlog_traces(self._h, C.byref(h), err, 512) != 0:
            raise VgpuError(err.value.decode())
        return MachineTraces(h)

    def witness_device(self, ctx):
        """Chip::generate_trace x14 on the GPU: ([14 DeviceMatrix], [2 DeviceMatrix]) for prove_machine(device_resident=...)."""
        main = (C.c_void_p * NUM_CHIPS)()
        prep = (C.c_void_p * 2)()
        ctx.check(lib().vgpu_witness_device(ctx._h, self._h, main, prep))
        return [DeviceMatrix(ctx, C.c_void_p(main[i])) for i in range(NUM_CHIPS)], [DeviceMatrix(ctx, C.c_void_p(prep[i])) for i in range(2)]

    def diff_witness(self, ctx, main, prep, cap=1 << 16):
        """diff_witness(ctx, self, main, prep, cap): the cells of a witness that differ from this run's."""
        return diff_witness(ctx, self, main, prep, cap)

    def free(self):
        if self._h:
            lib().vgpu_vmlog_free(self._h)
            self._h = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


def run_program_log(program, initial_fp=0x1000, initial_pc=0, max_cycles=1 << 30, static_data=None):
    """Machine::run only (host interpreter): returns the VmLog the host or the device expands into traces."""
    p = np.ascontiguousarray(program, dtype=np.int32)
    h = C.c_void_p()
    err = C.create_string_buffer(512)
    sa = np.array(sorted((static_data or {}).keys()), dtype=np.uint32)
    sv = np.array([(static_data or {})[int(a)] for a in sa], dtype=np.uint32)
    u32ptr = C.POINTER(C.c_uint32)
    rc = lib().vgpu_vm_run(p.ctypes.data_as(C.POINTER(C.c_int32)), p.shape[0], initial_pc, initial_fp, max_cycles,
                           sa.ctypes.data_as(u32ptr), sv.ctypes.data_as(u32ptr), len(sa), C.byref(h), err, 512)
    if rc != 0:
        raise VgpuError(err.value.decode())
    return VmLog(h)


def fib_program(n):
    """fib_program() of basic/tests/test_prover.rs:35-188 with the `imm32 -8(fp)` operand set to n."""
    words = (C.c_int32 * (23 * 6))()
    cnt = lib().vgpu_fib_program(n, words)
    return np.array(list(words), dtype=np.int32).reshape(int(cnt), 6)


def run_program(program, initial_fp=0x1000, initial_pc=0, max_cycles=1 << 30, static_data=None):
    """Machine::run + generate_trace for every chip (host).  static_data: {address: 32-bit cell} preloaded through the
    static-data chip (machine.static_data_mut().write(addr, Word(..)), basic/tests/test_static_data.rs:59-60)."""
    p = np.ascontiguousarray(program, dtype=np.int32)
    h = C.c_void_p()
    err = C.create_string_buffer(512)
    sa = np.array(sorted((static_data or {}).keys()), dtype=np.uint32)
    sv = np.array([(static_data or {})[int(a)] for a in sa], dtype=np.uint32)
    u32ptr = C.POINTER(C.c_uint32)
    rc = lib().vgpu_machine_run_static(p.ctypes.data_as(C.POINTER(C.c_int32)), p.shape[0], initial_pc, initial_fp, max_cycles,
                                       sa.ctypes.data_as(u32ptr), sv.ctypes.data_as(u32ptr), len(sa), C.byref(h), err, 512)
    if rc != 0:
        raise VgpuError(err.value.decode())
    return MachineTraces(h)
