"""Cost of diff_witness (every cell of a witness that differs from its run's): python profiles/prof_diff_witness.py [log_rows] [reps]

On the Fibonacci run with 2^log_rows CPU rows (default 22: memory chip 2^24 rows, 2.06 GB per witness), on one GPU, medians over reps
after a warm-up of each:
  witness_device   vgpu_witness_device alone (the build diff_witness repeats, one chip at a time);
  clean            diff_witness of the device witness of the same run;
  one change       the same with one memory-chip value byte changed.
Each as the host clock around the synchronising call, and, in separate runs under torch.profiler, the device time of the kernels by
group: "compare" (diff_count_kernel, diff_write_kernel and the CTA scan), "build" (the row kernels and the address sort of the
witness builder) and the copies.  The compare kernels read both witnesses once, so their rate is 2 x witness bytes / compare time.
Prints the GPU's name and power limit read in the same run, and the call's peak device memory above the witness."""
import os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from torch.profiler import ProfilerActivity, profile
import valida_b200 as vb

args = sys.argv[1:]
log_rows = int(args[0]) if args else 22
reps = int(args[1]) if len(args) > 1 else 10
P = vb.BABYBEAR_P
q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
print("gpu:", q.stdout.strip() or "(nvidia-smi unavailable)", flush=True)
ctx = vb.Context(0)
log = vb.run_program_log(vb.fib_program(((1 << log_rows) - 17) // 7))
dm, dp = log.witness_device(ctx)
witness_bytes = sum(m.shape[0] * m.shape[1] * 4 for m in dm + dp)
print("cpu rows 2^%d, memory rows %d, witness %.2f GB" % (log_rows, dm[2].shape[0], witness_bytes / 1e9), flush=True)
med = lambda v: float(np.median(v))


def wall_ms(fn):
    fn()
    t = []
    for _ in range(reps):
        ctx.synchronize()
        t0 = time.perf_counter()
        fn()
        t.append((time.perf_counter() - t0) * 1e3)
    return med(t)


def group(name):
    if "diff_" in name or "fail_scan" in name:
        return "compare"
    if "rows_kernel" in name or "sort_" in name or "addr_bits" in name or "scan_u32" in name or "rm_to_cm" in name:
        return "build"
    if "memcpy" in name.lower() or "memset" in name.lower():
        return "copies"
    return "other"


def kernel_ms(fn, n=3):
    """device ms per call by group, from torch.profiler over n calls"""
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        us = getattr(e, "self_device_time_total", None)
        if us is None:
            us = e.self_cuda_time_total
        if us:
            out[group(e.key)] = out.get(group(e.key), 0.0) + us / 1e3 / n
    return out


def report(name, fn):
    wall = wall_ms(fn)
    k = kernel_ms(fn)
    rate = " compare rate %.2f TB/s" % (2 * witness_bytes / (k["compare"] * 1e-3) / 1e12) if k.get("compare") else ""
    print("%-34s call %8.2f ms   %s%s" % (name, wall, "  ".join("%s %.2f ms" % kv for kv in sorted(k.items())), rate), flush=True)


def build_only():
    m, p = log.witness_device(ctx)
    del m, p


res = vb.diff_witness(ctx, log, dm, dp)
assert res.total == 0, "the device witness differs from its own run"
ctx.memory_stats(reset=True)
vb.diff_witness(ctx, log, dm, dp)
print("diff_witness peak live device memory above the witness: %.1f MB" % ((ctx.memory_stats()["peak"] - ctx.memory_stats()["live"]) / 1e6), flush=True)
report("witness_device", build_only)
report("clean: diff_witness", lambda: vb.diff_witness(ctx, log, dm, dp))

h = dm[2].shape[0]
mem = dm[2].to_tensor()
r = h // 2 + 12345
mem[r, 1] = (mem[r, 1].to(torch.int64) + 1) % P
torch.cuda.synchronize()
bad = dm[:2] + [ctx.import_tensor(mem)] + dm[3:]
del mem
res = vb.diff_witness(ctx, log, bad, dp)
print("changed row %d: %s" % (r, [(e.chip_name, e.column_name, e.row, e.have, e.want) for e in res.cells]), flush=True)
report("one change: diff_witness", lambda: vb.diff_witness(ctx, log, bad, dp))
