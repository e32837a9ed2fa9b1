"""Cost of cell_alternatives (the other values the AIR accepts in a cell): python profiles/prof_cell_alternatives.py [log_rows] [reps]

On the device witness of the Fibonacci run with 2^log_rows CPU rows (default 22: memory chip 2^24 rows), on one GPU, per chip with the
default cap (2^16):
  call      the host clock around the synchronising call (median over reps after a warm-up);
  kernels   the KC_CHECK kernel time of one call (kernel_stats(): the count pass, the CTA scan and the write pass);
  peak      the call's peak device memory above what was live before it;
  listed    the cells with another value, of them bus-free, and the columns of the bus-free ones.
Prints the GPU's name and power limit read in the same run."""
import os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import valida_b200 as vb

args = sys.argv[1:]
log_rows = int(args[0]) if args else 22
reps = int(args[1]) if len(args) > 1 else 5
PREP = {1: 0, 12: 1}
q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
print("gpu:", q.stdout.strip() or "(nvidia-smi unavailable)", flush=True)
ctx = vb.Context(0)
log = vb.run_program_log(vb.fib_program(((1 << log_rows) - 17) // 7))
dm, dp = log.witness_device(ctx)
print("cpu rows 2^%d, memory rows %d" % (log_rows, dm[2].shape[0]), flush=True)
total_ms = 0.0
for chip in range(14):
    prep = dp[PREP[chip]] if chip in PREP else None
    call = lambda: vb.cell_alternatives(ctx, chip, dm[chip], prep)
    res = call()
    t = []
    for _ in range(reps):
        ctx.synchronize()
        t0 = time.perf_counter()
        call()
        t.append((time.perf_counter() - t0) * 1e3)
    ctx.set_kernel_timing(True)
    ctx.kernel_stats()
    call()
    k = sum(ms for name, _, ms, _ in ctx.kernel_stats() if name == "check_kernel")
    ctx.set_kernel_timing(False)
    ctx.memory_stats(reset=True)
    live = ctx.memory_stats()["live"]
    call()
    peak = ctx.memory_stats()["peak"] - live
    h = dm[chip].shape[0]
    cols = ["%s (%d)" % (n, f) for n, (_, f) in res.per_column.items() if f]
    total_ms += float(np.median(t))
    print("%-12s rows %9d  call %8.2f ms  kernels %8.2f ms  peak %8.1f KB  listed %10d  bus-free %10d  bus-free columns: %s"
          % (vb.CHIP_NAMES[chip], h, float(np.median(t)), k, peak / 1e3, res.total, res.bus_free, cols or "-"), flush=True)
print("all 14 chips: %.2f ms" % total_ms, flush=True)
