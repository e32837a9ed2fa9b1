"""Cost of check_buses (every unbalanced bus tuple of a witness): python profiles/prof_check_buses.py [log_rows] [reps]

On the Fibonacci device witness with 2^log_rows CPU rows (default 22: memory chip 2^24 rows), times on one GPU, after a warm-up of
each, beside check_witness (LogUp traces + check of the 14 chips) in the same process:
  clean     check_buses of the clean witness;
  tampered  the same with one memory-chip value byte changed (two unbalanced tuples).
Each as the host clock around the synchronising call and as the kernels' CUDA-event time (kernel_stats(), class "check_kernel", which
holds the bus kernels), medians over reps.  Prints the GPU's name and power limit read in the same run."""
import os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
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
print("cpu rows 2^%d, memory rows %d" % (log_rows, dm[2].shape[0]), flush=True)
ch = np.random.default_rng(8).integers(0, P, 15, dtype=np.uint32)
med = lambda v: float(np.median(v))


def timed(fn, kernel_names):
    """(host ms, event-timed kernel ms) of fn(), medians over reps after one warm-up."""
    fn()
    wall, kern = [], []
    for timing in (False, True):
        ctx.set_kernel_timing(timing)
        ctx.kernel_stats()
        for _ in range(reps):
            ctx.synchronize()
            t0 = time.perf_counter()
            fn()
            if timing:
                kern.append(sum(ms for name, _, ms, _ in ctx.kernel_stats() if name in kernel_names))
            else:
                wall.append((time.perf_counter() - t0) * 1e3)
    ctx.set_kernel_timing(False)
    return med(wall), med(kern)


def report(name, fn, kernel_names=("check_kernel",)):
    wall, kern = timed(fn, kernel_names)
    print("%-50s call %8.2f ms   kernels %8.2f ms" % (name, wall, kern), flush=True)


res = vb.check_buses(ctx, dm, dp, ch)
assert res.tuples == [] and res.complete, "the Fibonacci witness is unbalanced"
ctx.memory_stats(reset=True)
vb.check_buses(ctx, dm, dp, ch)
print("check_buses peak live device memory above the witness: %.1f MB" % ((ctx.memory_stats()["peak"] - ctx.memory_stats()["live"]) / 1e6), flush=True)
report("clean: check_buses", lambda: vb.check_buses(ctx, dm, dp, ch))
report("clean: check_witness (check kernels only)", lambda: vb.check_witness(ctx, dm, dp, ch))
report("clean: check_witness (LogUp + check kernels)", lambda: vb.check_witness(ctx, dm, dp, ch), ("check_kernel", "perm trace kernels"))

h = dm[2].shape[0]
mem = dm[2].to_tensor()
near = mem[h // 2:h // 2 + 4096].cpu().numpy()
r = h // 2 + next(k for k in range(len(near)) if int(near[k, 7]) + int(near[k, 8]) == 1 and not near[k, 6])
mem[r, 1] = (mem[r, 1].to(torch.int64) + 1) % P
torch.cuda.synchronize()
bad = dm[:2] + [ctx.import_tensor(mem)] + dm[3:]
del mem
res = vb.check_buses(ctx, bad, dp, ch)
print("tampered row %d: %s" % (r, [(t.bus_name, t.fields, t.net, [(e.chip_name, e.row) for e in t.events]) for t in res.tuples]), flush=True)
report("one memory byte changed: check_buses", lambda: vb.check_buses(ctx, bad, dp, ch))
report("one memory byte changed: check_witness (check kernels)", lambda: vb.check_witness(ctx, bad, dp, ch))
