"""Cost of check_failures (every failing row and constraint of a chip): python profiles/prof_check_failures.py [log_rows] [reps]

On the Fibonacci device witness with 2^log_rows CPU rows (default 22: memory chip 2^24 rows), with every chip's honest permutation
trace built beforehand, times on one GPU, after a warm-up of each:
  clean    check_failures of the 14 chips (the clean witness), against check_constraints of the same 14 chips;
  ten      the memory chip with ten words of its permutation trace changed (ten rows reached), against check_constraints;
  all      the CPU chip checked with other challenges than its permutation trace was built with (every row fails), cap 2^16.
Each as the host clock around the synchronising calls and as the kernels' CUDA-event time (kernel_stats(), KC_CHECK class), medians
over reps.  Prints the GPU's name and power limit read in the same run."""
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
prep = {1: dp[0], 12: dp[1]}
perm = [vb.generate_permutation_trace(ctx, c, dm[c], prep.get(c), ch)[0] for c in range(14)]
med = lambda v: float(np.median(v))


def timed(fn):
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
                kern.append(sum(ms for name, _, ms, _ in ctx.kernel_stats() if name == "check_kernel"))
            else:
                wall.append((time.perf_counter() - t0) * 1e3)
    ctx.set_kernel_timing(False)
    return med(wall), med(kern)


def report(name, fn):
    wall, kern = timed(fn)
    print("%-52s call %8.2f ms   kernels %8.2f ms" % (name, wall, kern), flush=True)


def failures(chips, cap, challenges=ch, perms=perm):
    out = []
    for c in chips:
        arr, total, _ = vb.check_failures(ctx, c, dm[c], prep.get(c), perms[c], challenges, cap=cap)
        out.append((len(arr), total))
    return out


assert failures(range(14), 1 << 16) == [(0, 0)] * 14, "the Fibonacci witness fails its check"
report("clean, 14 chips: check_failures (cap 2^16)", lambda: failures(range(14), 1 << 16))
report("clean, 14 chips: check_constraints", lambda: [vb.check_constraints(ctx, c, dm[c], prep.get(c), perm[c], ch) for c in range(14)])

h = dm[2].shape[0]
t = perm[2].to_tensor()
for r, col in [(0, 3), (1, 0), (h // 3, 7), (h // 2, 5), (h // 2 + 1, 9), ((h >> 4) + 17, 2), (h - 5, 4), (h - 3, 8), (h - 1, 1), (h // 5, 6)]:
    t[r, col] = (t[r, col].to(torch.int64) + 1) % P
torch.cuda.synchronize()
bad = list(perm)
bad[2] = ctx.import_tensor(t)
del t
print("ten words: (listed, total) =", failures([2], 1 << 16, perms=bad), flush=True)
report("ten words changed, memory chip: check_failures", lambda: failures([2], 1 << 16, perms=bad))
report("ten words changed, memory chip: check_constraints", lambda: vb.check_constraints(ctx, 2, dm[2], None, bad[2], ch))
del bad

other = np.random.default_rng(9).integers(0, P, 15, dtype=np.uint32)
print("every row of the cpu chip: (listed, total) =", failures([0], 1 << 16, challenges=other), flush=True)
report("every cpu row fails: check_failures (cap 2^16)", lambda: failures([0], 1 << 16, challenges=other))
report("every cpu row fails: check_constraints", lambda: vb.check_constraints(ctx, 0, dm[0], None, perm[0], other))
