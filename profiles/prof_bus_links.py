"""Cost of bus_links (every event carrying each item's bus tuple): python profiles/prof_bus_links.py [log_rows] [reps]

On the Fibonacci device witness with 2^log_rows CPU rows (default 22: memory chip 2^24 rows), on one GPU, with 1, 2^10 and 2^16 items
(add rows' general-bus receives spread over the trace, cap 2^20 so every tuple is listed), after a warm-up of each: the host clock
around the synchronising call and the kernels' CUDA-event time per class (kernel_stats()), medians over reps; the peak device memory
the call adds above the witness (memory_stats); and check_buses of the same witness for scale.  Prints the GPU's name and power limit
read in the same run."""
import os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import valida_b200 as vb

args = sys.argv[1:]
log_rows = int(args[0]) if args else 22
reps = int(args[1]) if len(args) > 1 else 10
q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
print("gpu:", q.stdout.strip() or "(nvidia-smi unavailable)", flush=True)
ctx = vb.Context(0)
log = vb.run_program_log(vb.fib_program(((1 << log_rows) - 17) // 7))
dm, dp = log.witness_device(ctx)
print("cpu rows 2^%d, memory rows %d" % (log_rows, dm[2].shape[0]), flush=True)
real = np.nonzero(dm[3].to_tensor()[:, 15].cpu().numpy())[0]
med = lambda v: float(np.median(v))


def measure(name, fn):
    fn()
    ctx.memory_stats(reset=True)
    fn()
    st = ctx.memory_stats()
    wall, kern = [], {}
    for timing in (False, True):
        ctx.set_kernel_timing(timing)
        ctx.kernel_stats()
        for _ in range(reps):
            ctx.synchronize()
            t0 = time.perf_counter()
            fn()
            if timing:
                for cls, _, ms, _ in ctx.kernel_stats():
                    kern.setdefault(cls, []).append(ms)
            else:
                wall.append((time.perf_counter() - t0) * 1e3)
    ctx.set_kernel_timing(False)
    print("%-28s call %8.2f ms   kernels %s   peak extra %.1f MB" % (name, med(wall), {k: round(med(v), 3) for k, v in kern.items()},
                                                                      (st["peak"] - st["live"]) / 1e6), flush=True)


for k in (1, 1 << 10, 1 << 16):
    rows = real[np.linspace(0, len(real) - 1, k).astype(np.int64)]
    items = np.zeros(k, dtype=vb.BUS_EVENT_DTYPE)
    items["chip"], items["interaction"], items["row"] = 3, 4, rows
    res = vb.bus_links(ctx, dm, dp, items, cap=1 << 20)
    assert res.complete and all(x.multiplicity == 1 and x.sends >= 1 for x in res.links)
    measure("bus_links, %d items" % k, lambda: vb.bus_links(ctx, dm, dp, items, cap=1 << 20))
ch = np.random.default_rng(8).integers(0, vb.BABYBEAR_P, 15, dtype=np.uint32)
measure("check_buses", lambda: vb.check_buses(ctx, dm, dp, ch))
