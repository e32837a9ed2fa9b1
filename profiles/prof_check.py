"""Cost of the debug mode (check_constraints on every chip before the commitments): python profiles/prof_check.py [log_rows] [reps]

Proves Fibonacci with 2^log_rows CPU rows (default 22: memory chip 2^24 rows) device-resident, with the debug mode off and on in
alternation after a warm-up of each, and prints the median proof time of each, the check kernels' own time from kernel_stats()
(the check_kernel class), and the GPU's name and power limit read in the same run."""
import os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import valida_b200 as vb

log_rows = int(sys.argv[1]) if len(sys.argv) > 1 else 22
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5
q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
print("gpu:", q.stdout.strip() or "(nvidia-smi unavailable)", flush=True)
ctx = vb.Context(0)
cfg = vb.StarkConfig(ctx, np.random.default_rng(7).integers(0, vb.BABYBEAR_P, 480, dtype=np.uint32))
log = vb.run_program_log(vb.fib_program(((1 << log_rows) - 17) // 7))
dm, dp = log.witness_device(ctx)
print("cpu rows 2^%d, memory rows %d" % (log_rows, dm[2].shape[0]), flush=True)


def prove(debug):
    ctx.set_debug_checks(debug)
    ctx.synchronize()
    t0 = time.perf_counter()
    proof = vb.prove_machine(cfg, None, device_resident=(dm, dp))
    return proof, (time.perf_counter() - t0) * 1e3


ref, _ = prove(False)
assert prove(True)[0] == ref, "the debug mode changed the proof bytes"
times = {False: [], True: []}
for _ in range(reps):
    for debug in (False, True):
        proof, ms = prove(debug)
        assert proof == ref
        times[debug].append(ms)
# the check's own time, in separate proofs: kernel timing adds an event pair per launch, so it stays out of the proof times above
check_ms = []
ctx.set_kernel_timing(True)
for _ in range(reps):
    ctx.kernel_stats()                          # drop earlier records
    prove(True)
    check_ms.append(sum(t for name, _, t, _ in ctx.kernel_stats() if name == "check_kernel"))
ctx.set_kernel_timing(False)
ctx.set_debug_checks(False)
med = lambda v: float(np.median(v))
print("proof, debug mode off: median %.1f ms  %s" % (med(times[False]), ["%.1f" % t for t in times[False]]))
print("proof, debug mode on:  median %.1f ms  %s" % (med(times[True]), ["%.1f" % t for t in times[True]]))
print("check_kernel (14 launches per proof, event-timed): median %.2f ms  %s" % (med(check_ms), ["%.2f" % t for t in check_ms]))
