"""Cost of the debug mode (check_constraints on every chip before the commitments): python profiles/prof_check.py [log_rows] [reps]

Proves Fibonacci with 2^log_rows CPU rows (default 22: memory chip 2^24 rows) device-resident, with the debug mode off and on in
alternation after a warm-up of each, and prints the median proof time of each, the check kernels' own time from kernel_stats()
(the check_kernel class), and the GPU's name and power limit read in the same run.

--witness: times check_witness (the witness check without a proof) of the same device witness on one GPU instead: the call (it ends
in a synchronisation) by the host clock, and its kernels by CUDA events (kernel_stats(), per class)."""
import os, subprocess, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import valida_b200 as vb

witness = "--witness" in sys.argv[1:]
args = [a for a in sys.argv[1:] if a != "--witness"]
log_rows = int(args[0]) if args else 22
reps = int(args[1]) if len(args) > 1 else 5
q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
print("gpu:", q.stdout.strip() or "(nvidia-smi unavailable)", flush=True)
ctx = vb.Context(0)
cfg = vb.StarkConfig(ctx, np.random.default_rng(7).integers(0, vb.BABYBEAR_P, 480, dtype=np.uint32))
log = vb.run_program_log(vb.fib_program(((1 << log_rows) - 17) // 7))
dm, dp = log.witness_device(ctx)
print("cpu rows 2^%d, memory rows %d" % (log_rows, dm[2].shape[0]), flush=True)

med = lambda v: float(np.median(v))

if witness:
    ch = np.random.default_rng(8).integers(0, vb.BABYBEAR_P, 15, dtype=np.uint32)
    reports, cancel = vb.check_witness(ctx, dm, dp, ch)         # warm-up
    assert cancel and all(r[0] == -1 for r in reports), "the Fibonacci witness fails its check"
    wall = []
    for _ in range(reps):
        ctx.synchronize()
        t0 = time.perf_counter()
        vb.check_witness(ctx, dm, dp, ch)
        wall.append((time.perf_counter() - t0) * 1e3)
    ctx.set_kernel_timing(True)
    ctx.kernel_stats()
    per_class = {}
    for _ in range(reps):
        vb.check_witness(ctx, dm, dp, ch)
        for name, n, ms, _ in ctx.kernel_stats():
            per_class.setdefault(name, []).append(ms)
    ctx.set_kernel_timing(False)
    print("check_witness: median %.2f ms per call (host clock around the synchronising call)  %s" % (med(wall), ["%.2f" % t for t in wall]))
    for name, v in sorted(per_class.items(), key=lambda kv: -med(kv[1])):
        print("  %-28s median %.2f ms per call (event-timed)" % (name, med(v)))
    sys.exit(0)


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
print("proof, debug mode off: median %.1f ms  %s" % (med(times[False]), ["%.1f" % t for t in times[False]]))
print("proof, debug mode on:  median %.1f ms  %s" % (med(times[True]), ["%.1f" % t for t in times[True]]))
print("check_kernel (14 launches per proof, event-timed): median %.2f ms  %s" % (med(check_ms), ["%.2f" % t for t in check_ms]))
