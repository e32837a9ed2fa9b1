"""One Fibonacci proof at a chosen size, checked by the library's verifier: python profiles/prove_big.py <log_rows>
(BASELINE config 4 is log_rows = 24: CPU 2^24 rows, memory chip 2^26 rows, LDE 2^27 = the field's two-adicity)."""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import valida_b200 as vb

log_rows = int(sys.argv[1]) if len(sys.argv) > 1 else 24
ctx = vb.Context(0)
cfg = vb.StarkConfig(ctx, np.random.default_rng(7).integers(0, vb.BABYBEAR_P, 480, dtype=np.uint32))
n = ((1 << log_rows) - 17) // 7
t0 = time.perf_counter()
t = vb.run_program(vb.fib_program(n), initial_fp=0x1000)
print("tracegen %.1f s, heights" % (time.perf_counter() - t0), [m.shape[0] for m in t.main[:4]], flush=True)
dm = [ctx.upload(m) for m in t.main]; dp = [ctx.upload(m) for m in t.preprocessed]
ctx.synchronize()
for i in range(3):
    ctx.memory_stats(reset=True)
    t0 = time.perf_counter()
    proof = vb.prove_machine(cfg, t, device_resident=(dm, dp))
    dt = time.perf_counter() - t0
    print("prove %d: %.1f ms  %.2f Mrows/s  proof %d bytes" % (i, dt * 1e3, (1 << log_rows) / dt / 1e6, len(proof)), flush=True)
    print("  phases:", ["%s %.1f" % p for p in vb.last_prove_phases(ctx)], flush=True)
    ms = ctx.memory_stats()
    print("  memory (GB): live %.2f  peak live %.2f  cached %.2f  symmetric-heap peak %.2f"
          % tuple(ms[k] / 1e9 for k in ("live", "peak", "cached", "symm_peak")), flush=True)
t0 = time.perf_counter()
vb.verify_machine(cfg, proof, t.preprocessed)
print("verified in %.1f ms" % ((time.perf_counter() - t0) * 1e3))
