"""Traces from caller device memory against host uploads, on one GPU, in one process:

  python profiles/prof_device_import.py [--log-rows 22] [--reps 5] [--out FILE.json]

* the card's name and power limit;
* the 14 + 2 Fibonacci traces (2^22 CPU rows by default, BASELINE config 3) as row-major torch.int32 tensors: CUDA-event time of
  importing all of them (vgpu_dmat_import, which synchronises once per matrix to read its verdict) and the import kernels' own time
  (per-kernel event timing);
* the same traces as column-major Montgomery tensors: event time of borrowing them (one validation pass, no copy);
* the same traces from page-locked host memory: event time of vgpu_dmat_upload (H2D copy + transpose);
* end-to-end proofs, alternated --reps times each: import from the tensors + vgpu_prove_device, borrow + vgpu_prove_device, and
  vgpu_prove from the page-locked host traces (bench.py's e2e path); host wall clock around calls that return after a synchronise.
The context and torch share one side stream (torch's default stream is the legacy stream, which a context cannot enqueue on), so
torch's CUDA events time the context's work directly."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import valida_b200 as vb  # noqa: E402
from oracle_binding import Oracle  # noqa: E402

P = 2013265921


def smi(q):
    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader,nounits"], capture_output=True, text=True)
    return r.stdout.strip() if r.returncode == 0 else None


def event_ms(fn, ctx):
    """(event ms of fn on the context's stream, ms of its import / export kernels)."""
    ctx.kernel_stats()
    ctx.set_kernel_timing(True)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    ctx.set_kernel_timing(False)
    io = sum(ms for name, _, ms, _ in ctx.kernel_stats() if name.startswith("import_kernel"))
    return a.elapsed_time(b), io, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-rows", type=int, default=22)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    gpu = {"name": torch.cuda.get_device_name(0), "power_limit_w": smi("power.limit"), "sm_clock_max_mhz": smi("clocks.max.sm")}
    print("gpu:", gpu, flush=True)

    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        run(args, gpu, stream)


def run(args, gpu, stream):
    orc = Oracle()
    ctx = vb.Context(0, stream=stream.cuda_stream)
    cfg = vb.StarkConfig(ctx, orc.rc480)
    t = vb.run_program(vb.fib_program(((1 << args.log_rows) - 17) // 7), initial_fp=0x1000)
    mats = t.main + t.preprocessed
    nbytes = sum(m.nbytes for m in mats)
    rm = [torch.from_numpy(np.ascontiguousarray(m).view(np.int32)).cuda() for m in mats]
    cm = []
    for m in mats:
        mt = ((np.ascontiguousarray(m.T).astype(np.uint64) << np.uint64(32)) % np.uint64(P)).astype(np.uint32)
        cm.append(torch.from_numpy(mt.view(np.int32)).cuda().t())
    for m in mats:
        ctx.host_register(m)
    torch.cuda.synchronize()
    res = {"gpu": gpu, "log_rows": args.log_rows, "trace_bytes": nbytes, "matrices": len(mats)}

    def free(ms):
        for m in ms:
            m.free()

    # warm-up of every path, then one timed pass each
    free([ctx.import_tensor(x) for x in rm]); free([ctx.borrow_tensor(x) for x in cm]); free([ctx.upload(m) for m in mats])
    ms, io, out = event_ms(lambda: [ctx.import_tensor(x) for x in rm], ctx)
    free(out)
    res["import"] = {"event_ms": ms, "kernel_ms": io, "kernel_GBps_in_plus_out": 2 * nbytes / io / 1e6}
    ms, io, out = event_ms(lambda: [ctx.borrow_tensor(x) for x in cm], ctx)
    free(out)
    res["borrow_validation"] = {"event_ms": ms, "kernel_ms": io, "kernel_GBps_read": nbytes / io / 1e6}
    ms, _, out = event_ms(lambda: [ctx.upload(m) for m in mats], ctx)
    free(out)
    res["upload_pinned"] = {"event_ms": ms, "GBps": nbytes / ms / 1e6}
    print(json.dumps(res, indent=1), flush=True)

    ref = vb.prove_machine(cfg, t)

    def from_import():
        dm = [ctx.import_tensor(x) for x in rm]
        p = vb.prove_machine(cfg, None, device_resident=(dm[:14], dm[14:]))
        free(dm)
        return p

    def from_borrow():
        dm = [ctx.borrow_tensor(x) for x in cm]
        p = vb.prove_machine(cfg, None, device_resident=(dm[:14], dm[14:]))
        free(dm)
        return p

    paths = {"import_tensors+prove_device": from_import, "borrow_tensors+prove_device": from_borrow,
             "prove_pinned_host": lambda: vb.prove_machine(cfg, t)}
    times = {k: [] for k in paths}
    for k, fn in paths.items():
        assert fn() == ref, k                         # warm-up, and the bytes of every path agree
    for _ in range(args.reps):
        for k, fn in paths.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            times[k].append((time.perf_counter() - t0) * 1e3)
    res["proof_ms"] = {k: {"median": statistics.median(v), "min": min(v), "max": max(v), "all": v} for k, v in times.items()}
    for k, v in res["proof_ms"].items():
        print("%-32s median %.1f ms  (min %.1f, max %.1f)" % (k, v["median"], v["min"], v["max"]), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    for m in mats:
        ctx.host_unregister(m)
    ctx.close()


if __name__ == "__main__":
    main()
