"""Split proofs from traces in the ranks' own device memory, three ways, alternated in one process:

  python profiles/prof_local_shards.py [--log-rows 22] [--ranks 2 4 8] [--reps 3] [--out FILE.json]

For N ranks (threads, one context each, rank r on GPU r % device_count) and the Fibonacci traces (2^22 CPU rows by default):
* import_rows:  every rank holds the WHOLE traces (row-major torch.int32) and imports its run of rows (vgpu_dmat_import_rows);
* import_local: every rank holds only its local_rows(H) rows (row-major) and imports them (vgpu_dmat_import_local);
* borrow_local: every rank holds only its rows as column-major Montgomery tensors and proves from them in place
                (vgpu_dmat_borrow_local).
Per rank and path it reports the caller's tensor bytes, the context's peak live bytes over import + proof (memory_stats), the
CUDA-event time of the imports or borrows on the rank's stream, and the median proof time (host wall clock; a proof returns after
a synchronise).  The card's name, power limit and SM clock are printed in the same run.  When ranks share a GPU the times are
shared-GPU times (the ranks' kernels compete for one device), not multi-GPU figures; the run labels them so."""
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


def monty_cm(a, device):
    """Column-major (stride(0) == 1) Montgomery words of host matrix a, on device."""
    mt = ((np.ascontiguousarray(a.T).astype(np.uint64) << np.uint64(32)) % np.uint64(P)).astype(np.uint32)
    return torch.from_numpy(mt.view(np.int32)).to(device).t()


def row_major(a, device):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.int32)).to(device)


def run_n(n, t, orc, reps, single):
    mats = t.main + t.preprocessed
    ndev = torch.cuda.device_count()
    devs = [r % ndev for r in range(n)]
    streams = [torch.cuda.Stream(device=d) for d in devs]
    ctxs = [vb.Context(d, stream=s.cuda_stream) for d, s in zip(devs, streams)]
    vb.comm_init_local(ctxs)
    cfgs = [vb.StarkConfig(c, orc.rc480) for c in ctxs]
    whole, local_rm, local_cm = [], [], []
    for c in ctxs:
        dev = "cuda:%d" % c.device
        whole.append([row_major(a, dev) for a in mats])
        spans = [c.local_rows(a.shape[0]) for a in mats]
        local_rm.append([row_major(a[r0:r0 + k], dev) for a, (r0, k) in zip(mats, spans)])
        local_cm.append([monty_cm(a[r0:r0 + k], dev) for a, (r0, k) in zip(mats, spans)])
    torch.cuda.synchronize()
    paths = {
        "import_rows": (whole, lambda c, x, a: c.import_tensor_rows(x)),
        "import_local": (local_rm, lambda c, x, a: c.import_tensor_local(x, a.shape[0])),
        "borrow_local": (local_cm, lambda c, x, a: c.borrow_tensor_local(x, a.shape[0])),
    }

    def one(path):
        tens, make = paths[path]

        def rank(r, c):
            s = streams[r]
            c.release_cached()
            c.memory_stats(reset=True)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(s)
            dm = [make(c, x, a) for x, a in zip(tens[r], mats)]
            e1.record(s)
            t0 = time.perf_counter()
            p = vb.prove_machine(cfgs[r], None, device_resident=(dm[:14], dm[14:]))
            ms = (time.perf_counter() - t0) * 1e3
            peak = c.memory_stats()["peak"]
            for m in dm:
                m.free()
            e1.synchronize()
            return p, e0.elapsed_time(e1), ms, peak

        return vb.run_ranks(rank, ctxs)

    res = {}
    for path in paths:                                   # warm-up; every path gives the single-GPU bytes on every rank
        assert all(o[0] == single for o in one(path)), path
    samples = {p: [] for p in paths}
    for _ in range(reps):
        for path in paths:
            samples[path].append(one(path))
    for path, (tens, _) in paths.items():
        res[path] = [{"rank": r, "device": devs[r],
                      "tensor_bytes": sum(x.numel() * 4 for x in tens[r]),
                      "peak_live_bytes": max(s[r][3] for s in samples[path]),
                      "import_event_ms_median": statistics.median(s[r][1] for s in samples[path]),
                      "proof_ms_median": statistics.median(s[r][2] for s in samples[path])} for r in range(n)]
    for c in ctxs:
        c.close()
    del whole, local_rm, local_cm
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--log-rows", type=int, default=22)
    ap.add_argument("--ranks", type=int, nargs="+", default=[2, 4, 8])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    gpu = {"name": torch.cuda.get_device_name(0), "count": torch.cuda.device_count(), "power_limit_w": smi("power.limit"),
           "sm_clock_mhz": smi("clocks.sm"), "sm_clock_max_mhz": smi("clocks.max.sm")}
    print("gpu:", gpu, flush=True)
    orc = Oracle()
    t = vb.run_program(vb.fib_program(((1 << args.log_rows) - 17) // 7), initial_fp=0x1000)
    ctx = vb.Context(0)
    single = vb.prove_machine(vb.StarkConfig(ctx, orc.rc480), t)
    ctx.close()
    out = {"gpu": gpu, "log_rows": args.log_rows, "trace_bytes": sum(a.nbytes for a in t.main + t.preprocessed), "runs": {}}
    for n in args.ranks:
        shared = n > gpu["count"]
        r = run_n(n, t, orc, args.reps, single)
        out["runs"][str(n)] = {"ranks_share_a_gpu": shared, "paths": r}
        label = "SHARED-GPU times (%d ranks on %d GPU%s)" % (n, gpu["count"], "s" if gpu["count"] > 1 else "") if shared else "one rank per GPU"
        print("N = %d, %s" % (n, label), flush=True)
        for path, ranks in r.items():
            for x in ranks:
                print("  %-12s rank %d  tensors %6.3f GB  peak %6.3f GB  import %7.2f ms  proof %8.1f ms" % (
                    path, x["rank"], x["tensor_bytes"] / 1e9, x["peak_live_bytes"] / 1e9, x["import_event_ms_median"], x["proof_ms_median"]), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
