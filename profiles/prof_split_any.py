"""Split proofs on thread ranks, this tree against another build of the library (the parent commit), alternated:

  python profiles/prof_split_any.py --other /path/to/parent/checkout [--ranks 8] [--log-rows 20] [--reps 3] [--out FILE.json]

Both trees must have their library built (python -m valida_b200.build).  Each measurement runs in a fresh process that imports the
package of one tree, makes N contexts on the visible GPUs (rank r on GPU r % device_count; on a one-GPU box all ranks SHARE it, so
the times are shared-GPU times, not multi-GPU figures), proves Fibonacci once to warm up, and then reports the median proof time
(host wall clock; a proof returns after a synchronise) and, from one proof with per-launch CUDA-event timing, rank 0's quotient-sweep
and exchange kernel times.  Processes alternate between the two trees, `reps` each.  A rank count the other tree refuses (a count
that is not a power of two, before uneven runs) is reported as refused.  The card's name, power limit and SM clock are printed in
the same run."""
import argparse
import json
import os
import statistics
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def smi(q):
    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader,nounits"], capture_output=True, text=True)
    return r.stdout.strip() if r.returncode == 0 else None


def worker(tree, n, log_rows, proofs):
    sys.path.insert(0, tree)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import time

    import torch

    import valida_b200 as vb
    from oracle_binding import Oracle

    assert os.path.dirname(os.path.dirname(os.path.abspath(vb.__file__))) == os.path.abspath(tree)
    orc = Oracle()
    t = vb.run_program(vb.fib_program(((1 << log_rows) - 17) // 7), initial_fp=0x1000)
    ndev = torch.cuda.device_count()
    ctxs = [vb.Context(r % ndev) for r in range(n)]
    try:
        vb.comm_init_local(ctxs)
    except vb.VgpuError as e:
        return {"refused": str(e)}
    cfgs = [vb.StarkConfig(c, orc.rc480) for c in ctxs]
    first = vb.run_ranks(lambda r, c: vb.prove_machine(cfgs[r], t), ctxs)
    times = []
    for _ in range(proofs):
        t0 = time.perf_counter()
        out = vb.run_ranks(lambda r, c: vb.prove_machine(cfgs[r], t), ctxs)
        times.append((time.perf_counter() - t0) * 1e3)
        assert out == first
    for c in ctxs:
        c.set_kernel_timing(True)
        c.kernel_stats()
    vb.run_ranks(lambda r, c: vb.prove_machine(cfgs[r], t), ctxs)
    ks = {name: ms for name, _, ms, _ in ctxs[0].kernel_stats()}
    for c in ctxs:
        c.close()
    return {"proof_ms": statistics.median(times), "quotient_ms": ks.get("quotient_kernel"), "exchange_ms": ks.get("peer-store exchange"),
            "proof_bytes": len(first[0])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--other", required=True, help="root of the other tree (built)")
    ap.add_argument("--ranks", type=int, nargs="+", default=[8])
    ap.add_argument("--log-rows", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--proofs", type=int, default=3)
    ap.add_argument("--out")
    ap.add_argument("--worker", nargs=3, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        print(json.dumps(worker(a.worker[0], int(a.worker[1]), int(a.worker[2]), a.proofs)))
        return
    import torch

    res = {"gpu": smi("name"), "power_limit_w": smi("power.limit"), "sm_clock_mhz": smi("clocks.sm"),
           "devices": torch.cuda.device_count(), "log_rows": a.log_rows, "runs": []}
    trees = {"this": ROOT, "other": os.path.abspath(a.other)}
    for n in a.ranks:
        for rep in range(a.reps):
            for name, tree in trees.items():
                p = subprocess.run([sys.executable, __file__, "--other", a.other, "--proofs", str(a.proofs), "--worker", tree, str(n), str(a.log_rows)],
                                   capture_output=True, text=True)
                r = json.loads(p.stdout.strip().splitlines()[-1]) if p.returncode == 0 else {"error": p.stderr[-2000:]}
                r.update(tree=name, ranks=n, rep=rep, shared_gpu=res["devices"] < n)
                res["runs"].append(r)
                print(json.dumps(r), flush=True)
    summary = {}
    for n in a.ranks:
        for name in trees:
            rs = [r for r in res["runs"] if r["ranks"] == n and r["tree"] == name and "proof_ms" in r]
            if rs:
                summary["%s@%d" % (name, n)] = {k: statistics.median(r[k] for r in rs) for k in ("proof_ms", "quotient_ms", "exchange_ms")}
    res["summary"] = summary
    print(json.dumps({"gpu": res["gpu"], "power_limit_w": res["power_limit_w"], "summary": summary}, indent=1))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
