"""Keccak-256 against Poseidon-16 Merkle trees (vgpu_ctx_set_merkle_hash) on one GPU, in one process:

  python profiles/prof_merkle_hash.py [--proofs 10] [--log-rows 22]

* the card's name and power limit;
* after a warm-up, device-resident Fibonacci proofs (2^22 CPU rows by default, BASELINE config 3) alternating between the two
  hashes, --proofs of each: median and spread of the step time;
* one more proof per hash with per-kernel event timing: the leaf, compression / tail, FRI-leaf and path classes;
* Poseidon permutations per second in a tree of 2^21 one-permutation leaves (a 2^20 x 8 matrix, LDE 2^21 rows; 2^22 - 1
  permutations), against the issue-rate floor: SASS instructions of one permutation (the round loop of p16_layer_kernel, partial
  and full rounds counted apart) x permutations / (SMs x 4 schedulers x 32 lanes x clock)."""
import argparse
import os
import re
import shutil
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

HASHES = {vb.MERKLE_KECCAK256: "keccak256", vb.MERKLE_POSEIDON16: "poseidon16"}


def smi(q):
    r = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader,nounits"], capture_output=True, text=True)
    return r.stdout.strip() if r.returncode == 0 else None


def permutation_instructions():
    """(instructions of one permutation, how they were counted) from the SASS of p16_layer_kernel's first round loop (the first
    backward branch over more than 100 instructions): the block a forward branch inside it skips is the S-box layer of lanes 1..15,
    run in the 8 full rounds only."""
    cuobjdump = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    sass = subprocess.run([cuobjdump, "-sass", vb.lib_path], capture_output=True, text=True).stdout
    fn = re.search(r"Function : (\S*p16_layer_kernel\S*)\n(.*?)(?=\n\s+Function : |\Z)", sass, flags=re.S)
    ins = [(int(m.group(1), 16), m.group(2)) for m in re.finditer(r"/\*([0-9a-f]{4,})\*/\s+([^;]*);", fn.group(2))]
    at = {a: k for k, (a, _) in enumerate(ins)}
    loops = []
    for k, (a, text) in enumerate(ins):
        m = re.search(r"BRA\s+(?:`\(\.L_x_\d+\)\s*)?\(?0x([0-9a-f]+)", text)
        if m and int(m.group(1), 16) < a and int(m.group(1), 16) in at:
            loops.append((at[int(m.group(1), 16)], k))
    if not loops:
        return None, "no round loop found"
    loops = [l for l in loops if l[1] - l[0] > 100]
    if not loops:
        return None, "no round loop found"
    lo, hi = loops[0]
    body = hi - lo + 1
    blocks = []
    for k in range(lo, hi):
        m = re.search(r"@!?U?P\w*\s+BRA\s+(?:`\(\.L_x_\d+\)\s*)?\(?0x([0-9a-f]+)", ins[k][1])
        if m and int(m.group(1), 16) in at and lo < at[int(m.group(1), 16)] <= hi:
            blocks.append(at[int(m.group(1), 16)] - k - 1)
    if len(blocks) == 1:
        full = blocks[0]
        return 30 * (body - full) + 8 * full, "round loop %d instructions, of which %d run in the full rounds only" % (body, full)
    return 30 * body, "round loop %d instructions x 30 rounds (blocks not separated: an upper bound)" % body


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--proofs", type=int, default=10)
    ap.add_argument("--log-rows", type=int, default=22)
    a = ap.parse_args()
    print("gpu:", smi("name,power.limit") or "(nvidia-smi unavailable)", flush=True)
    props = torch.cuda.get_device_properties(0)
    orc = Oracle()
    t = vb.run_program(vb.fib_program(((1 << a.log_rows) - 17) // 7), initial_fp=0x1000)
    ctx = vb.Context(0)
    cfg = vb.StarkConfig(ctx, orc.rc480)
    dm = [ctx.upload(m) for m in t.main]
    dp = [ctx.upload(m) for m in t.preprocessed]

    def prove(h):
        ctx.set_merkle_hash(h)
        t0 = time.perf_counter()
        p = vb.prove_machine(cfg, t, device_resident=(dm, dp))
        return time.perf_counter() - t0, p

    for _ in range(2):
        for h in HASHES:
            prove(h)
    times = {h: [] for h in HASHES}
    proofs = {}
    for _ in range(a.proofs):
        for h in HASHES:
            dt, proofs[h] = prove(h)
            times[h].append(dt * 1e3)
    for h, name in HASHES.items():
        v = sorted(times[h])
        print("%-10s step %8.2f ms median, %.2f .. %.2f ms over %d proofs, %d proof bytes" % (name, statistics.median(v), v[0], v[-1], len(v), len(proofs[h])))
    ctx.set_merkle_hash(vb.MERKLE_POSEIDON16)
    vb.verify_machine(cfg, proofs[vb.MERKLE_POSEIDON16], t.preprocessed)

    classes = ("leaf_hash_kernel", "compress_layer_kernel", "fri_leaf_hash_kernel", "query_path_kernel",
               "p16_leaf_kernel", "p16_layer_kernel + p16_tail_kernel", "p16_fri_leaf_kernel", "p16_path_kernel")
    ctx.set_kernel_timing(True)
    for h, name in HASHES.items():
        ctx.kernel_stats()
        prove(h)
        for cls, n, ms, _ in ctx.kernel_stats():
            if cls in classes:
                print("%-10s %-36s %5d launches %9.3f ms" % (name, cls, n, ms))

    # permutation rate: one tree of 2^21 leaves of 8 words (one permutation each) and 2^21 - 1 compressions
    m = ctx.upload(np.random.default_rng(9).integers(0, vb.BABYBEAR_P, (1 << 20, 8), dtype=np.uint32))
    pcs = cfg.pcs()
    ctx.set_merkle_hash(vb.MERKLE_POSEIDON16)
    for _ in range(2):
        ctx.kernel_stats()
        _, pd = pcs.commit_batches([m])
        pd.free()
        ms = sum(v for c, _, v, _ in ctx.kernel_stats() if c.startswith("p16_"))
    perms = (1 << 22) - 1
    rate = perms / (ms * 1e-3)
    clock = smi("clocks.max.sm")
    n_ins, how = permutation_instructions()
    print("poseidon16 permutations: %d in %.3f ms of p16 kernels = %.3g /s" % (perms, ms, rate))
    if n_ins and clock:
        floor = props.multi_processor_count * 4 * 32 * float(clock) * 1e6 / n_ins
        print("issue-rate floor: %d instructions per permutation (%s); %d SMs x 128 lanes x %s MHz (max SM clock) = %.3g /s; "
              "measured %.0f %% of it" % (n_ins, how, props.multi_processor_count, clock, floor, 100 * rate / floor))
    ctx.close()


if __name__ == "__main__":
    main()
