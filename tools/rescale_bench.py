"""Time DivideAndRoundQLast (NTT form) against the same rescale chained from the library's existing calls.

    python tools/rescale_bench.py --out DIR [--reps 5]

Workloads: 64 ciphertexts (count = 128 polynomials) of 31 limbs at N = 2^16 and at N = 2^15, device buffers.  Both
implementations run on the same buffers in one process, alternated rep by rep, each rep timed with CUDA events.  The
JSON written to DIR/rescale_bench.json (and printed) holds per workload: the time per ciphertext of both, the
kernel launches per call, the algorithmic bytes (2L + 1) * 8 * N per polynomial -- read L + 1 limbs, write L -- and
their share of the H100's 3.35 TB/s, plus the card's name and power limit."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

import hexl_b200 as hb  # noqa: E402
import rescale_exact as rx  # noqa: E402

PEAK_BYTES_PER_S = 3.35e12


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return {"name": name, "power_limit": power}


def time_ms(fn):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    fn()
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop)


def workload(log_n, limbs, ciphertexts, reps):
    n, count = 1 << log_n, 2 * ciphertexts
    mods = hb.GeneratePrimes(1, 59, False, n) + hb.GeneratePrimes(limbs - 2, 39, True, n) + \
        hb.GeneratePrimes(1, 49, True, n)
    ntts = [hb.GetNTT(n, q) for q in mods]
    x = rx.random_operand(log_n, n, mods, count)
    src = torch.from_numpy(x.view(np.int64)).cuda()
    out = torch.empty_like(src)
    out_chain = torch.empty_like(src)

    def fused():
        hb.DivideAndRoundQLast(out, src, n, mods, limbs, count, True)

    def chained():
        rx.rescale_chain(hb, out_chain, src, n, mods, count, True, ntts)

    fused(); chained()  # warm: tables, pool
    torch.cuda.synchronize()
    same = bool(torch.equal(out.view(count, limbs, n)[:, :-1], out_chain.view(count, limbs, n)[:, :-1]))
    l0 = hb.launch_count(); fused(); torch.cuda.synchronize(); launches = hb.launch_count() - l0
    l0 = hb.launch_count(); chained(); torch.cuda.synchronize(); launches_chain = hb.launch_count() - l0
    t_fused, t_chain = [], []
    for _ in range(reps):
        t_fused.append(time_ms(fused))
        t_chain.append(time_ms(chained))
    L = limbs - 1
    alg_bytes = (2 * L + 1) * 8 * n * count
    best = min(t_fused)
    return {
        "n": n, "limbs": limbs, "ciphertexts": ciphertexts, "count": count,
        "ms_per_call": t_fused, "us_per_ciphertext": [1e3 * t / ciphertexts for t in t_fused],
        "chain_ms_per_call": t_chain, "chain_us_per_ciphertext": [1e3 * t / ciphertexts for t in t_chain],
        "launches_per_call": launches, "chain_launches_per_call": launches_chain,
        "algorithmic_bytes": alg_bytes, "best_share_of_3.35TBps": alg_bytes / (best * 1e-3) / PEAK_BYTES_PER_S,
        "chain_equals_fused": same,
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    res = {"card": card(), "workloads": [workload(16, 31, 64, args.reps), workload(15, 31, 64, args.reps)]}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "rescale_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
