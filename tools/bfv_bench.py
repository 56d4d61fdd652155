"""Time BfvMultiply and BfvMultiplyRelinearizeHybrid with device-resident data.

    python tools/bfv_bench.py --out DIR [--reps 20]

Shapes: n = 2^13, 2^14 and 2^15 with moduli of the bit sizes of SEAL's default BFV moduli at the top level (the last
one the special prime, digit size 1), t = 65537 and the 20-bit batching prime 786433, and one hybrid shape (n = 2^15,
digit size 5, 3 special primes).  B and m_sk follow SEAL's rule (61-bit primes, |B| = l or l + 1).  One ciphertext pair
per call, alternating rep by rep after a warm-up, each rep timed with CUDA events:
  * bfv:        BfvMultiply (three components);
  * bfv_relin:  BfvMultiplyRelinearizeHybrid;
  * ckks_relin: MultiplyRelinearizeHybrid (NTT form, rescale = 0) at the same (n, l, digit size, K): what BEHZ adds.
Then, in a run of its own, torch.profiler's kernel time of one bfv_relin call split by kernel name: extension,
transforms, tensor, scaling and relinearization (everything else).  The JSON written to DIR/bfv_bench.json (and printed)
also holds the card's name and power limit, read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

import hexl_b200 as hb  # noqa: E402
from galois_bench import alternate, card  # noqa: E402

SEAL_BITS = {8192: [43, 43, 44, 44, 44], 16384: [48, 48, 48, 49, 49, 49, 49, 49, 49], 32768: [55] * 13 + [56] * 3}
SHAPES = [(8192, 1, 1), (16384, 1, 1), (32768, 1, 1), (32768, 5, 3)]  # (n, digit size, special primes)
PLAIN = (65537, 786433)


def moduli(n, K):
    bits = SEAL_BITS[n]
    data = []
    for b in sorted(set(bits[:-1])):
        data += [int(q) for q in hb.GeneratePrimes(bits[:-1].count(b), b - 1, False, n)]  # [2^(b-1), 2^b)
    special = [int(q) for q in hb.GeneratePrimes(K + len(data), bits[-1] - 1, True, n) if int(q) not in data][:K]
    return data, special


def seal_bases(n, Q, t):
    bits = 1
    for q in Q:
        bits *= q
    k = len(Q) + (1 if 32 + t.bit_length() + bits.bit_length() >= 61 * (len(Q) + 1) else 0)
    primes = [int(p) for p in hb.GeneratePrimes(k + 1 + len(Q), 60, True, n) if int(p) not in Q][:k + 1]
    return primes[:k], primes[k]


def category(name):
    for key, cat in (("bfv_extend", "extension"), ("bfv_scale", "scaling"), ("dyadic", "tensor"), ("ntt", "transforms")):
        if key in name:
            return cat
    return "relinearization"


def kernel_split(fn):
    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    split = {}
    for evt in prof.key_averages():
        us = getattr(evt, "device_time_total", None)
        if us is None:
            us = evt.cuda_time_total
        if us:
            cat = category(evt.key)
            split[cat] = split.get(cat, 0.0) + us / 1000.0
    return {k: round(v, 4) for k, v in sorted(split.items())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    rows = []
    for n, alpha, K in SHAPES:
        data, special = moduli(n, K)
        L = len(data)
        mods = data + special
        rng = np.random.default_rng(n + alpha)
        keys = [rng.integers(0, 1 << 62, size=2 * (L + K) * n, dtype=np.uint64) % np.repeat(
            np.array(mods * 2, dtype=np.uint64), n) for _ in range(-(-L // alpha))]
        handle = hb.KeySwitchKeys(keys, n, len(keys), L + K, 2)
        cts = [torch.from_numpy((rng.integers(0, 1 << 62, size=2 * L * n, dtype=np.uint64) % np.repeat(
            np.array(data * 2, dtype=np.uint64), n)).view(np.int64)).cuda() for _ in range(2)]
        d = torch.empty(3 * L * n, dtype=torch.int64, device="cuda")
        r = torch.empty(2 * L * n, dtype=torch.int64, device="cuda")
        for t in PLAIN if alpha == 1 else PLAIN[:1]:
            B, m_sk = seal_bases(n, data, t)
            fns = {
                "bfv": lambda: hb.BfvMultiply(d, cts[0], cts[1], n, data, L, B, m_sk, t),
                "bfv_relin": lambda: hb.BfvMultiplyRelinearizeHybrid(r, cts[0], cts[1], n, L, L, K, alpha, mods, B,
                                                                     m_sk, t, handle),
                "ckks_relin": lambda: hb.MultiplyRelinearizeHybrid(r, cts[0], cts[1], n, L, L, K, alpha, mods, handle),
            }
            times = alternate(args.reps, **fns)
            row = {"n": n, "l": L, "k": len(B), "digit_size": alpha, "K": K, "t": t}
            for name, ts in times.items():
                row[name + "_ms_median"] = round(statistics.median(ts), 4)
                row[name + "_ms_min"] = round(min(ts), 4)
            row["bfv_relin_kernel_ms"] = kernel_split(fns["bfv_relin"])
            rows.append(row)
            print(json.dumps(row), flush=True)
    out = {"card": card(), "reps": args.reps, "rows": rows}
    with open(os.path.join(args.out, "bfv_bench.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out["card"]))


if __name__ == "__main__":
    main()
