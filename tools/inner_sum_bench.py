"""Time InnerSumHybrid against the chain of existing calls that computes the same slot sum.

    python tools/inner_sum_bench.py --out DIR [--reps 7]

Shape: N = 2^16, L = 30 data primes of 50 bits, (digit size, special primes) in {(5, 5), (10, 10)} with 50-bit special
primes, levels 30 and 15, g = 5, k in {2, 4, 8, 16, 64, 2^15}, rescale 0 and 1, device buffers, resident keys (random
words: only the time is measured).  Alternating rep by rep after a warm-up, each rep timed with CUDA events:
  * fused: InnerSumHybrid, one call;
  * chain: the same log-step recurrence from existing calls, per bit one ApplyGaloisKeySwitchHybridHoisted for the
           bit's keyed elements (the doubling and the shift share the call), then EltwiseAddModMulti for A + Rot(A) and
           R + Rot(A); with rescale = 1, DivideAndRoundQLast of both components at the end;
  * bsgs (k = 16 only): LinearTransformHybridBSGS over babies {1, g, g^2, g^3} and giants {1, g^4, g^8, g^12} with
           4 x 4 unit diagonals.
Reported: median and min ms per call and launches per call.  The JSON written to DIR/inner_sum_bench.json (and printed)
also holds the card's name and power limit, read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import hexl_b200 as hb  # noqa: E402
from galois_bench import alternate, card  # noqa: E402

N, L, G = 1 << 16, 30, 5
SHAPES = ((5, 5), (10, 10))
LEVELS = (30, 15)
COUNTS = (2, 4, 8, 16, 64, 1 << 15)


def bits(g, k):
    """per bit of k: (doubling element or None, shift element or None), as hexl_b200_inner_sum_hybrid walks them"""
    out, power, shift, i = [], g % (2 * N), 1, 0
    while k >> i:
        sh = None
        if (k >> i) & 1:
            sh, shift = shift, shift * power % (2 * N)
        out.append((power if k >> (i + 1) else None, sh))
        power, i = power * power % (2 * N), i + 1
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    gen = torch.Generator(device="cuda").manual_seed(17)

    def rows(moduli):
        return torch.cat([torch.randint(0, q, (N,), dtype=torch.int64, device="cuda", generator=gen) for q in moduli])

    work = []
    for alpha, K in SHAPES:
        primes = [int(q) for q in hb.GeneratePrimes(L + K, 50, True, N)]
        data = primes[:L]
        elts = sorted({e for k in COUNTS for bit in bits(G, k) for e in bit if e not in (None, 1)}
                      | {pow(G, e, 2 * N) for e in (1, 2, 3, 4, 8, 12)})
        handles = {e: hb.KeySwitchKeys([rows(primes * 2) for _ in range(-(-L // alpha))], N, -(-L // alpha), L + K, 2)
                   for e in elts}
        torch.cuda.synchronize()
        key_elts, key_handles = list(handles), list(handles.values())
        for level in LEVELS:
            comp = level * N
            ct = rows(data[:level] * 2)
            a = [torch.empty(2 * comp, dtype=torch.int64, device="cuda") for _ in range(2)]
            r = torch.empty(2 * comp, dtype=torch.int64, device="cuda")
            rot = torch.empty(2 * 2 * comp, dtype=torch.int64, device="cuda")
            ones = torch.ones((level + K) * N, dtype=torch.int64, device="cuda")
            mods2 = data[:level] * 2
            for k in COUNTS:
                for rescale in (False, True):
                    out_level = level - int(rescale)
                    out = torch.empty(2 * out_level * N, dtype=torch.int64, device="cuda")

                    def fused():
                        hb.InnerSumHybrid(out, ct, N, level, L, K, alpha, primes, G, k, key_handles, key_elts, rescale)

                    def chain():
                        cur, nxt, have_r = ct, 0, False
                        for dbl, shift in bits(G, k):
                            keyed = [e for e in (dbl, shift) if e not in (None, 1)]
                            if keyed:
                                hb.ApplyGaloisKeySwitchHybridHoisted(rot, cur, N, level, L, K, alpha, primes,
                                                                     [handles[e] for e in keyed], keyed)
                            rots = {e: rot[i * 2 * comp:(i + 1) * 2 * comp] for i, e in enumerate(keyed)}
                            if shift is not None:
                                term = rots.get(shift, cur)
                                if have_r:
                                    hb.EltwiseAddModMulti(r, r, term, N, mods2)
                                else:
                                    r.copy_(term)
                                have_r = True
                            if dbl is not None:
                                hb.EltwiseAddModMulti(a[nxt], cur, rots.get(dbl, cur), N, mods2)
                                cur, nxt = a[nxt], 1 - nxt
                        if rescale:
                            hb.DivideAndRoundQLast(r, r, N, data[:level], level, 2)

                    fns = {"fused": fused, "chain": chain}
                    if k == 16:
                        babies = [pow(G, e, 2 * N) for e in range(4)]
                        giants = [pow(G, 4 * e, 2 * N) for e in range(4)]
                        grid = [[ones] * 4 for _ in range(4)]

                        def bsgs():
                            hb.LinearTransformHybridBSGS(out, ct, N, level, L, K, alpha, primes,
                                                         [None] + [handles[e] for e in babies[1:]], babies,
                                                         [None] + [handles[e] for e in giants[1:]], giants, grid,
                                                         rescale)
                        fns["bsgs"] = bsgs
                    times = alternate(args.reps, **fns)
                    launches = {}
                    for name, fn in fns.items():
                        l0 = hb.launch_count(); fn(); torch.cuda.synchronize(); launches[name] = hb.launch_count() - l0
                    med = {name: statistics.median(v) for name, v in times.items()}
                    work.append({"digit_size": alpha, "special_primes": K, "level": level, "sum_count": k,
                                 "rescale": int(rescale), "ms_per_call": times, "median_ms": med,
                                 "min_ms": {name: min(v) for name, v in times.items()},
                                 "fused_over": {name: med["fused"] / med[name] for name in med if name != "fused"},
                                 "launches_per_call": launches})
                    print(json.dumps({key: work[-1][key] for key in ("digit_size", "special_primes", "level",
                                                                     "sum_count", "rescale", "median_ms", "fused_over",
                                                                     "launches_per_call")}), flush=True)
                    del out
            del ct, a, r, rot, ones
        del handles, key_handles
        torch.cuda.empty_cache()
    res = {"card": card(), "shape": {"n": N, "q_size": L, "moduli_bits": 50, "galois_elt": G,
                                     "sum_counts": list(COUNTS)}, "workloads": work}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "inner_sum_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({"card": res["card"]}))


if __name__ == "__main__":
    main()
