"""Time MultiplyRelinearizeHybrid against the chains of existing calls it replaces.

    python tools/mul_relin_bench.py --out DIR [--reps 15]

Shape: N = 2^16, L = 30 data primes of 50 bits, (digit size, special primes) in {(5, 5), (10, 10)} with 50-bit special
primes, levels 30 and 15, one ciphertext pair, device buffers, resident keys.  Alternating rep by rep after a warm-up,
each rep timed with CUDA events:
  * fused_rescale: MultiplyRelinearizeHybrid with rescale = 1;
  * chain_rescale: DyadicMultiply, KeySwitchHybrid of d2 into (d0, d1), DivideAndRoundQLast of both polynomials;
  * fused:         MultiplyRelinearizeHybrid with rescale = 0;
  * chain:         DyadicMultiply, KeySwitchHybrid.
Reported: median and min ms per call, launches per call, and the HBM words per coefficient slot of each path by the
shapes (not measured).  The JSON written to DIR/mul_relin_bench.json (and printed) also holds the card's name and
power limit, read in the same run."""
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

N, L = 1 << 16, 30
SHAPES = ((5, 5), (10, 10))
LEVELS = (30, 15)


def words_per_slot(level, alpha, K):
    """HBM words per coefficient slot, from the shapes (the accounting of tools/hybrid_rotation_bench.py).  D digits,
    B = level + K.  KeySwitchHybrid: the target's inverse transform 2l, the mod-up's conversion and transform l + 3DB,
    keys 2DB, the digits once per component 2DB, the products 2B, the mod-down (special limbs' inverse 4K, conversion
    2K + 2l, transform 4l, finish reading and rewriting the result 8l).  DyadicMultiply 7l.  DivideAndRoundQLast of two
    polynomials 2 (6 (l - 1) + 5).  Fused: the inverse transform reads both operands 3l, the digits are read once for
    both components DB, the tensor reads 4l, and the mod-down from K' = K + rescale limbs into l' = l - rescale moduli
    stores its result: 6K' + 2l' + 4l' + 6l'."""
    D, B = -(-level // alpha), level + K

    def mod_down(k, lv, finish):
        return 4 * k + 2 * k + 2 * lv + 4 * lv + finish * lv

    ks = 2 * level + level + 3 * D * B + 2 * D * B + 2 * D * B + 2 * B + mod_down(K, level, 8)
    fused_common = 3 * level + level + 3 * D * B + 2 * D * B + D * B + 4 * level + 2 * B
    return {"chain": 7 * level + ks,
            "chain_rescale": 7 * level + ks + 2 * (6 * (level - 1) + 5),
            "fused": fused_common + mod_down(K, level, 6),
            "fused_rescale": fused_common + mod_down(K + 1, level - 1, 6)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=15)
    args = ap.parse_args()
    rng = np.random.default_rng(13)

    def rows(moduli):
        return torch.from_numpy(np.concatenate([rng.integers(0, q, N, dtype=np.uint64) for q in moduli])
                                .view(np.int64)).cuda()

    work = []
    for alpha, K in SHAPES:
        primes = [int(q) for q in hb.GeneratePrimes(L + K, 50, True, N)]
        data = primes[:L]
        keys = [rows(primes * 2) for _ in range(-(-L // alpha))]
        handle = hb.KeySwitchKeys(keys, N, len(keys), L + K, 2)
        del keys
        for level in LEVELS:
            comp = level * N
            ct1, ct2 = rows(data[:level] * 2), rows(data[:level] * 2)
            out0 = torch.empty(2 * comp, dtype=torch.int64, device="cuda")
            out1 = torch.empty(2 * (level - 1) * N, dtype=torch.int64, device="cuda")
            d = torch.empty(3 * comp, dtype=torch.int64, device="cuda")

            def fused_rescale():
                hb.MultiplyRelinearizeHybrid(out1, ct1, ct2, N, level, L, K, alpha, primes, handle, True)

            def fused():
                hb.MultiplyRelinearizeHybrid(out0, ct1, ct2, N, level, L, K, alpha, primes, handle, False)

            def chain():
                hb.DyadicMultiply(d, ct1, ct2, N, data[:level], level)
                hb.KeySwitchHybrid(d[:2 * comp], d[2 * comp:], N, level, L, K, alpha, 2, primes, handle)

            def chain_rescale():
                chain()
                hb.DivideAndRoundQLast(d[:2 * comp], d[:2 * comp], N, data[:level], level, 2)

            fns = {"fused_rescale": fused_rescale, "chain_rescale": chain_rescale, "fused": fused, "chain": chain}
            times = alternate(args.reps, **fns)
            launches = {}
            for k, fn in fns.items():
                l0 = hb.launch_count(); fn(); torch.cuda.synchronize(); launches[k] = hb.launch_count() - l0
            med = {k: statistics.median(v) for k, v in times.items()}
            work.append({"digit_size": alpha, "special_primes": K, "level": level, "ms_per_call": times,
                         "median_ms": med, "min_ms": {k: min(v) for k, v in times.items()},
                         "fused_over_chain": {"rescale": med["fused_rescale"] / med["chain_rescale"],
                                              "no_rescale": med["fused"] / med["chain"]},
                         "launches_per_call": launches, "words_per_slot_by_shape": words_per_slot(level, alpha, K)})
            print(json.dumps({k: work[-1][k] for k in ("digit_size", "special_primes", "level", "median_ms",
                                                        "fused_over_chain", "launches_per_call")}), flush=True)
            del ct1, ct2, out0, out1, d
        del handle
        torch.cuda.empty_cache()
    res = {"card": card(), "shape": {"n": N, "q_size": L, "moduli_bits": 50, "pairs": 1}, "workloads": work}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "mul_relin_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({"card": res["card"]}))


if __name__ == "__main__":
    main()
