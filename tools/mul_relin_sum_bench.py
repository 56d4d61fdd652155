"""Time MultiplyRelinearizeSumHybrid against the two ways of computing a sum of ciphertext products without it.

    python tools/mul_relin_sum_bench.py --out DIR [--reps 9]

Shape: N = 2^16, L = 30 data primes of 50 bits, (digit size, special primes) in {(5, 5), (10, 10)} with 50-bit special
primes, levels 30 and 15, k in {1, 2, 4, 8, 16} pairs of distinct ciphertexts, rescale 0 and 1, device buffers,
resident keys.  Alternating rep by rep after a warm-up, each rep timed with CUDA events:
  * fused:    MultiplyRelinearizeSumHybrid;
  * per_pair: k x MultiplyRelinearizeHybrid, the products summed with k - 1 EltwiseAddModMulti;
  * chain:    k x DyadicMultiply, the tensors summed with k - 1 EltwiseAddModMulti, KeySwitchHybrid of the summed d2
              into the summed (d0, d1), and with rescale = 1 DivideAndRoundQLast of both polynomials.
Reported: median and min ms per call, launches per call, and the HBM words per coefficient slot of each path by the
shapes (not measured).  The JSON written to DIR/mul_relin_sum_bench.json (and printed) also holds the card's name and
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
from mul_relin_bench import words_per_slot as single_words  # noqa: E402

N, L = 1 << 16, 30
SHAPES = ((5, 5), (10, 10))
LEVELS = (30, 15)
PAIRS = (1, 2, 4, 8, 16)


def words_per_slot(level, alpha, K, k, rescale):
    """HBM words per coefficient slot, from the shapes, on the accounting of tools/mul_relin_bench.py.  An
    EltwiseAddModMulti reads two words and writes one per limb.  Fused with k > 1: the tensor sum reads 4 l words per
    pair and stores 3 l; the relinearization then reads t in its inverse transform (2 l with the store, against 3 l
    with the multiply on load) and d0, d1 in the multiply-accumulate (2 l, against the 4 l of a0, a1, b0, b1)."""
    one = single_words(level, alpha, K)
    key = "_rescale" if rescale else ""
    out_level = level - int(rescale)
    fused = one["fused" + key] if k == 1 else one["fused" + key] + 4 * level * k + 3 * level - level - 2 * level
    return {"fused": fused,
            "per_pair": k * one["fused" + key] + (k - 1) * 3 * 2 * out_level,
            "chain": one["chain" + key] + (k - 1) * (7 * level + 3 * 3 * level)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=9)
    args = ap.parse_args()
    rng = np.random.default_rng(17)

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
            pool1 = [rows(data[:level] * 2) for _ in range(max(PAIRS))]
            pool2 = [rows(data[:level] * 2) for _ in range(max(PAIRS))]
            acc = torch.empty(3 * comp, dtype=torch.int64, device="cuda")
            d = torch.empty(3 * comp, dtype=torch.int64, device="cuda")
            for k in PAIRS:
                ct1s, ct2s = pool1[:k], pool2[:k]
                for rescale in (False, True):
                    out_level = level - int(rescale)
                    out = torch.empty(2 * out_level * N, dtype=torch.int64, device="cuda")
                    tmp = torch.empty(2 * out_level * N, dtype=torch.int64, device="cuda")

                    def fused():
                        hb.MultiplyRelinearizeSumHybrid(out, ct1s, ct2s, N, level, L, K, alpha, primes, handle,
                                                        rescale)

                    def per_pair():
                        hb.MultiplyRelinearizeHybrid(out, ct1s[0], ct2s[0], N, level, L, K, alpha, primes, handle,
                                                     rescale)
                        for r in range(1, k):
                            hb.MultiplyRelinearizeHybrid(tmp, ct1s[r], ct2s[r], N, level, L, K, alpha, primes, handle,
                                                         rescale)
                            hb.EltwiseAddModMulti(out, out, tmp, N, data[:out_level] * 2)

                    def chain():
                        hb.DyadicMultiply(acc, ct1s[0], ct2s[0], N, data[:level], level)
                        for r in range(1, k):
                            hb.DyadicMultiply(d, ct1s[r], ct2s[r], N, data[:level], level)
                            hb.EltwiseAddModMulti(acc, acc, d, N, data[:level] * 3)
                        hb.KeySwitchHybrid(acc[:2 * comp], acc[2 * comp:], N, level, L, K, alpha, 2, primes, handle)
                        if rescale:
                            hb.DivideAndRoundQLast(acc[:2 * comp], acc[:2 * comp], N, data[:level], level, 2)

                    fns = {"fused": fused, "per_pair": per_pair, "chain": chain}
                    times = alternate(args.reps, **fns)
                    launches = {}
                    for name, fn in fns.items():
                        l0 = hb.launch_count(); fn(); torch.cuda.synchronize(); launches[name] = hb.launch_count() - l0
                    med = {name: statistics.median(v) for name, v in times.items()}
                    work.append({"digit_size": alpha, "special_primes": K, "level": level, "pairs": k,
                                 "rescale": int(rescale), "ms_per_call": times, "median_ms": med,
                                 "min_ms": {name: min(v) for name, v in times.items()},
                                 "fused_over": {"per_pair": med["fused"] / med["per_pair"],
                                                "chain": med["fused"] / med["chain"]},
                                 "launches_per_call": launches,
                                 "words_per_slot_by_shape": words_per_slot(level, alpha, K, k, rescale)})
                    print(json.dumps({key: work[-1][key] for key in ("digit_size", "special_primes", "level", "pairs",
                                                                     "rescale", "median_ms", "fused_over",
                                                                     "launches_per_call")}), flush=True)
                    del out, tmp
            del pool1, pool2, acc, d
        del handle
        torch.cuda.empty_cache()
    res = {"card": card(), "shape": {"n": N, "q_size": L, "moduli_bits": 50, "pairs": list(PAIRS)}, "workloads": work}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "mul_relin_sum_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({"card": res["card"]}))


if __name__ == "__main__":
    main()
