"""Time the BGV calls against their CKKS counterparts, and the merged modulus switch against the chain, with
device-resident data.

    python tools/bgv_bench.py --out DIR [--reps 15]

Shapes: n = 2^15 and 2^16, L = 30 data moduli of 50 bits, (digit size, K) in {(1, 1), (5, 5), (10, 10)} with 55-bit
special primes, levels 30 and 15, plain modulus 65537.  One ciphertext (pair) per call; every comparison alternates
its calls rep by rep after a warm-up, each rep timed with CUDA events:
  * multiply:  BgvMultiplyRelinearizeHybrid vs MultiplyRelinearizeHybrid (no modulus switch / rescale);
  * switch:    BgvKeySwitchHybrid vs KeySwitchHybrid (key component count 2);
  * hoisted:   BgvApplyGaloisKeySwitchHybridHoisted vs ApplyGaloisKeySwitchHybridHoisted (one element);
  * modswitch: BgvModSwitch vs DivideAndRoundQLast (NTT form, two polynomials);
  * merged:    BgvMultiplyRelinearizeHybrid with mod_switch = 1 vs DyadicMultiply + BgvKeySwitchHybrid + BgvModSwitch.
Per comparison the JSON holds each call's median and the median, min and max of the rep-by-rep ratio (first / second):
the spread of the ratio is the noise of the comparison.  DIR/bgv_bench.json also holds the card's name and power
limit, read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

import hexl_b200 as hb  # noqa: E402
from galois_bench import alternate, card  # noqa: E402

L, TAU = 30, 65537
SHAPES = [(1, 1), (5, 5), (10, 10)]


def uniform(mods, comps, n, gen):
    """comps x len(mods) limbs of n canonical words, on the GPU"""
    m = torch.tensor(mods, dtype=torch.int64, device="cuda").repeat(comps).repeat_interleave(n)
    return torch.randint(0, 1 << 62, (comps * len(mods) * n,), dtype=torch.int64, device="cuda", generator=gen) % m


def compare(reps, first, second):
    times = alternate(reps, a=first, b=second)
    ratios = [x / y for x, y in zip(times["a"], times["b"])]
    return {"first_ms": round(statistics.median(times["a"]), 4), "second_ms": round(statistics.median(times["b"]), 4),
            "ratio_median": round(statistics.median(ratios), 4), "ratio_min": round(min(ratios), 4),
            "ratio_max": round(max(ratios), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=15)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(2026)
    rows = []
    for n in (1 << 15, 1 << 16):
        data = [int(q) for q in hb.GeneratePrimes(L, 49, True, n)]
        for alpha, K in SHAPES:
            special = [int(q) for q in hb.GeneratePrimes(K, 54, True, n)]
            mods = data + special
            keys = [uniform(mods, 2, n, gen) for _ in range(-(-L // alpha))]
            handle = hb.KeySwitchKeys(keys, n, len(keys), L + K, 2)
            del keys
            for level in (30, 15):
                comp = level * n
                ct1, ct2 = uniform(data[:level], 2, n, gen), uniform(data[:level], 2, n, gen)
                out = torch.zeros(2 * comp, dtype=torch.int64, device="cuda")
                rot = torch.empty(2 * comp, dtype=torch.int64, device="cuda")
                d = torch.empty(3 * comp, dtype=torch.int64, device="cuda")
                ms = torch.empty(2 * comp, dtype=torch.int64, device="cuda")
                lm = data[:level]

                def chain():
                    hb.DyadicMultiply(d, ct1, ct2, n, lm, level)
                    hb.BgvKeySwitchHybrid(d[:2 * comp], d[2 * comp:], n, level, L, K, alpha, 2, mods, TAU, handle)
                    hb.BgvModSwitch(d[:2 * comp], d[:2 * comp], n, lm, level, TAU, 2, True)

                row = {"n": n, "level": level, "digit_size": alpha, "K": K}
                row["multiply"] = compare(
                    args.reps,
                    lambda: hb.BgvMultiplyRelinearizeHybrid(out, ct1, ct2, n, level, L, K, alpha, mods, TAU, handle),
                    lambda: hb.MultiplyRelinearizeHybrid(out, ct1, ct2, n, level, L, K, alpha, mods, handle))
                row["switch"] = compare(
                    args.reps,
                    lambda: hb.BgvKeySwitchHybrid(out, ct2[:comp], n, level, L, K, alpha, 2, mods, TAU, handle),
                    lambda: hb.KeySwitchHybrid(out, ct2[:comp], n, level, L, K, alpha, 2, mods, handle))
                row["hoisted"] = compare(
                    args.reps,
                    lambda: hb.BgvApplyGaloisKeySwitchHybridHoisted(rot, ct1, n, level, L, K, alpha, mods, TAU,
                                                                    [handle], [5]),
                    lambda: hb.ApplyGaloisKeySwitchHybridHoisted(rot, ct1, n, level, L, K, alpha, mods, [handle],
                                                                 [5]))
                row["modswitch"] = compare(
                    args.reps,
                    lambda: hb.BgvModSwitch(ms, ct1, n, lm, level, TAU, 2, True),
                    lambda: hb.DivideAndRoundQLast(ms, ct1, n, lm, level, 2, True))
                row["merged"] = compare(
                    args.reps,
                    lambda: hb.BgvMultiplyRelinearizeHybrid(out[:2 * (level - 1) * n], ct1, ct2, n, level, L, K,
                                                            alpha, mods, TAU, handle, True),
                    chain)
                rows.append(row)
                print(json.dumps(row), flush=True)
            del handle
            torch.cuda.empty_cache()
    out = {"card": card(), "reps": args.reps, "rows": rows}
    with open(os.path.join(args.out, "bgv_bench.json"), "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out["card"]))


if __name__ == "__main__":
    main()
