"""Time KeySwitchHybrid against KeySwitchResident.

    python tools/hybrid_bench.py --out DIR [--reps 15]

Shape: N = 2^15 and 2^16, level = L = 30 data primes of 50 bits, key_component_count 2, resident keys, one ciphertext,
device buffers.  For (alpha, K) in {(1, 1), (2, 2), (3, 3), (5, 5), (10, 10), (15, 15), (30, 30)} (K special primes of
50 bits, digits of alpha moduli), one KeySwitchHybrid call alternates rep by rep with one KeySwitchResident call at the
same level with one special prime (SEAL's decomposition: 30 digits), each rep timed with CUDA events after a warm-up.
Reported: ms per switch, launches per switch, resident key bytes, and the bytes per switch the hybrid call moves by
the shapes.  The (1, 1) output is checked against KeySwitchResident's in the same run.  The JSON written to
DIR/hybrid_bench.json (and printed) also holds the card's name and power limit, read in the same run."""
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

PEAK_BYTES_PER_S = 3.35e12
L, KCC = 30, 2
SHAPES = ((1, 1), (2, 2), (3, 3), (5, 5), (10, 10), (15, 15), (30, 30))


def key_bytes(n, alpha, K):
    return -(-L // alpha) * KCC * (L + K) * n * 8


def bytes_per_switch(n, alpha, K):
    """HBM words each step reads and writes, from the shapes"""
    D, B = -(-L // alpha), L + K
    words = {
        "inverse": 2 * L * n,                                    # the target's limbs in and out
        "mod_up": (L + D * B) * n + 2 * D * B * n,               # conversion (digits in, D x B limbs out), transform
        "multiply_accumulate": KCC * D * B * n + KCC * B * n,    # digits once per component, products out
        "keys": D * KCC * B * n,
        "mod_down": (2 * KCC * K + KCC * K + KCC * L + 2 * KCC * L + 4 * KCC * L) * n,
    }
    out = {k: 8 * v for k, v in words.items()}
    out["total"] = sum(out.values())
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=15)
    args = ap.parse_args()
    rng = np.random.default_rng(7)
    work = []
    for log_n in (15, 16):
        n = 1 << log_n
        primes = [int(q) for q in hb.GeneratePrimes(L + max(k for _, k in SHAPES), 50, True, n)]

        def rows(moduli):
            return torch.from_numpy(np.concatenate([rng.integers(0, q, n, dtype=np.uint64) for q in moduli])
                                    .view(np.int64)).cuda()

        target = rows(primes[:L])
        result0 = rows(primes[:L] * KCC)
        # SEAL's decomposition: 30 digits and one special prime, the keys KeySwitchResident takes
        seal_mods = primes[:L + 1]
        modswitch = [pow(seal_mods[-1] % q, -1, q) for q in primes[:L]]
        rk = [rows([q for _ in range(KCC) for q in seal_mods]) for _ in range(L)]
        resident_keys = hb.KeySwitchKeys(rk, n, L, L + 1, KCC)  # also the hybrid keys of (1, 1)
        del rk
        for alpha, K in SHAPES:
            mods = primes[:L + K]
            if (alpha, K) == (1, 1):
                handle = resident_keys
            else:
                keys = [rows([q for _ in range(KCC) for q in mods]) for _ in range(-(-L // alpha))]
                handle = hb.KeySwitchKeys(keys, n, len(keys), L + K, KCC)
                del keys
            out_h, out_r = result0.clone(), result0.clone()

            def hybrid():
                hb.KeySwitchHybrid(out_h, target, n, L, L, K, alpha, KCC, mods, handle)

            def resident():
                hb.KeySwitchResident(out_r, target, n, L, L + 1, L + 1, KCC, seal_mods, resident_keys, modswitch)

            times = alternate(args.reps, hybrid=hybrid, resident=resident)
            launches = {}
            for k, fn in (("hybrid", hybrid), ("resident", resident)):
                l0 = hb.launch_count(); fn(); torch.cuda.synchronize(); launches[k] = hb.launch_count() - l0
            entry = {"n": n, "alpha": alpha, "K": K, "digits": -(-L // alpha), "ms_per_switch": times,
                     "median_ms": {k: statistics.median(v) for k, v in times.items()},
                     "min_ms": {k: min(v) for k, v in times.items()}, "launches_per_switch": launches,
                     "key_bytes": {"hybrid": key_bytes(n, alpha, K), "resident": key_bytes(n, 1, 1)},
                     "hybrid_bytes_per_switch": bytes_per_switch(n, alpha, K)}
            entry["hybrid_share_of_3.35TBps_at_median"] = (entry["hybrid_bytes_per_switch"]["total"]
                                                           / (entry["median_ms"]["hybrid"] * 1e-3) / PEAK_BYTES_PER_S)
            if (alpha, K) == (1, 1):
                a, b = result0.clone(), result0.clone()
                hb.KeySwitchHybrid(a, target, n, L, L, 1, 1, KCC, mods, handle)
                hb.KeySwitchResident(b, target, n, L, L + 1, L + 1, KCC, seal_mods, handle, modswitch)
                torch.cuda.synchronize()
                entry["equals_key_switch_resident"] = bool(torch.equal(a, b))
            work.append(entry)
            print(json.dumps({k: entry[k] for k in ("n", "alpha", "K", "median_ms", "launches_per_switch")}),
                  flush=True)
            del handle, out_h, out_r
            torch.cuda.empty_cache()
        del resident_keys
    res = {"card": card(), "shape": {"level": L, "q_size": L, "moduli_bits": 50, "kcc": KCC, "ciphertexts": 1},
           "workloads": work}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "hybrid_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({"card": res["card"], "equals": [w.get("equals_key_switch_resident") for w in work
                                                     if w["alpha"] == 1]}))


if __name__ == "__main__":
    main()
