"""Time ApplyGaloisKeySwitchHoisted against one ApplyGaloisKeySwitch call per element.

    python tools/hoist_bench.py --out DIR [--reps 15]

Shape: bench.py's C5 (N = 2^15, 29 digits + the special prime, 50-bit moduli, resident keys), one ciphertext, device
buffers.  For G in {1, 2, 4, 8, 16} elements (3, 5, 7, ..., each with a key handle of its own):
  * hoisted: one ApplyGaloisKeySwitchHoisted call rotating the ciphertext by the G elements;
  * separate: G ApplyGaloisKeySwitch calls, each on its own copy of the same ciphertext.
The two alternate rep by rep after a warm-up, each rep timed with CUDA events.  Reported: ms per call and per
rotation, launches per call, and the bytes per rotation the hoisted call moves by the shapes (keys streamed once,
the permuted digits as the multiply-accumulate reads them, once per key component, and the mod-down with the c0
permutation and c1 memset).  The JSON written to DIR/hoist_bench.json (and printed) also holds the card's name and
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

PEAK_BYTES_PER_S = 3.35e12
N, DECOMP, KCC = 1 << 15, 29, 2
ELEMENTS = (1, 2, 4, 8, 16)


def bytes_per_rotation():
    rns, w = DECOMP + 1, 8
    keys = DECOMP * KCC * rns * N * w
    digits = KCC * rns * DECOMP * N * w            # the MAC reads every digit once per key component
    products = KCC * rns * N * w                    # the MAC's output, written once
    # mod-down: inverse transform of the special part (read + write), round (write), forward transform (read + write),
    # finish (products, round and result read, result written); plus sigma(c0) (read + write) and the c1 memset
    mod_down = (2 * KCC * N + DECOMP * KCC * N * (1 + 2 + 4)) * w + 3 * DECOMP * N * w
    return {"keys": keys, "permuted_digits": digits, "products": products, "mod_down": mod_down,
            "total": keys + digits + products + mod_down}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=15)
    args = ap.parse_args()
    kms = rns = DECOMP + 1
    mods = hb.GeneratePrimes(kms, 50, True, N)
    modswitch = [hb.InverseMod(mods[-1] % mods[i], mods[i]) for i in range(DECOMP)]
    rng = np.random.default_rng(5)

    def rows(moduli):
        return np.concatenate([rng.integers(0, q, N, dtype=np.uint64) for q in moduli])

    keys = [torch.from_numpy(rows([mods[i] for _ in range(KCC) for i in range(kms)]).view(np.int64)).cuda()
            for _ in range(DECOMP)]
    handles = [hb.KeySwitchKeys(keys, N, DECOMP, kms, KCC) for _ in range(max(ELEMENTS))]  # one copy per element
    del keys
    comp = DECOMP * N
    ct = torch.from_numpy(rows(mods[:DECOMP] * KCC).view(np.int64)).cuda()
    shape = (N, DECOMP, kms, rns, KCC, mods)
    work = []
    for G in ELEMENTS:
        elts = [3 + 2 * r for r in range(G)]
        out = torch.empty(G * 2 * comp, dtype=torch.int64, device="cuda")
        copies = ct.repeat(G)

        def hoisted():
            hb.ApplyGaloisKeySwitchHoisted(out, ct, *shape, handles[:G], modswitch, elts)

        def separate():
            for r, g in enumerate(elts):
                hb.ApplyGaloisKeySwitch(copies[r * 2 * comp:(r + 1) * 2 * comp], *shape, handles[r], modswitch, g)

        times = alternate(args.reps, hoisted=hoisted, separate=separate)
        launches = {}
        for k, fn in (("hoisted", hoisted), ("separate", separate)):
            l0 = hb.launch_count(); fn(); torch.cuda.synchronize(); launches[k] = hb.launch_count() - l0
        med = {k: statistics.median(v) for k, v in times.items()}
        b = bytes_per_rotation()
        work.append({"elements": G, "ms_per_call": times, "launches_per_call": launches,
                     "median_ms_per_rotation": {k: v / G for k, v in med.items()},
                     "min_ms_per_rotation": {k: min(v) / G for k, v in times.items()},
                     "hoisted_bytes_per_rotation": b,
                     "hoisted_share_of_3.35TBps_at_median": b["total"] / (med["hoisted"] / G * 1e-3) / PEAK_BYTES_PER_S})
        del out, copies
        torch.cuda.empty_cache()
    res = {"card": card(), "shape": {"n": N, "decomp": DECOMP, "rns": rns, "moduli_bits": 50, "ciphertexts": 1},
           "workloads": work}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "hoist_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
