"""Time the rotations with hybrid keys: ApplyGaloisKeySwitchHybridHoisted against the SEAL-shaped hoisted rotations, and
LinearTransformHybrid against the hoisted hybrid rotations followed by the weighting and the sum.

    python tools/hybrid_rotation_bench.py --out DIR [--reps 15]

Shape: N = 2^16, level = L = 30 data primes of 50 bits, digit size 10 with 10 special primes of 50 bits, one
ciphertext, device buffers.  For G in {1, 2, 4, 8, 16} elements (5, 25, 125, ... mod 2N, each with a key handle of its
own), alternating rep by rep after a warm-up, each rep timed with CUDA events:
  * hoisted_hybrid: one ApplyGaloisKeySwitchHybridHoisted call rotating the ciphertext by the G elements;
  * hoisted_seal:   one ApplyGaloisKeySwitchHoisted call, SEAL's decomposition (30 digits, one special prime);
  * linear:         one LinearTransformHybrid call with G random diagonals;
  * chain:          hoisted_hybrid, then one EltwiseMultModMulti of every rotation by its diagonal and G - 1
                    EltwiseAddModMulti into the sum.
Reported: median and min ms per element, launches per call, key bytes per element, and the words per coefficient slot
each hybrid call moves by the shapes (not measured).  The JSON written to DIR/hybrid_rotation_bench.json (and printed)
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

N, L, ALPHA, K = 1 << 16, 30, 10, 10
ELEMENTS = (1, 2, 4, 8, 16)


def words_per_slot(G):
    """HBM words per coefficient slot of each hybrid call, from the shapes.  D digits, B = L + K moduli of the
    extended basis, two key components.  Paid once per ciphertext: the target's inverse transform (2L), the mod-up's
    conversion and transform (L + 3 D B).  Per element, hoisted: keys 2 D B, the permuted digits once per component
    2 D B, the products 2 B, the mod-down (special limbs' inverse 4K, conversion 2K + 2L, transform 4L, finish 8L) and
    sigma(c0) plus the c1 memset 3L.  Linear: keys 2 D B, the permuted digits once D B, the diagonal B, the
    permuted-sum read of c0 and its diagonal limbs 2L; once: the accumulator 2 B and one mod-down."""
    D, B = -(-L // ALPHA), L + K
    once = 2 * L + L + 3 * D * B
    mod_down = 4 * K + 2 * K + 2 * L + 4 * L + 8 * L
    hoisted = once + G * (2 * D * B + 2 * D * B + 2 * B + mod_down + 3 * L)
    linear = once + G * (2 * D * B + D * B + B + 2 * L) + 2 * B + 2 * L + mod_down
    return {"hoisted_hybrid": hoisted, "linear": linear}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=15)
    args = ap.parse_args()
    rng = np.random.default_rng(11)
    primes = [int(q) for q in hb.GeneratePrimes(L + K, 50, True, N)]
    data, basis = primes[:L], primes
    seal_mods = primes[:L + 1]
    modswitch = [pow(seal_mods[-1] % q, -1, q) for q in data]

    def rows(moduli):
        return torch.from_numpy(np.concatenate([rng.integers(0, q, N, dtype=np.uint64) for q in moduli])
                                .view(np.int64)).cuda()

    G_max = max(ELEMENTS)
    keys = [rows([q for _ in range(2) for q in basis]) for _ in range(-(-L // ALPHA))]
    hybrid_handles = [hb.KeySwitchKeys(keys, N, len(keys), L + K, 2) for _ in range(G_max)]  # one copy per element
    del keys
    keys = [rows([q for _ in range(2) for q in seal_mods]) for _ in range(L)]
    seal_handles = [hb.KeySwitchKeys(keys, N, L, L + 1, 2) for _ in range(G_max)]
    del keys
    comp = L * N
    ct = rows(data * 2)
    diag_all = rows(basis * G_max)
    work = []
    for G in ELEMENTS:
        elts = [pow(5, r + 1, 2 * N) for r in range(G)]
        out_h = torch.empty(G * 2 * comp, dtype=torch.int64, device="cuda")
        out_s = torch.empty_like(out_h)
        res = torch.empty(2 * comp, dtype=torch.int64, device="cuda")
        diag = diag_all[:G * (L + K) * N]
        # the data limbs of each diagonal, once per component, for the chain's weighting
        w2 = diag.view(G, L + K, N)[:, :L].unsqueeze(1).expand(G, 2, L, N).reshape(-1).contiguous()
        weighted = torch.empty_like(out_h)
        chain_sum = torch.empty(2 * comp, dtype=torch.int64, device="cuda")

        def hoisted_hybrid():
            hb.ApplyGaloisKeySwitchHybridHoisted(out_h, ct, N, L, L, K, ALPHA, basis, hybrid_handles[:G], elts)

        def hoisted_seal():
            hb.ApplyGaloisKeySwitchHoisted(out_s, ct, N, L, L + 1, L + 1, 2, seal_mods, seal_handles[:G], modswitch,
                                           elts)

        def linear():
            hb.LinearTransformHybrid(res, ct, N, L, L, K, ALPHA, basis, hybrid_handles[:G], elts, diag)

        def chain():
            hoisted_hybrid()
            hb.EltwiseMultModMulti(weighted, out_h, w2, N, data * 2 * G)
            chain_sum.copy_(weighted[:2 * comp])
            for r in range(1, G):
                hb.EltwiseAddModMulti(chain_sum, chain_sum, weighted[r * 2 * comp:(r + 1) * 2 * comp], N, data * 2)

        times = alternate(args.reps, hoisted_hybrid=hoisted_hybrid, hoisted_seal=hoisted_seal, linear=linear,
                          chain=chain)
        launches = {}
        for k, fn in (("hoisted_hybrid", hoisted_hybrid), ("hoisted_seal", hoisted_seal), ("linear", linear),
                      ("chain", chain)):
            l0 = hb.launch_count(); fn(); torch.cuda.synchronize(); launches[k] = hb.launch_count() - l0
        med = {k: statistics.median(v) for k, v in times.items()}
        wps = words_per_slot(G)
        work.append({"elements": G, "ms_per_call": times, "launches_per_call": launches,
                     "median_ms_per_element": {k: v / G for k, v in med.items()},
                     "min_ms_per_element": {k: min(v) / G for k, v in times.items()},
                     "words_per_slot_by_shape": wps,
                     "bytes_by_shape": {k: v * 8 * N for k, v in wps.items()}})
        print(json.dumps({"elements": G, "median_ms_per_element": work[-1]["median_ms_per_element"],
                          "launches_per_call": launches}), flush=True)
        del out_h, out_s, res, w2, weighted, chain_sum
        torch.cuda.empty_cache()
    res = {"card": card(),
           "shape": {"n": N, "level": L, "digit_size": ALPHA, "special_primes": K, "moduli_bits": 50,
                     "ciphertexts": 1},
           "key_bytes_per_element": {"hybrid": -(-L // ALPHA) * 2 * (L + K) * N * 8, "seal": L * 2 * (L + 1) * N * 8},
           "workloads": work}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "hybrid_rotation_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({"card": res["card"], "key_bytes_per_element": res["key_bytes_per_element"]}))


if __name__ == "__main__":
    main()
