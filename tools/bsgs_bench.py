"""Time LinearTransformHybridBSGS against the chain of existing calls and against the flat LinearTransformHybrid.

    python tools/bsgs_bench.py --out DIR [--reps 15]

Shape: N = 2^16, level = L = 30 data primes of 50 bits, digit size 10 with K = 10 special primes of 50 bits, one
ciphertext, device buffers.  For the grids n1 x n2 in {4 x 4, 8 x 8} (babies b_i = 5^i, giants h_j = 5^(n1 j), so baby
0 and giant 0 are identity terms without keys), alternating rep by rep after a warm-up, each rep timed with CUDA
events:
  * bsgs:  one LinearTransformHybridBSGS call, n1 + n2 - 2 key handles;
  * chain: per giant step one LinearTransformHybrid over the babies, one ApplyGaloisKeySwitchHybridHoisted by h_j
           (none for h_0 = 1) and one EltwiseAddModMulti into the sum;
  * flat:  one LinearTransformHybrid over the n1 n2 elements h_j b_i with diagonals sigma_{h_j}(w_{j,i}),
           n1 n2 - 1 key handles.
The three compute the same plaintext-matrix product, each with its own roundings.  The keys switch from s = 0 (the
key's component 0 is the NTT of a small error, component 1 uniform) and the diagonals are small integer polynomials,
so the phase of each output is its c0 and the three outputs must agree within a small noise: the report gives the
largest centred difference of c0 under q_0 between bsgs and each of the others.  Also reported: median and min ms,
launches per call, key bytes, the words per coefficient slot each call moves by the shapes (not measured), and the
card's name and power limit, read in the same run.  Everything goes to DIR/bsgs_bench.json and is printed."""
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
GRIDS = ((4, 4), (8, 8))
BOUND_W, BOUND_E = 4, 8


def words_per_slot(n1, n2):
    """HBM words per coefficient slot, from the shapes (D digits, B = L + K moduli, two key components).  A mod-up:
    inverse transform 2L plus conversion and transform L + 3 D B; its multiply-accumulate per keyed element: keys 2 D B
    and digits D B (+ B diagonal and nothing stored in the linear transform, + 2B stored in the BSGS baby products).
    A mod-down of c components: c (6K + 14L).  BSGS: one baby mod-up with n1 - 1 stored products; per giant the sum
    (n1 diagonals B, products 2B, c0 L, outputs 8B); per keyed giant a 1-component mod-down, a mod-up and one keyed
    multiply-accumulate; one final mod-down.  Chain: per giant a linear transform over n1 babies and a hoisted rotation
    (mod-up, one multiply-accumulate, products 2B, a 2-component mod-down, 3L) and an add 6L.  Flat: one linear
    transform over n1 n2 elements."""
    D, B = -(-L // ALPHA), L + K
    mod_up = 2 * L + L + 3 * D * B
    down1, down2 = 6 * K + 14 * L, 2 * (6 * K + 14 * L)

    def linear(G):
        return mod_up + (G - 1) * (2 * D * B + D * B + B) + G * 2 * L + 2 * B + down2

    bsgs = mod_up + (n1 - 1) * (3 * D * B + 2 * B)
    bsgs += n2 * (n1 * (B + 2 * B + L) + 8 * B) + (n2 - 1) * (down1 + mod_up + 3 * D * B) + down2
    chain = n2 * linear(n1) + (n2 - 1) * (mod_up + 3 * D * B + 2 * B + down2 + 3 * L) + (n2 - 1) * 6 * L
    return {"bsgs": bsgs, "chain": chain, "flat": linear(n1 * n2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=15)
    args = ap.parse_args()
    rng = np.random.default_rng(12)
    basis = [int(q) for q in hb.GeneratePrimes(L + K, 50, True, N)]
    data = basis[:L]
    ntts = [hb.NTT(N, q) for q in basis]

    def small_ntt(count, bound):
        """count small integer polynomials in NTT form under every modulus of B: count x (L + K) x N words"""
        coef = rng.integers(-bound, bound + 1, size=(count, N), dtype=np.int64)
        out = torch.empty((len(basis), count, N), dtype=torch.int64, device="cuda")
        for b, q in enumerate(basis):
            x = torch.from_numpy((coef % q).astype(np.uint64).view(np.int64).reshape(-1)).cuda()
            ntts[b].ComputeForward(out[b].view(-1), x, 1, 1)
        return out.permute(1, 0, 2).contiguous().view(-1)

    def uniform(moduli):
        return torch.from_numpy(np.concatenate([rng.integers(0, q, N, dtype=np.uint64) for q in moduli])
                                .view(np.int64)).cuda()

    D = -(-L // ALPHA)
    errors = small_ntt(D, BOUND_E).view(D, L + K, N)
    keys = [torch.cat([errors[d].reshape(-1), uniform(basis)]) for d in range(D)]  # switch from s = 0
    n_max = max(a * b for a, b in GRIDS)
    handles = [hb.KeySwitchKeys(keys, N, D, L + K, 2) for _ in range(n_max - 1)]  # one copy per element
    del keys, errors
    comp = L * N
    ct = uniform(data * 2)
    work = []
    for n1, n2 in GRIDS:
        G = n1 * n2
        babies = [pow(5, i, 2 * N) for i in range(n1)]
        giants = [pow(5, n1 * j, 2 * N) for j in range(n2)]
        bkeys = [None] + handles[:n1 - 1]
        gkeys = [None] + handles[n1 - 1:n1 + n2 - 2]
        w = small_ntt(G, BOUND_W).view(n2, n1, (L + K) * N)
        grid = [[w[j, i] for i in range(n1)] for j in range(n2)]
        rows = [w[j].reshape(-1) for j in range(n2)]  # the diagonals of row j back to back, for the chain
        flat_elts = [giants[j] * babies[i] % (2 * N) for j in range(n2) for i in range(n1)]
        flat_keys = [None] + handles[:G - 1]
        flat_diag = torch.empty(G * (L + K) * N, dtype=torch.int64, device="cuda")
        for j in range(n2):
            dst = flat_diag[j * n1 * (L + K) * N:(j + 1) * n1 * (L + K) * N]
            hb.ApplyGalois(dst, rows[j], N, basis, L + K, n1, giants[j], True)
        out_b, out_c, out_f = (torch.empty(2 * comp, dtype=torch.int64, device="cuda") for _ in range(3))
        part, rot = (torch.empty(2 * comp, dtype=torch.int64, device="cuda") for _ in range(2))

        def bsgs():
            hb.LinearTransformHybridBSGS(out_b, ct, N, L, L, K, ALPHA, basis, bkeys, babies, gkeys, giants, grid)

        def chain():
            hb.LinearTransformHybrid(out_c, ct, N, L, L, K, ALPHA, basis, bkeys, babies, rows[0])
            for j in range(1, n2):
                hb.LinearTransformHybrid(part, ct, N, L, L, K, ALPHA, basis, bkeys, babies, rows[j])
                hb.ApplyGaloisKeySwitchHybridHoisted(rot, part, N, L, L, K, ALPHA, basis, [gkeys[j]], [giants[j]])
                hb.EltwiseAddModMulti(out_c, out_c, rot, N, data * 2)

        def flat():
            hb.LinearTransformHybrid(out_f, ct, N, L, L, K, ALPHA, basis, flat_keys, flat_elts, flat_diag)

        times = alternate(args.reps, bsgs=bsgs, chain=chain, flat=flat)
        launches = {}
        for k, fn in (("bsgs", bsgs), ("chain", chain), ("flat", flat)):
            l0 = hb.launch_count(); fn(); torch.cuda.synchronize(); launches[k] = hb.launch_count() - l0

        def c0_distance(a, b):
            """the largest |a0 - b0| over the coefficients, centred under q_0 (the phases are the c0 under s = 0)"""
            q0 = data[0]
            d = torch.empty(N, dtype=torch.int64, device="cuda")
            hb.EltwiseSubMod(d, a[:N], b[:N], N, q0)
            ntts[0].ComputeInverse(d, d, 1, 1)
            x = d.cpu().numpy().view(np.uint64).astype(object)
            return int(max(min(int(v), q0 - int(v)) for v in x))

        med = {k: statistics.median(v) for k, v in times.items()}
        wps = words_per_slot(n1, n2)
        work.append({"grid": [n1, n2], "ms_per_call": times, "median_ms": med,
                     "min_ms": {k: min(v) for k, v in times.items()}, "launches_per_call": launches,
                     "key_handles": {"bsgs": n1 + n2 - 2, "chain": n1 + n2 - 2, "flat": G - 1},
                     "key_bytes": {k: v * D * 2 * (L + K) * N * 8 for k, v in
                                   (("bsgs", n1 + n2 - 2), ("chain", n1 + n2 - 2), ("flat", G - 1))},
                     "words_per_slot_by_shape": wps, "bytes_by_shape": {k: v * 8 * N for k, v in wps.items()},
                     "c0_distance_from_bsgs": {"chain": c0_distance(out_b, out_c), "flat": c0_distance(out_b, out_f)}})
        print(json.dumps({"grid": [n1, n2], "median_ms": med, "launches_per_call": launches,
                          "c0_distance_from_bsgs": work[-1]["c0_distance_from_bsgs"]}), flush=True)
        del w, grid, rows, flat_diag, out_b, out_c, out_f, part, rot
        torch.cuda.empty_cache()
    res = {"card": card(),
           "shape": {"n": N, "level": L, "digit_size": ALPHA, "special_primes": K, "moduli_bits": 50,
                     "ciphertexts": 1, "diagonal_coefficient_bound": BOUND_W, "key_error_bound": BOUND_E},
           "workloads": work}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "bsgs_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({"card": res["card"]}))


if __name__ == "__main__":
    main()
