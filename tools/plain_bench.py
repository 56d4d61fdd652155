"""Time PlainLift, BfvAddPlain and BfvMultiplyPlain with device-resident data.

    python tools/plain_bench.py --out DIR [--reps 30]

Shapes: n = 2^13 to 2^16 with l = 3, 15 and 30 data moduli of 50 bits, t = 65537, a full plaintext (plain_coeff_count =
n) broadcast to a batch of 8 ciphertexts.  All calls of one shape alternate rep by rep after a warm-up, each rep timed
with CUDA events:
  * lift:       PlainLift of one plaintext in NTT form;
  * add:        BfvAddPlain in place;
  * mul:        BfvMultiplyPlain with the plaintext in coefficient form (lifted and transformed once per call);
  * mul_ntt:    BfvMultiplyPlain with the plaintext PlainLift already produced;
  * chain:      the four-call chain the fused multiply replaces: PlainLift (NTT form), ComputeForwardMulti of the
                ciphertexts, EltwiseMultModMulti by the lifted plaintext, ComputeInverseMulti.
Achieved bytes/s use the algorithmic bytes of each call, computed below: lift n + l n words; add (in place) l n + n
words read and l n written per ciphertext; both multiplies 2 l n read and 2 l n written per ciphertext plus the
plaintext (n words, or l n in NTT form).  The JSON written to DIR/plain_bench.json (and printed) also holds the card's
name and power limit, read in the same run."""
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

LOGN = (13, 14, 15, 16)
LEVELS = (3, 15, 30)
BATCH = 8
T = 65537


def algorithmic_bytes(n, l, batch):
    return {"lift": 8 * (n + l * n), "add": 8 * batch * (2 * l * n + n),
            "mul": 8 * (batch * 4 * l * n + n), "mul_ntt": 8 * (batch * 4 * l * n + l * n),
            "chain": 8 * (batch * 4 * l * n + n)}


def shape(n, l, reps):
    mods = [int(q) for q in hb.GeneratePrimes(l, 50, True, n)]
    ntts = [hb.GetNTT(n, q) for q in mods]
    g = torch.Generator(device="cuda").manual_seed(n + l)
    ct = torch.cat([torch.randint(0, q, (n,), device="cuda", generator=g) for _ in range(2 * BATCH) for q in mods])
    plain = torch.randint(0, T, (n,), device="cuda", generator=g)
    out, x = torch.empty_like(ct), torch.empty_like(ct)
    fp = torch.empty(l * n, dtype=torch.int64, device="cuda")
    fp2 = torch.empty(2 * BATCH * l * n, dtype=torch.int64, device="cuda")
    lifted = torch.empty(l * n, dtype=torch.int64, device="cuda")
    hb.PlainLift(fp, plain, n, n, mods, l, T, 1, True)
    work = ct.clone()

    def chain():
        hb.PlainLift(lifted, plain, n, n, mods, l, T, 1, True)
        hb.ComputeForwardMulti(ntts * 2 * BATCH, x, ct)
        hb.EltwiseMultModMulti(x, x, fp2, n, mods * 2 * BATCH)
        hb.ComputeInverseMulti(ntts * 2 * BATCH, x, x)

    fp2.copy_(fp.repeat(2 * BATCH))  # the chain's operand layout: the lifted plaintext once per component
    fns = {
        "lift": lambda: hb.PlainLift(lifted, plain, n, n, mods, l, T, 1, True),
        "add": lambda: hb.BfvAddPlain(work, work, plain, n, n, mods, l, T, False, 1, BATCH),
        "mul": lambda: hb.BfvMultiplyPlain(out, ct, plain, n, n, mods, l, T, False, 1, BATCH),
        "mul_ntt": lambda: hb.BfvMultiplyPlain(out, ct, fp, n, n, mods, l, T, True, 1, BATCH),
        "chain": chain,
    }
    times = alternate(reps, **fns)
    hb.BfvMultiplyPlain(out, ct, plain, n, n, mods, l, T, False, 1, BATCH)
    chain()
    torch.cuda.synchronize()
    same = bool(torch.equal(out, x))
    nbytes = algorithmic_bytes(n, l, BATCH)
    row = {"n": n, "l": l, "batch": BATCH, "fused_equals_chain": same}
    for k, v in times.items():
        med = statistics.median(v)
        row[k] = {"median_ms": round(med, 4), "min_ms": round(min(v), 4),
                  "GB_per_s": round(nbytes[k] / (med * 1e-3) / 1e9, 1)}
    row["mul_over_chain"] = round(row["mul"]["median_ms"] / row["chain"]["median_ms"], 3)
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=30)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("plain_bench needs a CUDA device")
    result = {"card": card(), "rows": [shape(1 << lg, l, args.reps) for lg in LOGN for l in LEVELS]}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "plain_bench.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
