"""Time ApplyGalois and ApplyGaloisKeySwitch.

    python tools/galois_bench.py --out DIR [--reps 7]

Every workload runs after a warm-up, each rep timed with CUDA events and alternated rep by rep with its comparison:
  * ApplyGalois, 128 polynomials of 31 limbs, device buffers, out of place: NTT form at N = 2^16, coefficient form at
    N = 2^14 (the largest degree staged in shared memory), 2^15 (the smallest served by L2 gathers) and 2^16.  The
    comparison is a device-to-device copy of the same buffer (the floor for a permutation).  Reported: time, achieved
    bytes/s at 16 B per word (read once, written once) and their share of the H100's 3.35 TB/s.
  * ApplyGaloisKeySwitch at bench.py's C5 shape (N = 2^15, 29 digits + the special prime, 50-bit moduli, 8
    ciphertexts per call, resident keys): time per ciphertext next to KeySwitchResident on the same buffers and next to
    the chain of existing calls (ApplyGalois of both components, copy and zero, KeySwitchResident); device buffers and
    pinned host buffers.
The JSON written to DIR/galois_bench.json (and printed) also holds the card's name and power limit, read in the same
run."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import torch  # noqa: E402

import hexl_b200 as hb  # noqa: E402
import rescale_exact as rx  # noqa: E402

PEAK_BYTES_PER_S = 3.35e12


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return {"name": name, "power_limit": power}


def time_ms(fn):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    fn()
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop)


def alternate(reps, **fns):
    for fn in fns.values():
        fn()
    torch.cuda.synchronize()
    times = {k: [] for k in fns}
    for _ in range(reps):
        for k, fn in fns.items():
            times[k].append(time_ms(fn))
    return times


def permutation(log_n, ntt_form, reps, limbs=31, count=128):
    n = 1 << log_n
    mods = rx.chain(hb.GeneratePrimes, n, "seal", limbs)
    src = torch.from_numpy(rx.random_operand(log_n, n, mods, count).view(np.int64)).cuda()
    out, copy = torch.empty_like(src), torch.empty_like(src)
    g = 2 * n - 5
    times = alternate(reps, galois=lambda: hb.ApplyGalois(out, src, n, mods, limbs, count, g, ntt_form),
                      copy=lambda: copy.copy_(src))
    l0 = hb.launch_count(); hb.ApplyGalois(out, src, n, mods, limbs, count, g, ntt_form); torch.cuda.synchronize()
    launches = hb.launch_count() - l0
    nbytes = 16 * src.numel()
    best = min(times["galois"])
    return {"op": "ApplyGalois", "form": "ntt" if ntt_form else "coefficient", "n": n, "limbs": limbs,
            "polynomials": count, "galois_elt": g, "ms": times["galois"], "copy_ms": times["copy"],
            "launches_per_call": launches, "bytes": nbytes, "best_bytes_per_s": nbytes / (best * 1e-3),
            "best_share_of_3.35TBps": nbytes / (best * 1e-3) / PEAK_BYTES_PER_S}


def rotation(reps):
    n, decomp, kcc, cts = 1 << 15, 29, 2, 8
    kms = rns = decomp + 1
    mods = hb.GeneratePrimes(kms, 50, True, n)
    modswitch = [hb.InverseMod(mods[-1] % mods[i], mods[i]) for i in range(decomp)]
    rng = np.random.default_rng(5)

    def rows(moduli):
        return np.concatenate([rng.integers(0, q, n, dtype=np.uint64) for q in moduli])

    keys = [torch.from_numpy(rows([mods[i] for _ in range(kcc) for i in range(kms)]).view(np.int64)).cuda()
            for _ in range(decomp)]
    handle = hb.KeySwitchKeys(keys, n, decomp, kms, kcc)
    comp = decomp * n
    ct0 = torch.from_numpy(rows(mods[:decomp] * (kcc * cts)).view(np.int64)).cuda()
    ct = ct0.clone()
    t = torch.from_numpy(rows(mods[:decomp] * cts).view(np.int64)).cuda()
    res = ct0.clone()
    perm = torch.empty_like(ct0)
    g = 3

    def chain():
        hb.ApplyGalois(perm, ct, n, mods, decomp, kcc * cts, g, True)
        p = perm.view(cts, kcc, comp)
        c = ct.view(cts, kcc, comp)
        c[:, 0].copy_(p[:, 0])
        c[:, 1].zero_()
        t.view(cts, comp).copy_(p[:, 1])
        hb.KeySwitchResident(ct, t, n, decomp, kms, rns, kcc, mods, handle, modswitch, cts)

    fns = {"rotation": lambda: hb.ApplyGaloisKeySwitch(ct, n, decomp, kms, rns, kcc, mods, handle, modswitch, g, cts),
           "key_switch": lambda: hb.KeySwitchResident(res, t, n, decomp, kms, rns, kcc, mods, handle, modswitch, cts),
           "chain": chain}
    # the composite and the chain compute the same words
    a = ct0.clone(); b = ct0.clone()
    ct.copy_(a); fns["rotation"](); a.copy_(ct)
    ct.copy_(b); chain(); b.copy_(ct)
    torch.cuda.synchronize()
    same = bool(torch.equal(a, b))
    times = alternate(reps, **fns)
    launches = {}
    for k, fn in fns.items():
        l0 = hb.launch_count(); fn(); torch.cuda.synchronize(); launches[k] = (hb.launch_count() - l0) / cts
    # host buffers (pinned), same shape
    h_ct = hb.pinned_empty(ct0.numel()); h_ct[:] = ct0.cpu().numpy().view(np.uint64)
    h_res = hb.pinned_empty(ct0.numel()); h_res[:] = h_ct
    h_t = hb.pinned_empty(t.numel()); h_t[:] = t.cpu().numpy().view(np.uint64)
    host_times = alternate(
        reps,
        rotation=lambda: hb.ApplyGaloisKeySwitch(h_ct, n, decomp, kms, rns, kcc, mods, handle, modswitch, g, cts),
        key_switch=lambda: hb.KeySwitchResident(h_res, h_t, n, decomp, kms, rns, kcc, mods, handle, modswitch, cts))
    per = {k: [1e3 * v / cts for v in vs] for k, vs in times.items()}
    host_per = {k: [1e3 * v / cts for v in vs] for k, vs in host_times.items()}
    return {"op": "ApplyGaloisKeySwitch", "n": n, "decomp": decomp, "rns": rns, "ciphertexts_per_call": cts,
            "device_us_per_ciphertext": per, "host_us_per_ciphertext": host_per,
            "launches_per_ciphertext": launches, "composite_equals_chain": same}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=7)
    args = ap.parse_args()
    work = [permutation(16, True, args.reps), permutation(14, False, args.reps), permutation(15, False, args.reps),
            permutation(16, False, args.reps)]
    torch.cuda.empty_cache()
    work.append(rotation(args.reps))
    res = {"card": card(), "workloads": work}
    os.makedirs(args.out, exist_ok=True)
    with open(os.path.join(args.out, "galois_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
