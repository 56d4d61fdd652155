"""Rescale by the last RNS modulus (DivideAndRoundQLast) for the tests: SEAL's composition of
RNSTool::divide_and_round_q_last(_ntt)_inplace from single-modulus operations, its integer definition, the same
composition chained from this library's existing public calls, and the moduli chains the tests run.

Layout everywhere: `count` polynomials back to back, each of rns = L + 1 limbs of n words, limb i under moduli[i].
Output limb i (i < L) is floor((X + h) / q_L) mod q_i, with X the CRT lift of the coefficient's limbs and
h = floor(q_L / 2); limb L is left as the operand had it.
"""
from __future__ import annotations

import numpy as np

from util import uniform_below

U64 = np.uint64


def rescale_exact(ops, operand, n, moduli, count, ntt_form):
    """SEAL's sequence on `ops` (the C restatement or the compiled reference): inverse transform of the last limb,
    add h under q_L, then per modulus q_i: reduce, subtract h mod q_i, forward transform, subtract from limb i and
    multiply by q_L^-1 mod q_i.  Returns a new array in the operand's layout."""
    moduli = [int(q) for q in moduli]
    rns = len(moduli)
    L, q_last = rns - 1, moduli[-1]
    half = q_last >> 1
    x = np.asarray(operand, dtype=U64).reshape(count, rns, n)
    out = x.copy()
    last = np.ascontiguousarray(x[:, L]).reshape(-1)
    if ntt_form:
        last = ops.ntt_inverse(last, n, q_last)
    last = ops.add_mod(last, half, q_last)
    for i in range(L):
        q = moduli[i]
        t = ops.sub_mod(last % U64(q), half % q, q)
        if ntt_form:
            t = ops.ntt_forward(t, n, q)
        d = ops.sub_mod(np.ascontiguousarray(x[:, i]).reshape(-1), t, q)
        inv = ops.inverse_mod(q_last % q, q)
        out[:, i] = ops.mult_mod(d, np.full(d.size, inv, dtype=U64), q).reshape(count, n)
    return out.reshape(-1)


def rescale_integer(operand, n, moduli, count):
    """The definition in coefficient form, with Python integers: CRT lift, divide and round, reduce."""
    moduli = [int(q) for q in moduli]
    rns = len(moduli)
    Q = 1
    for q in moduli:
        Q *= q
    basis = [(Q // q) * pow(Q // q, -1, q) for q in moduli]
    q_last, half = moduli[-1], moduli[-1] >> 1
    x = np.asarray(operand, dtype=U64).reshape(count, rns, n)
    out = x.copy()
    for p in range(count):
        for l in range(n):
            X = sum(int(x[p, i, l]) * basis[i] for i in range(rns)) % Q
            y = (X + half) // q_last
            for i in range(rns - 1):
                out[p, i, l] = y % moduli[i]
    return out.reshape(-1)


def rescale_per_limb(operand, n, moduli, count):
    """Coefficient form limb by limb, with Python integers: (x_i + h - ((x_L + h) mod q_L)) * q_L^-1 mod q_i.  Equal to
    rescale_integer() where the CRT lift exists, and still defined where the q_i share factors with each other (each
    q_i coprime to q_L)."""
    moduli = [int(q) for q in moduli]
    rns = len(moduli)
    q_last, half = moduli[-1], moduli[-1] >> 1
    x = np.asarray(operand, dtype=U64).reshape(count, rns, n)
    out = x.copy()
    t = (x[:, -1].astype(object) + half) % q_last
    for i, q in enumerate(moduli[:-1]):
        out[:, i] = ((x[:, i].astype(object) + half - t) * pow(q_last, -1, q) % q).astype(U64)
    return out.reshape(-1)


def edge_values(moduli, n, seed):
    """One polynomial per edge class, as integers ([row][n]): X = 0, X = Q - 1, and X mod q_L in {h - 1, h, h + 1}
    (a random multiple of q_L below Q added), so (X + h) / q_L falls just below, on and just above an integer"""
    Q = 1
    for q in moduli:
        Q *= q
    q_last = moduli[-1]
    half = q_last >> 1
    ks = [int(v) for v in uniform_below(seed, 3 * n, 1 << 63)]
    rows = [[0] * n, [Q - 1] * n]
    for j, off in enumerate((half - 1, half, half + 1)):
        rows.append([(ks[j * n + l] * (Q // q_last) >> 63) * q_last + off for l in range(n)])
    return rows


def limbs_of(values, moduli):
    """Integers (one per coefficient, [count][n]) -> the operand layout [count][rns][n]"""
    values = [[int(v) for v in row] for row in values]
    return np.array([[[v % q for v in row] for q in moduli] for row in values], dtype=U64).reshape(-1)


def random_operand(seed, n, moduli, count):
    return np.concatenate([uniform_below(seed * 7919 + 100 * p + i, n, int(q))
                           for p in range(count) for i, q in enumerate(moduli)])


def chain(primes, n, name, limbs=6):
    """Named moduli chains (every one NTT-friendly for n); the last modulus is the one dropped.
    primes(num, b, prefer_small, n) is GeneratePrimes: b + 1-bit primes, just above 2^b or just below 2^(b+1).

    seal        a 60-bit first prime, 40-bit middles and a 50-bit last prime (SEAL's CKKS shape), `limbs` in all
    classes     a 58-bit, a 29-bit and a 50-bit prime (the transforms' three word classes), then a 45-bit last prime
                larger than one of them and smaller than the others
    wide        primes just below 2^61 (the largest modulus accepted)
    small       primes just above 2^29
    blocks      70 limbs: more than one 64-modulus parameter block
    """
    if name == "seal":
        mods = primes(1, 59, False, n) + primes(limbs - 2, 39, True, n) + primes(1, 49, True, n)
    elif name == "classes":
        mods = primes(1, 57, True, n) + primes(1, 28, True, n) + primes(1, 49, True, n) + primes(1, 44, True, n)
    elif name == "wide":
        mods = primes(4, 60, False, n)
    elif name == "small":
        mods = primes(4, 29, True, n)
    elif name == "blocks":
        mods = primes(69, 44, True, n) + primes(1, 49, True, n)
    else:
        raise ValueError(name)
    assert len(set(mods)) == len(mods)
    return [int(q) for q in mods]


def rescale_chain(hb, result, operand, n, moduli, count, ntt_form, ntts):
    """The rescale chained from the library's existing single-modulus calls, as a caller without
    DivideAndRoundQLast builds it: per polynomial ComputeInverse and EltwiseAddMod on the last limb, then per modulus
    EltwiseReduceMod and EltwiseSubMod, one ComputeForwardMulti over all moduli, and per modulus EltwiseSubMod and
    EltwiseFMAMod.  result / operand: torch CUDA int64 tensors; ntts: GetNTT(n, q) of every modulus."""
    import torch
    moduli = [int(q) for q in moduli]
    rns = len(moduli)
    L, q_last = rns - 1, moduli[-1]
    half = q_last >> 1
    x = operand.view(count, rns, n)
    r = result.view(count, rns, n)
    last = torch.empty(n, dtype=torch.int64, device=operand.device)
    t = torch.empty(L * n, dtype=torch.int64, device=operand.device)
    tv = t.view(L, n)
    for p in range(count):
        if ntt_form:
            ntts[L].ComputeInverse(last, x[p, L], 1, 1)
        else:
            last.copy_(x[p, L])
        hb.EltwiseAddMod(last, last, half, n, q_last)
        for i in range(L):
            hb.EltwiseReduceMod(tv[i], last, n, moduli[i], moduli[i], 1)
            hb.EltwiseSubMod(tv[i], tv[i], half % moduli[i], n, moduli[i])
        if ntt_form:
            hb.ComputeForwardMulti(ntts[:L], t, t, 1, 1, 1)
        for i in range(L):
            q = moduli[i]
            hb.EltwiseSubMod(tv[i], x[p, i], tv[i], n, q)
            hb.EltwiseFMAMod(r[p, i], tv[i], hb.InverseMod(q_last % q, q), None, n, q)
    return result
