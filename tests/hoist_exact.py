"""The hoisted rotations (hexl_b200_apply_galois_key_switch_hoisted) exactly, for the tests.

For a ciphertext (c0, c1) in NTT form, element g and its keys K:
    a_j        = INTT_{q_j}(c1_j)                       digit j, in [0, q_j)
    D_{j,i}    = NTT_{q_i}(a_j mod q_i)                 every modulus i of the switch
    prod_{i,k} = sum_j pi_g(D_{j,i}) K[j][k][slot(i)]  mod q_i
    out        = [sigma_g(c0), 0] + ModDown(prod)        (the mod-down of tests/ks_exact.py:key_switch_exact)
hoisted_exact() computes it in that order, as the GPU does: the digits are transformed once and only permuted per
element.  signed_lift_exact() computes the same thing the other way round, on Python integers: digit j's coefficients
are lifted to the signed integers sigma_g(a_j) (entries +-a_j[t]) and then switched like key_switch_exact.  Both use
the C restatement's canonical NTT, mult_mod, add_mod and sub_mod, as ks_exact does.  tests/test_hoist_exact.py shows
that the two agree, that at g = 1 they equal the rotation [sigma(c0), 0] + KS(sigma(c1)), and that elsewhere they do
not, because sigma_g of the unsigned lift is the signed lift plus q_j wherever sigma_g negates a nonzero coefficient.
"""
from __future__ import annotations

import numpy as np

import galois_exact as gx
from util import uniform_below

U64 = np.uint64


def _slot(i, decomp, kms):
    return kms - 1 if i == decomp else i


def _switch(port, result, ops, n, decomp, kms, kcc, moduli, keys, modswitch):
    """result + ModDown(prod) with prod[i, k] = sum_j ops[i][j] * key_j[k, slot(i)] mod q; ops[i]: [decomp][n] array of
    transformed digits under the modulus of slot(i).  The arithmetic of key_switch_exact, step for step."""
    prod = {}
    for i in range(decomp + 1):
        s = _slot(i, decomp, kms)
        q = moduli[s]
        for k in range(kcc):
            off = (k * kms + s) * n
            acc = np.zeros(n, dtype=U64)
            for j in range(decomp):
                key = np.asarray(keys[j][off:off + n], dtype=U64) % U64(q)
                acc = port.add_mod(acc, port.mult_mod(ops[i][j], key, q), q)
            prod[i, k] = acc
    q_last = moduli[kms - 1]
    half = q_last >> 1
    out = np.array(result, dtype=U64, copy=True)
    for k in range(kcc):
        t_last = port.add_mod(port.ntt_inverse(prod[decomp, k], n, q_last), half, q_last)
        for i in range(decomp):
            qi = moduli[i]
            centred = port.sub_mod(t_last % U64(qi), half % qi, qi)
            d = port.sub_mod(prod[i, k], port.ntt_forward(centred, n, qi), qi)
            d = port.mult_mod(d, np.full(n, int(modswitch[i]) % qi, dtype=U64), qi)
            dst = slice(n * (decomp * k + i), n * (decomp * k + i + 1))
            out[dst] = port.add_mod(out[dst], d, qi)
    return out


def _digits(port, c1, n, decomp, moduli):
    """a_j = INTT_{q_j}(c1_j), canonical"""
    return [port.ntt_inverse(np.asarray(c1[j * n:(j + 1) * n], dtype=U64) % U64(moduli[j]), n, moduli[j])
            for j in range(decomp)]


def hoisted_exact(port, ct, n, decomp, kms, moduli, elts, keys, modswitch):
    """One ciphertext (2 x decomp x n words) rotated by every element of `elts` with keys[r] (a list of KeySwitch key
    lists), transforms first and permutation after, as the GPU runs it.  Returns the rotations back to back."""
    moduli = [int(q) for q in moduli]
    comp = decomp * n
    ct = np.asarray(ct, dtype=U64)
    coef = _digits(port, ct[comp:2 * comp], n, decomp, moduli)
    transformed = []
    for i in range(decomp + 1):  # D_{j,i}: once for every element
        q = moduli[_slot(i, decomp, kms)]
        transformed.append(port.ntt_forward(np.concatenate([c % U64(q) for c in coef]), n, q).reshape(decomp, n))
    out = []
    for g, key in zip(elts, keys):
        p = gx.pi(n, g)
        ops = [d[:, p] for d in transformed]
        r = np.concatenate([gx.sigma_ntt(ct[:comp], n, g), np.zeros(comp, dtype=U64)])
        out.append(_switch(port, r, ops, n, decomp, kms, 2, moduli, key, modswitch))
    return np.concatenate(out)


def signed_lift_exact(port, ct, n, decomp, kms, moduli, g, keys, modswitch):
    """The same rotation on Python integers: digit j lifted to sigma_g(a_j) over Z[X]/(X^n + 1) (coefficients
    +-a_j[t]), reduced into every modulus, transformed and switched"""
    moduli = [int(q) for q in moduli]
    comp = decomp * n
    ct = np.asarray(ct, dtype=U64)
    lifted = [gx.sigma_int([int(v) for v in a], n, g) for a in _digits(port, ct[comp:2 * comp], n, decomp, moduli)]
    ops = []
    for i in range(decomp + 1):
        q = moduli[_slot(i, decomp, kms)]
        ops.append([port.ntt_forward(np.array([v % q for v in a], dtype=U64), n, q) for a in lifted])
    r = np.concatenate([gx.sigma_ntt(ct[:comp], n, g), np.zeros(comp, dtype=U64)])
    return _switch(port, r, ops, n, decomp, kms, 2, moduli, keys, modswitch)


def ciphertexts(case, batch, seed):
    """batch ciphertexts of two canonical components of decomp limbs"""
    n, d = case.n, case.decomp
    return np.concatenate([uniform_below(seed * 7919 + 100 * c + i, n, case.mods[i])
                           for c in range(2 * batch) for i in range(d)])
