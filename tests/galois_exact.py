"""The Galois automorphism sigma_g : a(X) -> a(X^g) for the tests, by definition, and the Galois keys a rotation
key-switches with.

Layout everywhere: `count` polynomials back to back, each of rns limbs of n words, limb i under moduli[i].
    coefficient form  coefficient i moves to k = i g mod 2n; negated (mod q) when k >= n, because X^n = -1
    NTT form          result[j] = operand[pi_g(j)], pi_g(j) = rev(((g (2 rev(j) + 1)) mod 2n - 1) / 2)
The NTT form is the forward-transform order of ntt_exact.forward (slot j holds a(psi^(2 rev(j) + 1))), so
forward(sigma_coef(a)) == sigma_ntt(forward(a)); tests/test_galois_exact.py pins that.

rotation_exact() is ApplyGaloisKeySwitch exactly: the exact key switch (tests/ks_exact.py) of [sigma(c0), 0] with the
digits sigma(c1).
"""
from __future__ import annotations

import numpy as np

import ks_exact
from ntt_exact import _brv
from util import uniform_below

U64 = np.uint64


def pi(n, g):
    """pi_g as an index array: slot j of the NTT-form result reads slot pi[j] of the operand"""
    assert g % 2 == 1 and 1 <= g < 2 * n
    rev = _brv(n)
    k = (g * (2 * rev + 1)) % (2 * n)
    return rev[(k - 1) // 2]


def sigma_ntt(x, n, g):
    """NTT form: every polynomial of x (back to back, any modulus) permuted by pi_g"""
    return np.ascontiguousarray(np.asarray(x, dtype=U64).reshape(-1, n)[:, pi(n, g)]).reshape(-1)


def sigma_coef(x, n, g, moduli, count=1):
    """coefficient form, by definition: result[i g mod 2n] = x[i], or -x[i] mod q at (i g mod 2n) - n"""
    assert g % 2 == 1 and 1 <= g < 2 * n
    moduli = [int(q) for q in moduli]
    a = np.asarray(x, dtype=U64).reshape(count, len(moduli), n)
    q = np.array(moduli, dtype=U64)[None, :, None]
    k = (np.arange(n, dtype=np.int64) * g) % (2 * n)
    pos = k < n
    out = np.empty_like(a)
    out[:, :, k[pos]] = a[:, :, pos]
    neg = a[:, :, ~pos]
    out[:, :, k[~pos] - n] = np.where(neg == 0, U64(0), q - neg)
    return out.reshape(-1)


def sigma_int(coeffs, n, g):
    """sigma_g of one polynomial of Python integers (no modulus): the coefficient rule over Z[X]/(X^n + 1)"""
    out = [0] * n
    for i, c in enumerate(coeffs):
        k = i * g % (2 * n)
        if k < n:
            out[k] = c
        else:
            out[k - n] = -c
    return out


def rotation_exact(port, case, ct, g, batch):
    """ks_exact of r = [sigma(c0), 0] with t = sigma(c1), per ciphertext: `batch` ciphertexts of the ks_exact.Case
    `case` (two components of decomp limbs each, NTT form) back to back"""
    comp = case.decomp * case.n
    out = []
    for c in range(batch):
        c0 = ct[2 * c * comp:(2 * c + 1) * comp]
        c1 = ct[(2 * c + 1) * comp:(2 * c + 2) * comp]
        r = np.concatenate([sigma_ntt(c0, case.n, g), np.zeros(comp, dtype=U64)])
        out.append(ks_exact.key_switch_exact(port, r, sigma_ntt(c1, case.n, g), *case.shape, case.keys,
                                             case.modswitch))
    return np.concatenate(out)


def galois_keys(port, s, g, n, mods, decomp, error_seed, bound_e):
    """Key-switch keys that move a ciphertext under sigma_g(s) back under s, in the layout KeySwitch takes.

    s: the ternary secret (Python ints, n coefficients).  mods: the key moduli, the special prime P last
    (key_modulus_size = len(mods)).  Key j (digit j), in NTT form under every key modulus:
        component 1: a_j, uniform;
        component 0: -a_j s + e_j + [i == j] P sigma_g(s) in limb i < decomp, and -a_j s + e_j under P,
    with e_j an integer polynomial of coefficients in [-bound_e, bound_e].  Returns (keys, modswitch), modswitch_i =
    P^-1 mod q_i."""
    kms = len(mods)
    P = mods[-1]
    sg = sigma_int(s, n, g)

    def ntt(coeffs, q):
        return port.ntt_forward(np.array([c % q for c in coeffs], dtype=U64), n, q)

    s_ntt = [ntt(s, q) for q in mods]
    sg_ntt = [ntt(sg, q) for q in mods]
    keys = []
    for j in range(decomp):
        e = [int(v) - bound_e for v in uniform_below(error_seed + j, n, 2 * bound_e + 1)]
        c0, c1 = [], []
        for i, q in enumerate(mods):
            a = uniform_below(error_seed * 31 + 1000 * j + i, n, q)
            b = port.sub_mod(ntt(e, q), port.mult_mod(a, s_ntt[i], q), q)
            if i == j:
                b = port.add_mod(b, port.mult_mod(sg_ntt[i], np.full(n, P % q, dtype=U64), q), q)
            c0.append(b)
            c1.append(a)
        keys.append(np.concatenate(c0 + c1))
    modswitch = [port.inverse_mod(P % q, q) for q in mods[:decomp]]
    return keys, modswitch
