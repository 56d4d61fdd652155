"""Ciphertext multiplication with relinearization by hybrid keys (hexl_b200_multiply_relinearize_hybrid) exactly, for
the tests.

The definitions of include/hexl_b200.h restated with the C restatement's canonical NTT, mult_mod, add_mod and sub_mod,
as tests/hybrid_exact.py does, from the pieces of tests/hybrid_rotation_exact.py (the mod-up, the key products and the
rounded mod-down).  For ct1 = (a0, a1), ct2 = (b0, b1) in NTT form at level l:
    d0 = a0 b0,  d1 = a0 b1 + a1 b0,  t = a1 b1                       per data limb
    prod = sum_d D_d(t) K[d]                                          mod-up of t, every m in B
    ext_{q_i} = prod_{q_i} + [P]_{q_i} d,  ext_{p_j} = prod_{p_j}
    result    = ModDown_T(ext), stored                                T = {p_j} or {q_{l-1}, p_j} (rescale)
The mod-down by T = {q_{l-1}, p_0..p_{K-1}} is the mod-down of hybrid_rotation_exact with the limbs of B read as l - 1
data moduli followed by K + 1 special ones: q_{l-1} sits right before the special limbs in B.
"""
from __future__ import annotations

import numpy as np

import hybrid_rotation_exact as hr

U64 = np.uint64


def tensor(port, ct1, ct2, n, level, moduli):
    """(d0, d1, d2) of two ciphertexts, each level x n words: hexl_b200_dyadic_multiply restated"""
    c1 = np.asarray(ct1, dtype=U64).reshape(2, level, n)
    c2 = np.asarray(ct2, dtype=U64).reshape(2, level, n)
    d = np.zeros((3, level, n), dtype=U64)
    for i in range(level):
        q = int(moduli[i])
        d[0, i] = port.mult_mod(c1[0, i], c2[0, i], q)
        d[1, i] = port.add_mod(port.mult_mod(c1[0, i], c2[1, i], q), port.mult_mod(c1[1, i], c2[0, i], q), q)
        d[2, i] = port.mult_mod(c1[1, i], c2[1, i], q)
    return d.reshape(3, level * n)


def multiply_relinearize(port, ct1, ct2, n, level, q_size, p_size, alpha, moduli, keys, rescale):
    """one pair of ciphertexts (2 x level x n words each) with the argument layout of
    hexl_b200_multiply_relinearize_hybrid; returns the product, 2 x (level - rescale) x n words"""
    moduli = [int(q) for q in moduli]
    basis, _ = hr._basis(moduli, level, q_size, p_size)
    d0, d1, t = tensor(port, ct1, ct2, n, level, moduli)
    D = hr.mod_up(port, t, n, level, q_size, p_size, alpha, moduli)
    ext = hr.products(port, D, n, 1, keys, level, q_size, p_size, moduli)  # pi_1 is the identity
    P = 1
    for p in moduli[q_size:q_size + p_size]:
        P *= p
    for i in range(level):
        q = moduli[i]
        for k, d in enumerate((d0, d1)):
            ext[i, k] = port.add_mod(ext[i, k], port.mult_mod(d[i * n:(i + 1) * n], np.full(n, P % q, dtype=U64), q),
                                     q)
    out_level = level - int(rescale)
    return hr.mod_down(port, np.zeros(2 * out_level * n, dtype=U64), ext, n, out_level, out_level,
                       p_size + int(rescale), basis)


def negacyclic_product(a, b, n):
    """a b in Z[X]/(X^n + 1), integer coefficients"""
    out = [0] * n
    for i, x in enumerate(a):
        if x == 0:
            continue
        for j, y in enumerate(b):
            k = i + j
            if k < n:
                out[k] += x * y
            else:
                out[k - n] -= x * y
    return out
