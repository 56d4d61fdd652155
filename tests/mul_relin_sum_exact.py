"""A sum of ciphertext products relinearized once with hybrid keys (hexl_b200_multiply_relinearize_sum_hybrid) exactly,
for the tests.

The definitions of include/hexl_b200.h restated with the C restatement's canonical mult_mod and add_mod, from the
tensor of tests/mul_relin_exact.py and the pieces of tests/hybrid_rotation_exact.py (the mod-up, the key products and
the rounded mod-down).  For pairs (ct1_r, ct2_r) = ((a0_r, a1_r), (b0_r, b1_r)) in NTT form at level l:
    d0 = sum_r a0_r b0_r,  d1 = sum_r (a0_r b1_r + a1_r b0_r),  t = sum_r a1_r b1_r       per data limb, mod q_i
    prod = sum_d D_d(t) K[d]                                                                mod-up of t, every m in B
    ext_{q_i} = prod_{q_i} + [P]_{q_i} d,  ext_{p_j} = prod_{p_j}
    result    = ModDown_T(ext), stored                                  T = {p_j} or {q_{l-1}, p_j} (rescale)
"""
from __future__ import annotations

import numpy as np

import hybrid_rotation_exact as hr
import mul_relin_exact as mr

U64 = np.uint64


def tensor_sum(port, ct1s, ct2s, n, level, moduli):
    """(d0, d1, t) summed over the pairs, 3 x level x n words: DyadicMultiply of every pair and EltwiseAddModMulti"""
    moduli = [int(q) for q in moduli]
    d = None
    for a, b in zip(ct1s, ct2s):
        t = mr.tensor(port, a, b, n, level, moduli)
        if d is None:
            d = t
            continue
        for k in range(3):
            for i in range(level):
                s = slice(i * n, (i + 1) * n)
                d[k, s] = port.add_mod(d[k, s], t[k, s], moduli[i])
    return d


def relinearize(port, d, n, level, q_size, p_size, alpha, moduli, keys, rescale):
    """the steps of hexl_b200_multiply_relinearize_hybrid from the mod-up of t on, for a tensor d = (d0, d1, t)"""
    moduli = [int(q) for q in moduli]
    basis, _ = hr._basis(moduli, level, q_size, p_size)
    d0, d1, t = d
    D = hr.mod_up(port, t, n, level, q_size, p_size, alpha, moduli)
    ext = hr.products(port, D, n, 1, keys, level, q_size, p_size, moduli)  # pi_1 is the identity
    P = 1
    for p in moduli[q_size:q_size + p_size]:
        P *= p
    for i in range(level):
        q = moduli[i]
        for k, dk in enumerate((d0, d1)):
            ext[i, k] = port.add_mod(ext[i, k], port.mult_mod(dk[i * n:(i + 1) * n], np.full(n, P % q, dtype=U64), q),
                                     q)
    out_level = level - int(rescale)
    return hr.mod_down(port, np.zeros(2 * out_level * n, dtype=U64), ext, n, out_level, out_level,
                       p_size + int(rescale), basis)


def multiply_relinearize_sum(port, ct1s, ct2s, n, level, q_size, p_size, alpha, moduli, keys, rescale):
    """one output: the pairs (ct1s[r], ct2s[r]) (2 x level x n words each) with the argument layout of
    hexl_b200_multiply_relinearize_sum_hybrid; returns the relinearized sum, 2 x (level - rescale) x n words"""
    d = tensor_sum(port, ct1s, ct2s, n, level, moduli)
    return relinearize(port, d, n, level, q_size, p_size, alpha, moduli, keys, rescale)
