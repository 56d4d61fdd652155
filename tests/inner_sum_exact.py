"""The inner sum of k rotations with hybrid keys (hexl_b200_inner_sum_hybrid) exactly, for the tests, and its launch
plan.

Built from the pieces of tests/hybrid_rotation_exact.py (mod-up, key products, rounded mod-down) and the automorphism of
tests/galois_exact.py, with the C restatement's canonical arithmetic.  A pair (X, Y): X two components on the data limbs,
Y two components over B = {q_0..q_{l-1}, p_0..p_{K-1}} or None (empty); val(X, Y) = X + ModDown_P(Y).
    Rot_1(X, Y) = (X, Y)
    Rot_e(X, Y) = ((sigma_e X0, 0), (pi_e Y0 + M_e,0, M_e,1)),  M_e = products(mod_up(c1'), e),
                  c1' = X1 + ModDown_P(Y1)  (X1 while Y is empty)
    A = (ct, None); R = None; s = 0
    for i = 0 .. floor(log2 k):
        bit i of k set:   R = Rot_{g^s}(A) or R + Rot_{g^s}(A);  s += 2^i
        2^(i+1) <= k:     A = A + Rot_{g^(2^i)}(A)
    rescale = 0:  X_R + ModDown_P(Y_R)   (X_R while Y_R is empty)
    rescale = 1:  the mod-down of Y_R + [P] X_R (data limbs) by q_{l-1} P, as tests/bsgs_exact.py folds it
Both rotations of one bit read the same A, so they share c1' and its mod-up.
"""
from __future__ import annotations

import numpy as np

import composite_plan as cp
import galois_exact as gx
import hybrid_rotation_exact as hr

U64 = np.uint64


def inner_sum_bits(g, k, n):
    """per bit i of k: (doubling element g^(2^i) when 2^(i+1) <= k else None, shift element g^s when bit i is set else
    None), elements mod 2n"""
    bits, power, shift = [], g % (2 * n), 1
    i = 0
    while k >> i:
        sh = None
        if (k >> i) & 1:
            sh, shift = shift, shift * power % (2 * n)
        bits.append((power if k >> (i + 1) else None, sh))
        power = power * power % (2 * n)
        i += 1
    return bits


def needed_elements(g, k, n):
    """the elements other than 1 the call needs keys for, sorted"""
    return sorted({e for bit in inner_sum_bits(g, k, n) for e in bit if e is not None and e != 1})


def inner_sum_exact(port, ct, n, level, q_size, p_size, alpha, moduli, g, k, keys, rescale=False):
    """one ciphertext (2 x level x n words); keys maps each element of needed_elements to its hybrid key buffers.
    Returns 2 x (level - rescale) x n words."""
    moduli = [int(q) for q in moduli]
    basis, _ = hr._basis(moduli, level, q_size, p_size)
    nb, comp = len(basis), level * n
    ct = np.asarray(ct, dtype=U64)
    assert k >= 1

    def add_x(a, b):
        return np.stack([np.stack([port.add_mod(a[c, i], b[c, i], basis[i]) for i in range(level)]) for c in range(2)])

    def add_y(a, b):
        if a is None:
            return b
        if b is None:
            return a
        return {key: port.add_mod(a[key], b[key], basis[key[0]]) for key in a}

    def rot(pair, e):
        X, Y = pair
        if e == 1:
            return X, Y
        c1 = X[1].reshape(-1)
        if Y is not None:
            half = {(b, 0): np.zeros(n, dtype=U64) for b in range(nb)}
            half.update({(b, 1): Y[b, 1] for b in range(nb)})
            start = np.concatenate([np.zeros(comp, dtype=U64), c1])
            c1 = hr.mod_down(port, start, half, n, level, q_size, p_size, moduli)[comp:]
        D = hr.mod_up(port, c1, n, level, q_size, p_size, alpha, moduli)
        M = hr.products(port, D, n, e, keys[e], level, q_size, p_size, moduli)
        X2 = np.zeros_like(X)
        X2[0] = gx.sigma_ntt(X[0], n, e).reshape(level, n)
        Y2 = {}
        for b in range(nb):
            y0 = gx.sigma_ntt(Y[b, 0], n, e) if Y is not None else np.zeros(n, dtype=U64)
            Y2[b, 0] = port.add_mod(y0, M[b, 0], basis[b])
            Y2[b, 1] = M[b, 1]
        return X2, Y2

    A = (ct[:2 * comp].reshape(2, level, n).copy(), None)
    R = None
    for dbl, shift in inner_sum_bits(g, k, n):
        if shift is not None:
            r = rot(A, shift)
            R = r if R is None else (add_x(R[0], r[0]), add_y(R[1], r[1]))
        if dbl is not None:
            r = rot(A, dbl)
            A = (add_x(A[0], r[0]), add_y(A[1], r[1]))
    X, Y = R
    if not rescale:
        out = X.reshape(-1)
        return out if Y is None else hr.mod_down(port, out, Y, n, level, q_size, p_size, moduli)
    ext = Y if Y is not None else {(b, c): np.zeros(n, dtype=U64) for b in range(nb) for c in range(2)}
    ext = dict(ext)
    P = 1
    for p in moduli[q_size:q_size + p_size]:
        P *= p
    for b in range(level):
        for c in range(2):
            w = port.mult_mod(X[c, b], np.full(n, P % basis[b], dtype=U64), basis[b])
            ext[b, c] = port.add_mod(ext[b, c], w, basis[b])
    return hr.mod_down(port, np.zeros(2 * (level - 1) * n, dtype=U64), ext, n, level - 1, level - 1, p_size + 1, basis)


def inner_sum_launches(n, level, K, alpha, basis, ntt, g, k, rescale=False):
    """InnerSumHybrid: kernel launches of one ciphertext (basis: the moduli of B; ntt(forward, units) as in
    composite_plan.hybrid_launches).  Per bit: one step launch per block of 64 moduli of the span (B when Y is read or
    written, else the data moduli); with a keyed element, the one-component mod-down of Y_A1 when Y_A is non-empty and
    one mod-up with a multiply-accumulate set per keyed element; then the final mod-down (none while Y_R is empty, or
    over (level - 1, K + 1) with the merged rescale)."""
    bits = inner_sum_bits(g, k, n)
    total, y_a, y_r = 0, False, False
    for i, (dbl, shift) in enumerate(bits):
        fold = rescale and i + 1 == len(bits)
        keyed = [e for e in (dbl, shift) if e is not None and e != 1]
        next_y = dbl is not None and (y_a or dbl != 1)
        r_y = shift is not None and (y_a or shift != 1 or fold)
        copy1 = y_a and bool(keyed)
        span = level + K if (next_y or r_y or copy1) else level
        total += -(-span // cp.PARAM_BLOCK)
        if keyed:
            if y_a:
                total += cp.hybrid_mod_down_launches(level, K, 1, ntt)
            total += cp.hybrid_mod_up_launches(n, level, K, alpha, basis, ntt,
                                               lambda D, q: len(keyed) * len(cp.ks_mac_launches(D, q)))
        if dbl is not None:
            y_a = next_y
        y_r = y_r or r_y
    if rescale:
        return total + cp.hybrid_mod_down_launches(level, K, 2, ntt, True)
    return total + (cp.hybrid_mod_down_launches(level, K, 2, ntt) if y_r else 0)
