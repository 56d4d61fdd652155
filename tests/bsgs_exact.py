"""The baby-step giant-step linear transform with hybrid keys (hexl_b200_linear_transform_hybrid_bsgs) exactly, for the
tests.

Built from the pieces of tests/hybrid_rotation_exact.py (the mod-up, the key products and the rounded mod-down) and the
automorphism of tests/galois_exact.py, with the C restatement's canonical arithmetic.  For ct = (c0, c1) in NTT form at
level l, R_j the babies with a diagonal in row j, X on the data limbs (from 0) and Y two components over B (from empty):
    x0_j  = sum_{i in R_j} w_{j,i} sigma_{b_i}(c0),  x1_j = sum_{i in R_j, b_i identity} w_{j,i} c1     data limbs
    y_j,k = sum_{i in R_j, b_i keyed} w_{j,i} prod^{b_i}_k                                             every m in B
    identity giant:  X += (x0_j, x1_j);  Y += y_j
    keyed giant h:   c1'_j = x1_j + ModDown_P(y_j,1)      (no ModDown without a keyed baby in R_j)
                     X0 += sigma_h(x0_j);  Y0 += sigma_h(y_j,0);  Y += products(mod_up(c1'_j), h)
    rescale = 0:     result = X + ModDown_P(Y)            (result = X while Y is empty)
    rescale = 1:     ext = Y + [P] X on the data limbs;  result = the mod-down of ext by q_{l-1} P
X and Y stay apart: the mod-down of P x alone need not give x back when K > 1.
"""
from __future__ import annotations

import numpy as np

import galois_exact as gx
import hybrid_rotation_exact as hr

U64 = np.uint64


def _add(port, acc, key, v, m):
    acc[key] = port.add_mod(acc[key], v, m)


def bsgs_exact(port, ct, n, level, q_size, p_size, alpha, moduli, baby_elts, baby_keys, giant_elts, giant_keys,
               diagonals, rescale=False):
    """one ciphertext (2 x level x n words) with the argument layout of hexl_b200_linear_transform_hybrid_bsgs;
    keys[i] is None for an identity term (element 1); diagonals[j][i] is None (absent) or (level + p_size) x n words.
    Returns 2 x (level - rescale) x n words."""
    moduli = [int(q) for q in moduli]
    basis, _ = hr._basis(moduli, level, q_size, p_size)
    nb, comp = len(basis), level * n
    ct = np.asarray(ct, dtype=U64)
    c0, c1 = ct[:comp].reshape(level, n), ct[comp:2 * comp].reshape(level, n)
    n1, n2 = len(baby_elts), len(giant_elts)
    used = [i for i in range(n1) if baby_keys[i] is not None and any(diagonals[j][i] is not None for j in range(n2))]
    prods = {}
    if used:
        D = hr.mod_up(port, ct[comp:2 * comp], n, level, q_size, p_size, alpha, moduli)
        for i in used:
            prods[i] = hr.products(port, D, n, baby_elts[i], baby_keys[i], level, q_size, p_size, moduli)
    X = np.zeros((2, level, n), dtype=U64)
    Y = None

    def zeros_y():
        return {(b, k): np.zeros(n, dtype=U64) for b in range(nb) for k in range(2)}

    for j in range(n2):
        present = [i for i in range(n1) if diagonals[j][i] is not None]
        if not present:
            continue
        x = np.zeros((2, level, n), dtype=U64)
        y = zeros_y()
        keyed_baby = False
        for i in present:
            w = np.asarray(diagonals[j][i], dtype=U64).reshape(nb, n)
            s0 = gx.sigma_ntt(c0, n, baby_elts[i]).reshape(level, n)
            for b in range(level):
                x[0, b] = port.add_mod(x[0, b], port.mult_mod(w[b], s0[b], basis[b]), basis[b])
            if baby_keys[i] is None:
                for b in range(level):
                    x[1, b] = port.add_mod(x[1, b], port.mult_mod(w[b], c1[b], basis[b]), basis[b])
                continue
            keyed_baby = True
            for (b, k), v in prods[i].items():
                _add(port, y, (b, k), port.mult_mod(w[b], v, basis[b]), basis[b])
        if Y is None and (keyed_baby or giant_keys[j] is not None):
            Y = zeros_y()
        if giant_keys[j] is None:
            for b in range(level):
                for k in range(2):
                    X[k, b] = port.add_mod(X[k, b], x[k, b], basis[b])
            if keyed_baby:
                for key, v in y.items():
                    _add(port, Y, key, v, basis[key[0]])
            continue
        h = giant_elts[j]
        c1p = x[1].reshape(-1)
        if keyed_baby:  # the c1 part alone down to Q: component 1 of a two-component mod-down
            half = {(b, 0): np.zeros(n, dtype=U64) for b in range(nb)}
            half.update({(b, 1): y[b, 1] for b in range(nb)})
            start = np.concatenate([np.zeros(comp, dtype=U64), c1p])
            c1p = hr.mod_down(port, start, half, n, level, q_size, p_size, moduli)[comp:]
        rot = gx.sigma_ntt(x[0], n, h).reshape(level, n)
        for b in range(level):
            X[0, b] = port.add_mod(X[0, b], rot[b], basis[b])
        for b in range(nb):
            _add(port, Y, (b, 0), gx.sigma_ntt(y[b, 0], n, h), basis[b])
        D = hr.mod_up(port, c1p, n, level, q_size, p_size, alpha, moduli)
        for key, v in hr.products(port, D, n, h, giant_keys[j], level, q_size, p_size, moduli).items():
            _add(port, Y, key, v, basis[key[0]])
    if not rescale:
        out = X.reshape(-1)
        return out if Y is None else hr.mod_down(port, out, Y, n, level, q_size, p_size, moduli)
    ext = Y if Y is not None else zeros_y()
    P = 1
    for p in moduli[q_size:q_size + p_size]:
        P *= p
    for b in range(level):
        for k in range(2):
            _add(port, ext, (b, k), port.mult_mod(X[k, b], np.full(n, P % basis[b], dtype=U64), basis[b]), basis[b])
    return hr.mod_down(port, np.zeros(2 * (level - 1) * n, dtype=U64), ext, n, level - 1, level - 1, p_size + 1, basis)


def grid_diagonals(basis, n, n2, n1, present, seed, fill=None):
    """an n2 x n1 grid of diagonals: (j, i) in `present` (a set, or None for every pair) gets a hr.random_diagonals
    diagonal, the others None"""
    grid = []
    for j in range(n2):
        row = []
        for i in range(n1):
            ok = present is None or (j, i) in present
            row.append(hr.random_diagonals(basis, n, 1, seed * 1009 + 31 * j + i, fill) if ok else None)
        grid.append(row)
    return grid
