"""The rotations with hybrid keys exactly, for the tests: hexl_b200_apply_galois_key_switch_hybrid_hoisted and
hexl_b200_linear_transform_hybrid.

Built from the hybrid switch's pieces (tests/hybrid_exact.py: fast_base_convert, digits) and the automorphism
(tests/galois_exact.py: pi, sigma_ntt), with the C restatement's canonical NTT, mult_mod, add_mod and sub_mod: every
product and every sum reduced, so nothing can wrap.  For a ciphertext (c0, c1) in NTT form at level l:
    a_i         = INTT_{q_i}(c1_i)
    D_{d,m}     = NTT_m(Conv_{S_d -> m}(a))                                  mod-up, once, every m in B
    prod^r_{m,k} = sum_d pi_{g_r}(D_{d,m}) K_r[d][k][slot(m)]  mod m
    hoisted:    out_r  = [sigma_{g_r}(c0), 0] + ModDown_P(prod^r)
    linear:     acc    = sum_{r keyed} w_{r,m} prod^r_{m,k}  mod m
                result = [sum_r w_r sigma_{g_r}(c0), sum_{r identity} w_r c1] + ModDown_P(acc)   (no ModDown term when
                         every element is an identity term)
ModDown_P is the rounded mod-down of hybrid_exact.key_switch_hybrid.
"""
from __future__ import annotations

import numpy as np

import galois_exact as gx
import hybrid_exact as hx
from util import uniform_below

U64 = np.uint64


def _basis(moduli, level, q_size, p_size):
    """the moduli of B = {q_0..q_{l-1}, p_0..p_{K-1}} and their key slots"""
    moduli = [int(q) for q in moduli]
    basis = moduli[:level] + moduli[q_size:q_size + p_size]
    slots = list(range(level)) + [q_size + j for j in range(p_size)]
    return basis, slots


def mod_up(port, c1, n, level, q_size, p_size, alpha, moduli):
    """D[d][b]: digit d of c1 converted into modulus b of B and transformed, canonical"""
    moduli = [int(q) for q in moduli]
    basis, _ = _basis(moduli, level, q_size, p_size)
    c1 = np.asarray(c1, dtype=U64)
    a = [port.ntt_inverse(c1[i * n:(i + 1) * n], n, moduli[i]) for i in range(level)]
    out = []
    for S in hx.digits(level, alpha):
        ext = hx.fast_base_convert(port, np.concatenate([a[i] for i in S]), n, [moduli[i] for i in S],
                                   basis).reshape(-1, n)
        out.append([port.ntt_forward(ext[b], n, m) for b, m in enumerate(basis)])
    return out


def products(port, D, n, g, keys, level, q_size, p_size, moduli):
    """prod[b, k] = sum_d pi_g(D[d][b]) keys[d][k][slot(b)] mod m_b"""
    basis, slots = _basis(moduli, level, q_size, p_size)
    kms = q_size + p_size
    p = gx.pi(n, g)
    prod = {}
    for b, m in enumerate(basis):
        for k in range(2):
            off = (k * kms + slots[b]) * n
            acc = np.zeros(n, dtype=U64)
            for d in range(len(D)):
                key = np.asarray(keys[d][off:off + n], dtype=U64) % U64(m)
                acc = port.add_mod(acc, port.mult_mod(np.ascontiguousarray(D[d][b][p]), key, m), m)
            prod[b, k] = acc
    return prod


def mod_down(port, out, prod, n, level, q_size, p_size, moduli):
    """out (2 x level x n) + ModDown_P(prod), rounded, as a new array"""
    moduli = [int(q) for q in moduli]
    special = moduli[q_size:q_size + p_size]
    P = 1
    for p in special:
        P *= p
    half = P // 2
    out = np.array(out, dtype=U64, copy=True)
    for k in range(2):
        x = np.concatenate([port.ntt_inverse(prod[level + j, k], n, p) for j, p in enumerate(special)])
        c = hx.fast_base_convert(port, x, n, special, moduli[:level], add=[half % p for p in special],
                                 sub=[half % q for q in moduli[:level]]).reshape(level, n)
        for i in range(level):
            q = moduli[i]
            d = port.sub_mod(prod[i, k], port.ntt_forward(c[i], n, q), q)
            d = port.mult_mod(d, np.full(n, pow(P % q, -1, q), dtype=U64), q)
            dst = slice(n * (level * k + i), n * (level * k + i + 1))
            out[dst] = port.add_mod(out[dst], d, q)
    return out


def hoisted_exact(port, ct, n, level, q_size, p_size, alpha, moduli, elts, keys):
    """one ciphertext (2 x level x n words) rotated by every element of `elts` with keys[r] (a list of hybrid key
    buffers); the rotations back to back"""
    ct = np.asarray(ct, dtype=U64)
    comp = level * n
    D = mod_up(port, ct[comp:2 * comp], n, level, q_size, p_size, alpha, moduli)
    out = []
    for g, key in zip(elts, keys):
        prod = products(port, D, n, g, key, level, q_size, p_size, moduli)
        start = np.concatenate([gx.sigma_ntt(ct[:comp], n, g), np.zeros(comp, dtype=U64)])
        out.append(mod_down(port, start, prod, n, level, q_size, p_size, moduli))
    return np.concatenate(out)


def linear_transform_exact(port, ct, n, level, q_size, p_size, alpha, moduli, elts, keys, diagonals):
    """one ciphertext: sum_r w_r (.) Rot_{g_r}(ct) under one mod-down.  keys[r] is None for an identity term (g = 1);
    diagonals: len(elts) x (level + p_size) x n words"""
    moduli = [int(q) for q in moduli]
    basis, _ = _basis(moduli, level, q_size, p_size)
    nb = len(basis)
    ct = np.asarray(ct, dtype=U64)
    w = np.asarray(diagonals, dtype=U64).reshape(len(elts), nb, n)
    comp = level * n
    c0, c1 = ct[:comp].reshape(level, n), ct[comp:2 * comp].reshape(level, n)
    start = np.zeros(2 * comp, dtype=U64)
    for r, g in enumerate(elts):
        s0 = gx.sigma_ntt(c0, n, g).reshape(level, n)
        for i in range(level):
            q = moduli[i]
            dst = slice(i * n, (i + 1) * n)
            start[dst] = port.add_mod(start[dst], port.mult_mod(w[r, i], s0[i], q), q)
            if keys[r] is None:
                dst = slice(comp + i * n, comp + (i + 1) * n)
                start[dst] = port.add_mod(start[dst], port.mult_mod(w[r, i], c1[i], q), q)
    keyed = [r for r in range(len(elts)) if keys[r] is not None]
    if not keyed:
        return start
    D = mod_up(port, ct[comp:2 * comp], n, level, q_size, p_size, alpha, moduli)
    acc = {(b, k): np.zeros(n, dtype=U64) for b in range(nb) for k in range(2)}
    for r in keyed:
        prod = products(port, D, n, elts[r], keys[r], level, q_size, p_size, moduli)
        for (b, k), v in prod.items():
            acc[b, k] = port.add_mod(acc[b, k], port.mult_mod(w[r, b], v, basis[b]), basis[b])
    return mod_down(port, start, acc, n, level, q_size, p_size, moduli)


def random_diagonals(basis, n, count, seed, fill=None):
    """count diagonals of len(basis) canonical limbs; fill="q-1": every word q - 1, fill="one": every word 1"""
    rows = []
    for r in range(count):
        for b, m in enumerate(int(q) for q in basis):
            if fill == "q-1":
                rows.append(np.full(n, m - 1, dtype=U64))
            elif fill == "one":
                rows.append(np.ones(n, dtype=U64))
            else:
                rows.append(uniform_below(seed * 7717 + 131 * r + b, n, m))
    return np.concatenate(rows)


def small_diagonals(port, basis, n, count, bound, seed):
    """count integer polynomials of coefficients in [-bound, bound] and their NTT forms under every modulus of B:
    (list of coefficient lists, count x len(basis) x n words)"""
    polys, rows = [], []
    for r in range(count):
        w = [int(v) - bound for v in uniform_below(seed * 613 + r, n, 2 * bound + 1)]
        polys.append(w)
        rows += [port.ntt_forward(np.array([c % int(m) for c in w], dtype=U64), n, int(m)) for m in basis]
    return polys, np.concatenate(rows)
