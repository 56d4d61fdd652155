"""BFV multiplication by BEHZ (hexl_b200_bfv_multiply) and its relinearized form
(hexl_b200_bfv_multiply_relinearize_hybrid) exactly, for the tests.

The definitions of include/hexl_b200.h restated with the C restatement's canonical NTT, mult_mod, add_mod and sub_mod,
as tests/mul_relin_exact.py does, and the fast base conversion of tests/hybrid_exact.py.  Every value is canonical, so
the GPU's lazy and 128-bit intermediates must give the same words.  For a ciphertext pair in coefficient form:
    lift      x'_m = [(FBC([x m~]; Q -> m) + [Q]_m r_c) m~^-1]_m over Bsk = B u {m_sk}, x'_{q_i} = x_i
    tensor    D0 = a0 b0, D1 = a0 b1 + a1 b0, D2 = a1 b1 per modulus of Q u Bsk (NTT, dyadic, inverse NTT)
    scale     w = fast floor of t D / Q over Bsk, then Shenoy-Kumaresan from B u {m_sk} back to Q
    relin     (d0, d1) + KS(d2) with the hybrid switch taken in coefficient form
"""
from __future__ import annotations

import numpy as np

import hybrid_exact as hx
import hybrid_rotation_exact as hr

U64 = np.uint64
MT = 1 << 32  # m~, SEAL's fixed Montgomery modulus of the lift


def _prod(values):
    out = 1
    for v in values:
        out *= int(v)
    return out


def _full(n, v):
    return np.full(n, int(v), dtype=U64)


def bound_holds(n, t, Q, B, m_sk):
    """n t Q (m~ + 2l)^2 + 2 (l + 1) m~^2 <= B (m_sk - 1 - 2k) m~^2, in integers"""
    l, k = len(Q), len(B)
    lhs = n * t * _prod(Q) * (MT + 2 * l) ** 2 + 2 * (l + 1) * MT * MT
    return m_sk - 1 - 2 * k > 0 and lhs <= _prod(B) * (m_sk - 1 - 2 * k) * MT * MT


def largest_plain_modulus(n, Q, B, m_sk):
    """the largest t the bound accepts for these bases (may be below 2)"""
    l, k = len(Q), len(B)
    room = _prod(B) * (m_sk - 1 - 2 * k) * MT * MT - 2 * (l + 1) * MT * MT
    return room // (n * _prod(Q) * (MT + 2 * l) ** 2)


def seal_base_b_size(Q, t):
    """SEAL's rule: |B| = l, or l + 1 when 32 + bits(t) + bits(Q) >= 61 (l + 1)"""
    l = len(Q)
    return l + 1 if 32 + int(t).bit_length() + _prod(Q).bit_length() >= 61 * (l + 1) else l


def seal_bases(port, n, Q, t):
    """(B, m_sk) as SEAL picks them: 61-bit primes = 1 mod 2n (generate_primes(., 60, .) draws from [2^60, 2^61)),
    distinct from Q"""
    k = seal_base_b_size(Q, t)
    primes = [int(p) for p in port.generate_primes(k + 1 + len(Q), 60, True, n) if int(p) not in Q][:k + 1]
    return primes[:k], primes[k]


def lift(port, x, n, Q, B, m_sk):
    """one polynomial of len(Q) limbs (coefficient form) -> len(Q) + len(B) + 1 limbs over Q u Bsk"""
    Q = [int(q) for q in Q]
    bsk = [int(b) for b in B] + [int(m_sk)]
    x = np.asarray(x, dtype=U64).reshape(len(Q), n)
    y = np.concatenate([port.mult_mod(x[i], _full(n, MT % q), q) for i, q in enumerate(Q)])
    z = hx.fast_base_convert(port, y, n, Q, bsk).reshape(len(bsk), n)
    Qp = _prod(Q)
    # z_m~ = FBC(y; Q -> 2^32): the same staged products, summed modulo 2^32
    zt = np.zeros(n, dtype=U64)
    for i, q in enumerate(Q):
        v = port.mult_mod(y[i * n:(i + 1) * n], _full(n, pow(Qp // q % q, -1, q)), q)
        zt = (zt + (v & U64(MT - 1)) * U64(Qp // q % MT)) & U64(MT - 1)
    r = ((U64(MT) - zt) * U64(pow(Qp, -1, MT))) & U64(MT - 1)  # [-z Q^-1]_{m~}
    out = [x[i] for i in range(len(Q))]
    for e, m in enumerate(bsk):
        rc = port.sub_mod(r % U64(m), np.where(r >= U64(MT // 2), U64(MT % m), U64(0)), m)  # r_c mod m
        s = port.add_mod(z[e], port.mult_mod(_full(n, Qp % m), rc, m), m)
        out.append(port.mult_mod(s, _full(n, pow(MT, -1, m)), m))
    return np.concatenate(out)


def tensor(port, a, b, n, mods):
    """(D0, D1, D2) of the lifted pairs a = (a0, a1), b = (b0, b1), each len(mods) limbs: per modulus forward NTT,
    dyadic products, inverse NTT"""
    M = len(mods)
    a = np.asarray(a, dtype=U64).reshape(2, M, n)
    b = np.asarray(b, dtype=U64).reshape(2, M, n)
    D = np.zeros((3, M, n), dtype=U64)
    for j, m in enumerate(int(q) for q in mods):
        fa = [port.ntt_forward(a[c, j], n, m) for c in range(2)]
        fb = [port.ntt_forward(b[c, j], n, m) for c in range(2)]
        prods = [port.mult_mod(fa[0], fb[0], m),
                 port.add_mod(port.mult_mod(fa[0], fb[1], m), port.mult_mod(fa[1], fb[0], m), m),
                 port.mult_mod(fa[1], fb[1], m)]
        for c in range(3):
            D[c, j] = port.ntt_inverse(prods[c], n, m)
    return D


def scale(port, D, n, Q, B, m_sk, t):
    """one tensor polynomial over Q u Bsk -> len(Q) limbs: the fast floor into Bsk, Shenoy-Kumaresan back to Q"""
    Q = [int(q) for q in Q]
    B = [int(b) for b in B]
    m_sk = int(m_sk)
    bsk = B + [m_sk]
    l, k = len(Q), len(B)
    D = np.asarray(D, dtype=U64).reshape(l + k + 1, n)
    Qp, Bp = _prod(Q), _prod(B)
    u = np.concatenate([port.mult_mod(D[i], _full(n, t % q), q) for i, q in enumerate(Q)])
    f = hx.fast_base_convert(port, u, n, Q, bsk).reshape(k + 1, n)
    w = []
    for e, m in enumerate(bsk):
        tD = port.mult_mod(D[l + e], _full(n, t % m), m)
        w.append(port.mult_mod(port.sub_mod(tD, f[e], m), _full(n, pow(Qp, -1, m)), m))
    c = hx.fast_base_convert(port, np.concatenate(w[:k]), n, B, Q + [m_sk]).reshape(l + 1, n)
    alpha = port.mult_mod(port.sub_mod(c[l], w[k], m_sk), _full(n, pow(Bp, -1, m_sk)), m_sk)
    neg = alpha > U64(m_sk // 2)
    out = []
    for i, q in enumerate(Q):
        up = port.add_mod(c[i], port.mult_mod(_full(n, Bp % q), (U64(m_sk) - alpha) % U64(q), q), q)
        down = port.sub_mod(c[i], port.mult_mod(_full(n, Bp % q), alpha % U64(q), q), q)
        out.append(np.where(neg, up, down))
    return np.concatenate(out)


def bfv_multiply(port, ct1, ct2, n, Q, B, m_sk, t):
    """one pair (2 x l x n words each, coefficient form) with the argument layout of hexl_b200_bfv_multiply; returns
    (d0, d1, d2), 3 x l x n words"""
    Q = [int(q) for q in Q]
    l = len(Q)
    mods = Q + [int(b) for b in B] + [int(m_sk)]
    c1 = np.asarray(ct1, dtype=U64).reshape(2, l * n)
    c2 = np.asarray(ct2, dtype=U64).reshape(2, l * n)
    a = np.concatenate([lift(port, c1[c], n, Q, B, m_sk) for c in range(2)])
    b = np.concatenate([lift(port, c2[c], n, Q, B, m_sk) for c in range(2)])
    D = tensor(port, a, b, n, mods)
    return np.concatenate([scale(port, D[c], n, Q, B, m_sk, t) for c in range(3)])


def _ntt_limbs(port, x, n, mods, forward):
    x = np.asarray(x, dtype=U64).reshape(-1, len(mods), n)
    f = port.ntt_forward if forward else port.ntt_inverse
    return np.concatenate([f(x[c, i], n, int(q)) for c in range(x.shape[0]) for i, q in enumerate(mods)])


def relinearize_chain(port, d, n, level, q_size, p_size, alpha, moduli, keys):
    """the anchor: NTT of d2, hexl_b200_key_switch_hybrid into zeros, inverse NTT, plus (d0, d1)"""
    mods = [int(q) for q in moduli[:level]]
    d = np.asarray(d, dtype=U64).reshape(3, level * n)
    t = _ntt_limbs(port, d[2], n, mods, True)
    ks = hx.key_switch_hybrid(port, np.zeros(2 * level * n, dtype=U64), t, n, level, q_size, p_size, alpha, 2,
                              moduli, keys)
    ks = _ntt_limbs(port, ks, n, mods, False).reshape(2, level, n)
    out = np.zeros((2, level, n), dtype=U64)
    for k in range(2):
        for i, q in enumerate(mods):
            out[k, i] = port.add_mod(d[k, i * n:(i + 1) * n], ks[k, i], q)
    return out.reshape(-1)


def relinearize(port, d, n, level, q_size, p_size, alpha, moduli, keys):
    """(d0, d1) + KS(d2) in coefficient form as the call computes it: the mod-up reads d2's limbs, the mod-down brings
    the products' data limbs back to coefficients and adds (INTT(prod) - c) P^-1"""
    moduli = [int(q) for q in moduli]
    basis, _ = hr._basis(moduli, level, q_size, p_size)
    d = np.asarray(d, dtype=U64).reshape(3, level, n)
    D = []
    for S in hx.digits(level, alpha):
        ext = hx.fast_base_convert(port, np.concatenate([d[2, i] for i in S]), n, [moduli[i] for i in S],
                                   basis).reshape(-1, n)
        D.append([port.ntt_forward(ext[b], n, m) for b, m in enumerate(basis)])
    prod = hr.products(port, D, n, 1, keys, level, q_size, p_size, moduli)
    special = moduli[q_size:q_size + p_size]
    P = _prod(special)
    half = P // 2
    out = np.zeros((2, level, n), dtype=U64)
    for k in range(2):
        x = np.concatenate([port.ntt_inverse(prod[level + j, k], n, p) for j, p in enumerate(special)])
        c = hx.fast_base_convert(port, x, n, special, moduli[:level], add=[half % p for p in special],
                                 sub=[half % q for q in moduli[:level]]).reshape(level, n)
        for i in range(level):
            q = moduli[i]
            v = port.sub_mod(port.ntt_inverse(prod[i, k], n, q), c[i], q)
            v = port.mult_mod(v, _full(n, pow(P % q, -1, q)), q)
            out[k, i] = port.add_mod(d[k, i], v, q)
    return out.reshape(-1)


def bfv_multiply_relinearize(port, ct1, ct2, n, level, q_size, p_size, alpha, moduli, B, m_sk, t, keys):
    """one pair with the argument layout of hexl_b200_bfv_multiply_relinearize_hybrid; 2 x level x n words"""
    d = bfv_multiply(port, ct1, ct2, n, [int(q) for q in moduli[:level]], B, m_sk, t)
    return relinearize(port, d, n, level, q_size, p_size, alpha, moduli, keys)
