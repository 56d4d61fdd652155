"""Hybrid key switching (hexl_b200_key_switch_hybrid) and fast base conversion (hexl_b200_fast_base_convert) exactly,
for the tests.

The definitions of include/hexl_b200.h restated with the C restatement's canonical NTT, mult_mod, add_mod and sub_mod,
as tests/ks_exact.py does: every product and every sum reduced, so nothing can wrap, and the GPU's unreduced 128-bit
sums must give the same canonical words.

    fast_base_convert   result_m = [sum_i [(x_i + add_i) (Q/q_i)^-1]_{q_i} [Q/q_i]_m - sub_m]_m
    key_switch_hybrid   mod-up of every digit by fast base conversion, inner product with the keys, mod-down by P with
                        rounding (add = sub = floor(P/2))
    hybrid_keys         keys that switch a ciphertext from s_new to s, gadget P (Q/Q_d) [(Q/Q_d)^-1]_{Q_d}
"""
from __future__ import annotations

import numpy as np

from util import uniform_below

U64 = np.uint64


def _prod(values):
    out = 1
    for v in values:
        out *= int(v)
    return out


def fast_base_convert(port, x, n, from_moduli, to_moduli, add=None, sub=None):
    """One polynomial: x holds len(from_moduli) limbs of n canonical words; returns len(to_moduli) limbs.  add[i] is
    added to source limb i, sub[e] subtracted from target limb e (the mod-down's rounding; default none)."""
    src = [int(q) for q in from_moduli]
    x = np.asarray(x, dtype=U64).reshape(len(src), n)
    Q = _prod(src)
    y = []
    for i, q in enumerate(src):
        v = x[i] if add is None else port.add_mod(x[i], int(add[i]) % q, q)
        y.append(port.mult_mod(v, np.full(n, pow(Q // q % q, -1, q), dtype=U64), q))
    out = []
    for e, t in enumerate(int(t) for t in to_moduli):
        acc = np.zeros(n, dtype=U64)
        for i, q in enumerate(src):
            acc = port.add_mod(acc, port.mult_mod(y[i] % U64(t), np.full(n, Q // q % t, dtype=U64), t), t)
        if sub is not None:
            acc = port.sub_mod(acc, int(sub[e]) % t, t)
        out.append(acc)
    return np.concatenate(out)


def fast_base_convert_int(x, n, from_moduli, to_moduli):
    """The definition of hexl_b200_fast_base_convert in plain Python integers, for its whole domain (pairwise-coprime
    sources and any targets in (1, 2^61), neither needing to be prime, odd or NTT-friendly):
        result_t = (sum_i [x_i (Q/q_i)^-1]_{q_i} (Q/q_i)) mod t
    One polynomial of len(from_moduli) limbs of n words; returns len(to_moduli) limbs."""
    src = [int(q) for q in from_moduli]
    Q = _prod(src)
    x = np.asarray(x, dtype=U64).reshape(len(src), n).astype(object)
    total = np.zeros(n, dtype=object)
    for i, q in enumerate(src):
        total = total + (x[i] * pow(Q // q, -1, q)) % q * (Q // q)
    return np.concatenate([(total % int(t)).astype(U64) for t in to_moduli])


def digits(level, alpha):
    """S_d = [d alpha, min((d + 1) alpha, level)) for d < ceil(level / alpha)"""
    return [list(range(lo, min(lo + alpha, level))) for lo in range(0, level, alpha)]


def key_switch_hybrid(port, result, target, n, level, q_size, p_size, alpha, kcc, moduli, keys):
    """The hybrid switch of one ciphertext with the argument layout of hexl_b200_key_switch_hybrid; returns the
    updated result (kcc x level x n) as a new array.  keys[d]: kcc x (q_size + p_size) x n words."""
    moduli = [int(q) for q in moduli]
    kms = q_size + p_size
    special = moduli[q_size:kms]
    basis = moduli[:level] + special
    slots = list(range(level)) + [q_size + j for j in range(p_size)]
    target = np.asarray(target, dtype=U64)
    a = [port.ntt_inverse(target[i * n:(i + 1) * n], n, moduli[i]) for i in range(level)]
    groups = digits(level, alpha)
    # mod-up: D_{d,m} = NTT_m(conv_d(a)_m) for every m in B
    ext = [fast_base_convert(port, np.concatenate([a[i] for i in S]), n, [moduli[i] for i in S], basis).reshape(-1, n)
           for S in groups]
    prod = {}
    for b, m in enumerate(basis):
        ops = [port.ntt_forward(ext[d][b], n, m) for d in range(len(groups))]
        for k in range(kcc):
            off = (k * kms + slots[b]) * n
            acc = np.zeros(n, dtype=U64)
            for d in range(len(groups)):
                key = np.asarray(keys[d][off:off + n], dtype=U64) % U64(m)
                acc = port.add_mod(acc, port.mult_mod(ops[d], key, m), m)
            prod[b, k] = acc
    # mod-down by P with rounding
    P = _prod(special)
    half = P // 2
    out = np.array(result, dtype=U64, copy=True)
    for k in range(kcc):
        x = np.concatenate([port.ntt_inverse(prod[level + j, k], n, p) for j, p in enumerate(special)])
        c = fast_base_convert(port, x, n, special, moduli[:level], add=[half % p for p in special],
                              sub=[half % q for q in moduli[:level]]).reshape(level, n)
        for i in range(level):
            q = moduli[i]
            d = port.sub_mod(prod[i, k], port.ntt_forward(c[i], n, q), q)
            d = port.mult_mod(d, np.full(n, pow(P % q, -1, q), dtype=U64), q)
            dst = slice(n * (level * k + i), n * (level * k + i + 1))
            out[dst] = port.add_mod(out[dst], d, q)
    return out


def hybrid_keys(port, s, s_new, n, moduli, q_size, alpha, error_seed, bound_e):
    """Keys that switch from s_new to s, in the layout hexl_b200_key_switch_hybrid takes.

    s, s_new: integer polynomials (Python ints, n coefficients).  moduli: q_size data moduli, then the special primes.
    Key d (digit d < ceil(q_size / alpha)), in NTT form under every key modulus m:
        component 1: a_d, uniform;
        component 0: -a_d s + e_d + g_d s_new,  g_d = P (Q/Q_d) [(Q/Q_d)^-1]_{Q_d} mod m,
    Q the product of the data moduli, Q_d of digit d's, P of the special primes, e_d of coefficients in
    [-bound_e, bound_e].  g_d is P mod the moduli of digit d and 0 mod every other modulus, at every level."""
    moduli = [int(q) for q in moduli]
    Q, P = _prod(moduli[:q_size]), _prod(moduli[q_size:])

    def ntt(coeffs, q):
        return port.ntt_forward(np.array([c % q for c in coeffs], dtype=U64), n, q)

    s_ntt = [ntt(s, q) for q in moduli]
    new_ntt = [ntt(s_new, q) for q in moduli]
    keys = []
    for d, S in enumerate(digits(q_size, alpha)):
        Qd = _prod(moduli[i] for i in S)
        g = P * (Q // Qd) * pow(Q // Qd % Qd, -1, Qd)
        e = [int(v) - bound_e for v in uniform_below(error_seed + d, n, 2 * bound_e + 1)]
        c0, c1 = [], []
        for i, q in enumerate(moduli):
            a = uniform_below(error_seed * 31 + 1000 * d + i, n, q)
            b = port.sub_mod(ntt(e, q), port.mult_mod(a, s_ntt[i], q), q)
            b = port.add_mod(b, port.mult_mod(new_ntt[i], np.full(n, g % q, dtype=U64), q), q)
            c0.append(b)
            c1.append(a)
        keys.append(np.concatenate(c0 + c1))
    return keys


def random_keys(moduli, n, q_size, alpha, kcc, seed, fill=None):
    """ceil(q_size / alpha) key buffers of kcc x len(moduli) x n words, limb i below moduli[i]; fill="q-1": every word
    q - 1"""
    out = []
    for d in range(len(digits(q_size, alpha))):
        rows = []
        for k in range(kcc):
            for i, q in enumerate(moduli):
                rows.append(np.full(n, int(q) - 1, dtype=U64) if fill == "q-1"
                            else uniform_below(seed + 100000 * d + 1000 * k + i, n, int(q)))
        out.append(np.concatenate(rows))
    return out


def noise(port, result, target, s, s_new, n, level, moduli):
    """max |u0 + u1 s - t s_new| over the coefficients, centred mod Q_level: how far the switched pair (u0, u1) in
    result (kcc = 2, NTT form) is from decrypting to target x s_new"""
    moduli = [int(q) for q in moduli[:level]]
    Q = _prod(moduli)
    res = np.asarray(result, dtype=U64).reshape(2, level, n)
    t = np.asarray(target, dtype=U64).reshape(level, n)
    limbs = []
    for i, q in enumerate(moduli):
        s_i = port.ntt_forward(np.array([c % q for c in s], dtype=U64), n, q)
        new_i = port.ntt_forward(np.array([c % q for c in s_new], dtype=U64), n, q)
        v = port.add_mod(res[0, i], port.mult_mod(res[1, i], s_i, q), q)
        v = port.sub_mod(v, port.mult_mod(t[i], new_i, q), q)
        limbs.append(port.ntt_inverse(v, n, q))
    basis = [(Q // q) * pow(Q // q % q, -1, q) for q in moduli]
    worst = 0
    for col in range(n):
        X = sum(int(limbs[i][col]) * basis[i] for i in range(level)) % Q
        worst = max(worst, abs(X - Q if X > Q // 2 else X))
    return worst
