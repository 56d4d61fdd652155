"""The BGV calls exactly, for the tests: hexl_b200_bgv_mod_switch, hexl_b200_bgv_key_switch_hybrid,
hexl_b200_bgv_apply_galois_key_switch_hybrid_hoisted and hexl_b200_bgv_multiply_relinearize_hybrid, and BGV keys,
encryption and decryption.

Built from the hybrid switch's pieces (tests/hybrid_rotation_exact.py: the mod-up and the key products) with the C
restatement's canonical NTT, mult_mod, add_mod and sub_mod under the data and special moduli, and Python integers under
the plain modulus tau (any value in [2, 2^61)).  The only new piece is the t-corrected conversion of include/hexl_b200.h:
    y_t     = [x_t (P_T/t)^-1]_t
    X~_m    = [sum_t y_t [P_T/t]_m]_m                     every target m and m = tau
    k       = [-X~_tau P_T^-1]_tau
    delta_m = [X~_m + [P_T]_m k]_m
and the mod-down that subtracts it: out_i = (ext_i - NTT(delta_i)) P_T^-1 mod q_i.
"""
from __future__ import annotations

import numpy as np

import galois_exact as gx
import hybrid_exact as hx
import hybrid_rotation_exact as hr
import mul_relin_exact as mr
from util import uniform_below

U64 = np.uint64


def _prod(values):
    out = 1
    for v in values:
        out *= int(v)
    return out


def t_corrected_convert(port, x, n, from_moduli, to_moduli, tau):
    """delta of one polynomial: x holds len(from_moduli) canonical limbs of n words (coefficient form); returns
    len(to_moduli) limbs, canonical"""
    src = [int(q) for q in from_moduli]
    P = _prod(src)
    x = np.asarray(x, dtype=U64).reshape(len(src), n)
    y = [port.mult_mod(x[i], np.full(n, pow(P // q % q, -1, q), dtype=U64), q) for i, q in enumerate(src)]
    x_tau = sum(y[i].astype(object) * (P // q % tau) for i, q in enumerate(src)) % tau
    k = x_tau * ((-pow(P % tau, -1, tau)) % tau) % tau
    out = []
    for m in (int(m) for m in to_moduli):
        acc = np.zeros(n, dtype=U64)
        for i, q in enumerate(src):
            acc = port.add_mod(acc, port.mult_mod(y[i] % U64(m), np.full(n, P // q % m, dtype=U64), m), m)
        corr = port.mult_mod((k % m).astype(U64), np.full(n, P % m, dtype=U64), m)
        out.append(port.add_mod(acc, corr, m))
    return np.concatenate(out)


def mod_down(port, out, prod, n, level, p_size, basis, tau, kcc=2):
    """out (kcc x level x n) + ModDown^tau_T(prod) as a new array; T = the p_size limbs of `basis` after the first
    `level` (prod[b, k] over basis)"""
    basis = [int(m) for m in basis]
    special = basis[level:level + p_size]
    P = _prod(special)
    out = np.array(out, dtype=U64, copy=True)
    for k in range(kcc):
        x = np.concatenate([port.ntt_inverse(prod[level + j, k], n, p) for j, p in enumerate(special)])
        c = t_corrected_convert(port, x, n, special, basis[:level], tau).reshape(level, n)
        for i in range(level):
            q = basis[i]
            d = port.sub_mod(prod[i, k], port.ntt_forward(c[i], n, q), q)
            d = port.mult_mod(d, np.full(n, pow(P % q, -1, q), dtype=U64), q)
            dst = slice(n * (level * k + i), n * (level * k + i + 1))
            out[dst] = port.add_mod(out[dst], d, q)
    return out


def products(port, D, n, g, keys, level, q_size, p_size, moduli, kcc):
    """prod[b, k] = sum_d pi_g(D[d][b]) keys[d][k][slot(b)] mod m_b, k < kcc"""
    basis, slots = hr._basis(moduli, level, q_size, p_size)
    kms = q_size + p_size
    p = gx.pi(n, g)
    prod = {}
    for b, m in enumerate(basis):
        for k in range(kcc):
            off = (k * kms + slots[b]) * n
            acc = np.zeros(n, dtype=U64)
            for d in range(len(D)):
                key = np.asarray(keys[d][off:off + n], dtype=U64) % U64(m)
                acc = port.add_mod(acc, port.mult_mod(np.ascontiguousarray(D[d][b][p]), key, m), m)
            prod[b, k] = acc
    return prod


def key_switch(port, result, target, n, level, q_size, p_size, alpha, kcc, moduli, keys, tau):
    """hexl_b200_bgv_key_switch_hybrid of one target (level x n, NTT form): the updated result as a new array"""
    basis, _ = hr._basis(moduli, level, q_size, p_size)
    D = hr.mod_up(port, target, n, level, q_size, p_size, alpha, moduli)
    prod = products(port, D, n, 1, keys, level, q_size, p_size, moduli, kcc)
    return mod_down(port, result, prod, n, level, p_size, basis, tau, kcc)


def hoisted(port, ct, n, level, q_size, p_size, alpha, moduli, elts, keys, tau):
    """hexl_b200_bgv_apply_galois_key_switch_hybrid_hoisted of one ciphertext: the rotations back to back"""
    basis, _ = hr._basis(moduli, level, q_size, p_size)
    ct = np.asarray(ct, dtype=U64)
    comp = level * n
    D = hr.mod_up(port, ct[comp:2 * comp], n, level, q_size, p_size, alpha, moduli)
    out = []
    for g, key in zip(elts, keys):
        prod = products(port, D, n, g, key, level, q_size, p_size, moduli, 2)
        start = np.concatenate([gx.sigma_ntt(ct[:comp], n, g), np.zeros(comp, dtype=U64)])
        out.append(mod_down(port, start, prod, n, level, p_size, basis, tau))
    return np.concatenate(out)


def multiply_relinearize(port, ct1, ct2, n, level, q_size, p_size, alpha, moduli, keys, tau, mod_switch):
    """hexl_b200_bgv_multiply_relinearize_hybrid of one pair: 2 x (level - mod_switch) x n words"""
    moduli = [int(q) for q in moduli]
    basis, _ = hr._basis(moduli, level, q_size, p_size)
    d0, d1, t = mr.tensor(port, ct1, ct2, n, level, moduli)
    D = hr.mod_up(port, t, n, level, q_size, p_size, alpha, moduli)
    ext = products(port, D, n, 1, keys, level, q_size, p_size, moduli, 2)
    P = _prod(moduli[q_size:q_size + p_size])
    for i in range(level):
        q = moduli[i]
        for k, d in enumerate((d0, d1)):
            ext[i, k] = port.add_mod(ext[i, k], port.mult_mod(d[i * n:(i + 1) * n], np.full(n, P % q, dtype=U64), q),
                                     q)
    out_level = level - int(mod_switch)
    return mod_down(port, np.zeros(2 * out_level * n, dtype=U64), ext, n, out_level, p_size + int(mod_switch), basis,
                    tau)


def mod_switch(port, operand, n, moduli, count, ntt_form, tau):
    """hexl_b200_bgv_mod_switch: `count` polynomials of len(moduli) limbs; limb L of the result keeps the operand's"""
    moduli = [int(q) for q in moduli]
    rns = len(moduli)
    L, q_last = rns - 1, moduli[-1]
    x = np.asarray(operand, dtype=U64).reshape(count, rns, n)
    out = x.copy()
    for p in range(count):
        last = port.ntt_inverse(x[p, L], n, q_last) if ntt_form else x[p, L]
        delta = t_corrected_convert(port, last, n, [q_last], moduli[:L], tau).reshape(L, n)
        for i in range(L):
            q = moduli[i]
            d = port.ntt_forward(delta[i], n, q) if ntt_form else delta[i]
            d = port.sub_mod(x[p, i], d, q)
            out[p, i] = port.mult_mod(d, np.full(n, pow(q_last % q, -1, q), dtype=U64), q)
    return out.reshape(-1)


def seal_mod_switch(operand, n, moduli, count, tau):
    """SEAL's mod_t_and_divide_q_last_inplace written limb by limb in Python integers (coefficient form):
    k = [-x_L q_L^-1]_tau, delta = x_L + q_L k, out_i = (x_i - delta) q_L^-1 mod q_i"""
    moduli = [int(q) for q in moduli]
    rns = len(moduli)
    q_last = moduli[-1]
    x = np.asarray(operand, dtype=U64).reshape(count, rns, n)
    out = x.copy()
    neg_inv = (-pow(q_last % tau, -1, tau)) % tau
    xl = x[:, -1].astype(object)
    delta = xl + q_last * (xl * neg_inv % tau)
    for i, q in enumerate(moduli[:-1]):
        out[:, i] = ((x[:, i].astype(object) - delta) * pow(q_last, -1, q) % q).astype(U64)
    return out.reshape(-1)


# ------------------------------------------------------------------------------------------------ keys, encryption
def _ntt(port, coeffs, n, q):
    return port.ntt_forward(np.array([int(c) % q for c in coeffs], dtype=U64), n, q)


def bgv_keys(port, s, s_new, n, moduli, q_size, alpha, tau, error_seed, bound_e):
    """Hybrid keys that switch from s_new to s for BGV, in the layout hexl_b200_bgv_key_switch_hybrid takes: key d is
    (-a_d s + tau e_d + g_d s_new, a_d) under every key modulus, NTT form, with the gadget
    g_d = P (Q/Q_d) [(Q/Q_d)^-1]_{Q_d} of hybrid_exact.hybrid_keys"""
    moduli = [int(q) for q in moduli]
    Q, P = _prod(moduli[:q_size]), _prod(moduli[q_size:])
    s_ntt = [_ntt(port, s, n, q) for q in moduli]
    new_ntt = [_ntt(port, s_new, n, q) for q in moduli]
    keys = []
    for d, S in enumerate(hx.digits(q_size, alpha)):
        Qd = _prod(moduli[i] for i in S)
        g = P * (Q // Qd) * pow(Q // Qd % Qd, -1, Qd)
        e = [tau * (int(v) - bound_e) for v in uniform_below(error_seed + d, n, 2 * bound_e + 1)]
        c0, c1 = [], []
        for i, q in enumerate(moduli):
            a = uniform_below(error_seed * 31 + 1000 * d + i, n, q)
            b = port.sub_mod(_ntt(port, e, n, q), port.mult_mod(a, s_ntt[i], q), q)
            b = port.add_mod(b, port.mult_mod(new_ntt[i], np.full(n, g % q, dtype=U64), q), q)
            c0.append(b)
            c1.append(a)
        keys.append(np.concatenate(c0 + c1))
    return keys


def secret(n, seed):
    """a ternary secret, integer coefficients"""
    return [int(v) - 1 for v in uniform_below(seed, n, 3)]


def encrypt(port, m, s, n, moduli, tau, seed, bound_e=8):
    """(-a s + tau e + m, a) in NTT form under every modulus of `moduli`: 2 x len(moduli) x n words"""
    e = [tau * (int(v) - bound_e) + int(mv) for v, mv in zip(uniform_below(seed, n, 2 * bound_e + 1), m)]
    c0, c1 = [], []
    for i, q in enumerate(int(q) for q in moduli):
        a = uniform_below(seed * 53 + i, n, q)
        c0.append(port.sub_mod(_ntt(port, e, n, q), port.mult_mod(a, _ntt(port, s, n, q), q), q))
        c1.append(a)
    return np.concatenate(c0 + c1)


def decrypt(port, ct, powers, n, moduli, tau):
    """[sum_j c_j s^j]_Q centred, mod tau; ct holds len(powers) components of len(moduli) limbs in NTT form, powers[j]
    the integer polynomial s^j (powers[0] unused: 1)"""
    moduli = [int(q) for q in moduli]
    level = len(moduli)
    Q = _prod(moduli)
    c = np.asarray(ct, dtype=U64).reshape(len(powers), level, n)
    limbs = []
    for i, q in enumerate(moduli):
        v = c[0, i]
        for j in range(1, len(powers)):
            v = port.add_mod(v, port.mult_mod(c[j, i], _ntt(port, powers[j], n, q), q), q)
        limbs.append(port.ntt_inverse(v, n, q))
    basis = [(Q // q) * pow(Q // q % q, -1, q) for q in moduli]
    out = []
    for col in range(n):
        X = sum(int(limbs[i][col]) * basis[i] for i in range(level)) % Q
        out.append((X - Q if X > Q // 2 else X) % tau)
    return out
