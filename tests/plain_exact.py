"""The plaintext calls exactly, for the tests: hexl_b200_plain_lift, hexl_b200_bfv_add_plain and
hexl_b200_bfv_multiply_plain, and BFV encryption and decryption in coefficient form.

Python integers under t and the q_i (any values below 2^61), and the C restatement's canonical NTT and mult_mod for the
products.  The fix of add_plain is computed the way the kernel computes it (a Shoup quotient corrected by one), so the
CPU tests can check that computation against the true quotient.
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


def _ints(a):
    return np.asarray(a, dtype=U64).astype(object)


def padded(plain, pcc, n):
    """the n coefficients of a plaintext of pcc words, as Python integers"""
    out = np.zeros(n, dtype=object)
    out[:pcc] = _ints(plain)[:pcc]
    return out


def lift(plain, pcc, n, moduli, t, correction_factor=1):
    """one plaintext into len(moduli) limbs of n words, coefficient form: m' = [m c]_t, centred into every q_i"""
    m = padded(plain, pcc, n) * int(correction_factor) % t
    neg = m >= (t + 1) // 2
    return np.concatenate([np.where(neg, (m - t) % int(q), m % int(q)).astype(U64) for q in moduli])


def plain_lift(port, plain, pcc, n, moduli, t, correction_factor=1, ntt_form=False, count=1):
    """hexl_b200_plain_lift of `count` plaintexts back to back"""
    out = []
    for p in range(count):
        x = lift(np.asarray(plain, dtype=U64)[p * pcc:(p + 1) * pcc], pcc, n, moduli, t, correction_factor)
        if ntt_form:
            x = np.concatenate([port.ntt_forward(x[i * n:(i + 1) * n], n, int(q)) for i, q in enumerate(moduli)])
        out.append(x)
    return np.concatenate(out)


def fix_quotient(m, r, t):
    """floor((m r + h) / t), h = floor((t + 1) / 2), as bfv_add_plain_kernel computes it: est = hi64(m floor(r 2^64 /
    t)) is floor(m r / t) or one less, rem = m r - est t < 2t, one correction, then [rem + h >= t]"""
    r_shoup = (r << 64) // t
    a = (m * r_shoup) >> 64
    rem = m * r - a * t
    assert 0 <= rem < 2 * t
    if rem >= t:
        rem -= t
        a += 1
    return a + (1 if rem + (t + 1) // 2 >= t else 0)


def add_plain(ct, plain, pcc, n, moduli, t, subtract=False):
    """hexl_b200_bfv_add_plain of one ciphertext (2 x len(moduli) x n words, coefficient form): SEAL's
    multiply_add_plain_with_scaling_variant, c0_i += [m floor(Q/t) + fix]_{q_i} (or -=)"""
    Q = _prod(moduli)
    r = Q % t
    m = padded(plain, pcc, n)
    fix = np.array([fix_quotient(int(v), r, t) for v in m], dtype=object)
    out = np.array(ct, dtype=U64, copy=True)
    for i, q in enumerate(int(q) for q in moduli):
        s = (m * (Q // t % q) + fix) % q
        c0 = _ints(out[i * n:(i + 1) * n])
        out[i * n:(i + 1) * n] = ((c0 - s if subtract else c0 + s) % q).astype(U64)
    return out


def multiply_plain(port, ct, plain, pcc, n, moduli, t, plain_ntt_form=False):
    """hexl_b200_bfv_multiply_plain of one ciphertext: INTT(NTT(ct_k,i) . NTT(lift(m)_i)) per component and limb"""
    l = len(moduli)
    fp = np.asarray(plain, dtype=U64) if plain_ntt_form else plain_lift(port, plain, pcc, n, moduli, t, ntt_form=True)
    ct = np.asarray(ct, dtype=U64)
    out = []
    for k in range(2):
        for i, q in enumerate(int(q) for q in moduli):
            x = port.ntt_forward(ct[(k * l + i) * n:(k * l + i + 1) * n], n, q)
            out.append(port.ntt_inverse(port.mult_mod(x, fp[i * n:(i + 1) * n], q), n, q))
    return np.concatenate(out)


# ------------------------------------------------------------------------------------------------ BFV encryption
def _poly_mul_mod(port, x, s, q, n):
    return port.ntt_inverse(port.mult_mod(port.ntt_forward(x, n, q), port.ntt_forward(s, n, q), q), n, q)


def encrypt(port, m, s, moduli, n, t, seed, bound_e=8):
    """(c0, c1) = (-a s + e + floor(Q/t) m, a) in coefficient form, e in [-bound_e, bound_e]"""
    delta = _prod(moduli) // t
    e = [int(v) - bound_e for v in uniform_below(seed, n, 2 * bound_e + 1)]
    c0, c1 = [], []
    for i, q in enumerate(int(q) for q in moduli):
        a = uniform_below(seed * 31 + i, n, q)
        s_q = np.array([v % q for v in s], dtype=U64)
        v = port.sub_mod(np.array([(x + delta * int(mm)) % q for x, mm in zip(e, m)], dtype=U64),
                         _poly_mul_mod(port, a, s_q, q, n), q)
        c0.append(v)
        c1.append(a)
    return np.concatenate(c0 + c1)


def decrypt(port, ct, s, moduli, n, t):
    """round(t [c0 + c1 s]_Q / Q) mod t"""
    moduli = [int(q) for q in moduli]
    l = len(moduli)
    c = np.asarray(ct, dtype=U64).reshape(2, l, n)
    Q = _prod(moduli)
    basis = [(Q // q) * pow(Q // q % q, -1, q) for q in moduli]
    limbs = [port.add_mod(c[0, i], _poly_mul_mod(port, c[1, i], np.array([v % q for v in s], dtype=U64), q, n), q)
             for i, q in enumerate(moduli)]
    out = []
    for col in range(n):
        X = sum(int(limbs[i][col]) * basis[i] for i in range(l)) % Q
        out.append(((t * X + Q // 2) // Q) % t)
    return out
