"""The model of BFV multiplication by BEHZ (tests/bfv_exact.py) against big-integer statements of its steps, against the
chain of existing calls, and against decryption; and the compiler's resource report of its two kernels.  CPU only.

(a) the lift x' is x mod Q with -Q/2 <= x' < lambda Q, lambda = 1/2 + l/m~, and every output coefficient is
    floor(t D / Q) - v mod Q with 0 <= v < l, D the exact integer tensor of the lifts; at bases the bound only just
    accepts and with every input word q - 1;
(b) the bound holds for SEAL's choice of B and m_sk, and its largest plain modulus is exact;
(c) the relinearized model is the chain: forward NTT of d2, the hybrid key switch, inverse NTT, plus (d0, d1);
(d) BFV ciphertexts of m1 and m2 under a ternary secret decrypt to m1 m2 in R_t, the product under (1, s, s^2) and the
    relinearized one under (1, s); relinearization keys for another secret do not."""
import numpy as np
import pytest

import bfv_exact as bx
import hybrid_exact as hx
from mul_relin_exact import negacyclic_product
from test_kernel_resources import kernel_resources
from util import uniform_below

U64 = np.uint64
T30 = 1073741789  # a 30-bit prime


def _crt(limbs, mods):
    """the integer in [0, prod mods) of each coefficient, limbs: len(mods) x n"""
    M = bx._prod(mods)
    basis = [(M // m) * pow(M // m % m, -1, m) for m in mods]
    n = len(limbs[0])
    return [sum(int(limbs[i][c]) * basis[i] for i in range(len(mods))) % M for c in range(n)]


def _ciphertext(Q, n, seed, fill=None):
    if fill == "q-1":
        return np.concatenate([np.full(n, q - 1, dtype=U64) for _ in range(2) for q in Q])
    return np.concatenate([uniform_below(seed * 97 + c * 13 + i, n, q) for c in range(2) for i, q in enumerate(Q)])


def _tight_case(port, n, l, k):
    """Q, B and m_sk of 61-bit primes (generate_primes(., 60, .) draws from [2^60, 2^61)), and the largest t the bound
    accepts for them"""
    primes = [int(q) for q in port.generate_primes(l + k + 1, 60, True, n)]
    Q, extra = primes[:l], primes[l:]
    B, m_sk = extra[:k], extra[k]
    return Q, B, m_sk, bx.largest_plain_modulus(n, Q, B, m_sk)


@pytest.mark.parametrize("l, k", [(2, 2), (3, 3), (1, 1)])
@pytest.mark.parametrize("fill", [None, "q-1"])
def test_lift_and_fast_floor_hold_at_the_tightest_plain_modulus(port, l, k, fill):
    n = 16
    Q, B, m_sk, t = _tight_case(port, n, l, k)
    assert 2 <= t < 1 << 61
    assert bx.bound_holds(n, t, Q, B, m_sk) and not bx.bound_holds(n, t + 1, Q, B, m_sk)
    mods = Q + B + [m_sk]
    Qp, Mp = bx._prod(Q), bx._prod(mods)
    ct1, ct2 = _ciphertext(Q, n, 1, fill), _ciphertext(Q, n, 2, fill)
    lifts = []
    for ct in (ct1, ct2):
        for c in range(2):
            x = ct[c * l * n:(c + 1) * l * n]
            xl = bx.lift(port, x, n, Q, B, m_sk).reshape(len(mods), n)
            ints = [v - Mp if v > Mp // 2 else v for v in _crt(xl, mods)]
            orig = _crt(x.reshape(l, n), Q)
            for v, o in zip(ints, orig):
                assert v % Qp == o
                assert -Qp <= 2 * v and v * 2 * bx.MT < (bx.MT + 2 * l) * Qp  # -Q/2 <= x' < lambda Q
            lifts.append(ints)
    a0, a1, b0, b1 = lifts
    d1 = [x + y for x, y in zip(negacyclic_product(a0, b1, n), negacyclic_product(a1, b0, n))]
    tensor = [negacyclic_product(a0, b0, n), d1, negacyclic_product(a1, b1, n)]
    out = bx.bfv_multiply(port, ct1, ct2, n, Q, B, m_sk, t).reshape(3, l, n)
    for c in range(3):
        got = _crt(out[c], Q)
        for g, D in zip(got, tensor[c]):
            v = ((t * D) // Qp - g) % Qp
            assert 0 <= v < l, f"component {c}: floor(tD/Q) - out = {v} mod Q"


# the bit sizes of SEAL's default BFV moduli (CoeffModulus::BFVDefault, 128-bit security), the last one special
SEAL_BITS = {4096: [36, 36, 37], 8192: [43, 43, 44, 44, 44], 16384: [48, 48, 48, 49, 49, 49, 49, 49, 49],
             32768: [55] * 13 + [56] * 3}


def seal_moduli(port, n):
    out = []
    for bits in sorted(set(SEAL_BITS[n])):
        count = SEAL_BITS[n].count(bits)
        out += [int(q) for q in port.generate_primes(count, bits - 1, False, n)]  # the largest below 2^bits
    return out


@pytest.mark.parametrize("n", sorted(SEAL_BITS))
@pytest.mark.parametrize("t", [2, 65537, 786433, (1 << 60) - 93])
def test_seal_bases_pass_the_bound_at_every_level(port, n, t):
    mods = seal_moduli(port, n)
    for level in range(1, len(mods)):
        Q = mods[:level]
        B, m_sk = bx.seal_bases(port, n, Q, t)
        assert len(B) == bx.seal_base_b_size(Q, t)
        assert bx.bound_holds(n, t, Q, B, m_sk), f"level {level}"
        tmax = bx.largest_plain_modulus(n, Q, B, m_sk)
        assert bx.bound_holds(n, tmax, Q, B, m_sk) and not bx.bound_holds(n, tmax + 1, Q, B, m_sk)


@pytest.mark.parametrize("L, K, alpha, level", [(3, 1, 1, 3), (4, 2, 2, 3), (5, 3, 2, 5), (3, 2, 3, 2)])
def test_relinearized_model_is_the_chain(port, L, K, alpha, level):
    n, t = 32, 65537
    mods = [int(q) for q in port.generate_primes(L, 50, True, n)] + [int(q) for q in port.generate_primes(K, 55, True, n)]
    Q = mods[:level]
    B, m_sk = bx.seal_bases(port, n, Q, t)
    keys = hx.random_keys(mods, n, L, alpha, 2, 7 + L)
    d = bx.bfv_multiply(port, _ciphertext(Q, n, 3), _ciphertext(Q, n, 4), n, Q, B, m_sk, t)
    got = bx.relinearize(port, d, n, level, L, K, alpha, mods, keys)
    exp = bx.relinearize_chain(port, d, n, level, L, K, alpha, mods, keys)
    assert (got == exp).all()


def _poly_mul_mod(port, x, s, q, n):
    return port.ntt_inverse(port.mult_mod(port.ntt_forward(x, n, q), port.ntt_forward(s, n, q), q), n, q)


def _encrypt(port, m, s, Q, n, t, seed):
    """(c0, c1) = (-a s + e + floor(Q/t) m, a) limb by limb, e in [-8, 8]"""
    delta = bx._prod(Q) // t
    e = [int(v) - 8 for v in uniform_below(seed, n, 17)]
    c0, c1 = [], []
    for i, q in enumerate(Q):
        a = uniform_below(seed * 31 + i, n, q)
        s_q = np.array([v % q for v in s], dtype=U64)
        v = port.sub_mod(np.array([(x + delta * mm) % q for x, mm in zip(e, m)], dtype=U64),
                         _poly_mul_mod(port, a, s_q, q, n), q)
        c0.append(v)
        c1.append(a)
    return np.concatenate(c0 + c1)


def _decrypt(port, ct, powers, Q, n, t):
    """round(t [sum_j c_j s^j]_Q / Q) mod t; powers[j] is s^j as integer coefficients"""
    l = len(Q)
    comps = np.asarray(ct, dtype=U64).reshape(len(powers), l, n)
    limbs = []
    for i, q in enumerate(Q):
        acc = comps[0, i]
        for j in range(1, len(powers)):
            acc = port.add_mod(acc, _poly_mul_mod(port, comps[j, i], np.array([v % q for v in powers[j]], dtype=U64),
                                                  q, n), q)
        limbs.append(acc)
    Qp = bx._prod(Q)
    return [((t * v + Qp // 2) // Qp) % t for v in _crt(limbs, Q)]


@pytest.mark.parametrize("n, l, t", [(16, 1, 2), (16, 1, 257), (64, 2, 65537), (256, 3, T30), (1024, 4, 65537),
                                     (128, 4, T30)])
def test_products_decrypt_to_the_message_product(port, n, l, t):
    K, alpha = (2, 2) if l == 4 else (1, 1)
    mods = [int(q) for q in port.generate_primes(l + K, 60, True, n)]
    Q = mods[:l]
    B, m_sk = bx.seal_bases(port, n, Q, t)
    s = [int(v) - 1 for v in uniform_below(5 + n, n, 3)]
    s2 = negacyclic_product(s, s, n)
    m1 = [int(v) for v in uniform_below(11 + l, n, t)]
    m2 = [int(v) for v in uniform_below(12 + l, n, t)]
    expect = [v % t for v in negacyclic_product(m1, m2, n)]
    ct1, ct2 = _encrypt(port, m1, s, Q, n, t, 21), _encrypt(port, m2, s, Q, n, t, 22)
    assert _decrypt(port, ct1, [None, s], Q, n, t) == m1
    d = bx.bfv_multiply(port, ct1, ct2, n, Q, B, m_sk, t)
    assert _decrypt(port, d, [None, s, s2], Q, n, t) == expect
    keys = hx.hybrid_keys(port, s, s2, n, mods, l, alpha, 30 + n, 8)
    r = bx.relinearize(port, d, n, l, l, K, alpha, mods, keys)
    assert _decrypt(port, r, [None, s], Q, n, t) == expect
    other = [int(v) - 1 for v in uniform_below(6 + n, n, 3)]
    wrong = hx.hybrid_keys(port, other, negacyclic_product(other, other, n), n, mods, l, alpha, 30 + n, 8)
    r = bx.relinearize(port, d, n, l, l, K, alpha, mods, wrong)
    assert _decrypt(port, r, [None, s], Q, n, t) != expect


@pytest.mark.parametrize("kernel", ["bfv_extend_kernel", "bfv_scale_kernel"])
def test_bfv_kernels_keep_no_local_memory(kernel):
    res = {name: r for name, r in kernel_resources("bfv.cu").items() if kernel in name}
    assert res, f"no ptxas report for {kernel}"
    for name, (frame, stores, loads) in res.items():
        assert frame == 0 and stores == 0 and loads == 0, f"{name}: stack {frame}, spills {stores}/{loads}"
