"""The model of the multiply-relinearize call (tests/mul_relin_exact.py) against the existing exact models and against
decryption; and the compiler's resource report of its multiply-accumulate kernel.  CPU only.

(a) rescale = 0 is DyadicMultiply followed by KeySwitchHybrid of d2 into (d0, d1), bit for bit;
(b) at digit size 1 with one special prime that is the SEAL-shaped key switch of tests/ks_exact.py;
(c) with keys for s^2 the product decrypts to phase(ct1) phase(ct2), and with rescale = 1 to that divided by q_{l-1},
    within bounds derived from the hybrid switch's; keys for another secret miss both by far."""
import numpy as np
import pytest

import hybrid_exact as hx
import ks_exact
import mul_relin_exact as mr
from test_hybrid_exact import noise_bound
from test_kernel_resources import kernel_resources
from util import uniform_below

U64 = np.uint64


def _ciphertext(mods, level, n, seed):
    return np.concatenate([uniform_below(seed * 7919 + 100 * c + i, n, mods[i]) for c in range(2)
                           for i in range(level)])


def _primes(port, n, L, K):
    return [int(q) for q in port.generate_primes(L, 50, True, n)] + [int(q) for q in port.generate_primes(K, 55, True, n)]


def _chain(port, ct1, ct2, n, level, L, K, alpha, mods, keys):
    """DyadicMultiply, then KeySwitchHybrid of d2 accumulated into (d0, d1)"""
    d0, d1, d2 = mr.tensor(port, ct1, ct2, n, level, mods)
    return hx.key_switch_hybrid(port, np.concatenate([d0, d1]), d2, n, level, L, K, alpha, 2, mods, keys)


@pytest.mark.parametrize("L, K, alpha, level", [(6, 2, 2, 6), (7, 3, 3, 5), (5, 2, 5, 5), (8, 4, 2, 3), (4, 1, 3, 1)])
def test_no_rescale_is_the_chain(port, L, K, alpha, level):
    """a partial last digit at (7, 3, 3, 5), one digit at (5, 2, 5), level 1 at (4, 1, 3, 1)"""
    n = 32
    mods = _primes(port, n, L, K)
    keys = hx.random_keys(mods, n, L, alpha, 2, L + K)
    ct1, ct2 = _ciphertext(mods, level, n, 1), _ciphertext(mods, level, n, 2)
    got = mr.multiply_relinearize(port, ct1, ct2, n, level, L, K, alpha, mods, keys, False)
    assert (got == _chain(port, ct1, ct2, n, level, L, K, alpha, mods, keys)).all()


@pytest.mark.parametrize("L, level", [(4, 4), (5, 3), (3, 1)])
def test_alpha_one_k_one_is_the_seal_shaped_switch(port, L, level):
    """SEAL's multiply + relinearize: (d0, d1) + KeySwitch(d2) with one special prime and one-modulus digits"""
    n = 32
    mods = _primes(port, n, L, 1)
    keys = hx.random_keys(mods, n, L, 1, 2, 5)
    ct1, ct2 = _ciphertext(mods, level, n, 3), _ciphertext(mods, level, n, 4)
    got = mr.multiply_relinearize(port, ct1, ct2, n, level, L, 1, 1, mods, keys, False)
    d0, d1, d2 = mr.tensor(port, ct1, ct2, n, level, mods)
    modswitch = [pow(mods[-1] % q, -1, q) for q in mods[:level]]
    exp = ks_exact.key_switch_exact(port, np.concatenate([d0, d1]), d2, n, level, L + 1, level + 1, 2, mods,
                                    keys[:level], modswitch)
    assert (got == exp).all()


@pytest.mark.parametrize("rescale", [False, True])
def test_squaring_is_the_product_of_two_copies(port, rescale):
    n, L, K, alpha, level = 32, 6, 2, 4, 5
    mods = _primes(port, n, L, K)
    keys = hx.random_keys(mods, n, L, alpha, 2, 9)
    ct = _ciphertext(mods, level, n, 6)
    got = mr.multiply_relinearize(port, ct, ct, n, level, L, K, alpha, mods, keys, rescale)
    assert (got == mr.multiply_relinearize(port, ct, ct.copy(), n, level, L, K, alpha, mods, keys, rescale)).all()
    if not rescale:
        assert (got == _chain(port, ct, ct.copy(), n, level, L, K, alpha, mods, keys)).all()


# ------------------------------------------------------------------------------------------------ decryption
def _prod(values):
    out = 1
    for v in values:
        out *= int(v)
    return out


def _encrypt(port, m, s, mods, level, n, seed):
    """(c0, c1) = (m - a s, a) in NTT form at level `level`: a ciphertext of phase m"""
    c0, c1 = [], []
    for i, q in enumerate(mods[:level]):
        a = uniform_below(seed * 131 + i, n, q)
        s_i = port.ntt_forward(np.array([c % q for c in s], dtype=U64), n, q)
        m_i = port.ntt_forward(np.array([c % q for c in m], dtype=U64), n, q)
        c0.append(port.sub_mod(m_i, port.mult_mod(a, s_i, q), q))
        c1.append(a)
    return np.concatenate(c0 + c1)


def _ntt_limbs(port, coeffs, mods, level, n):
    return np.concatenate([port.ntt_forward(np.array([c % q for c in coeffs], dtype=U64), n, q)
                           for q in mods[:level]])


def relin_bound(mods, L, K, alpha, level, n, bound_e, rescale):
    """rescale = 0: the hybrid switch's bound (noise_bound).  rescale = 1: its key-switch term divided by q_{l-1},
    plus the rounding term of a mod-down from K + 1 sources, plus one for rounding phase(ct1) phase(ct2) / q_{l-1}"""
    if not rescale:
        return noise_bound(mods, L, K, alpha, level, n, bound_e)
    switch = noise_bound(mods, L, K, alpha, level, n, bound_e) - K * (n + 1)
    return switch // mods[level - 1] + 1 + (K + 1) * (n + 1) + 1


@pytest.mark.parametrize("L, K, alpha", [(6, 2, 2), (7, 3, 3), (5, 5, 5)])
def test_product_decrypts_within_the_bound(port, L, K, alpha):
    """phases of 30-bit coefficients, so that the product (up to n 2^60) is far above q_{l-1} and far below Q_l"""
    n, bound_m = 64, 1 << 30
    mods = [int(q) for q in port.generate_primes(L, 40, True, n)] + [int(q) for q in port.generate_primes(K, 45, True, n)]
    s = [int(v) - 1 for v in uniform_below(40 + L, n, 3)]
    keys = hx.hybrid_keys(port, s, mr.negacyclic_product(s, s, n), n, mods, L, alpha, 42 + L, 8)
    wrong = hx.hybrid_keys(port, s, s, n, mods, L, alpha, 42 + L, 8)  # switch s, not s^2
    one = [1] + [0] * (n - 1)
    m1 = [int(v) - bound_m for v in uniform_below(7, n, 2 * bound_m + 1)]
    m2 = [int(v) - bound_m for v in uniform_below(8, n, 2 * bound_m + 1)]
    m = mr.negacyclic_product(m1, m2, n)
    for level in sorted({L, L - 1, 2}):
        ct1, ct2 = _encrypt(port, m1, s, mods, level, n, 1), _encrypt(port, m2, s, mods, level, n, 2)
        for rescale in (False, True):
            out_level = level - int(rescale)
            q_last = mods[level - 1]
            exp = [(c + q_last // 2) // q_last for c in m] if rescale else m
            exp = _ntt_limbs(port, exp, mods, out_level, n)
            bound = relin_bound(mods, L, K, alpha, level, n, 8, rescale)
            assert bound < _prod(mods[:out_level]) >> 20
            res = mr.multiply_relinearize(port, ct1, ct2, n, level, L, K, alpha, mods, keys, rescale)
            got = hx.noise(port, res, exp, s, one, n, out_level, mods)
            assert got <= bound, f"level {level} rescale {rescale}: noise {got} above {bound}"
            res = mr.multiply_relinearize(port, ct1, ct2, n, level, L, K, alpha, mods, wrong, rescale)
            assert hx.noise(port, res, exp, s, one, n, out_level, mods) > bound << 20


# ------------------------------------------------------------------------------------------------ compiler report
def test_relin_mac_kernel_keeps_no_local_memory():
    res = {name: r for name, r in kernel_resources("seal.cu").items() if "ks_relin_mac_kernel" in name}
    assert len(res) == 1, f"expected one ks_relin_mac_kernel, found {sorted(res)}"
    for name, (frame, st, ld) in res.items():
        assert frame == 0 and st == 0 and ld == 0, f"{name}: {frame} B stack frame, {st} B spill stores, {ld} B loads"
