"""The model of the sum-of-products call (tests/mul_relin_sum_exact.py) against the existing exact models and against
decryption; and the compiler's resource report of its tensor-sum kernel.  CPU only.

(a) one pair is the multiply-relinearize model of tests/mul_relin_exact.py bit for bit, in both rescale modes;
(b) rescale = 0 is DyadicMultiply of every pair, the sums, then KeySwitchHybrid of the summed d2 into the summed
    (d0, d1), bit for bit, with the sums formed here in integers;
(c) with keys for s^2 the result decrypts to sum_r phase(ct1_r) phase(ct2_r), and with rescale = 1 to that divided by
    q_{l-1}, within the bound of one relinearization; keys for another secret miss by far, and the sum of the pairs'
    separately relinearized products carries a larger error."""
import numpy as np
import pytest

import hybrid_exact as hx
import mul_relin_exact as mr
import mul_relin_sum_exact as ms
from test_kernel_resources import kernel_resources
from test_mul_relin_exact import _ciphertext, _encrypt, _ntt_limbs, _primes, _prod, relin_bound
from util import uniform_below

U64 = np.uint64


@pytest.mark.parametrize("rescale", [False, True])
@pytest.mark.parametrize("L, K, alpha, level", [(6, 2, 2, 6), (7, 3, 3, 5), (4, 1, 3, 2)])
def test_one_pair_is_multiply_relinearize(port, L, K, alpha, level, rescale):
    n = 32
    mods = _primes(port, n, L, K)
    keys = hx.random_keys(mods, n, L, alpha, 2, L + K)
    ct1, ct2 = _ciphertext(mods, level, n, 1), _ciphertext(mods, level, n, 2)
    got = ms.multiply_relinearize_sum(port, [ct1], [ct2], n, level, L, K, alpha, mods, keys, rescale)
    assert (got == mr.multiply_relinearize(port, ct1, ct2, n, level, L, K, alpha, mods, keys, rescale)).all()


def _integer_tensor_sum(ct1s, ct2s, n, level, mods):
    """(d0, d1, t) of the pairs summed in Python integers and reduced once"""
    out = np.zeros((3, level * n), dtype=U64)
    for i in range(level):
        q, s = mods[i], slice(i * n, (i + 1) * n)
        acc = [[0] * n for _ in range(3)]
        for a, b in zip(ct1s, ct2s):
            a0, a1 = a[s].tolist(), a[level * n:][s].tolist()
            b0, b1 = b[s].tolist(), b[level * n:][s].tolist()
            for l in range(n):
                acc[0][l] += a0[l] * b0[l]
                acc[1][l] += a0[l] * b1[l] + a1[l] * b0[l]
                acc[2][l] += a1[l] * b1[l]
        for k in range(3):
            out[k, s] = np.array([v % q for v in acc[k]], dtype=U64)
    return out


@pytest.mark.parametrize("pairs", [2, 5])
@pytest.mark.parametrize("L, K, alpha, level", [(6, 2, 2, 6), (7, 3, 3, 5), (5, 2, 5, 5), (4, 1, 3, 1)])
def test_no_rescale_is_the_chain(port, L, K, alpha, level, pairs):
    """a partial last digit at (7, 3, 3, 5), one digit at (5, 2, 5), level 1 at (4, 1, 3, 1); a repeated ciphertext and
    a square among the pairs"""
    n = 32
    mods = _primes(port, n, L, K)
    keys = hx.random_keys(mods, n, L, alpha, 2, L + K + pairs)
    cts = [_ciphertext(mods, level, n, 10 + r) for r in range(pairs + 1)]
    ct1s = [cts[r] for r in range(pairs)]
    ct2s = [cts[0]] + [cts[r + 1] if r % 2 else cts[r] for r in range(1, pairs)]
    d0, d1, d2 = _integer_tensor_sum(ct1s, ct2s, n, level, mods)
    assert (np.stack([d0, d1, d2]) == ms.tensor_sum(port, ct1s, ct2s, n, level, mods)).all()
    chain = hx.key_switch_hybrid(port, np.concatenate([d0, d1]), d2, n, level, L, K, alpha, 2, mods, keys)
    got = ms.multiply_relinearize_sum(port, ct1s, ct2s, n, level, L, K, alpha, mods, keys, False)
    assert (got == chain).all()


# ------------------------------------------------------------------------------------------------ decryption
def _add(port, x, y, mods, level, n):
    """x + y for two ciphertexts of 2 x level x n words"""
    out = x.copy()
    for c in range(2):
        for i in range(level):
            s = slice((c * level + i) * n, (c * level + i + 1) * n)
            out[s] = port.add_mod(x[s], y[s], mods[i])
    return out


@pytest.mark.parametrize("pairs", [1, 3, 8])
@pytest.mark.parametrize("L, K, alpha", [(6, 2, 2), (7, 3, 3)])
def test_sum_decrypts_within_one_relinearization(port, L, K, alpha, pairs):
    """phases of 30-bit coefficients: the sum of products (up to 8 n 2^60) is far above q_{l-1} and far below Q_l"""
    n, bound_m = 64, 1 << 30
    mods = [int(q) for q in port.generate_primes(L, 40, True, n)] + [int(q) for q in port.generate_primes(K, 45, True, n)]
    s = [int(v) - 1 for v in uniform_below(40 + L, n, 3)]
    keys = hx.hybrid_keys(port, s, mr.negacyclic_product(s, s, n), n, mods, L, alpha, 42 + L, 8)
    wrong = hx.hybrid_keys(port, s, s, n, mods, L, alpha, 42 + L, 8)  # switch s, not s^2
    one = [1] + [0] * (n - 1)
    m1 = [[int(v) - bound_m for v in uniform_below(7 + 2 * r, n, 2 * bound_m + 1)] for r in range(pairs)]
    m2 = [[int(v) - bound_m for v in uniform_below(8 + 2 * r, n, 2 * bound_m + 1)] for r in range(pairs)]
    m = [sum(col) for col in zip(*[mr.negacyclic_product(a, b, n) for a, b in zip(m1, m2)])]
    for level in sorted({L, 3}):
        ct1s = [_encrypt(port, m1[r], s, mods, level, n, 1 + 2 * r) for r in range(pairs)]
        ct2s = [_encrypt(port, m2[r], s, mods, level, n, 2 + 2 * r) for r in range(pairs)]
        for rescale in (False, True):
            out_level = level - int(rescale)
            q_last = mods[level - 1]
            exp = [(c + q_last // 2) // q_last for c in m] if rescale else m
            exp = _ntt_limbs(port, exp, mods, out_level, n)
            bound = relin_bound(mods, L, K, alpha, level, n, 8, rescale)
            assert bound < _prod(mods[:out_level]) >> 20
            res = ms.multiply_relinearize_sum(port, ct1s, ct2s, n, level, L, K, alpha, mods, keys, rescale)
            got = hx.noise(port, res, exp, s, one, n, out_level, mods)
            assert got <= bound, f"level {level} rescale {rescale}: noise {got} above {bound}"
            res = ms.multiply_relinearize_sum(port, ct1s, ct2s, n, level, L, K, alpha, mods, wrong, rescale)
            assert hx.noise(port, res, exp, s, one, n, out_level, mods) > bound << 20
            if pairs == 8 and not rescale:
                separate = mr.multiply_relinearize(port, ct1s[0], ct2s[0], n, level, L, K, alpha, mods, keys, False)
                for r in range(1, pairs):
                    separate = _add(port, separate, mr.multiply_relinearize(port, ct1s[r], ct2s[r], n, level, L, K,
                                                                            alpha, mods, keys, False), mods, level, n)
                worse = hx.noise(port, separate, exp, s, one, n, out_level, mods)
                assert worse > got, f"level {level}: {pairs} relinearizations {worse}, one {got}"


# ------------------------------------------------------------------------------------------------ compiler report
def test_tensor_sum_kernel_keeps_no_local_memory():
    res = {name: r for name, r in kernel_resources("seal.cu").items() if "relin_tensor_sum_kernel" in name}
    assert len(res) == 1, f"expected one relin_tensor_sum_kernel, found {sorted(res)}"
    for name, (frame, st, ld) in res.items():
        assert frame == 0 and st == 0 and ld == 0, f"{name}: {frame} B stack frame, {st} B spill stores, {ld} B loads"
