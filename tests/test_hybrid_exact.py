"""The hybrid key-switch model (tests/hybrid_exact.py) against big-integer arithmetic, against the exact key switch, and
against decryption; the plain-integer base conversion of the GPU domain tests against the modular model; and the
compiler's resource report of the base-conversion kernel.  CPU only."""
import numpy as np
import pytest

import hybrid_exact as hx
import ks_exact
from test_kernel_resources import kernel_resources
from util import uniform_below

U64 = np.uint64


def _prod(values):
    out = 1
    for v in values:
        out *= int(v)
    return out


@pytest.mark.parametrize("shape", [(1, 50, 3), (3, 40, 5), (8, 60, 70), (64, 60, 2)])
@pytest.mark.parametrize("fill", ["uniform", "q-1"])
def test_base_conversion_is_the_lift_plus_a_multiple_of_q(port, shape, fill):
    """result_m = X + e Q mod m with X the CRT lift of the inputs in [0, Q) and 0 <= e < from_count, for every slot"""
    count, bits, to_count = shape
    n = 8
    mods = [int(q) for q in port.generate_primes(count + to_count, bits, False, n)]
    src, dst = mods[:count], mods[count:]
    x = np.concatenate([np.full(n, q - 1, dtype=U64) if fill == "q-1" else uniform_below(7 + i, n, q)
                        for i, q in enumerate(src)])
    got = hx.fast_base_convert(port, x, n, src, dst).reshape(to_count, n)
    Q = _prod(src)
    basis = [(Q // q) * pow(Q // q % q, -1, q) for q in src]
    for col in range(n):
        X = sum(int(x[i * n + col]) * basis[i] for i in range(count)) % Q
        ys = [int(x[i * n + col]) * pow(Q // q % q, -1, q) % q for i, q in enumerate(src)]
        e = (sum(y * (Q // q) for y, q in zip(ys, src)) - X) // Q
        assert 0 <= e < count
        assert [int(got[j, col]) for j in range(to_count)] == [(X + e * Q) % t for t in dst]


def test_base_conversion_returns_a_source_limb_in_its_own_modulus(port):
    n = 16
    mods = [int(q) for q in port.generate_primes(5, 50, True, n)]
    x = np.concatenate([uniform_below(3 + i, n, q) for i, q in enumerate(mods)])
    got = hx.fast_base_convert(port, x, n, mods, mods[::-1])
    assert (got == np.concatenate([x[i * n:(i + 1) * n] for i in range(4, -1, -1)])).all()


# the ks_exact cases whose key_modulus_size equals rns_modulus_size: SEAL's layout is then the hybrid one at alpha = 1,
# K = 1 (the special prime in slot L)
ANCHOR_CASES = ["uniform", "kcc1", "kcc3", "one_digit", "small_special", "word_classes", "wrap17", "wrap_keys",
                "wrap_blocks"]


@pytest.mark.parametrize("name", ANCHOR_CASES)
def test_alpha_one_k_one_is_the_exact_key_switch(port, name):
    case = ks_exact.make_case(port, name, 16)
    assert case.kms == case.rns and case.digit_factor == 1
    L, n, kcc = case.decomp, case.n, case.kcc
    result, t = ks_exact.ciphertext(case, 5)
    for level in sorted({L, max(1, L // 2), 1}):
        res = result.reshape(kcc, L, n)[:, :level].reshape(-1)
        exp = ks_exact.key_switch_exact(port, res, t[:level * n], n, level, case.kms, level + 1, kcc, case.mods,
                                        case.keys[:level], case.modswitch[:level])
        got = hx.key_switch_hybrid(port, res, t[:level * n], n, level, L, 1, 1, kcc, case.mods, case.keys)
        assert (got == exp).all(), f"{name} at level {level}"


def hybrid_case(port, L, K, alpha, n, seed):
    """40-bit data primes, 45-bit special primes, a ternary secret and keys from it to a second ternary secret"""
    mods = [int(q) for q in port.generate_primes(L, 40, True, n)] + [int(q) for q in port.generate_primes(K, 45, True, n)]
    s = [int(v) - 1 for v in uniform_below(seed, n, 3)]
    s_new = [int(v) - 1 for v in uniform_below(seed + 1, n, 3)]
    keys = hx.hybrid_keys(port, s, s_new, n, mods, L, alpha, seed + 2, 8)
    return mods, s, s_new, keys


def noise_bound(mods, L, K, alpha, level, n, bound_e):
    """D alpha n B_e max Q_d / P from the digits' lifts (each below alpha Q_d) times the key errors, plus K (n + 1) from
    the mod-down, whose base conversion rounds to within K of the exact quotient in each component"""
    groups = hx.digits(level, alpha)
    max_qd = max(_prod(mods[i] for i in S) for S in groups)
    P = _prod(mods[L:L + K])
    return len(groups) * alpha * n * bound_e * max_qd // P + K * (n + 1)


@pytest.mark.parametrize("L, K, alpha", [(6, 2, 2), (7, 3, 3), (5, 5, 5)])
def test_switched_ciphertext_decrypts_within_the_bound(port, L, K, alpha):
    n = 64
    mods, s, s_new, keys = hybrid_case(port, L, K, alpha, n, 40 + L)
    for level in sorted({L, L - 1, 1 + alpha // 2}):
        t = np.concatenate([uniform_below(90 + i, n, q) for i, q in enumerate(mods[:level])])
        res = hx.key_switch_hybrid(port, np.zeros(2 * level * n, dtype=U64), t, n, level, L, K, alpha, 2, mods, keys)
        got = hx.noise(port, res, t, s, s_new, n, level, mods)
        bound = noise_bound(mods, L, K, alpha, level, n, 8)
        assert got <= bound, f"level {level}: noise {got} above {bound}"
        # the wrong secret misses by far
        assert hx.noise(port, res, t, s, s, n, level, mods) > bound << 20


def test_base_conversion_kernel_keeps_no_local_memory():
    res = {name: r for name, r in kernel_resources("rns.cu").items() if "base_conv_kernel" in name}
    assert len(res) == 2, f"expected the two base_conv_kernel instances, found {sorted(res)}"
    bad = [f"{name}: {frame} B frame, {st} B spill stores" for name, (frame, st, ld) in res.items()
           if frame > max(st, ld)]
    assert not bad, bad


@pytest.mark.parametrize("sizes, bits", [((1, 3), 50), ((3, 5), 50), ((10, 29), 60), ((64, 3), 60)])
def test_integer_base_conversion_equals_the_modular_model_on_primes(port, sizes, bits):
    """the plain-integer reference of the GPU's base-conversion domain tests, pinned to the modular model on NTT primes
    (where both apply), with every word q - 1 and with uniform words"""
    mods = [int(q) for q in port.generate_primes(sum(sizes), bits, bits < 60, 2)]
    src, dst = mods[:sizes[0]], mods[sizes[0]:]
    n = 65
    for x in (np.concatenate([uniform_below(7 * i + 1, n, q) for i, q in enumerate(src)]),
              np.concatenate([np.full(n, q - 1, dtype=np.uint64) for q in src])):
        assert (hx.fast_base_convert_int(x, n, src, dst) == hx.fast_base_convert(port, x, n, src, dst)).all()


def test_integer_base_conversion_on_small_numbers():
    """sources 3, 5 (Q = 15) into 2, 4, 7 and 15 itself: the sum of y_i (Q/q_i) over the integers, reduced"""
    x = np.array([2, 1, 0, 4], dtype=np.uint64)  # limb 3: 5 and 4 mod 3, limb 5: 5 and 4 mod 5
    out = hx.fast_base_convert_int(x, 2, [3, 5], [2, 4, 7, 15]).reshape(4, 2)
    # X = 5: y = (2 * 5^-1 mod 3, 0) = (1, 0), sum 5;  X = 4: y = (1 * 2 mod 3, 4 * 3^-1 mod 5) = (2, 3), sum 10 + 9 = 19
    assert out.tolist() == [[1, 1], [1, 3], [5, 5], [5, 4]]
