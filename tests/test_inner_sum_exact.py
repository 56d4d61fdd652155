"""The model of the inner sum (tests/inner_sum_exact.py) against the models of the existing calls and against decryption;
and the compiler's resource report of its step kernel.  CPU only.

(a) k = 1 is the BSGS model with one identity baby, one identity giant and a unit diagonal (with rescale = 0, a copy of
    ct); k = 2 is the hoisted rotation by g plus ct, and the linear transform over {1, g} with unit diagonals; k = 3 and
    k = 4 are the BSGS model with unit diagonals over babies {1, g} and giants {1, g} (one pair absent) or {1, g^2},
    in both rescale modes;
(b) the needed elements are the powers g^(2^i) and the partial sums g^s, and an element of order 2 needs no key for its
    square;
(c) with Galois keys for s the result decrypts to sum_{j<k} sigma_{g^j}(phase(ct)) (divided by q_{l-1} and rounded with
    the rescale) within a bound built per keyed rotation from one key switch and one rounding; keys for another secret
    miss by far."""
import numpy as np
import pytest

import bsgs_exact as bx
import galois_exact as gx
import hybrid_exact as hx
import hybrid_rotation_exact as hr
import inner_sum_exact as ix
from test_bsgs_exact import _rescaled
from test_hybrid_exact import hybrid_case, noise_bound
from test_hybrid_rotation_exact import _ciphertext, _galois_keys, _phase, _primes
from test_kernel_resources import kernel_resources

U64 = np.uint64


def _random_keys(mods, n, L, alpha, elts, seed):
    return {e: hx.random_keys(mods, n, L, alpha, 2, seed + 7 * e) for e in elts}


def _ones(basis, n):
    return np.ones(len(basis) * n, dtype=U64)


SHAPES = [(6, 2, 2, 6), (7, 3, 3, 5), (5, 5, 5, 5), (4, 1, 3, 2), (5, 2, 1, 3)]


@pytest.mark.parametrize("L, K, alpha, level", SHAPES)
def test_one_and_two_terms(port, L, K, alpha, level):
    n, g = 32, 5
    mods = _primes(port, n, L, K)
    basis = mods[:level] + mods[L:]
    keys = _random_keys(mods, n, L, alpha, [g], L)
    ct = _ciphertext(mods, level, n, level)
    one = [[_ones(basis, n)]]
    for rescale in (False, True):
        got = ix.inner_sum_exact(port, ct, n, level, L, K, alpha, mods, g, 1, keys, rescale)
        exp = bx.bsgs_exact(port, ct, n, level, L, K, alpha, mods, [1], [None], [1], [None], one, rescale)
        assert (got == exp).all()
        if not rescale:
            assert (got == ct).all()
    got = ix.inner_sum_exact(port, ct, n, level, L, K, alpha, mods, g, 2, keys)
    rot = hr.hoisted_exact(port, ct, n, level, L, K, alpha, mods, [g], [keys[g]])
    exp = np.concatenate([port.add_mod(rot[i * n:(i + 1) * n], ct[i * n:(i + 1) * n], mods[i % level])
                          for i in range(2 * level)])
    assert (got == exp).all()
    ones = np.concatenate([_ones(basis, n)] * 2)
    lt = hr.linear_transform_exact(port, ct, n, level, L, K, alpha, mods, [1, g], [None, keys[g]], ones)
    assert (got == lt).all()


@pytest.mark.parametrize("rescale", [False, True])
@pytest.mark.parametrize("L, K, alpha, level", SHAPES)
def test_three_and_four_terms_are_bsgs(port, L, K, alpha, level, rescale):
    n, g = 32, 3
    mods = _primes(port, n, L, K)
    basis = mods[:level] + mods[L:]
    g2 = g * g % (2 * n)
    keys = _random_keys(mods, n, L, alpha, [g, g2], 2 * L)
    ct = _ciphertext(mods, level, n, 5 + level)
    w = _ones(basis, n)
    got = ix.inner_sum_exact(port, ct, n, level, L, K, alpha, mods, g, 3, keys, rescale)
    exp = bx.bsgs_exact(port, ct, n, level, L, K, alpha, mods, [1, g], [None, keys[g]], [1, g], [None, keys[g]],
                        [[w, None], [w, w]], rescale)
    assert (got == exp).all()
    got = ix.inner_sum_exact(port, ct, n, level, L, K, alpha, mods, g, 4, keys, rescale)
    exp = bx.bsgs_exact(port, ct, n, level, L, K, alpha, mods, [1, g], [None, keys[g]], [1, g2], [None, keys[g2]],
                        [[w, w], [w, w]], rescale)
    assert (got == exp).all()


def test_needed_elements():
    n = 64
    assert ix.needed_elements(5, 1, n) == []
    assert ix.needed_elements(5, 2, n) == [5]
    assert ix.needed_elements(5, 3, n) == [5]                        # g^1 as doubling and as shift
    assert ix.needed_elements(5, 4, n) == [5, 25]
    assert ix.needed_elements(5, 7, n) == sorted({5, 25, 5 ** 3 % 128})
    assert ix.needed_elements(2 * n - 1, 6, n) == [2 * n - 1]        # g^2 = 1: the doubling at bit 1 and g^2 shift
    assert ix.inner_sum_bits(2 * n - 1, 6, n) == [(2 * n - 1, None), (1, 1), (None, 1)]
    assert ix.inner_sum_bits(3, 5, n) == [(3, 1), (9, None), (None, 3)]


def test_order_two_element_sums_with_identities(port):
    """g = 2n - 1 (conjugation): sum_{j<k} sigma_{g^j} is ceil(k/2) ct + floor(k/2) sigma_g(ct) in phase; k = 6 has an
    identity doubling and an identity shift after the first"""
    n, L, K, alpha = 32, 4, 2, 2
    mods, s, _, _ = hybrid_case(port, L, K, alpha, n, 11)
    g = 2 * n - 1
    keys = dict(zip([g], _galois_keys(port, s, mods, L, K, alpha, n, [g], 3)))
    one = [1] + [0] * (n - 1)
    ct = _ciphertext(mods, L, n, 2)
    ph = _phase(port, ct, n, L, mods, s)
    rot = gx.sigma_ntt(ph, n, g)
    for k in (5, 6):
        exp = np.zeros(L * n, dtype=U64)
        for j in range(k):
            for i, q in enumerate(mods[:L]):
                dst = slice(i * n, (i + 1) * n)
                exp[dst] = port.add_mod(exp[dst], (rot if j % 2 else ph)[dst], q)
        res = ix.inner_sum_exact(port, ct, n, L, L, K, alpha, mods, g, k, keys)
        assert hx.noise(port, res, exp, s, one, n, L, mods) <= 4 * noise_bound(mods, L, K, alpha, L, n, 8)


def inner_sum_bound(mods, L, K, alpha, level, n, bound_e, g, k, rescale):
    """t = one key switch plus the rounding of c1' times s (K (n + 1)) per keyed rotation; the automorphism keeps the
    norm.  A's error doubles with each doubling and gains t when the doubling is keyed; each update of R adds A's error
    plus t when keyed.  Then one rounding K (n + 1) for the final mod-down; with the rescale, the sum divided by
    q_{l-1} plus one, a mod-down rounding from K + 1 sources, and one for rounding the reference."""
    rounding = K * (n + 1)
    t = noise_bound(mods, L, K, alpha, level, n, bound_e) + rounding
    err_a = err_r = 0
    for dbl, shift in ix.inner_sum_bits(g, k, n):
        if shift is not None:
            err_r += err_a + (t if shift != 1 else 0)
        if dbl is not None:
            err_a = 2 * err_a + (t if dbl != 1 else 0)
    total = err_r + rounding
    if not rescale:
        return total
    return total // mods[level - 1] + 1 + (K + 1) * (n + 1) + 1


@pytest.mark.parametrize("k", list(range(1, 10)) + [16, 17, 31])
def test_inner_sum_decrypts_within_the_bound(port, k):
    n, L, K, alpha, g = 64, 5, 2, 2, 5
    mods, s, _, _ = hybrid_case(port, L, K, alpha, n, 70)
    other = hybrid_case(port, L, K, alpha, n, 71)[1]  # another secret
    elts = ix.needed_elements(g, k, n)
    keys = dict(zip(elts, _galois_keys(port, s, mods, L, K, alpha, n, elts, 13)))
    wrong = dict(zip(elts, _galois_keys(port, other, mods, L, K, alpha, n, elts, 13)))
    one = [1] + [0] * (n - 1)
    level = L - (k % 2)
    ct = _ciphertext(mods, level, n, k)
    ph = _phase(port, ct, n, level, mods, s)
    exp = np.zeros(level * n, dtype=U64)
    for j in range(k):
        rot = gx.sigma_ntt(ph, n, pow(g, j, 2 * n))
        for i, q in enumerate(mods[:level]):
            dst = slice(i * n, (i + 1) * n)
            exp[dst] = port.add_mod(exp[dst], rot[dst], q)
    for rescale in (False, True):
        out_level = level - int(rescale)
        ref = _rescaled(port, exp, n, level, mods) if rescale else exp
        bound = inner_sum_bound(mods, L, K, alpha, level, n, 8, g, k, rescale)
        res = ix.inner_sum_exact(port, ct, n, level, L, K, alpha, mods, g, k, keys, rescale)
        got = hx.noise(port, res, ref, s, one, n, out_level, mods)
        assert got <= bound, f"k {k} rescale {rescale}: noise {got} above {bound}"
        if elts:
            res = ix.inner_sum_exact(port, ct, n, level, L, K, alpha, mods, g, k, wrong, rescale)
            assert hx.noise(port, res, ref, s, one, n, out_level, mods) > bound << 20, f"k {k} rescale {rescale}"


# ------------------------------------------------------------------------------------------------ compiler report
def test_inner_sum_step_kernel_keeps_no_local_memory():
    res = {name: r for name, r in kernel_resources("seal.cu").items() if "inner_sum_step_kernel" in name}
    assert len(res) == 1, f"expected one inner_sum_step_kernel, found {sorted(res)}"
    for name, (frame, st, ld) in res.items():
        assert frame == 0 and st == 0 and ld == 0, f"{name}: {frame} B stack frame, {st} B spill stores, {ld} B loads"
