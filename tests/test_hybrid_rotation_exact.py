"""The model of the rotations with hybrid keys (tests/hybrid_rotation_exact.py) against the existing exact models, and
against decryption; and the compiler's resource report of the linear transform's two kernels.  CPU only.

(a) at digit size 1 with one special prime the hoisted hybrid rotation is the hoisted SEAL-shaped rotation;
(b) at g = 1 it is [c0, 0] + KeySwitchHybrid(c1);
(c) the linear transform of one element with a diagonal of ones is the hoisted rotation."""
import numpy as np
import pytest

import galois_exact as gx
import hoist_exact
import hybrid_exact as hx
import hybrid_rotation_exact as hr
from test_hybrid_exact import hybrid_case, noise_bound
from test_kernel_resources import kernel_resources
from util import uniform_below

U64 = np.uint64


def _ciphertext(mods, level, n, seed):
    return np.concatenate([uniform_below(seed * 7919 + 100 * c + i, n, mods[i]) for c in range(2)
                           for i in range(level)])


def _primes(port, n, L, K):
    return [int(q) for q in port.generate_primes(L, 50, True, n)] + [int(q) for q in port.generate_primes(K, 55, True, n)]


@pytest.mark.parametrize("L, level", [(4, 4), (5, 3), (3, 1)])
def test_alpha_one_k_one_is_the_hoisted_rotation(port, L, level):
    n = 32
    mods = _primes(port, n, L, 1)
    elts = [3, 2 * n - 1, 5, 3]
    keys = [hx.random_keys(mods, n, L, 1, 2, 10 + r) for r in range(len(elts))]
    ct = _ciphertext(mods, level, n, L)
    got = hr.hoisted_exact(port, ct, n, level, L, 1, 1, mods, elts, keys)
    modswitch = [pow(mods[-1] % q, -1, q) for q in mods[:level]]
    exp = hoist_exact.hoisted_exact(port, ct, n, level, L + 1, mods, elts, [k[:level] for k in keys], modswitch)
    assert (got == exp).all()


@pytest.mark.parametrize("L, K, alpha, level", [(6, 2, 2, 6), (7, 3, 3, 5), (5, 5, 5, 5), (4, 1, 3, 4)])
def test_identity_element_is_the_hybrid_key_switch(port, L, K, alpha, level):
    n = 32
    mods = _primes(port, n, L, K)
    keys = hx.random_keys(mods, n, L, alpha, 2, 3)
    ct = _ciphertext(mods, level, n, 7)
    comp = level * n
    got = hr.hoisted_exact(port, ct, n, level, L, K, alpha, mods, [1], [keys])
    start = np.concatenate([ct[:comp], np.zeros(comp, dtype=U64)])
    exp = hx.key_switch_hybrid(port, start, ct[comp:], n, level, L, K, alpha, 2, mods, keys)
    assert (got == exp).all()


@pytest.mark.parametrize("g", [1, 3, 25, 63])
def test_one_element_with_unit_diagonal_is_the_hoisted_rotation(port, g):
    n, L, K, alpha, level = 32, 6, 2, 4, 5
    mods = _primes(port, n, L, K)
    keys = hx.random_keys(mods, n, L, alpha, 2, g)
    ct = _ciphertext(mods, level, n, g)
    basis = mods[:level] + mods[L:]
    ones = hr.random_diagonals(basis, n, 1, 0, fill="one")
    got = hr.linear_transform_exact(port, ct, n, level, L, K, alpha, mods, [g], [keys], ones)
    assert (got == hr.hoisted_exact(port, ct, n, level, L, K, alpha, mods, [g], [keys])).all()


def test_identity_terms_alone_weight_the_ciphertext(port):
    """no keyed element: no key switch, result = sum_r w_r (.) ct"""
    n, L, K, alpha, level = 16, 3, 2, 2, 3
    mods = _primes(port, n, L, K)
    basis = mods[:level] + mods[L:]
    ct = _ciphertext(mods, level, n, 1)
    w = hr.random_diagonals(basis, n, 2, 4).reshape(2, len(basis), n)
    got = hr.linear_transform_exact(port, ct, n, level, L, K, alpha, mods, [1, 1], [None, None], w.reshape(-1))
    for c in range(2):
        for i, q in enumerate(mods[:level]):
            x = ct[(c * level + i) * n:(c * level + i + 1) * n]
            exp = port.add_mod(port.mult_mod(w[0, i], x, q), port.mult_mod(w[1, i], x, q), q)
            assert (got[(c * level + i) * n:(c * level + i + 1) * n] == exp).all()


# ------------------------------------------------------------------------------------------------ decryption
def _galois_keys(port, s, mods, L, K, alpha, n, elts, seed):
    """hybrid keys that switch s(X^g) back to s, one set per element"""
    return [hx.hybrid_keys(port, s, gx.sigma_int(s, n, g), n, mods, L, alpha, seed + 17 * r, 8)
            for r, g in enumerate(elts)]


@pytest.mark.parametrize("L, K, alpha", [(6, 2, 2), (7, 3, 3), (5, 5, 5)])
def test_hoisted_rotation_decrypts_within_the_bound(port, L, K, alpha):
    """out_r - [sigma(c0), 0] is the switch of sigma(c1) from sigma(s) to s: within the hybrid switch's bound (the
    signed lift is below alpha Q_d like the unsigned one), and with the keys of another element far off"""
    n = 64
    mods, s, _, _ = hybrid_case(port, L, K, alpha, n, 40 + L)
    elts = [3, 2 * n - 1, 25]
    keys = _galois_keys(port, s, mods, L, K, alpha, n, elts, 5)
    for level in sorted({L, L - 1}):
        ct = _ciphertext(mods, level, n, level)
        comp = level * n
        out = hr.hoisted_exact(port, ct, n, level, L, K, alpha, mods, elts, keys).reshape(len(elts), 2 * comp)
        swapped = hr.hoisted_exact(port, ct, n, level, L, K, alpha, mods, elts, keys[1:] + keys[:1])
        swapped = swapped.reshape(len(elts), 2 * comp)
        bound = noise_bound(mods, L, K, alpha, level, n, 8)
        for r, g in enumerate(elts):
            c1g = gx.sigma_ntt(ct[comp:], n, g)
            for res, ok in ((out[r], True), (swapped[r], False)):
                ks = res.copy()
                ks[:comp] = np.concatenate([port.sub_mod(ks[i * n:(i + 1) * n],
                                                         gx.sigma_ntt(ct[i * n:(i + 1) * n], n, g), mods[i])
                                            for i in range(level)])
                got = hx.noise(port, ks, c1g, s, gx.sigma_int(s, n, g), n, level, mods)
                if ok:
                    assert got <= bound, f"level {level}, g = {g}: noise {got} above {bound}"
                else:
                    assert got > bound << 20, f"level {level}, g = {g}: swapped keys give noise {got}"


def linear_transform_bound(mods, L, K, alpha, level, n, bound_e, elts, bound_w):
    """G n B_w times the key-switch term of noise_bound (each element's error E_r/P, below D alpha n B_e max Q_d / P,
    multiplied by a diagonal of n coefficients below B_w), plus one rounding term K (n + 1) for the single mod-down"""
    rounding = K * (n + 1)
    switch = noise_bound(mods, L, K, alpha, level, n, bound_e) - rounding
    return elts * n * bound_w * switch + rounding


def _phase(port, ct, n, level, mods, s):
    """c0 + c1 s per limb, NTT form"""
    out = []
    for i, q in enumerate(mods[:level]):
        s_i = port.ntt_forward(np.array([c % q for c in s], dtype=U64), n, q)
        c0, c1 = ct[i * n:(i + 1) * n], ct[(level + i) * n:(level + i + 1) * n]
        out.append(port.add_mod(c0, port.mult_mod(c1, s_i, q), q))
    return np.concatenate(out)


@pytest.mark.parametrize("L, K, alpha", [(6, 2, 2), (7, 3, 3), (5, 5, 5)])
def test_linear_transform_decrypts_within_the_bound(port, L, K, alpha):
    """the phase of the result is sum_r w_r sigma_r(c0 + c1 s) up to the derived bound, with small integer
    diagonals, an identity term and a repeated element; the keys of another element miss it by far"""
    n, bound_w = 64, 4
    mods, s, _, _ = hybrid_case(port, L, K, alpha, n, 40 + L)
    elts = [3, 1, 2 * n - 1, 3]
    keys = _galois_keys(port, s, mods, L, K, alpha, n, elts, 9)
    keys[1] = None
    swapped = [keys[2], None, keys[0], keys[2]]
    one = [1] + [0] * (n - 1)
    for level in sorted({L, L - 1}):
        basis = mods[:level] + mods[L:L + K]
        _, w = hr.small_diagonals(port, basis, n, len(elts), bound_w, level)
        w3 = w.reshape(len(elts), len(basis), n)
        ct = _ciphertext(mods, level, n, 3 + level)
        ph = _phase(port, ct, n, level, mods, s)
        exp = np.zeros(level * n, dtype=U64)
        for r, g in enumerate(elts):
            rot = gx.sigma_ntt(ph, n, g)
            for i, q in enumerate(mods[:level]):
                dst = slice(i * n, (i + 1) * n)
                exp[dst] = port.add_mod(exp[dst], port.mult_mod(w3[r, i], rot[dst], q), q)
        bound = linear_transform_bound(mods, L, K, alpha, level, n, 8, len(elts), bound_w)
        res = hr.linear_transform_exact(port, ct, n, level, L, K, alpha, mods, elts, keys, w)
        got = hx.noise(port, res, exp, s, one, n, level, mods)
        assert got <= bound, f"level {level}: noise {got} above {bound}"
        res = hr.linear_transform_exact(port, ct, n, level, L, K, alpha, mods, elts, swapped, w)
        assert hx.noise(port, res, exp, s, one, n, level, mods) > bound << 20


# ------------------------------------------------------------------------------------------------ compiler report
@pytest.mark.parametrize("kernel", ["ks_weighted_mac_kernel", "ks_permuted_sum_kernel"])
def test_linear_transform_kernels_keep_no_local_memory(kernel):
    res = {name: r for name, r in kernel_resources("seal.cu").items() if kernel in name}
    assert len(res) == 1, f"expected one {kernel}, found {sorted(res)}"
    for name, (frame, st, ld) in res.items():
        assert frame == 0 and st == 0 and ld == 0, f"{name}: {frame} B stack frame, {st} B spill stores, {ld} B loads"
