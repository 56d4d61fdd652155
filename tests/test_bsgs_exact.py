"""The model of the baby-step giant-step linear transform (tests/bsgs_exact.py) against the models of the existing
calls and against decryption; and the compiler's resource report of its sum kernel.  CPU only.

(a) with one identity giant it is LinearTransformHybrid over the babies, the absent diagonals as zero ones;
(b) with one identity baby and diagonals of ones it is LinearTransformHybrid over the giants with unit diagonals, and
    with one keyed giant, the hoisted rotation;
(c) its phase is sum_j sigma_{h_j}(sum_i w_{j,i} sigma_{b_i}(phase(ct))) within a derived bound (divided by q_{l-1}
    and rounded with the rescale), and swapped giant keys miss that bound by far."""
import numpy as np
import pytest

import bsgs_exact as bx
import galois_exact as gx
import hybrid_exact as hx
import hybrid_rotation_exact as hr
from test_hybrid_exact import hybrid_case, noise_bound
from test_hybrid_rotation_exact import _ciphertext, _galois_keys, _phase, _primes
from test_kernel_resources import kernel_resources

U64 = np.uint64


def _zero_filled(grid, basis, n):
    return np.concatenate([np.asarray(w, dtype=U64) if w is not None else np.zeros(len(basis) * n, dtype=U64)
                           for w in grid])


@pytest.mark.parametrize("L, K, alpha, level", [(6, 2, 2, 6), (7, 3, 3, 5), (5, 5, 5, 5), (4, 1, 3, 4), (5, 2, 1, 2)])
def test_one_identity_giant_is_the_linear_transform(port, L, K, alpha, level):
    n = 32
    mods = _primes(port, n, L, K)
    basis = mods[:level] + mods[L:]
    babies = [3, 1, 2 * n - 1, 5, 3, 1]
    keys = [hx.random_keys(mods, n, L, alpha, 2, 10 + i) for i in range(len(babies))]
    keys[1] = keys[5] = None
    ct = _ciphertext(mods, level, n, level)
    grid = bx.grid_diagonals(basis, n, 1, len(babies), {(0, 0), (0, 1), (0, 2), (0, 4)}, L)
    for rescale in (False, True):
        got = bx.bsgs_exact(port, ct, n, level, L, K, alpha, mods, babies, keys, [1], [None], grid, rescale)
        if rescale:  # the rescale merged into the final mod-down: (X, Y) folded as P X + Y, checked in (c)
            assert got.size == 2 * (level - 1) * n
            continue
        exp = hr.linear_transform_exact(port, ct, n, level, L, K, alpha, mods, babies, keys,
                                        _zero_filled(grid[0], basis, n))
        assert (got == exp).all()


@pytest.mark.parametrize("L, K, alpha, level", [(6, 2, 2, 6), (7, 3, 3, 5), (4, 1, 1, 3)])
def test_one_identity_baby_is_the_linear_transform_over_the_giants(port, L, K, alpha, level):
    n = 32
    mods = _primes(port, n, L, K)
    basis = mods[:level] + mods[L:]
    giants = [5, 1, 2 * n - 1, 5]
    keys = [hx.random_keys(mods, n, L, alpha, 2, 20 + j) for j in range(len(giants))]
    keys[1] = None
    ct = _ciphertext(mods, level, n, 3)
    grid = bx.grid_diagonals(basis, n, len(giants), 1, None, 0, fill="one")
    got = bx.bsgs_exact(port, ct, n, level, L, K, alpha, mods, [1], [None], giants, keys, grid)
    ones = hr.random_diagonals(basis, n, len(giants), 0, fill="one")
    assert (got == hr.linear_transform_exact(port, ct, n, level, L, K, alpha, mods, giants, keys, ones)).all()
    one = bx.bsgs_exact(port, ct, n, level, L, K, alpha, mods, [1], [None], [giants[2]], [keys[2]], grid[:1])
    assert (one == hr.hoisted_exact(port, ct, n, level, L, K, alpha, mods, [giants[2]], [keys[2]])).all()


def test_absent_rows_and_identity_terms_alone(port):
    """no keyed element at all: result = sum_j sum_i w_{j,i} ct; an absent row adds nothing"""
    n, L, K, alpha, level = 16, 3, 2, 2, 3
    mods = _primes(port, n, L, K)
    basis = mods[:level] + mods[L:]
    ct = _ciphertext(mods, level, n, 1)
    grid = bx.grid_diagonals(basis, n, 3, 2, {(0, 0), (2, 0), (2, 1)}, 5)
    got = bx.bsgs_exact(port, ct, n, level, L, K, alpha, mods, [1, 1], [None, None], [1, 1, 1], [None] * 3, grid)
    for c in range(2):
        for i, q in enumerate(mods[:level]):
            x = ct[(c * level + i) * n:(c * level + i + 1) * n]
            exp = np.zeros(n, dtype=U64)
            for j, b in ((0, 0), (2, 0), (2, 1)):
                w = np.asarray(grid[j][b]).reshape(len(basis), n)[i]
                exp = port.add_mod(exp, port.mult_mod(w, x, q), q)
            assert (got[(c * level + i) * n:(c * level + i + 1) * n] == exp).all()


# ------------------------------------------------------------------------------------------------ decryption
def bsgs_bound(mods, L, K, alpha, level, n, bound_e, grid, baby_keyed, giant_keyed, bound_w, rescale):
    """Per present row j: n B_w times the key-switch term of noise_bound per keyed baby (as linear_transform_bound),
    plus for a keyed giant one key-switch term and, when the row has a keyed baby, the rounding of c1'_j's mod-down
    times s (K (n + 1)); the giant automorphism keeps the norm.  Then one rounding term K (n + 1) for the final
    mod-down; with the rescale, the sum divided by q_{l-1} plus one, the rounding of a mod-down from K + 1 sources,
    plus one for rounding the reference."""
    rounding = K * (n + 1)
    switch = noise_bound(mods, L, K, alpha, level, n, bound_e) - rounding
    total = 0
    for j, row in enumerate(grid):
        present = [i for i, w in enumerate(row) if w is not None]
        if not present:
            continue
        kb = sum(1 for i in present if baby_keyed[i])
        total += kb * n * bound_w * switch
        if giant_keyed[j]:
            total += switch + (rounding if kb else 0)
    if not rescale:
        return total + rounding
    return total // mods[level - 1] + 1 + (K + 1) * (n + 1) + 1


def _rescaled(port, limbs, n, level, mods):
    """round(v / q_{level-1}) for v the centred lift of `limbs` (level x n, NTT form), NTT form under level - 1 moduli"""
    ms = mods[:level]
    Q = 1
    for q in ms:
        Q *= q
    coef = [port.ntt_inverse(limbs[i * n:(i + 1) * n], n, q) for i, q in enumerate(ms)]
    basis = [(Q // q) * pow(Q // q % q, -1, q) for q in ms]
    q_last = ms[-1]
    out = []
    for col in range(n):
        v = sum(int(coef[i][col]) * basis[i] for i in range(level)) % Q
        v = v - Q if v > Q // 2 else v
        out.append((v + q_last // 2) // q_last)
    return np.concatenate([port.ntt_forward(np.array([c % q for c in out], dtype=U64), n, q) for q in ms[:-1]])


@pytest.mark.parametrize("L, K, alpha", [(6, 2, 2), (7, 3, 3), (5, 5, 5)])
def test_bsgs_decrypts_within_the_bound(port, L, K, alpha):
    """a sparse 3 x 4 grid with an identity baby, an identity giant and a repeated element (3 as baby and giant)"""
    n, bound_w = 64, 4
    mods, s, _, _ = hybrid_case(port, L, K, alpha, n, 40 + L)
    babies, giants = [1, 3, 2 * n - 1, 3], [1, 9, 3]
    bkeys = _galois_keys(port, s, mods, L, K, alpha, n, babies, 9)
    bkeys[0] = None
    gkeys = _galois_keys(port, s, mods, L, K, alpha, n, giants, 31)
    gkeys[0] = None
    swapped = [None, gkeys[2], gkeys[1]]
    present = {(0, 1), (0, 2), (1, 0), (1, 1), (1, 3), (2, 0), (2, 2), (2, 3)}
    one = [1] + [0] * (n - 1)
    for level in sorted({L, L - 1}):
        basis = mods[:level] + mods[L:L + K]
        _, w = hr.small_diagonals(port, basis, n, len(babies) * len(giants), bound_w, level)
        w = w.reshape(len(giants), len(babies), -1)
        grid = [[w[j, i] if (j, i) in present else None for i in range(len(babies))] for j in range(len(giants))]
        ct = _ciphertext(mods, level, n, 3 + level)
        ph = _phase(port, ct, n, level, mods, s)
        exp = np.zeros(level * n, dtype=U64)
        for j, h in enumerate(giants):
            inner = np.zeros(level * n, dtype=U64)
            for i, b in enumerate(babies):
                if grid[j][i] is None:
                    continue
                rot = gx.sigma_ntt(ph, n, b)
                for r, q in enumerate(mods[:level]):
                    dst = slice(r * n, (r + 1) * n)
                    inner[dst] = port.add_mod(inner[dst], port.mult_mod(grid[j][i][dst], rot[dst], q), q)
            rot = gx.sigma_ntt(inner, n, h)
            for r, q in enumerate(mods[:level]):
                dst = slice(r * n, (r + 1) * n)
                exp[dst] = port.add_mod(exp[dst], rot[dst], q)
        for rescale in (False, True):
            out_level = level - int(rescale)
            ref = _rescaled(port, exp, n, level, mods) if rescale else exp
            bound = bsgs_bound(mods, L, K, alpha, level, n, 8, grid, [k is not None for k in bkeys],
                               [k is not None for k in gkeys], bound_w, rescale)
            res = bx.bsgs_exact(port, ct, n, level, L, K, alpha, mods, babies, bkeys, giants, gkeys, grid, rescale)
            got = hx.noise(port, res, ref, s, one, n, out_level, mods)
            assert got <= bound, f"level {level} rescale {rescale}: noise {got} above {bound}"
            res = bx.bsgs_exact(port, ct, n, level, L, K, alpha, mods, babies, bkeys, giants, swapped, grid, rescale)
            assert hx.noise(port, res, ref, s, one, n, out_level, mods) > bound << 20, f"level {level} {rescale}"


# ------------------------------------------------------------------------------------------------ compiler report
def test_bsgs_sum_kernel_keeps_no_local_memory():
    res = {name: r for name, r in kernel_resources("seal.cu").items() if "ks_bsgs_sum_kernel" in name}
    assert len(res) == 1, f"expected one ks_bsgs_sum_kernel, found {sorted(res)}"
    for name, (frame, st, ld) in res.items():
        assert frame == 0 and st == 0 and ld == 0, f"{name}: {frame} B stack frame, {st} B spill stores, {ld} B loads"
