"""Range and congruence claims of the device arithmetic (hexl_b200/csrc/ntt_kernels.cuh), checked on exact-integer
models of the same word-level formulas (tests/arith_model.py).  No GPU: this is the host-side proof obligation behind
the lazy ranges the kernels use; the GPU parity tests then show the CUDA code computes what the model says."""
import random

import pytest

import arith_model as am
from eltwise_exact import BARRETT_62_BIT_WITNESSES

M64 = am.M64


def _moduli(lo_bits, hi_bits, rng, count=6):
    """odd moduli across [2^lo_bits, 2^hi_bits): the extremes of the range plus random ones"""
    out = [(1 << lo_bits) + 1, (1 << hi_bits) - 1, (1 << hi_bits) - 59, (1 << (hi_bits - 1)) + 1]
    while len(out) < count + 4:
        out.append(rng.randrange(1 << lo_bits, 1 << hi_bits) | 1)
    return out


def _operands(bound, rng, count=200):
    """values below `bound`: its edges, words of all ones / zeros, then random"""
    edge = [0, 1, 2, bound - 1, bound - 2, bound >> 1, (bound >> 1) + 1,
            0xFFFFFFFF, 0x100000000, 0xFFFFFFFF00000000, 0x00000000FFFFFFFF, 0xFFFFFFFFFFFFFFFF, 0x8000000000000000,
            0x7FFFFFFFFFFFFFFF, 0xFFFFFFFEFFFFFFFF]
    vals = [v for v in edge if 0 <= v < bound]
    while len(vals) < count:
        vals.append(rng.randrange(bound))
    return vals


def test_quotient_estimate_is_low_by_at_most_two():
    rng = random.Random(1)
    worst = 0
    for a in _operands(1 << 64, rng, 400):
        for b in _operands(1 << 64, rng, 60):
            d = am.mulhi(a, b) - am.mulhi_approx(a, b)
            assert 0 <= d <= 2
            worst = max(worst, d)
    assert worst == 2  # the bound is attained: the [0,4q) range below is tight in principle


@pytest.mark.parametrize("lo_bits,hi_bits,in_bound_q,approx,out_bound_q", [
    (32, 56, 84, True, 4),    # FAST: forward values grow to 84q, product in [0,4q)
    (56, 61, 8, True, 4),     # WIDE: lazy ranges doubled, three-product quotient
    (2, 62, 4, False, 2),     # GENERIC: Harvey's exact quotient, [0,2q)
])
def test_twiddle_product_ranges(lo_bits, hi_bits, in_bound_q, approx, out_bound_q):
    rng = random.Random(2)
    for q in _moduli(lo_bits, hi_bits, rng):
        assert in_bound_q * q < (1 << 64)
        for w in [1, 2, q - 1, q - 2, q >> 1] + [rng.randrange(1, q) for _ in range(8)]:
            wp = am.shoup(w, q)
            for x in _operands(min(in_bound_q * q, 1 << 64), rng, 60) + _operands(1 << 64, rng, 20):
                r = am.mul_tw(x, w, wp, q, approx)   # valid for ANY 64-bit x (the inverse's folded root stage relies on it)
                assert r < out_bound_q * q and (r - x * w) % q == 0


def test_barrett_variants_reach_their_ranges():
    rng = random.Random(3)
    for q in _moduli(32, 62, rng, 10):
        for x in _operands(1 << 64, rng, 300):
            r2 = am.barrett_lazy_bigq(x, q)
            r3 = am.barrett_lazy3_bigq(x, q)
            rg = am.barrett_lazy(x, q)
            assert r2 < 2 * q and r3 < 3 * q and rg < 2 * q
            assert (r2 - x) % q == 0 and (r3 - x) % q == 0 and (rg - x) % q == 0
    for q in [3, 5, 17, 65537, (1 << 30) - 35, (1 << 31) + 11]:       # generic Barrett below 2^32 as well
        for x in _operands(1 << 64, rng, 100):
            r = am.barrett_lazy(x, q)
            assert r < 2 * q and (r - x) % q == 0


def test_sign_bit_conditional_subtraction():
    rng = random.Random(4)
    for b in [1, 2, (1 << 63) - 1, (1 << 62) + 12345, 4 * ((1 << 56) - 5), 8 * ((1 << 60) - 93)]:
        assert b < (1 << 63)
        for x in _operands(2 * b, rng, 200):
            assert am.csub_s(x, b) == am.csub(x, b)


@pytest.mark.parametrize("lo_bits,hi_bits,approx,out_bound_q",
                         [(32, 56, True, 4), (56, 61, True, 4), (3, 61, False, 2), (61, 62, False, 3)])
def test_product_multiplied_on_load_ranges(lo_bits, hi_bits, approx, out_bound_q):
    """prod_lazy: canonical operands -> [0,2q) with the exact quotient for every q < 2^61 (all PolyMultiplyMulti
    accepts), [0,4q) with the three-product estimate; at 62 bits the exact quotient's estimate can be low by two, so
    only [0,3q) holds.  The 128-bit product and the shifted word c1 are formed without losing
    bits for every q < 2^62."""
    rng = random.Random(5)
    witnesses = [q for q in BARRETT_62_BIT_WITNESSES if (1 << lo_bits) <= q < (1 << hi_bits)]
    for q in _moduli(lo_bits, hi_bits, rng, 8) + witnesses:
        for x in _operands(q, rng, 40):
            for y in _operands(q, rng, 40):
                r = am.prod_lazy(x, y, q, approx)
                assert r < out_bound_q * q and (r - x * y) % q == 0


def test_fast_forward_growth_stays_below_2_63():
    # FAST forward: X' = X + T, Y' = X + 4q - T with T < 4q: +4q per stage, inputs < 4q (in_mf <= 4), at most 20 stages
    q = (1 << 56) - 1
    bound = 4
    for _ in range(20):
        bound += 4
    assert bound == 84 and bound * q < (1 << 63)


@pytest.mark.parametrize("K", [1, 2, 3, 4])
def test_fast_inverse_slot_bounds(K):
    bounds, worst, cover_ok = am.simulate_inverse_pass_bounds(K)
    assert cover_ok                                   # the multiple of q added before each subtraction covers Y
    for e, b in enumerate(bounds):
        assert b == am.inv_slot_bound(K, e & ((1 << K) - 1))
    assert worst * ((1 << 56) - 1) < (1 << 64)        # largest transient (128q at K = 4; the kernel header budgets 256q) fits 64 bits
    over = [e for e, b in enumerate(bounds) if b > am.K_FAST_BOUND]
    if K == 4:
        assert len(over) == 4 and worst == 128        # the 4 of 16 slots the pass-boundary fix-up reduces
    # after the fix-up (barrett_lazy3_bigq -> < 3q) every slot is below 8q again: the next pass may start
    assert all(min(b, 3) <= am.K_FAST_BOUND for b in bounds)


def test_small_mode_words():
    rng = random.Random(6)
    for q in [3, 5, 12289, (1 << 29) + 11, (1 << 30) - 35]:
        for w in [1, q - 1, q >> 1] + [rng.randrange(1, q) for _ in range(6)]:
            for x in _operands(1 << 32, rng, 120):
                r = am.mul_tw32(x, w, q)                      # any 32-bit x -> [0,2q)
                assert r < 2 * q and (r - x * w) % q == 0
        for c in [q, 2 * q]:
            for x in _operands(2 * c, rng, 100):
                assert am.csub32(x, c) == am.csub(x, c)       # min(x, x - c) with wrap-around == conditional subtraction


@pytest.mark.parametrize("r", [30, 46, 61, 62])
def test_montgomery_reduction(r):
    rng = random.Random(7)
    R = 1 << r
    for q in [3, (1 << (r - 1)) - 1 | 1, R - 1 if (R - 1) % 2 else R - 3] + [rng.randrange(3, R) | 1 for _ in range(6)]:
        if q >= R or q % 2 == 0:
            continue
        Rinv = pow(R, -1, q)
        for _ in range(300):
            a, b = rng.randrange(q), rng.randrange(q)
            t = a * b
            assert am.redc(t >> 64, t & M64, q, r) == (t * Rinv) % q
        for t in [0, 1, q - 1, q * R - 1, (q - 1) * (q - 1), R, R - 1]:
            if t < q * R:
                assert am.redc(t >> 64, t & M64, q, r) == (t * Rinv) % q


@pytest.mark.parametrize("in_mf", [1, 2, 4])
def test_eltwise_generalised_barrett(in_mf):
    """exact for every q < 2^62 with in_mf * q < 2^63, the 62-bit witnesses included, where operands within 2^20 of q
    need the second conditional subtraction"""
    rng = random.Random(8)
    qs = [3, 5, 65537, (1 << 40) + 15, (1 << 50) - 27, (1 << 60) - 93, (1 << 61) - 1, (1 << 62) - 57]
    qs += list(BARRETT_62_BIT_WITNESSES)
    for q in qs:
        if in_mf * q >= (1 << 63):
            continue
        band = [q - 1 - rng.randrange(min(q, 1 << 20)) for _ in range(40)]
        for a in _operands(in_mf * q, rng, 40) + band:
            for b in _operands(in_mf * q, rng, 40) + band:
                assert am.eltwise_mult(a, b, q, in_mf) == (a * b) % q, (a, b, q)


def test_key_switch_mac_chunk_never_wraps():
    """A ks_mac_kernel launch adds up at most J(q) products of (lazy transform output < 4q) x (key word < q) in 128 bits,
    q the largest modulus of the launch.  J(q) = 64 (the parameter block) for every q < 2^60; above 2^60 it shrinks so
    the sum still fits, and it is as large as it can be (one more product of the largest operands would wrap)."""
    rng = random.Random(10)
    qs = [3, 5, (1 << 32) + 15, (1 << 50) - 27, (1 << 60) - 93, (1 << 60) - 1, 1 << 60, (1 << 60) + 1,
          (1 << 60) + (1 << 59), (1 << 61) - 59, (1 << 61) - 1]
    qs += [rng.randrange(3, 1 << 61) for _ in range(2000)] + [rng.randrange(1 << 60, 1 << 61) for _ in range(2000)]
    prev = None
    for q in sorted(qs):
        J = am.ks_mac_digits_per_launch(q)
        largest = (4 * q - 1) * (q - 1)
        assert 16 <= J <= 64 and J * largest < (1 << 128), q
        assert J == 64 or (J + 1) * largest >= (1 << 128), q
        if q < (1 << 60):
            assert J == 64, q
        assert prev is None or J <= prev     # a larger modulus never allows more digits
        prev = J
        assert am.ks_mac_finish(J * largest, q) == (J * largest) % q
    assert am.ks_mac_digits_per_launch((1 << 61) - 1) == 16


def test_key_switch_glue():
    rng = random.Random(9)
    for q in [(1 << 32) + 15, (1 << 50) - 27, (1 << 60) - 93, (1 << 61) - 1]:
        # at most ks_mac_digits_per_launch(q) summands per launch, each (lazy transform output < 4q) x (key word < q),
        # so the accumulator is any value below 2^128; the reference adds up ALL digits in 128 bits without reduction
        # (key-switch-internal.cpp:93-113), which wraps for q > 2^60 and more than 16 digits
        for acc in [0, 1, (1 << 64) - 1, 1 << 64, (1 << 128) - 1] + [rng.randrange(1 << 128) for _ in range(300)]:
            assert am.ks_mac_finish(acc, q) == acc % q
        for _ in range(300):
            prod, t, ms = rng.randrange(q), rng.randrange(4 * q), rng.randrange(q)
            assert am.ks_finish(prod, t, ms, q) == ((prod - t) * ms) % q
        assert am.ks_finish(0, 4 * q - 1, q - 1, q) == ((-(4 * q - 1)) * (q - 1)) % q
