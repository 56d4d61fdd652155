"""The exact element-wise model (tests/eltwise_exact.py) against the checkers, and where the checkers are wrong.
CPU only.

The GPU tests of the element-wise kernels compare against the exact model, so the model is pinned here: below 2^61,
on the operands the GPU tests use, it equals the C restatement and the compiled reference word for word.  Above that
the checkers are not exact, so they cannot say what the right answer is:
  * at the 62-bit witness primes the generalised Barrett product of the C restatement and of the reference's scalar
    tier leaves words in [q, 2q), while the reference's AVX-512 tier (which reduces from [0, 4q)) is exact;
  * ReduceMod with input_mod_factor 4 and q >= 2^63 subtracts 2q, which wraps, in every tier."""
import numpy as np
import pytest

import eltwise_exact as ee

W = ee.BARRETT_62_BIT_WITNESSES
ONE_OF_EACH = [3, (1 << 30) + 3, ee.prime_below(1 << 32), ee.prime_above(1 << 56), ee.prime_below(1 << 60),
               *ee.COMPOSITE_MODULI]


class _Scalar:
    """the compiled reference's scalar tier (its AVX-512 CmpSubMod gets 64-bit inputs wrong at q = 3, for one)"""

    def __init__(self, ref):
        self.ref, self.has_seal = ref, ref.has_seal

    def __getattr__(self, name):
        fn = getattr(self.ref, name)
        return fn if name == "dyadic_multiply" else (lambda *a: fn(*a, native=True))


@pytest.mark.parametrize("q", ONE_OF_EACH, ids=str)
@pytest.mark.parametrize("checker_kind", ["port", "ref"])
def test_exact_model_equals_checkers_below_2_61(request, port, checker_kind, q):
    checker = port if checker_kind == "port" else _Scalar(request.getfixturevalue("ref"))
    n = 4099
    for in_mf in (1, 2, 4):
        a, b = ee.operands(q, in_mf * q, in_mf, n)
        assert (ee.mult_mod(a, b, q) == checker.mult_mod(a, b, q, in_mf)).all(), in_mf
    for in_mf in (1, 2, 4, 8):
        a, c = ee.operands(q, in_mf * q, 10 + in_mf, n)
        for s in (in_mf * q - 1, q - 1, 0):
            assert (ee.fma_mod(a, s, c, q) == checker.fma_mod(a, s, c, q, in_mf)).all(), (in_mf, s)
            assert (ee.fma_mod(a, s, None, q) == checker.fma_mod(a, s, None, q, in_mf)).all(), (in_mf, s)
    a, b = ee.operands(q, q, 20, n)
    assert (ee.add_mod(a, b, q) == checker.add_mod(a, b, q)).all()
    assert (ee.sub_mod(a, b, q) == checker.sub_mod(a, b, q)).all()
    assert (ee.add_mod(a, q - 1, q) == checker.add_mod(a, q - 1, q)).all()
    assert (ee.sub_mod(a, q - 1, q) == checker.sub_mod(a, q - 1, q)).all()
    x, _ = ee.operands(q, 1 << 64, 30, n)
    for cmp in range(8):
        assert (ee.cmp_sub_mod(x, q, cmp, q, q - 1) == checker.cmp_sub_mod(x, q, cmp, q, q - 1)).all(), cmp
        assert (ee.cmp_add(x, cmp, 1 << 63, (1 << 64) - 1) == checker.cmp_add(x, cmp, 1 << 63, (1 << 64) - 1)).all()
    for in_mf in (2, 4):
        x, _ = ee.operands(q, in_mf * q, 40 + in_mf, n)
        exp = ee.reduce_mod(x, q)
        assert (exp == checker.reduce_mod(x, q, in_mf, 1)).all(), in_mf
        assert ee.wrong_lazy_words(checker.reduce_mod(x, q, 4, 2), exp, q) == 0, in_mf
    m = [q, ee.prime_below(1 << 50)]
    op1 = np.concatenate([ee.operands(p, p, 50 + i, 64)[0] for i, p in enumerate(m * 2)])
    op2 = np.concatenate([ee.operands(p, p, 60 + i, 64)[1] for i, p in enumerate(m * 2)])
    if getattr(checker, "has_seal", True):
        assert (ee.dyadic_multiply(op1, op2, 64, m) == checker.dyadic_multiply(op1, op2, 64, m)).all()


def _unreduced(got, exp, q):
    """words the checker got wrong, asserting each is the exact result plus q"""
    wrong = np.asarray(got) != exp
    assert (got[wrong] == exp[wrong] + np.uint64(q)).all()
    return int(wrong.sum())


@pytest.mark.parametrize("q", W, ids=str)
def test_scalar_product_leaves_unreduced_words_at_the_witnesses(port, request, q):
    """The C restatement and the reference's scalar tier (native=True) leave some products of operands near q in
    [q, 2q), for input_mod_factor 1 and 2."""
    tiers = [("C restatement", lambda a, b, m: port.mult_mod(a, b, q, m))]
    import oracle
    if oracle.Ref.available():
        ref = request.getfixturevalue("ref")
        tiers.append(("reference scalar tier", lambda a, b, m: ref.mult_mod(a, b, q, m, native=True)))
    for in_mf in (1, 2):
        a, b = ee.operands(q, in_mf * q, in_mf, 4099)
        exp = ee.mult_mod(a, b, q)
        for name, fn in tiers:
            assert _unreduced(fn(a, b, in_mf), exp, q) > 0, (name, in_mf)


@pytest.mark.parametrize("q", W, ids=str)
def test_avx512_product_is_exact_at_the_witnesses(ref, q):
    """n is a multiple of 8: the reference hands the first n mod 8 elements to its scalar tier"""
    if not ref.avx512 or not ref.L.ref_has_avx512dq():
        pytest.skip("the compiled reference has no AVX-512DQ tier on this host")
    for in_mf in (1, 2):
        a, b = ee.operands(q, in_mf * q, in_mf, 4096)
        assert (ref.mult_mod(a, b, q, in_mf) == ee.mult_mod(a, b, q)).all(), in_mf


EDGE_64 = np.array([100, 0, 1, (1 << 63) - 1, 1 << 63, (1 << 64) - 2, (1 << 64) - 1], dtype=np.uint64)


def test_reduce_mod_4_above_2_63_is_wrong_in_every_tier(port, request):
    """q = 2^63 + 5: subtracting 2q wraps, so some results are not even congruent to their inputs (100 -> 90)"""
    q = (1 << 63) + 5
    exp = ee.reduce_mod(EDGE_64, q)
    tiers = [("C restatement", lambda mf: port.reduce_mod(EDGE_64, q, 4, mf))]
    import oracle
    if oracle.Ref.available():
        ref = request.getfixturevalue("ref")
        tiers += [("reference scalar tier", lambda mf: ref.reduce_mod(EDGE_64, q, 4, mf, native=True)),
                  ("reference dispatch", lambda mf: ref.reduce_mod(EDGE_64, q, 4, mf))]
    for name, fn in tiers:
        got = fn(1)
        assert got[0] == 90, name
        assert ee.wrong_words(got, exp) > 0, name
        assert ee.wrong_lazy_words(fn(2), exp, q) > 0, name
