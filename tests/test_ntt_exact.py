"""The exact NTT model (tests/ntt_exact.py) against the definition, and the checkers against the model at the moduli and
inputs of the multi-modulus GPU tests.  CPU only.

The GPU tests of the multi-modulus transforms compare against the checkers (the C restatement, or the compiled
reference), so the checkers are pinned here: at every moduli list those tests use, from N = 2 to N = 2^20, on inputs
at in_mf * q - 1, 0 alternating with that value, and uniform below in_mf * q, their canonical outputs equal the model's
word for word.  The same holds at the primes of the single-modulus GPU tests (ntt_exact.SINGLE_PRIMES) that the lists
do not hold, on those tests' inputs."""
import numpy as np
import pytest

import ntt_exact as nx

U64 = np.uint64
LIST_NAMES = [name for name, _ in nx.MODULUS_LISTS]
SPECS = dict(nx.MODULUS_LISTS)
# one modulus per word class of the transforms: FAST, WIDE, GENERIC, and below 2^30
CLASS_MODULI = [("fast_edges", 2), ("wide_small", 0), ("generic_mixed", 0), ("small_only", 0)]


@pytest.mark.parametrize("name,index", CLASS_MODULI, ids=[f"{n}-{i}" for n, i in CLASS_MODULI])
def test_model_equals_the_definition(port, name, index):
    q = nx.moduli(port.generate_primes, SPECS[name])[index]
    for logn in range(1, 7):
        n = 1 << logn
        root = nx.minimal_root(n, q)
        assert root == port.minimal_primitive_root(2 * n, q), (q, n)
        x = nx.operand(logn, n, [q], 3, 4)
        for p in range(3):
            xp = x[p * n:(p + 1) * n]
            fwd = nx.forward(xp, n, q)
            assert (fwd == nx.forward_definition(xp, n, q, root)).all(), (q, n, p)
            assert (nx.inverse(xp, n, q) == nx.inverse_definition(xp, n, q, root)).all(), (q, n, p)
            assert (nx.inverse(fwd, n, q) == xp % U64(q)).all(), (q, n, p)
        # a given root: another primitive 2n-th root (an odd power of the minimal one)
        other = pow(root, 3, q)
        assert (nx.forward(x, n, q, other) == np.concatenate(
            [nx.forward_definition(x[p * n:(p + 1) * n], n, q, other) for p in range(3)])).all(), (q, n)
        assert (nx.forward(x, n, q, other) == port.ntt_forward(x, n, q, 4, 1, root=other)).all(), (q, n)


_model = {}


def _expected(port, name, logn, group, fwd, in_mf):
    """(moduli, operand, model output), computed once for both checkers"""
    key = name, logn, group, fwd, in_mf
    if key not in _model:
        n = 1 << logn
        mods = nx.moduli(port.generate_primes, SPECS[name])
        x = nx.operand(logn, n, mods, group, in_mf)
        sz = group * n
        f = nx.forward if fwd else nx.inverse
        _model[key] = mods, x, np.concatenate([f(x[i * sz:(i + 1) * sz], n, q) for i, q in enumerate(mods)])
    return _model[key]


def _check(chk, port, name, logn, group, fwd, in_mf):
    n = 1 << logn
    mods, x, exp = _expected(port, name, logn, group, fwd, in_mf)
    sz = group * n
    run = chk.ntt_forward if fwd else chk.ntt_inverse
    for i, q in enumerate(mods):
        got = run(x[i * sz:(i + 1) * sz], n, q, in_mf, 1)
        wrong = int((got != exp[i * sz:(i + 1) * sz]).sum())
        assert wrong == 0, f"{chk.kind} {'fwd' if fwd else 'inv'} {name} q={q} n=2^{logn} in_mf={in_mf}: {wrong} words"


def _checker(request, port, kind):
    return port if kind == "port" else request.getfixturevalue("ref")


@pytest.mark.parametrize("checker_kind", ["port", "ref"])
@pytest.mark.parametrize("logn", [1, 2, 3, 4, 8, 11, 14])
@pytest.mark.parametrize("name", LIST_NAMES)
def test_checkers_equal_the_model(request, port, checker_kind, name, logn):
    """every lazy input factor, three polynomials (one of each kind) per modulus"""
    chk = _checker(request, port, checker_kind)
    for in_mf in (1, 2, 4):
        _check(chk, port, name, logn, 3, True, in_mf)
    for in_mf in (1, 2):
        _check(chk, port, name, logn, 3, False, in_mf)


@pytest.mark.parametrize("checker_kind", ["port", "ref"])
@pytest.mark.parametrize("logn", [18, 20])
@pytest.mark.parametrize("name", LIST_NAMES)
def test_checkers_equal_the_model_at_two_column_passes(request, port, checker_kind, name, logn):
    """one polynomial per modulus at the largest input factor, its kind cycling over the moduli"""
    chk = _checker(request, port, checker_kind)
    _check(chk, port, name, logn, 1, True, 4)
    _check(chk, port, name, logn, 1, False, 2)


# the primes of the single-modulus GPU tests that no moduli list above holds
SINGLE_PINNED = ["above_2^30", "above_2^56", "above_2^61", "smallest"]
_single_model = {}


def _single_expected(q, logn, kind, fwd):
    """the model's transform of one polynomial of `kind`; its residues, hence the model, do not depend on in_mf"""
    key = q, logn, kind, fwd
    if key not in _single_model:
        n = 1 << logn
        x = nx.single_polynomial(kind, logn, n, q, 1)
        _single_model[key] = (nx.forward if fwd else nx.inverse)(x, n, q)
    return _single_model[key]


@pytest.mark.parametrize("checker_kind", ["port", "ref"])
@pytest.mark.parametrize("logn", range(1, nx.MAX_LOGN + 1))
def test_checkers_equal_the_model_at_single_primes(request, port, checker_kind, logn):
    """tests/test_gpu_ntt_degrees.py's inputs: every input factor and kind at every degree"""
    chk = _checker(request, port, checker_kind)
    n = 1 << logn
    primes = dict(nx.single_primes(port.generate_primes, logn))
    for name in SINGLE_PINNED:
        q = primes[name]
        for fwd, in_mfs in ((True, (1, 2, 4)), (False, (1, 2))):
            run = chk.ntt_forward if fwd else chk.ntt_inverse
            for kind in nx.KINDS:
                exp = _single_expected(q, logn, kind, fwd)
                for in_mf in in_mfs:
                    got = run(nx.single_polynomial(kind, logn, n, q, in_mf), n, q, in_mf, 1)
                    wrong = int((got != exp).sum())
                    assert wrong == 0, (f"{chk.kind} {'fwd' if fwd else 'inv'} {name} q={q} n=2^{logn} {kind} "
                                        f"in_mf={in_mf}: {wrong} words")
