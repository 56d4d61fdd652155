"""The multi-modulus transforms (ComputeForwardMulti / ComputeInverseMulti, and PolyMultiplyMulti, whose transforms
are the same kernels) against the checker at every degree from 2 to 2^20, with every lazy input and output factor.

Every composite of the library (KeySwitch, DivideAndRoundQLast, PolyMultiplyMulti) runs on these kernels.  The shapes
reach each of their paths: N = 2, 4, 8 take one thread per polynomial; N = 16 to 2^13 a row kernel alone, whose CTAs
hold rows of several polynomials below N = 4096, under different moduli when a group is one polynomial; N = 2^14 to
2^17 one column pass before it (of 2 bits at 2^14); N = 2^18 to 2^20 two column passes, the second over sub-blocks
smaller than a polynomial; and the forward of 64 or more polynomials at N = 2^17 is one pipelined launch.  The moduli lists
(tests/ntt_exact.py) put each arithmetic mode at its edges: FAST just above 2^32 and just below 2^56, WIDE with moduli
below 2^32 and below 2^30 beside one just below 2^61, and GENERIC from just below 2^62 down to below 2^30.  Inputs hold
polynomials at in_mf * q - 1, 0 alternating with that value, and uniform below in_mf * q.  tests/test_ntt_exact.py pins
the checker to the exact model at these moduli and inputs.

Canonical outputs must equal the checker word for word; lazy outputs must be congruent to it and below out_mf * q."""
import numpy as np
import pytest

import ntt_exact as nx
from test_gpu_north_star import PIPE_SPREAD, _multi_mode

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

U64 = np.uint64
LOGNS = [1, 2, 3, 4, 8, 11, 13, 14, 15, 16, 17, 18, 19, 20]
# one degree per kernel shape for the host-pointer calls: tiny, row kernel alone, one column pass, two column passes
HOST_LOGNS = (3, 11, 15, 19)
SPECS = dict(nx.MODULUS_LISTS)
MODES = {"fast_edges": "fast", "wide_small": "wide", "small_only": "wide", "generic_mixed": "generic"}
FWD_FACTORS = ((1, 2, 4), (1, 4))   # (input factors, output factors)
INV_FACTORS = ((1, 2), (1, 2))


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=U64).view(np.int64)).to("cuda")


def host(t):
    return t.cpu().numpy().view(U64)


@pytest.fixture(scope="module", autouse=True)
def _need_cuda(hb):
    if not torch.cuda.is_available() or hb.device_count() == 0:
        pytest.fail("gpu-marked test collected on a machine without CUDA")


def _moduli(hb, name):
    mods = nx.moduli(hb.GeneratePrimes, SPECS[name])
    assert _multi_mode(mods) == MODES[name], (name, mods)
    return mods


def _expected(checker, fwd, x, n, mods, group, in_mf):
    """the checker's canonical output for every modulus block of x"""
    sz = group * n
    run = checker.ntt_forward if fwd else checker.ntt_inverse
    return np.concatenate([run(x[i * sz:(i + 1) * sz], n, q, in_mf, 1) for i, q in enumerate(mods)])


def _check(got, exp, mods, sz, out_mf, what):
    got = np.asarray(got)
    if out_mf == 1:
        wrong = int((got != exp).sum())
    else:
        qv = np.repeat(np.array(mods, dtype=U64), sz)
        wrong = int(((got % qv != exp) | (got >= U64(out_mf) * qv)).sum())
    assert wrong == 0, f"{what}: {wrong} of {exp.size} words wrong"


@pytest.mark.parametrize("logn", LOGNS)
@pytest.mark.parametrize("name", list(MODES))
def test_multi_transforms_match_checker(hb, checker, name, logn):
    """groups of 1 and 3 polynomials per modulus, every factor pair, on a non-default stream out of place and in place;
    host pointers at one degree per kernel shape"""
    n = 1 << logn
    mods = _moduli(hb, name)
    ntts = [hb.NTT(n, q) for q in mods]
    s = torch.cuda.Stream()
    for group in (1, 3):
        sz = group * n
        for fwd, (in_mfs, out_mfs) in ((True, FWD_FACTORS), (False, INV_FACTORS)):
            call = hb.ComputeForwardMulti if fwd else hb.ComputeInverseMulti
            for in_mf in in_mfs:
                x = nx.operand(100 * logn + 10 * group + in_mf + (0 if fwd else 5), n, mods, group, in_mf)
                exp = _expected(checker, fwd, x, n, mods, group, in_mf)
                for out_mf in out_mfs:
                    what = f"{'fwd' if fwd else 'inv'} {name} n=2^{logn} group={group} in_mf={in_mf} out_mf={out_mf}"
                    with torch.cuda.stream(s):
                        d = dev(x)
                        o = torch.zeros_like(d)
                        call(ntts, o, d, in_mf, out_mf, batch_per_modulus=group, stream=s)
                    s.synchronize()
                    _check(host(o), exp, mods, sz, out_mf, what)
                    assert (host(d) == x).all(), f"{what}: the operand was modified"
                    with torch.cuda.stream(s):
                        call(ntts, d, d, in_mf, out_mf, batch_per_modulus=group, stream=s)
                    s.synchronize()
                    _check(host(d), exp, mods, sz, out_mf, f"{what} in place")
                if logn in HOST_LOGNS and group == 3:
                    h = np.zeros_like(x)
                    call(ntts, h, x, in_mf, 1, batch_per_modulus=group)
                    _check(h, exp, mods, sz, 1, f"{'fwd' if fwd else 'inv'} {name} n=2^{logn} in_mf={in_mf} host")


def test_multi_transforms_cross_a_parameter_block(hb, checker):
    """66 moduli just below 2^61 at N = 2^18 (two column passes): the last two take a second 64-entry parameter block"""
    n = 1 << 18
    mods = hb.GeneratePrimes(66, 60, False, n)
    assert len(set(mods)) == 66 and _multi_mode(mods) == "wide"
    ntts = [hb.NTT(n, q) for q in mods]
    for fwd, in_mf, out_mf in ((True, 4, 4), (False, 2, 2)):
        x = nx.operand(7 + in_mf, n, mods, 1, in_mf)
        exp = _expected(checker, fwd, x, n, mods, 1, in_mf)
        d = dev(x)
        (hb.ComputeForwardMulti if fwd else hb.ComputeInverseMulti)(ntts, d, d, in_mf, out_mf, batch_per_modulus=1)
        _check(host(d), exp, mods, n, out_mf, f"{'fwd' if fwd else 'inv'} 66 moduli in_mf={in_mf} out_mf={out_mf}")


@pytest.mark.parametrize("name", list(MODES))
def test_multi_forward_n17_pipelined_lazy_inputs(hb, checker, name):
    """the pipelined forward (64 or more polynomials at N = 2^17, one launch) on inputs below 4q"""
    n = 1 << 17
    mods = _moduli(hb, name)
    group = -(-64 // len(mods))
    ntts = [hb.NTT(n, q).Prepare() for q in mods]
    x = nx.operand(17, n, mods, group, 4)
    exp = {u: checker.ntt_forward(x[u * n:(u + 1) * n], n, mods[u // group], 4, 1) for u in PIPE_SPREAD}
    d = dev(x)
    o = torch.zeros_like(d)
    for out_mf in (1, 4):
        launches = hb.launch_count()
        hb.ComputeForwardMulti(ntts, o, d, 4, out_mf, batch_per_modulus=group)
        assert hb.launch_count() - launches == 1
        got = host(o)
        for u in PIPE_SPREAD:
            q = mods[u // group]
            _check(got[u * n:(u + 1) * n], exp[u], [q], n, out_mf, f"{name} unit {u} out_mf={out_mf}")


@pytest.mark.parametrize("logn", [14, 18, 20])
@pytest.mark.parametrize("name", ["fast_edges", "wide_small"])
def test_poly_multiply_multi_extremes(hb, checker, name, logn):
    """the inverse that multiplies on load, then the column passes, with operands at q - 1"""
    n, group = 1 << logn, 3
    mods = _moduli(hb, name)
    ntts = [hb.NTT(n, q) for q in mods]
    sz = group * n
    parts_a, parts_b = [], []
    for i, q in enumerate(mods):
        a = nx.polynomial("uniform", 40 + i, sz, q)
        b = nx.polynomial("uniform", 50 + i, sz, q)
        a[:n] = q - 1                      # first polynomial: all q-1 times all q-1
        b[:n] = q - 1
        b[n:n + n // 2] = 0                # second: zeros, ones and q-1 mixed with random values
        b[n + n // 2:2 * n] = 1
        a[n:2 * n:2] = q - 1
        parts_a.append(a)
        parts_b.append(b)
    a, b = np.concatenate(parts_a), np.concatenate(parts_b)
    conv = np.concatenate([
        checker.ntt_inverse(checker.mult_mod(checker.ntt_forward(a[i * sz:(i + 1) * sz], n, q),
                                             checker.ntt_forward(b[i * sz:(i + 1) * sz], n, q), q), n, q)
        for i, q in enumerate(mods)])
    o = dev(np.zeros_like(a))
    hb.PolyMultiplyMulti(ntts, o, dev(a), dev(b), group)
    _check(host(o), conv, mods, sz, 1, f"poly multiply {name} n=2^{logn}")
