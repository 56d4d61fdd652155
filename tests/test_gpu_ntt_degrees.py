"""The single-modulus transforms (NTT::ComputeForward / ComputeInverse) against the checker at every degree from 2 to
2^20, at primes on both sides of every boundary between arithmetic modes, with every lazy input and output factor.

This is the library's headline path, and every host-pointer RNS call, the rescale and the key switch's mod-down run
through it too.  The cases (tests/ntt_plan.py) launch every kernel ntt.cu compiles, which tests/test_ntt_plan.py
checks against the compiler's report:
- N = 2, 4, 8: one stage kernel per stage.  N = 16 .. 2^13: one row kernel, with 4096 / N polynomials per CTA below
  N = 4096, so batches of 4096 / N + 1 fill one CTA and leave one row in the next.
- N = 2^14 .. 2^17: the single-pass kernels (distributed shared memory, fused through L2, pipelined from 64
  polynomials on) or the split of one radix-32 column pass and a row kernel; N = 2^18 .. 2^20: two column passes.
- Each mode has its own kernels: SMALL below 2^30 (32-bit words), GENERIC in [2^30, 2^32) and from 2^61, FAST in
  [2^32, 2^56), WIDE in [2^56, 2^61).  The primes (tests/ntt_exact.py) take each side of each boundary, one mid-range
  prime per mode, and the smallest prime the degree allows.

Inputs hold polynomials at in_mf * q - 1, 0 alternating with that value, and uniform below in_mf * q, with residues
that do not depend on in_mf; tests/test_ntt_exact.py pins the checker to the exact model on them.  Canonical outputs
must equal the checker word for word; lazy outputs must be congruent to it and below out_mf * q.  Device calls run on
a non-default stream, out of place (the operand checked unchanged) and in place, with sentinel words on both sides of
`result`, and launch exactly the kernels of ntt_plan.kernels."""
import numpy as np
import pytest

import ntt_exact as nx
import ntt_plan as plan
from test_gpu_north_star import PIPE_SPREAD

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

U64 = np.uint64
FWD_FACTORS = ((1, 2, 4), (1, 4))   # (input factors, output factors)
INV_FACTORS = ((1, 2), (1, 2))
GUARD = 64                          # sentinel words on each side of `result`: 512 bytes, so its alignment is kept
SENTINEL = U64(0xA5A5_5A5A_C3C3_3C3C)
THREADS = 4                         # checker threads


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=U64).view(np.int64)).to("cuda")


def host(t):
    return t.cpu().numpy().view(U64)


@pytest.fixture(scope="module", autouse=True)
def _need_cuda(hb):
    if not torch.cuda.is_available() or hb.device_count() == 0:
        pytest.fail("gpu-marked test collected on a machine without CUDA")


def _prime(hb, name, logn):
    return dict(nx.single_primes(hb.GeneratePrimes, logn))[name]


def _check(got, exp, q, out_mf, what):
    got = np.asarray(got)
    if out_mf == 1:
        wrong = int((got != exp).sum())
    else:
        wrong = int(((got % U64(q) != exp) | (got >= U64(out_mf * q))).sum())
    assert wrong == 0, f"{what}: {wrong} of {exp.size} words wrong"


def _guarded(size):
    """a device buffer of sentinels and the `size` words between its guard regions"""
    buf = torch.from_numpy(np.full(size + 2 * GUARD, SENTINEL, dtype=U64).view(np.int64)).to("cuda")
    return buf, buf[GUARD:GUARD + size]


def _check_guards(buf, what):
    b = host(buf)
    assert (b[:GUARD] == SENTINEL).all() and (b[-GUARD:] == SENTINEL).all(), f"{what}: written outside `result`"


def _call(hb, ntt, fwd, result, operand, in_mf, out_mf, s, launches):
    """one device call on stream s; it must launch `launches` kernels"""
    before = hb.launch_count()
    with torch.cuda.stream(s):
        (ntt.ComputeForward if fwd else ntt.ComputeInverse)(result, operand, in_mf, out_mf, stream=s)
    assert hb.launch_count() - before == launches
    s.synchronize()


def _device_calls(hb, ntt, q, logn, fwd, x, exp, in_mf, out_mfs, s, what):
    """every output factor, out of place then in place, `result` between guard regions"""
    batch = x.size >> logn
    launches = len(plan.kernels(q, logn, batch, fwd))
    for out_mf in out_mfs:
        w = f"{what} out_mf={out_mf}"
        with torch.cuda.stream(s):
            d = dev(x)
            buf, res = _guarded(x.size)
        _call(hb, ntt, fwd, res, d, in_mf, out_mf, s, launches)
        _check(host(res), exp, q, out_mf, w)
        assert (host(d) == x).all(), f"{w}: the operand was modified"
        _check_guards(buf, w)
        with torch.cuda.stream(s):
            buf, res = _guarded(x.size)
            res.copy_(d)
        _call(hb, ntt, fwd, res, res, in_mf, out_mf, s, launches)
        _check(host(res), exp, q, out_mf, f"{w} in place")
        _check_guards(buf, f"{w} in place")


@pytest.mark.parametrize("logn", plan.LOGNS)
@pytest.mark.parametrize("name", nx.SINGLE_NAMES)
def test_single_modulus_transforms_match_checker(hb, checker, name, logn):
    """batches of 1 and 3 (and a row CTA and one row more below N = 4096), every factor pair; host pointers at one
    degree per kernel shape, for one prime per mode in chunks on both sides of the pipelined forward's threshold at 2^15
    and 2^16"""
    n = 1 << logn
    q = _prime(hb, name, logn)
    ntt = hb.NTT(n, q)
    s = torch.cuda.Stream()
    for fwd, (in_mfs, out_mfs) in ((True, FWD_FACTORS), (False, INV_FACTORS)):
        run = checker.ntt_forward if fwd else checker.ntt_inverse
        for batch in plan.batches(logn):
            seed = 100 * logn + batch + (0 if fwd else 50)
            exp = None
            for in_mf in in_mfs:
                x = nx.single_operand(seed, n, q, batch, in_mf)
                if exp is None:  # the residues, so the transform, are the same at every input factor
                    exp = run(x, n, q, in_mf, 1, threads=THREADS)
                what = f"{'fwd' if fwd else 'inv'} {name} q={q} n=2^{logn} batch={batch} in_mf={in_mf}"
                _device_calls(hb, ntt, q, logn, fwd, x, exp, in_mf, out_mfs, s, what)
            if logn in plan.HOST_LOGNS and batch == 3:
                # the batch of 3 repeated: every polynomial is checked without another checker call
                total = plan.host_batch(logn, name) * n
                xh, eh = np.resize(x, total), np.resize(exp, total)
                h = np.zeros_like(xh)
                before = hb.launch_count()
                (ntt.ComputeForward if fwd else ntt.ComputeInverse)(h, xh, in_mf, 1)
                assert hb.launch_count() - before == sum(
                    len(plan.kernels(q, logn, b, fwd)) for b in plan.host_chunks(logn, plan.host_batch(logn, name)))
                _check(h, eh, q, 1, f"{'fwd' if fwd else 'inv'} {name} n=2^{logn} in_mf={in_mf} host")
                assert (xh == np.resize(x, total)).all()


@pytest.mark.parametrize("logn", plan.DEEP_LOGNS)
@pytest.mark.parametrize("name", plan.DEEP_PRIMES)
def test_forward_at_the_deep_threshold(hb, checker, name, logn):
    """63 and 64 polynomials below 4q: the 64-bit modes take the pipelined forward from 64 on, and below it the kernel
    of distributed shared memory (2^15), the fused kernel (2^16) or the split (2^17); SMALL takes one kernel of
    distributed shared memory at both.  Polynomials cycle through the kinds, so 0, 30, 45 and 63 are at 4q - 1."""
    n = 1 << logn
    q = _prime(hb, name, logn)
    ntt = hb.NTT(n, q)
    s = torch.cuda.Stream()
    x = nx.single_operand(logn, n, q, plan.DEEP, 4)
    spread = np.concatenate([x[u * n:(u + 1) * n] for u in PIPE_SPREAD])
    exp = checker.ntt_forward(spread, n, q, 4, 1, threads=THREADS).reshape(len(PIPE_SPREAD), n)
    with torch.cuda.stream(s):
        d = dev(x)
    for batch in plan.DEEP_BATCHES:
        launches = len(plan.kernels(q, logn, batch, True))
        split = logn == 17 and batch < plan.DEEP and plan.mode(q) != plan.SMALL
        assert launches == (2 if split else 1)
        for out_mf in (1, 4):
            what = f"{name} q={q} n=2^{logn} batch={batch} out_mf={out_mf}"
            with torch.cuda.stream(s):
                buf, res = _guarded(batch * n)
            _call(hb, ntt, True, res, d[:batch * n], 4, out_mf, s, launches)
            got = host(res)
            for i, u in enumerate(PIPE_SPREAD):
                if u < batch:
                    _check(got[u * n:(u + 1) * n], exp[i], q, out_mf, f"{what} polynomial {u}")
            _check_guards(buf, what)


@pytest.mark.parametrize("logn", plan.ROOT_LOGNS)
@pytest.mark.parametrize("name", plan.MODE_PRIMES)
def test_non_minimal_root(hb, name, logn):
    """NTT(n, q, root) with root = (minimal root)^5: the forward of a uniform input below 4q against the exact model
    with that root, then the inverse of that output, made lazy below 2q, back to the input mod q"""
    n = 1 << logn
    q = _prime(hb, name, logn)
    root = hb.PowMod(hb.MinimalPrimitiveRoot(2 * n, q), 5, q)
    ntt = hb.NTT(n, q, root)
    s = torch.cuda.Stream()
    x = nx.single_polynomial("uniform", logn, n, q, 4)
    exp = nx.forward(x, n, q, root)
    lazy = exp + U64(q) * (np.arange(n, dtype=U64) & U64(1))
    with torch.cuda.stream(s):
        res, d, dl = dev(np.zeros_like(x)), dev(x), dev(lazy)
    _call(hb, ntt, True, res, d, 4, 1, s, len(plan.kernels(q, logn, 1, True)))
    _check(host(res), exp, q, 1, f"fwd {name} n=2^{logn} root={root}")
    _call(hb, ntt, False, res, dl, 2, 1, s, len(plan.kernels(q, logn, 1, False)))
    _check(host(res), x % U64(q), q, 1, f"inv {name} n=2^{logn} root={root}")
