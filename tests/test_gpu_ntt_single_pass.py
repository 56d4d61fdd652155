"""The single-pass transforms of 64-bit moduli at N = 2^14..2^17, at the launch choice the library makes by default.

At N = 2^14..2^16 each transform is one kernel: the one that keeps the whole polynomial in its cluster's shared memory
(N = 2^14, the 2^15 inverse, the 2^15 forward of shallow batches), the pipelined one (the 2^15 and 2^16 forward of
batches of 64 or more) or the cluster kernel whose intermediate goes through L2 (the 2^16 inverse, and the forward of
shallow batches).  At N = 2^17 the forward of 64 or more polynomials is the pipelined kernel too; the 2^17 inverse, and
the forward of shallow batches, are the two-kernel split.  These tests hold those paths to the checker at the edges of
every 64-bit arithmetic mode (FAST just above 2^32 and just below 2^56, WIDE, GENERIC just below 2^62), for lazy and
extreme inputs, in place, for a single polynomial, a few, and a grid many waves deep (where the 2^15..2^17 forward
is one pipelined launch), and at the benchmark's own shape; and they hold the kernels to registers in the ptxas report.
"""
import numpy as np
import pytest

from test_kernel_resources import kernel_resources
from util import uniform_below

torch = pytest.importorskip("torch")

LOGNS = [14, 15, 16]
# (name, bits, first): GeneratePrimes(1, bits, first, n) -- just above 2^bits when `first`, else just below 2^(bits+1)
MODULI = [("bench55", 55, True), ("fast_low", 32, True), ("fast_high", 55, False), ("wide60", 60, True),
          ("generic62", 61, False)]
# batch 1000: the polynomials compared with the checker (first, last, and across the grid's waves)
SPREAD = [0, 1, 2, 127, 128, 333, 500, 511, 512, 777, 998, 999]


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64)).cuda()


def host(t):
    return t.cpu().numpy().view(np.uint64)


def modulus(hb, n, bits, first):
    q = hb.GeneratePrimes(1, bits, first, n)[0]
    assert q >= 1 << 32 and q < 1 << 62
    return q


@pytest.mark.gpu
@pytest.mark.parametrize("logn", LOGNS)
@pytest.mark.parametrize("name,bits,first", MODULI, ids=[m[0] for m in MODULI])
def test_single_pass_matches_checker(hb, checker, logn, name, bits, first):
    n = 1 << logn
    q = modulus(hb, n, bits, first)
    qq = np.uint64(q)
    t = hb.NTT(n, q)
    seed = logn * 100 + bits
    for batch in (1, 3):
        for out_mf in (1, 4):
            x = uniform_below(seed + out_mf, n * batch, q)
            exp = checker.ntt_forward(x, n, q, 1, 1)
            o = dev(np.zeros_like(x))
            t.ComputeForward(o, dev(x), 1, out_mf)
            got = host(o)
            if out_mf == 1:
                assert (got == exp).all(), ("fwd", name, logn, batch, int((got != exp).sum()))
            else:
                assert (got % qq == exp).all() and (got < np.uint64(4 * q)).all(), ("fwd lazy", name, logn, batch)
        for in_mf in (1, 2):
            x = uniform_below(seed + 10 * in_mf, n * batch, q * in_mf)
            exp = checker.ntt_inverse(x, n, q, in_mf, 1)
            for out_mf in (1, 2):
                o = dev(np.zeros_like(x))
                t.ComputeInverse(o, dev(x), in_mf, out_mf)
                got = host(o)
                if out_mf == 1:
                    assert (got == exp).all(), ("inv", name, logn, batch, in_mf, int((got != exp).sum()))
                else:
                    assert (got % qq == exp).all() and (got < np.uint64(2 * q)).all(), ("inv lazy", name, logn, in_mf)
        # in place: result == operand
        x = uniform_below(seed + 7, n * batch, q)
        d = dev(x)
        t.ComputeForward(d, d, 1, 1)
        assert (host(d) == checker.ntt_forward(x, n, q)).all(), ("fwd in place", name, logn, batch)
        t.ComputeInverse(d, d, 1, 1)
        assert (host(d) == x).all(), ("round trip in place", name, logn, batch)


@pytest.mark.gpu
@pytest.mark.parametrize("logn", LOGNS)
@pytest.mark.parametrize("name,bits,first", MODULI, ids=[m[0] for m in MODULI])
def test_single_pass_extreme_inputs(hb, checker, logn, name, bits, first):
    """every coefficient at in_mf * q - 1: the largest lazy growth inside the kernels"""
    n = 1 << logn
    q = modulus(hb, n, bits, first)
    t = hb.NTT(n, q)
    for in_mf in (1, 4):
        x = np.full(n, q * in_mf - 1, dtype=np.uint64)
        o = dev(np.zeros_like(x))
        t.ComputeForward(o, dev(x), in_mf, 1)
        assert (host(o) == checker.ntt_forward(x, n, q, in_mf, 1)).all(), ("fwd extreme", name, logn, in_mf)
    for in_mf in (1, 2):
        x = np.full(n, q * in_mf - 1, dtype=np.uint64)
        o = dev(np.zeros_like(x))
        t.ComputeInverse(o, dev(x), in_mf, 1)
        assert (host(o) == checker.ntt_inverse(x, n, q, in_mf, 1)).all(), ("inv extreme", name, logn, in_mf)


@pytest.mark.gpu
@pytest.mark.parametrize("logn", LOGNS + [17])
@pytest.mark.parametrize("name,bits,first", MODULI, ids=[m[0] for m in MODULI])
def test_single_pass_many_waves(hb, checker, logn, name, bits, first):
    """1000 polynomials: a grid several waves deep.  The forward is one launch (the pipelined kernel from N = 2^15 on;
    at 2^17 the split would be two)."""
    n, batch = 1 << logn, 1000
    q = modulus(hb, n, bits, first)
    t = hb.NTT(n, q).Prepare()
    g = torch.Generator(device="cuda").manual_seed(logn * 1000 + bits)
    x = torch.randint(0, q, (batch, n), dtype=torch.int64, device="cuda", generator=g)
    y = torch.empty_like(x)
    launches = hb.launch_count()
    t.ComputeForward(y, x, 1, 1)
    assert hb.launch_count() - launches == 1, ("fwd launches", name, logn)
    xs = host(x[SPREAD]).reshape(-1)
    assert (host(y[SPREAD]).reshape(-1) == checker.ntt_forward(xs, n, q)).all(), ("fwd", name, logn)
    z = torch.empty_like(x)
    t.ComputeInverse(z, y, 1, 1)
    assert torch.equal(z, x), ("round trip", name, logn)
    t.ComputeInverse(y, y, 1, 1)
    assert torch.equal(y, x), ("round trip in place", name, logn)
    u = torch.randint(0, 2 * q, (batch, n), dtype=torch.int64, device="cuda", generator=g)
    t.ComputeInverse(z, u, 2, 1)
    us = host(u[SPREAD]).reshape(-1)
    assert (host(z[SPREAD]).reshape(-1) == checker.ntt_inverse(us, n, q, 2, 1)).all(), ("inv", name, logn)


@pytest.mark.gpu
def test_benchmark_shape(hb, checker):
    """bench.py's flagship step: 8192 polynomials at N = 2^16 under its 55-bit prime"""
    n, batch = 1 << 16, 8192
    q = hb.GeneratePrimes(1, 55, True, n)[0]
    t = hb.NTT(n, q)
    g = torch.Generator(device="cuda").manual_seed(42)
    x = torch.randint(0, q, (batch, n), dtype=torch.int64, device="cuda", generator=g)
    y = torch.empty_like(x)
    t.ComputeForward(y, x, 1, 1)
    spread = torch.linspace(0, batch - 1, 64).round().long().cuda()
    xs = host(x[spread]).reshape(-1)
    assert (host(y[spread]).reshape(-1) == checker.ntt_forward(xs, n, q)).all()
    t.ComputeInverse(y, y, 1, 1)
    assert torch.equal(y, x)


# ntt_dsmem_fwd / ntt_dsmem_inv <kFast, 2 / 3>: the distributed-shared-memory kernels of 64-bit words (N = 2^14, 2^15);
# ntt_pipe_fwd<kFast, 4>: the forward at the benchmark's shape.  (Its inverse, ntt_fused_inv<kFast, 4>, has a genuine
# 24-byte spill, which test_kernel_resources.py allows.)
SINGLE_PASS = ["13ntt_dsmem_fwdILi1ELi2EE", "13ntt_dsmem_invILi1ELi2EE", "13ntt_dsmem_fwdILi1ELi3EE",
               "13ntt_dsmem_invILi1ELi3EE", "12ntt_pipe_fwdILi1ELi4EE"]
MAX_FRAME = 16


def test_single_pass_kernels_stay_in_registers():
    res = kernel_resources("ntt.cu")
    for frag in SINGLE_PASS:
        hits = [(name, r) for name, r in res.items() if frag in name]
        assert len(hits) == 1, f"{frag}: {len(hits)} kernels match"
        name, (frame, st, ld) = hits[0]
        assert frame <= MAX_FRAME, f"{name}: {frame} B stack frame ({st} B spill stores, {ld} B spill loads)"
