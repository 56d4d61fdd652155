"""The BGV calls on the GPU: BgvModSwitch, BgvKeySwitchHybrid, BgvApplyGaloisKeySwitchHybridHoisted and
BgvMultiplyRelinearizeHybrid.

All four are compared bit for bit with the exact model of tests/bgv_exact.py over the hybrid shapes at every level,
every degree from 2 to 2^17, plain moduli from 2 to 2^61 - 1, q - 1 words below 2^61, K = 63 with the merged modulus
switch (64 sources in one t-corrected conversion) and K = 64 without it, and 70 moduli (two parameter blocks).  Also:
the anchors (mod_switch = 0 is DyadicMultiply then BgvKeySwitchHybrid, the hoisted call at g = 1 is BgvKeySwitchHybrid
of c1 into (c0, 0), the NTT-form mod switch is the inverse transform, the coefficient-form call and the forward
transform) at N = 2^12 and at N = 2^16, L = 30, alpha = K = 10; SEAL's formula at alpha = K = 1; the mod switch in place
and with count > 1; squaring, batches and unchanged inputs; every buffer kind and wrapped host batches; graph replay
with new data; a held stream; launch counts; every refusal; and a C++ caller."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import bgv_exact as bx
import composite_plan as plan
import hybrid_exact as hx
from test_gpu_hybrid_key_switch import SENTINEL, _check, _levels, _ntt_launches, _primes, dev, host
from test_gpu_hybrid_rotation import _mod_up_launches
from util import uniform_below

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U64 = np.uint64
INVALID_ARG = -1
TAU = 65537


@pytest.fixture(scope="module", autouse=True)
def _need_cuda(hb):
    if not torch.cuda.is_available() or hb.device_count() == 0:
        pytest.fail("gpu-marked test collected on a machine without CUDA")


class Case:
    """L data moduli then K special primes, relinearization keys (key component count 2), one Galois key set and
    their handles"""

    def __init__(self, hb, port, L, K, alpha, n, tau=TAU, data_bits=(50,), special_bits=(50,), fill=None, seed=1):
        self.L, self.K, self.alpha, self.n, self.tau, self.fill = L, K, alpha, n, tau, fill
        self.mods = _primes(port, n, L, data_bits, False) + _primes(port, n, K, special_bits, True)
        assert len(set(self.mods)) == L + K and all(np.gcd(q, tau) == 1 for q in self.mods)
        self.keys = hx.random_keys(self.mods, n, L, alpha, 2, seed, fill)
        self.handle = hb.KeySwitchKeys(self.keys, n, len(self.keys), L + K, 2)
        self.gkeys = hx.random_keys(self.mods, n, L, alpha, 2, seed + 500, fill)
        self.ghandle = hb.KeySwitchKeys(self.gkeys, n, len(self.gkeys), L + K, 2)

    def ciphertexts(self, level, batch, seed, comps=2):
        n, q = self.n, self.mods
        if self.fill == "q-1":
            return np.concatenate([np.full(n, q[i] - 1, dtype=U64) for _ in range(comps * batch) for i in range(level)])
        return np.concatenate([uniform_below(seed * 7919 + 64 * c + i, n, q[i]) for c in range(comps * batch)
                               for i in range(level)])

    # the calls
    def multiply(self, hb, out, a, b, level, ms, batch=1, stream=None):
        hb.BgvMultiplyRelinearizeHybrid(out, a, b, self.n, level, self.L, self.K, self.alpha, self.mods, self.tau,
                                        self.handle, ms, batch, stream=stream)

    def switch(self, hb, out, t, level, batch=1, stream=None):
        hb.BgvKeySwitchHybrid(out, t, self.n, level, self.L, self.K, self.alpha, 2, self.mods, self.tau, self.handle,
                              batch, stream=stream)

    def rotate(self, hb, out, ct, level, elts, batch=1, stream=None):
        hb.BgvApplyGaloisKeySwitchHybridHoisted(out, ct, self.n, level, self.L, self.K, self.alpha, self.mods,
                                                self.tau, [self.ghandle] * len(elts), elts, batch, stream=stream)

    # the model
    def exp_multiply(self, port, a, b, level, ms, batch=1):
        per = 2 * level * self.n
        return np.concatenate([bx.multiply_relinearize(port, a[c * per:(c + 1) * per], b[c * per:(c + 1) * per],
                                                       self.n, level, self.L, self.K, self.alpha, self.mods, self.keys,
                                                       self.tau, ms) for c in range(batch)])

    def exp_switch(self, port, res, t, level, batch=1):
        per = level * self.n
        return np.concatenate([bx.key_switch(port, res[2 * c * per:2 * (c + 1) * per], t[c * per:(c + 1) * per],
                                             self.n, level, self.L, self.K, self.alpha, 2, self.mods, self.keys,
                                             self.tau) for c in range(batch)])

    def exp_rotate(self, port, ct, level, elts, batch=1):
        per = 2 * level * self.n
        return np.concatenate([bx.hoisted(port, ct[c * per:(c + 1) * per], self.n, level, self.L, self.K, self.alpha,
                                          self.mods, elts, [self.gkeys] * len(elts), self.tau) for c in range(batch)])


def _out(words, fill=-1):
    return torch.full((words,), fill, dtype=torch.int64, device="cuda")


def _run_all(hb, port, case, level, seed, batch=1, square=False, elts=(5,)):
    """every call at one level against the model; the inputs must not change"""
    n = case.n
    ct1 = case.ciphertexts(level, batch, seed)
    ct2 = ct1 if square else case.ciphertexts(level, batch, seed + 1000)
    a = dev(ct1)
    b = a if square else dev(ct2)
    for ms in (False, True) if level >= 2 and case.K < 64 else (False,):
        out = _out(batch * 2 * (level - ms) * n)
        case.multiply(hb, out, a, b, level, ms, batch)
        torch.cuda.synchronize()
        _check(host(out), case.exp_multiply(port, ct1, ct2, level, ms, batch), f"multiply level {level} ms {ms}")
    res = case.ciphertexts(level, batch, seed + 7)
    t = case.ciphertexts(level, batch, seed + 8, comps=1)
    out = dev(res)
    case.switch(hb, out, dev(t), level, batch)
    torch.cuda.synchronize()
    _check(host(out), case.exp_switch(port, res, t, level, batch), f"key switch level {level}")
    elts = [e % (2 * n) or 1 for e in elts]
    out = _out(batch * len(elts) * 2 * level * n)
    case.rotate(hb, out, a, level, elts, batch)
    torch.cuda.synchronize()
    _check(host(out), case.exp_rotate(port, ct1, level, elts, batch), f"rotation level {level}")
    assert torch.equal(a, dev(ct1)) and torch.equal(b, dev(ct2)), "the inputs changed"
    if level >= 2:
        mods = case.mods[:level]
        for ntt in (True, False):
            out = _out(batch * 2 * level * n)
            hb.BgvModSwitch(out, a, n, mods, level, case.tau, 2 * batch, ntt)
            torch.cuda.synchronize()
            exp = bx.mod_switch(port, ct1, n, mods, 2 * batch, ntt, case.tau).reshape(2 * batch, level, n)
            got = host(out).reshape(2 * batch, level, n)
            _check(got[:, :level - 1], exp[:, :level - 1], f"mod switch level {level} ntt {ntt}")
            assert (got[:, level - 1] == U64(2**64 - 1)).all(), "the last limb was written"


@pytest.mark.parametrize("L, K, alpha", [(4, 1, 1), (6, 2, 2), (7, 3, 3), (5, 2, 5), (8, 4, 2)])
def test_shapes_at_every_level(hb, port, L, K, alpha):
    case = Case(hb, port, L, K, alpha, 256, seed=L * 100 + K * 10 + alpha)
    for level in _levels(L, alpha):
        _run_all(hb, port, case, level, level, elts=(5, 2 * 256 - 1))


@pytest.mark.parametrize("logn", range(1, 18))
def test_every_degree(hb, port, logn):
    case = Case(hb, port, 5, 2, 2, 1 << logn, seed=logn)
    _run_all(hb, port, case, 4, logn, elts=(3,))


@pytest.mark.parametrize("tau", [2, 3, 256, 65537, 1073479681, (1 << 40) + 15, (1 << 61) - 1])
def test_plain_moduli(hb, port, tau):
    case = Case(hb, port, 5, 3, 2, 64, tau=tau, data_bits=(29, 50, 58), special_bits=(45, 60), seed=tau % 1000)
    _run_all(hb, port, case, 5, 2)


@pytest.mark.parametrize("L, K, alpha, level", [(20, 2, 1, 20), (6, 63, 3, 6), (6, 64, 6, 5)])
def test_worst_case_words_below_2_61(hb, port, L, K, alpha, level):
    """the largest NTT primes below 2^61, every ciphertext and key word q - 1, tau = 2^61 - 1.  (6, 63): the merged
    mod switch converts from 64 sources; (6, 64): 64 special primes without it"""
    case = Case(hb, port, L, K, alpha, 32, tau=(1 << 61) - 1, data_bits=(60,), special_bits=(60,), fill="q-1")
    assert min(case.mods) > 1 << 60
    _run_all(hb, port, case, level, 0)


def test_seventy_moduli(hb, port):
    case = Case(hb, port, 70, 2, 64, 16, data_bits=(55,), special_bits=(55,))
    for level in (70, 66, 5):
        _run_all(hb, port, case, level, level)


def test_squaring_and_batches(hb, port):
    case = Case(hb, port, 7, 3, 3, 1 << 11, seed=5)
    for level in (7, 5):
        _run_all(hb, port, case, level, 9, batch=2, square=True)
        _run_all(hb, port, case, level, 19, batch=3)


# ------------------------------------------------------------------------------------------------ anchors
@pytest.mark.parametrize("n, L, K, alpha", [(1 << 12, 9, 3, 4), (1 << 16, 30, 10, 10)])
def test_anchors(hb, port, n, L, K, alpha):
    case = Case(hb, port, L, K, alpha, n)
    for level in (L, L // 2 + 1):
        comp = level * n
        ct1, ct2 = dev(case.ciphertexts(level, 1, 4)), dev(case.ciphertexts(level, 1, 5))
        fused = _out(2 * comp, 0)
        case.multiply(hb, fused, ct1, ct2, level, False)
        d = _out(3 * comp, 1)
        hb.DyadicMultiply(d, ct1, ct2, n, case.mods[:level], level)
        chain = d[:2 * comp].clone()
        case.switch(hb, chain, d[2 * comp:].clone(), level)
        torch.cuda.synchronize()
        assert torch.equal(fused, chain), f"multiply = dyadic + key switch, n = {n}, level {level}"
        rot = _out(2 * comp)
        case.rotate(hb, rot, ct1, level, [1])
        chain = torch.cat([ct1[:comp], torch.zeros_like(ct1[:comp])])
        hb.BgvKeySwitchHybrid(chain, ct1[comp:].clone(), n, level, L, K, alpha, 2, case.mods, case.tau, case.ghandle)
        torch.cuda.synchronize()
        assert torch.equal(rot, chain), f"hoisted g = 1 = key switch of c1, n = {n}, level {level}"
        ntts = [hb.GetNTT(n, q) for q in case.mods[:level]]
        fwd = _out(2 * comp, 0)
        hb.BgvModSwitch(fwd, ct1, n, case.mods[:level], level, case.tau, 2, True)
        coef = torch.empty_like(ct1)
        for c in range(2):
            hb.ComputeInverseMulti(ntts, coef[c * comp:(c + 1) * comp], ct1[c * comp:(c + 1) * comp])
        hb.BgvModSwitch(coef, coef, n, case.mods[:level], level, case.tau, 2, False)
        for c in range(2):
            part = coef[c * comp:c * comp + (level - 1) * n]
            hb.ComputeForwardMulti(ntts[:level - 1], part, part.clone())
        torch.cuda.synchronize()
        for c in range(2):
            sl = slice(c * comp, c * comp + (level - 1) * n)
            assert torch.equal(fwd[sl], coef[sl]), f"NTT mod switch = inverse, coefficients, forward, level {level}"


def test_alpha_one_k_one_is_seal(hb, port):
    """the mod switch against SEAL's per-limb formula; the key switch and multiply at digit size 1 with one special
    prime against the model, whose one-prime conversion is that formula"""
    for tau in (2, 65537, (1 << 61) - 1):
        case = Case(hb, port, 8, 1, 1, 1 << 10, tau=tau, data_bits=(60,), special_bits=(60,), seed=3)
        ct = case.ciphertexts(8, 2, 6)
        coef = dev(ct)
        hb.BgvModSwitch(coef, coef, case.n, case.mods[:8], 8, tau, 4, False)
        torch.cuda.synchronize()
        exp = bx.seal_mod_switch(ct, case.n, case.mods[:8], 4, tau)
        _check(host(coef), exp, f"SEAL mod switch, tau {tau}")
        _run_all(hb, port, case, 8, 5)


def test_mod_switch_in_place_and_counts(hb, port):
    case = Case(hb, port, 6, 1, 1, 1 << 12)
    n, mods = case.n, case.mods[:6]
    for count in (1, 3, 8):
        x = np.concatenate([uniform_below(100 + i, n, mods[i % 6]) for i in range(6 * count)])
        for ntt in (True, False):
            buf = dev(x)
            hb.BgvModSwitch(buf, buf, n, mods, 6, case.tau, count, ntt)
            torch.cuda.synchronize()
            exp = bx.mod_switch(port, x, n, mods, count, ntt, case.tau)
            _check(host(buf), exp, f"in place, count {count}, ntt {ntt}")  # limb 5 keeps the operand's


# ------------------------------------------------------------------------------------------------ buffers
@pytest.fixture(scope="module")
def buffers_case(hb, port):
    case = Case(hb, port, 7, 3, 3, 1 << 11, seed=77)
    level, batch = 5, 3
    ct1, ct2 = case.ciphertexts(level, batch, 21), case.ciphertexts(level, batch, 22)
    exp = {ms: case.exp_multiply(port, ct1, ct2, level, ms, batch) for ms in (False, True)}
    exp["rot"] = case.exp_rotate(port, ct1, level, [5, 7], batch)
    exp["ms"] = bx.mod_switch(port, ct1, case.n, case.mods[:level], 2 * batch, True, case.tau)
    return case, level, batch, ct1, ct2, exp


def _call(case, hb, which, out, a, b, level, batch, stream=None):
    if which == "rot":
        case.rotate(hb, out, a, level, [5, 7], batch, stream=stream)
    elif which == "ms":
        hb.BgvModSwitch(out, a, case.n, case.mods[:level], level, case.tau, 2 * batch, True, stream=stream)
    else:
        case.multiply(hb, out, a, b, level, which, batch, stream=stream)


def _cmp(case, which, got, exp, level, what):
    if which == "ms":  # the last limb is not written
        got = np.asarray(got).reshape(-1, level, case.n)[:, :level - 1]
        exp = exp.reshape(-1, level, case.n)[:, :level - 1]
    _check(got, exp, what)


@pytest.mark.parametrize("which", [False, True, "rot", "ms"])
@pytest.mark.parametrize("entry", ["device", "host", "pinned", "managed", "host_split"])
def test_buffers(hb, buffers_case, entry, which):
    """batch 3 between sentinel words"""
    case, level, batch, ct1, ct2, exps = buffers_case
    exp = exps[which]
    size = exp.size
    try:
        if entry == "device":
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                buf = torch.full((size + 2,), SENTINEL - (1 << 64), dtype=torch.int64, device="cuda")
                _call(case, hb, which, buf[1:1 + size], dev(ct1), dev(ct2), level, batch, stream=s)
            s.synchronize()
            got = host(buf)
        elif entry in ("managed", "pinned"):
            alloc, free = ((hb.managed_empty, hb.managed_free) if entry == "managed"
                           else (hb.pinned_empty, hb.pinned_free))
            a, b, buf = alloc(ct1.size), alloc(ct2.size), alloc(size + 2)
            try:
                a[:], b[:], buf[:] = ct1, ct2, SENTINEL
                _call(case, hb, which, buf[1:1 + size], a, b, level, batch)
                got = buf.copy()
                assert (a == ct1).all() and (b == ct2).all(), "the ciphertexts changed"
            finally:
                for x in (a, b, buf):
                    free(x)
        else:
            if entry == "host_split":
                hb.set_host_devices([0, 0])
            buf = np.full(size + 2, SENTINEL, dtype=U64)
            a, b = ct1.copy(), ct2.copy()
            _call(case, hb, which, buf[1:1 + size], a, b, level, batch)
            assert (a == ct1).all() and (b == ct2).all(), "the ciphertexts changed"
            got = buf
    finally:
        hb.set_host_devices([])
    assert got[0] == SENTINEL and got[-1] == SENTINEL, "a word next to the output was written"
    _cmp(case, which, got[1:1 + size], exp, level, f"{entry} {which}")


def test_host_batches_wrap_the_staging_slots(hb, port):
    """7 pairs through the rotating staging slots, over one and two host devices"""
    case = Case(hb, port, 4, 2, 2, 1 << 10, seed=3)
    level, batch = 4, 7
    ct1, ct2 = case.ciphertexts(level, batch, 31), case.ciphertexts(level, batch, 32)
    exp = case.exp_multiply(port, ct1, ct2, level, True, batch)
    exp_rot = case.exp_rotate(port, ct1, level, [3], batch)
    for devices in ([], [0, 0]):
        try:
            hb.set_host_devices(devices)
            out = np.zeros(exp.size, dtype=U64)
            case.multiply(hb, out, ct1, ct2, level, True, batch)
            rot = np.zeros(exp_rot.size, dtype=U64)
            case.rotate(hb, rot, ct1, level, [3], batch)
        finally:
            hb.set_host_devices([])
        _check(out, exp, f"multiply over {devices}")
        _check(rot, exp_rot, f"rotation over {devices}")


@pytest.mark.parametrize("which", [False, True, "rot", "ms"])
def test_graph_replay(hb, port, buffers_case, which):
    case, level, batch, ct1, ct2, exps = buffers_case
    out = _out(exps[which].size, 0)
    a, b = dev(ct1), dev(ct2)
    _call(case, hb, which, out, a, b, level, batch)  # warm: tables and pool
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _call(case, hb, which, out, a, b, level, batch)
    out.fill_(0)
    graph.replay()
    torch.cuda.synchronize()
    _cmp(case, which, host(out), exps[which], level, "graph replay")
    n1, n2 = case.ciphertexts(level, batch, 23), case.ciphertexts(level, batch, 24)
    a.copy_(dev(n1))
    b.copy_(dev(n2))
    graph.replay()
    torch.cuda.synchronize()
    if which == "rot":
        exp = case.exp_rotate(port, n1, level, [5, 7], batch)
    elif which == "ms":
        exp = bx.mod_switch(port, n1, case.n, case.mods[:level], 2 * batch, True, case.tau)
    else:
        exp = case.exp_multiply(port, n1, n2, level, which, batch)
    _cmp(case, which, host(out), exp, level, "graph replay, new data")


@pytest.mark.parametrize("which", [False, True, "rot", "ms"])
def test_held_stream(hb, buffers_case, which):
    """the inputs are written behind a bounded spin on the call's stream, and the result read behind the call"""
    case, level, batch, ct1, ct2, exps = buffers_case
    out = _out(exps[which].size, 0)
    a, b = torch.zeros(ct1.size, dtype=torch.int64, device="cuda"), torch.zeros(ct2.size, dtype=torch.int64,
                                                                                device="cuda")
    src1, src2 = dev(ct1), dev(ct2)
    _call(case, hb, which, out, src1, src2, level, batch)  # warm
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)
        a.copy_(src1)
        b.copy_(src2)
        out.fill_(0)
        _call(case, hb, which, out, a, b, level, batch, stream=s)
        got = out.clone()
    s.synchronize()
    _cmp(case, which, host(got), exps[which], level, "held stream")


# ------------------------------------------------------------------------------------------------ launch counts
def bgv_mod_down_launches(level, K, fwd, inv):
    """the special limbs' inverse transform; per block of 64 data moduli the t-corrected conversions, a forward
    transform and the finish (composite_plan's t-corrected mod-down, fwd and inv launches per transform)"""
    return plan.hybrid_mod_down_launches(level, K, 2, lambda forward, units: fwd if forward else inv, tau=True)


@pytest.mark.parametrize("L, K, alpha, level", [(6, 2, 2, 6), (30, 10, 10, 30), (70, 2, 64, 70), (70, 2, 64, 65),
                                                (12, 1, 1, 12)])
def test_launch_counts(hb, port, L, K, alpha, level):
    n = 1 << 12
    case = Case(hb, port, L, K, alpha, n, data_bits=(45,), special_bits=(45,))
    ct1, ct2 = dev(case.ciphertexts(level, 2, 1)), dev(case.ciphertexts(level, 2, 2))
    fwd, inv = _ntt_launches(hb, n, True), _ntt_launches(hb, n, False)
    mods = case.mods[:level]
    blocks = -(-(level - 1) // 64)
    ks_out, rot, ms_out = _out(2 * 2 * level * n, 0), _out(2 * 2 * 2 * level * n), _out(4 * level * n)
    # (name, call, launches of the whole call): the first four run two ciphertexts or pairs
    runs = [("key switch", lambda: case.switch(hb, ks_out, ct1[:2 * level * n], level, 2),
             2 * (_mod_up_launches(n, level, K, alpha, fwd, inv, 1) + bgv_mod_down_launches(level, K, fwd, inv))),
            ("rotation", lambda: case.rotate(hb, rot, ct1, level, [3, 5], 2),
             2 * (2 + _mod_up_launches(n, level, K, alpha, fwd, inv, 2)
                  + 2 * bgv_mod_down_launches(level, K, fwd, inv))),
            # two polynomials in one chunk: the last limbs' inverse transform, then per block of 64 moduli one
            # conversion, a forward transform of delta and the finish; coefficient form: the conversion and the finish
            ("mod switch ntt", lambda: hb.BgvModSwitch(ms_out, ct1, n, mods, level, case.tau, 2, True),
             inv + blocks * (2 + fwd)),
            ("mod switch coef", lambda: hb.BgvModSwitch(ms_out, ct1, n, mods, level, case.tau, 2, False), 2 * blocks)]
    for ms in (False, True):
        out = _out(2 * 2 * (level - ms) * n)
        runs.append((f"multiply ms {ms}", lambda out=out, ms=ms: case.multiply(hb, out, ct1, ct2, level, ms, 2),
                     2 * (_mod_up_launches(n, level, K, alpha, fwd, inv, 1)
                          + bgv_mod_down_launches(level - ms, K + ms, fwd, inv))))
    for name, run, exp in runs:
        run()  # warm
        torch.cuda.synchronize()
        before = hb.launch_count()
        run()
        torch.cuda.synchronize()
        got = hb.launch_count() - before
        assert got == exp, (name, got, exp, fwd, inv)


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals(hb, port):
    case = Case(hb, port, 6, 2, 2, 64)
    n, L, K, alpha, tau = case.n, 6, 2, 2, case.tau
    ct1, ct2 = dev(case.ciphertexts(L, 1, 2)), dev(case.ciphertexts(L, 1, 3))
    res = _out(2 * L * n, 0)
    mods = np.ascontiguousarray(case.mods, dtype=U64)

    def refused(what, fn):
        before = res.clone()
        with pytest.raises(hb.HexlB200Error) as e:
            fn()
        assert e.value.code == INVALID_ARG, (what, e.value)
        torch.cuda.synchronize()
        assert torch.equal(res, before), f"{what}: output written"

    def mul(t=tau, ms=0, level=L, p_size=K, m=mods, keys=case.handle):
        return hb._check(hb._lib.hexl_b200_bgv_multiply_relinearize_hybrid(
            res.data_ptr(), ct1.data_ptr(), ct2.data_ptr(), n, level, L, p_size, alpha, m.ctypes.data, t,
            keys._h if keys is not None else None, ms, 1, None))

    def ks(t=tau, m=mods, keys=case.handle):
        return hb._check(hb._lib.hexl_b200_bgv_key_switch_hybrid(
            res.data_ptr(), ct2.data_ptr(), n, L, L, K, alpha, 2, m.ctypes.data, t,
            keys._h if keys is not None else None, 1, None))

    def rot(t=tau, m=mods):
        keys = (hb._vp * 1)(case.ghandle._h)
        elts = np.array([5], dtype=U64)
        big = _out(2 * L * n)
        return hb._check(hb._lib.hexl_b200_bgv_apply_galois_key_switch_hybrid_hoisted(
            big.data_ptr(), ct1.data_ptr(), n, L, L, K, alpha, m.ctypes.data, t, keys, elts.ctypes.data, 1, 1, None))

    def msw(t=tau, m=mods, ntt=1, rns=L):
        return hb._check(hb._lib.hexl_b200_bgv_mod_switch(res.data_ptr(), ct1.data_ptr(), n, m.ctypes.data, rns, t, 2,
                                                          ntt, None))

    shared = int(case.mods[3]) * 3
    for name, call in (("multiply", mul), ("key switch", ks), ("rotation", rot), ("mod switch", msw)):
        refused(f"{name}: tau 0", lambda: call(t=0))
        refused(f"{name}: tau 1", lambda: call(t=1))
        refused(f"{name}: tau 2^61", lambda: call(t=1 << 61))
        refused(f"{name}: tau sharing a factor with a data modulus", lambda: call(t=shared))
    refused("key switch: tau sharing a factor with a special prime", lambda: ks(t=int(case.mods[-1]) * 2))
    refused("multiply: mod_switch 2", lambda: mul(ms=2))
    refused("multiply: mod_switch -1", lambda: mul(ms=-1))
    refused("multiply: mod_switch at level 1", lambda: mul(ms=1, level=1))
    refused("multiply: null keys", lambda: mul(keys=None))
    many = [int(q) for q in port.generate_primes(64, 45, True, n)]
    keys64 = hb.KeySwitchKeys(hx.random_keys(case.mods[:L] + many, n, L, alpha, 2, 8), n, 3, L + 64, 2)
    m64 = np.ascontiguousarray(case.mods[:L] + many, dtype=U64)
    refused("multiply: mod_switch with 64 special primes", lambda: mul(ms=1, p_size=64, m=m64, keys=keys64))
    refused("mod switch: one modulus", lambda: msw(rns=1))
    refused("mod switch: ntt_form 2", lambda: msw(ntt=2))
    refused("key switch: null keys", lambda: ks(keys=None))
    try:
        hb.set_host_devices([0, 0])
        sharded = hb.KeySwitchKeys(case.keys, n, len(case.keys), L + K, 2, sharded_by_modulus=True)
    finally:
        hb.set_host_devices([])
    refused("multiply: a sharded handle", lambda: mul(keys=sharded))
    refused("key switch: a sharded handle", lambda: ks(keys=sharded))
    bad = case.ciphertexts(L, 1, 2)
    bad[(L + 1) * n + 3] = case.mods[1]
    hb.set_debug(True)
    try:
        b = dev(bad)
        refused("mod switch: a word = q under debug",
                lambda: hb._check(hb._lib.hexl_b200_bgv_mod_switch(res.data_ptr(), b.data_ptr(), n, mods.ctypes.data,
                                                                   L, tau, 2, 1, None)))
    finally:
        hb.set_debug(False)
    before = res.clone()
    case.multiply(hb, res, ct1, ct2, L, True, 0)
    torch.cuda.synchronize()
    assert torch.equal(res, before), "batch = 0 wrote"


def test_cpp_caller_runs(hb, tmp_path):
    if not shutil.which("g++"):
        pytest.skip("g++ not present")
    exe = tmp_path / "bgv_caller"
    libdir = os.path.dirname(hb.LIB_PATH)
    subprocess.run(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "cpp", "bgv_caller.cpp"), "-o", str(exe),
                    "-L", libdir, "-lhexl_b200", f"-Wl,-rpath,{libdir}"], check=True)
    res = subprocess.run([str(exe), "run"], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
