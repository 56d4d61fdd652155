"""PlainLift, BfvAddPlain and BfvMultiplyPlain on the GPU.

Every call is compared bit for bit with the exact model of tests/plain_exact.py: at every degree from 2 to 2^17, at
levels 1 to 64, with t from 2 to 2^61 - 1 (above some q_i too) and plain_coeff_count 1, n/2 + 1 and n; with broadcast
and per-ciphertext plaintexts, subtraction, in place and out of place, and both plaintext forms of the multiply; at
production shapes (N = 2^15 and 2^16, l = 30) with host batches that wrap the staging slots.  Also pinned: device,
pageable, pinned, split-host and managed buffers; graph replay with new data; a held stream; launch counts; every
refusal; the anchors PlainLift(NTT form) = EltwiseCmpAdd per modulus + ComputeForwardMulti where t is below every q_i
and BfvMultiplyPlain = lift + forward + EltwiseMultModMulti + inverse; the BGV chains decrypt; and a C++ caller."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import bgv_exact as gx
import plain_exact as px
from mul_relin_exact import negacyclic_product
from util import uniform_below

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U64 = np.uint64
INVALID_ARG = -1
SENTINEL = 0xA5A5A5A5A5A5A5A5
T61 = (1 << 61) - 1


@pytest.fixture(scope="module", autouse=True)
def _need_cuda(hb):
    if not torch.cuda.is_available() or hb.device_count() == 0:
        pytest.fail("gpu-marked test collected on a machine without CUDA")


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=U64).view(np.int64)).to("cuda")


def host(t):
    return t.cpu().numpy().view(U64)


def _check(got, exp, what):
    bad = int((np.asarray(got, dtype=U64) != exp).sum())
    assert bad == 0, f"{what}: {bad} of {exp.size} words differ"


def _primes(port, n, count, bits):
    return [int(q) for q in port.generate_primes(count, bits, True, n)]


def _cts(mods, n, batch, seed):
    return np.concatenate([uniform_below(seed * 7919 + 64 * c + i, n, q) for c in range(2 * batch)
                           for i, q in enumerate(mods)])


class Shape:
    """ciphertexts, plaintexts and the expected outputs of all three calls for one (n, moduli, t, pcc)"""

    def __init__(self, port, n, mods, t, pcc, batch=1, plain_count=1, seed=1, cf=1):
        self.n, self.mods, self.t, self.pcc, self.batch, self.pc, self.cf = n, mods, t, pcc, batch, plain_count, cf
        self.l = len(mods)
        self.ct = _cts(mods, n, batch, seed)
        self.plain = uniform_below(seed + 500, plain_count * pcc, t)
        self.plain[:min(3, pcc)] = [t - 1, 0, (t + 1) // 2][:min(3, pcc)]
        self.port = port

    def _p(self, c):
        c = 0 if self.pc == 1 else c
        return self.plain[c * self.pcc:(c + 1) * self.pcc]

    def _c(self, c):
        per = 2 * self.l * self.n
        return self.ct[c * per:(c + 1) * per]

    def lift(self, ntt_form):
        return px.plain_lift(self.port, self.plain, self.pcc, self.n, self.mods, self.t, self.cf, ntt_form, self.pc)

    def add(self, subtract):
        return np.concatenate([px.add_plain(self._c(c), self._p(c), self.pcc, self.n, self.mods, self.t, subtract)
                               for c in range(self.batch)])

    def mul(self):
        return np.concatenate([px.multiply_plain(self.port, self._c(c), self._p(c), self.pcc, self.n, self.mods,
                                                 self.t) for c in range(self.batch)])


def _run_all(hb, sh, what, in_place=True):
    """the three calls on device buffers, out of place (and in place), against the model"""
    n, l, t, pcc, b, pc = sh.n, sh.l, sh.t, sh.pcc, sh.batch, sh.pc
    p = dev(sh.plain)
    for ntt_form in (False, True):
        out = torch.full((pc * l * n,), -1, dtype=torch.int64, device="cuda")
        hb.PlainLift(out, p, pcc, n, sh.mods, l, t, sh.cf, ntt_form, pc)
        _check(host(out), sh.lift(ntt_form), f"{what}: PlainLift ntt_form {ntt_form}")
    fp = dev(px.plain_lift(sh.port, sh.plain, pcc, n, sh.mods, t, 1, True, pc))
    for sub in (False, True):
        exp = sh.add(sub)
        ct = dev(sh.ct)
        out = torch.full_like(ct, -1)
        hb.BfvAddPlain(out, ct, p, pcc, n, sh.mods, l, t, sub, pc, b)
        _check(host(out), exp, f"{what}: BfvAddPlain subtract {sub}")
        if in_place:
            hb.BfvAddPlain(ct, ct, p, pcc, n, sh.mods, l, t, sub, pc, b)
            _check(host(ct), exp, f"{what}: BfvAddPlain subtract {sub} in place")
    exp = sh.mul()
    for ready in (False, True):
        ct = dev(sh.ct)
        out = torch.full_like(ct, -1)
        hb.BfvMultiplyPlain(out, ct, fp if ready else p, pcc, n, sh.mods, l, t, ready, pc, b)
        _check(host(out), exp, f"{what}: BfvMultiplyPlain plain_ntt_form {ready}")
        assert torch.equal(ct, dev(sh.ct)), "the ciphertexts changed"
        if in_place:
            hb.BfvMultiplyPlain(ct, ct, fp if ready else p, pcc, n, sh.mods, l, t, ready, pc, b)
            _check(host(ct), exp, f"{what}: BfvMultiplyPlain plain_ntt_form {ready} in place")
    assert torch.equal(p, dev(sh.plain)), "the plaintexts changed"


@pytest.mark.parametrize("logn", range(1, 18))
def test_every_degree(hb, port, logn):
    n = 1 << logn
    mods = _primes(port, n, 3, 50)
    for pcc in sorted({1, n // 2 + 1, n}):
        _run_all(hb, Shape(port, n, mods, 65537, pcc, batch=2, plain_count=2, seed=logn, cf=3), f"n {n} pcc {pcc}")


@pytest.mark.parametrize("level", [1, 2, 17, 63, 64])
def test_levels(hb, port, level):
    n = 64
    mods = _primes(port, n, 64, 58)[:level]
    _run_all(hb, Shape(port, n, mods, 786433, n // 2 + 1, batch=3, plain_count=1, seed=level), f"level {level}")


@pytest.mark.parametrize("t", [2, 3, 65537, (1 << 45) + 9, T61])
def test_plain_moduli_around_the_q(hb, port, t):
    """t below every q_i, between 30- and 60-bit q_i, and above all of them; every ciphertext word q - 1 too"""
    n = 256
    mods = _primes(port, n, 2, 29) + _primes(port, n, 2, 60)
    sh = Shape(port, n, mods, t, n, batch=2, plain_count=2, seed=t % 1000, cf=max(1, t - 1))
    _run_all(hb, sh, f"t {t}")
    sh.ct = np.concatenate([np.full(n, q - 1, dtype=U64) for _ in range(4) for q in mods])
    sh.plain[:] = t - 1
    _run_all(hb, sh, f"t {t}, words q - 1 and t - 1")


@pytest.mark.parametrize("logn", [15, 16])
def test_production_shapes(hb, port, logn):
    """l = 30 at N = 2^15 and 2^16: device batches, and host batches of 4 that wrap the three staging slots"""
    n = 1 << logn
    mods = _primes(port, n, 30, 50 if logn == 15 else 55)
    sh = Shape(port, n, mods, 65537, n, batch=4, plain_count=1, seed=logn)
    exp_add, exp_mul = sh.add(False), sh.mul()
    ct, p = dev(sh.ct), dev(sh.plain)
    out = torch.empty_like(ct)
    hb.BfvAddPlain(out, ct, p, n, n, mods, 30, sh.t, False, 1, 4)
    _check(host(out), exp_add, "device add")
    hb.BfvMultiplyPlain(out, ct, p, n, n, mods, 30, sh.t, False, 1, 4)
    _check(host(out), exp_mul, "device multiply")
    for devices in ([], [0, 0]):
        try:
            hb.set_host_devices(devices)
            got = np.zeros_like(sh.ct)
            hb.BfvAddPlain(got, sh.ct, sh.plain, n, n, mods, 30, sh.t, False, 1, 4)
            _check(got, exp_add, f"host add over {devices}")
            hb.BfvMultiplyPlain(got, sh.ct, sh.plain, n, n, mods, 30, sh.t, False, 1, 4)
            _check(got, exp_mul, f"host multiply over {devices}")
        finally:
            hb.set_host_devices([])


# ------------------------------------------------------------------------------------------------ anchors
def test_lift_equals_cmp_add_and_forward_where_t_is_below_every_q(hb, port):
    n, t = 1 << 12, 65537
    mods = _primes(port, n, 5, 50)
    plain = uniform_below(4, n, t)
    ntts = [hb.GetNTT(n, q) for q in mods]
    chain = torch.empty(5 * n, dtype=torch.int64, device="cuda")
    p = dev(plain)
    for i, q in enumerate(mods):  # m >= (t+1)/2: m + (q - t)
        hb.EltwiseCmpAdd(chain[i * n:(i + 1) * n], p, n, hb.CMPINT.NLT, (t + 1) // 2, q - t)
    hb.ComputeForwardMulti(ntts, chain, chain)
    out = torch.empty_like(chain)
    hb.PlainLift(out, p, n, n, mods, 5, t, 1, True)
    torch.cuda.synchronize()
    assert torch.equal(out, chain)


@pytest.mark.parametrize("n, l", [(1 << 12, 6), (1 << 15, 30)])
def test_multiply_plain_equals_the_four_call_chain(hb, port, n, l):
    mods = _primes(port, n, l, 55)
    t = 786433
    ct = dev(_cts(mods, n, 1, 9))
    p = dev(uniform_below(10, n // 2 + 1, t))
    fp = torch.empty(l * n, dtype=torch.int64, device="cuda")
    hb.PlainLift(fp, p, n // 2 + 1, n, mods, l, t, 1, True)
    ntts = [hb.GetNTT(n, q) for q in mods]
    x = torch.empty_like(ct)
    hb.ComputeForwardMulti(ntts * 2, x, ct)
    hb.EltwiseMultModMulti(x, x, torch.cat([fp, fp]), n, mods * 2)
    hb.ComputeInverseMulti(ntts * 2, x, x)
    out = torch.empty_like(ct)
    hb.BfvMultiplyPlain(out, ct, p, n // 2 + 1, n, mods, l, t)
    torch.cuda.synchronize()
    assert torch.equal(out, x)


def test_bgv_chains_decrypt_on_the_gpu(hb, port):
    """BGV add_plain after BgvModSwitch (the correction factor) and multiply_plain, through the existing calls"""
    n, L, t = 1 << 10, 3, 65537
    mods = _primes(port, n, L + 1, 55)
    s = gx.secret(n, 77)
    m1, m2 = [int(v) for v in uniform_below(1, n, t)], uniform_below(2, n, t)
    ct = gx.encrypt(port, m1, s, n, mods, t, 3)
    sw = dev(ct)
    hb.BgvModSwitch(sw, sw, n, mods, L + 1, t, 2, True)
    sw = torch.cat([sw[:L * n], sw[(L + 1) * n:(2 * L + 1) * n]])
    c = pow(mods[L] % t, -1, t)
    lifted = torch.empty(L * n, dtype=torch.int64, device="cuda")
    hb.PlainLift(lifted, dev(m2), n, n, mods[:L], L, t, c, True)
    hb.EltwiseAddModMulti(sw[:L * n], sw[:L * n].clone(), lifted, n, mods[:L])
    dec = [v * pow(c, -1, t) % t for v in gx.decrypt(port, host(sw), [None, s], n, mods[:L], t)]
    assert dec == [(a + int(b)) % t for a, b in zip(m1, m2)]
    full = torch.empty((L + 1) * n, dtype=torch.int64, device="cuda")
    hb.PlainLift(full, dev(m2), n, n, mods, L + 1, t, 1, True)
    prod = dev(ct)
    hb.EltwiseMultModMulti(prod, prod.clone(), torch.cat([full, full]), n, mods * 2)
    assert gx.decrypt(port, host(prod), [None, s], n, mods, t) == [
        v % t for v in negacyclic_product(m1, [int(v) for v in m2], n)]


# ------------------------------------------------------------------------------------------------ buffers
@pytest.fixture(scope="module")
def small(port):
    n = 1 << 11
    return Shape(port, n, _primes(port, n, 4, 50), 65537, n // 2 + 1, batch=3, plain_count=3, seed=21)


CALLS = ["lift", "add", "sub", "mul", "mul_ntt"]


def _call(hb, sh, which, out, ct, plain, stream=None):
    n, l, t, pcc, b, pc = sh.n, sh.l, sh.t, sh.pcc, sh.batch, sh.pc
    if which == "lift":
        return hb.PlainLift(out, plain, pcc, n, sh.mods, l, t, 1, True, pc, stream=stream)
    if which in ("add", "sub"):
        return hb.BfvAddPlain(out, ct, plain, pcc, n, sh.mods, l, t, which == "sub", pc, b, stream=stream)
    return hb.BfvMultiplyPlain(out, ct, plain, pcc, n, sh.mods, l, t, which == "mul_ntt", pc, b, stream=stream)


def _inputs(sh, which):
    plain = sh.lift(True) if which == "mul_ntt" else sh.plain
    exp = {"lift": lambda: sh.lift(True), "add": lambda: sh.add(False), "sub": lambda: sh.add(True),
           "mul": sh.mul, "mul_ntt": sh.mul}[which]()
    return plain, exp


@pytest.mark.parametrize("which", CALLS)
@pytest.mark.parametrize("entry", ["device", "host", "pinned", "managed", "host_split"])
def test_buffers(hb, small, entry, which):
    sh = small
    plain, exp = _inputs(sh, which)
    size = exp.size
    try:
        if entry == "device":
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                buf = torch.full((size + 2,), SENTINEL - (1 << 64), dtype=torch.int64, device="cuda")
                _call(hb, sh, which, buf[1:1 + size], dev(sh.ct), dev(plain), stream=s)
            s.synchronize()
            got = host(buf)
        elif entry in ("managed", "pinned"):
            alloc, free = ((hb.managed_empty, hb.managed_free) if entry == "managed"
                           else (hb.pinned_empty, hb.pinned_free))
            a, p, buf = alloc(sh.ct.size), alloc(plain.size), alloc(size + 2)
            try:
                a[:], p[:], buf[:] = sh.ct, plain, SENTINEL
                _call(hb, sh, which, buf[1:1 + size], a, p)
                got = buf.copy()
                assert (a == sh.ct).all() and (p == plain).all(), "an input changed"
            finally:
                for x in (a, p, buf):
                    free(x)
        else:
            if entry == "host_split":
                hb.set_host_devices([0, 0])
            buf = np.full(size + 2, SENTINEL, dtype=U64)
            a, p = sh.ct.copy(), plain.copy()
            _call(hb, sh, which, buf[1:1 + size], a, p)
            assert (a == sh.ct).all() and (p == plain).all(), "an input changed"
            got = buf
    finally:
        hb.set_host_devices([])
    assert got[0] == SENTINEL and got[-1] == SENTINEL, "a word next to the output was written"
    _check(got[1:1 + size], exp, f"{entry} {which}")


@pytest.mark.parametrize("which", ["add", "mul", "mul_ntt"])
def test_host_in_place_and_broadcast_batches_wrap_the_slots(hb, port, which):
    n = 1 << 10
    sh = Shape(port, n, _primes(port, n, 3, 50), 65537, n, batch=7, plain_count=1, seed=5)
    plain, exp = _inputs(sh, which)
    for devices in ([], [0, 0]):
        try:
            hb.set_host_devices(devices)
            ct = sh.ct.copy()
            _call(hb, sh, which, ct, ct, plain.copy())
        finally:
            hb.set_host_devices([])
        _check(ct, exp, f"{which} over {devices}")


@pytest.mark.parametrize("which", CALLS)
def test_graph_replay(hb, small, port, which):
    sh = small
    plain, exp = _inputs(sh, which)
    ct, p = dev(sh.ct), dev(plain)
    out = torch.zeros(exp.size, dtype=torch.int64, device="cuda")
    _call(hb, sh, which, out, ct, p)  # warm: tables, transforms and pool
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        _call(hb, sh, which, out, ct, p)
    out.fill_(0)
    graph.replay()
    torch.cuda.synchronize()
    _check(host(out), exp, "graph replay")
    new = Shape(port, sh.n, sh.mods, sh.t, sh.pcc, sh.batch, sh.pc, seed=22)
    plain2, exp2 = _inputs(new, which)
    ct.copy_(dev(new.ct))
    p.copy_(dev(plain2))
    graph.replay()
    torch.cuda.synchronize()
    _check(host(out), exp2, "graph replay, new data")


@pytest.mark.parametrize("which", CALLS)
def test_held_stream(hb, small, which):
    """the inputs are written behind a bounded spin on the call's stream, and the result read behind the call"""
    sh = small
    plain, exp = _inputs(sh, which)
    src_ct, src_p = dev(sh.ct), dev(plain)
    ct, p = torch.zeros_like(src_ct), torch.zeros_like(src_p)
    out = torch.zeros(exp.size, dtype=torch.int64, device="cuda")
    _call(hb, sh, which, out, src_ct, src_p)  # warm
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)
        ct.copy_(src_ct)
        p.copy_(src_p)
        out.fill_(0)
        _call(hb, sh, which, out, ct, p, stream=s)
        got = out.clone()
    s.synchronize()
    _check(host(got), exp, "held stream")


# ------------------------------------------------------------------------------------------------ launch counts
def _ntt_launches(hb, n, count, forward):
    ntts = [hb.GetNTT(n, q) for q in hb.GeneratePrimes(count, 50, True, n)]
    x = torch.zeros(count * n, dtype=torch.int64, device="cuda")
    fn = hb.ComputeForwardMulti if forward else hb.ComputeInverseMulti
    fn(ntts, x, x)
    torch.cuda.synchronize()
    before = hb.launch_count()
    fn(ntts, x, x)
    torch.cuda.synchronize()
    return hb.launch_count() - before


def _count(hb, fn):
    fn()  # warm
    torch.cuda.synchronize()
    before = hb.launch_count()
    fn()
    torch.cuda.synchronize()
    return hb.launch_count() - before


@pytest.mark.parametrize("l", [3, 30, 40])
def test_launch_counts(hb, port, l):
    """lift: 1 (+ the forward transform of count x l limbs); add: 1 for the batch; multiply per ciphertext: the
    forward transform of 2l limbs and two inverse transforms of l limbs, plus 1 lift and one forward transform of l
    limbs per plaintext lifted"""
    n, batch = 1 << 12, 3
    sh = Shape(port, n, _primes(port, n, l, 50), 65537, n, batch=batch, plain_count=batch, seed=l)
    fwd = {k: _ntt_launches(hb, n, k, True) for k in (l, 2 * l, batch * l)}
    inv = _ntt_launches(hb, n, l, False)
    ct, p = dev(sh.ct), dev(sh.plain)
    fp = dev(sh.lift(True))
    out = torch.empty_like(ct)
    lifted = torch.empty(batch * l * n, dtype=torch.int64, device="cuda")
    runs = [
        ("lift", lambda: hb.PlainLift(lifted, p, n, n, sh.mods, l, sh.t, 1, False, batch), 1),
        ("lift ntt", lambda: hb.PlainLift(lifted, p, n, n, sh.mods, l, sh.t, 1, True, batch), 1 + fwd[batch * l]),
        ("add in place", lambda: hb.BfvAddPlain(ct, ct, p, n, n, sh.mods, l, sh.t, False, batch, batch), 1),
        ("add", lambda: hb.BfvAddPlain(out, ct, p, n, n, sh.mods, l, sh.t, False, batch, batch), 1),
        ("mul per ciphertext", lambda: hb.BfvMultiplyPlain(out, ct, p, n, n, sh.mods, l, sh.t, False, batch, batch),
         batch * (1 + fwd[l] + fwd[2 * l] + 2 * inv)),
        ("mul broadcast", lambda: hb.BfvMultiplyPlain(out, ct, p, n, n, sh.mods, l, sh.t, False, 1, batch),
         1 + fwd[l] + batch * (fwd[2 * l] + 2 * inv)),
        ("mul ntt form", lambda: hb.BfvMultiplyPlain(out, ct, fp, n, n, sh.mods, l, sh.t, True, batch, batch),
         batch * (fwd[2 * l] + 2 * inv)),
    ]
    for name, fn, exp in runs:
        got = _count(hb, fn)
        assert got == exp, (name, got, exp)


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals(hb, port):
    n, l, t = 64, 3, 65537
    mods = _primes(port, n, l, 50)
    ct = dev(_cts(mods, n, 1, 2))
    p = dev(uniform_below(3, n, t))
    out = torch.zeros(2 * l * n, dtype=torch.int64, device="cuda")
    lo = torch.zeros(l * n, dtype=torch.int64, device="cuda")

    def refused(what, calls=("lift", "add", "mul"), res=None, a=ct, plain=p, nn=n, level=l, qmods=None, tt=t,
                pcc=n, pc=1, cf=1, ntt=0, sub=0, batch=1, null_res=False):
        mp = np.ascontiguousarray(qmods if qmods is not None else mods, dtype=U64)
        ptr = lambda x: x.data_ptr() if x is not None else None  # noqa: E731
        for call in calls:
            o = res if res is not None else (lo if call == "lift" else out)
            before = o.clone()
            r = None if null_res else o
            with pytest.raises(hb.HexlB200Error) as e:
                if call == "lift":
                    hb._check(hb._lib.hexl_b200_plain_lift(ptr(r), ptr(plain), pcc, nn, mp.ctypes.data, level, tt,
                                                           cf, ntt, pc, None))
                elif call == "add":
                    hb._check(hb._lib.hexl_b200_bfv_add_plain(ptr(r), ptr(a), ptr(plain), pcc, pc, nn,
                                                              mp.ctypes.data, level, tt, sub, batch, None))
                else:
                    hb._check(hb._lib.hexl_b200_bfv_multiply_plain(ptr(r), ptr(a), ptr(plain), pcc, pc, ntt, nn,
                                                                   mp.ctypes.data, level, tt, batch, None))
            assert e.value.code == INVALID_ARG, (what, call, e.value)
            assert torch.equal(o, before), f"{what}: output written"

    refused("null result", null_res=True)
    refused("null plain", plain=None)
    refused("null ct", a=None, calls=("add", "mul"))
    refused("n = 1", nn=1)
    refused("n not a power of two", nn=48)
    refused("n = 2^21", nn=1 << 21)
    refused("level 0", level=0)
    refused("level 65", level=65, qmods=mods + _primes(port, n, 62, 40))
    refused("t = 1", tt=1)
    refused("t = 0", tt=0)
    refused("t = 2^61", tt=1 << 61)
    refused("a modulus >= 2^61", qmods=mods[:-1] + [int(port.generate_primes(1, 62, True, n)[0])])
    refused("a modulus of 1", qmods=mods[:-1] + [1])
    refused("a modulus not NTT-friendly", qmods=mods[:-1] + [(1 << 40) + 15], calls=("mul",))
    refused("a modulus not NTT-friendly, lift in NTT form", qmods=mods[:-1] + [(1 << 40) + 15], calls=("lift",),
            ntt=1)
    refused("plain_coeff_count 0", pcc=0)
    refused("plain_coeff_count > n", pcc=n + 1)
    refused("correction factor 0", cf=0, calls=("lift",))
    refused("correction factor = t", cf=t, calls=("lift",))
    refused("ntt_form 2", ntt=2, calls=("lift", "mul"))
    refused("subtract 2", sub=2, calls=("add",))
    refused("plain_count 2 for batch 1", pc=2, calls=("add", "mul"))
    big = torch.zeros(6 * l * n, dtype=torch.int64, device="cuda")
    refused("result partly overlapping ct", res=big[l * n:3 * l * n], a=big[:2 * l * n], calls=("add", "mul"))
    refused("result overlapping plain", res=big[:2 * l * n], plain=big[l * n:l * n + n], calls=("add", "mul"))
    refused("lift result overlapping plain", res=big[:l * n], plain=big[n:2 * n], calls=("lift",))
    hb.set_debug(True)
    try:
        bad = host(p).copy()
        bad[5] = t
        refused("a plaintext word = t under debug", plain=dev(bad))
        badct = host(ct).copy()
        badct[n + 3] = mods[1]
        refused("a ciphertext word = q under debug", a=dev(badct), calls=("add", "mul"))
        fp = torch.zeros(l * n, dtype=torch.int64, device="cuda")
        fp[2 * n + 1] = mods[2]
        refused("an NTT-form plaintext word = q under debug", plain=fp, calls=("mul",), ntt=1)
    finally:
        hb.set_debug(False)
    before = out.clone()
    hb.BfvAddPlain(out, ct, p, n, n, mods, l, t, False, 1, 0)
    hb.BfvMultiplyPlain(out, ct, p, n, n, mods, l, t, False, 1, 0)
    hb.PlainLift(lo, p, n, n, mods, l, t, 1, False, 0)
    torch.cuda.synchronize()
    assert torch.equal(out, before), "batch = 0 wrote"


def test_cpp_caller_runs(hb, tmp_path):
    if not shutil.which("g++"):
        pytest.skip("g++ not present")
    exe = tmp_path / "plain_caller"
    libdir = os.path.dirname(hb.LIB_PATH)
    subprocess.run(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "cpp", "plain_caller.cpp"), "-o", str(exe),
                    "-L", libdir, "-lhexl_b200", f"-Wl,-rpath,{libdir}"], check=True)
    res = subprocess.run([str(exe), "run"], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
