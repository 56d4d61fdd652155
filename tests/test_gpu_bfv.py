"""BfvMultiply and BfvMultiplyRelinearizeHybrid on the GPU.

Both calls are compared bit for bit with the exact model of tests/bfv_exact.py: at the bit sizes of SEAL's default BFV
moduli for n = 2^12 to 2^15 with SEAL's choice of B and m_sk and SEAL-shaped keys (alpha = K = 1); at two hybrid
shapes and every level of them; at every degree from 2 to 2^17; at l = 64 and k = 64; with every word q - 1 below 2^61;
with t from 2 to just below 2^61 (and at the largest t the bound accepts).  Also pinned: squaring, batch > 1 and
unchanged inputs; the relinearized call equals the chain BfvMultiply, forward NTT of d2, KeySwitchHybrid, inverse NTT
and the addition of (d0, d1) (at n = 2^15 too), and at digit size 1 with one special prime the chain with
KeySwitchResident; device, pageable, pinned, split-host and managed buffers; host batches that wrap the staging slots;
graph replay with new data; a held stream; launch counts; every refusal, the bound one step past what it accepts
included; and a C++ caller."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import bfv_exact as bx
import hybrid_exact as hx
from test_bfv_exact import SEAL_BITS, seal_moduli
from util import uniform_below

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U64 = np.uint64
INVALID_ARG = -1
SENTINEL = 0xA5A5A5A5A5A5A5A5


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


class Case:
    """L data moduli then K special primes, BEHZ bases per level (SEAL's rule unless given), one set of relinearization
    keys and its handle"""

    def __init__(self, hb, port, n, mods, L, K, alpha, t, bases=None, fill=None, seed=1):
        self.n, self.mods, self.L, self.K, self.alpha, self.t, self.fill = n, [int(q) for q in mods], L, K, alpha, t, fill
        self.bases = bases or {}
        self.keys = hx.random_keys(self.mods, n, L, alpha, 2, seed, fill)
        self.handle = hb.KeySwitchKeys(self.keys, n, len(self.keys), L + K, 2)
        self.port = port

    def base(self, level):
        if level not in self.bases:
            self.bases[level] = bx.seal_bases(self.port, self.n, self.mods[:level], self.t)
        return self.bases[level]

    def ciphertexts(self, level, batch, seed):
        n, q = self.n, self.mods
        if self.fill == "q-1":
            return np.concatenate([np.full(n, q[i] - 1, dtype=U64) for _ in range(2 * batch) for i in range(level)])
        return np.concatenate([uniform_below(seed * 7919 + 64 * c + i, n, q[i]) for c in range(2 * batch)
                               for i in range(level)])

    def multiply(self, hb, out, ct1, ct2, level, batch=1, stream=None):
        B, m_sk = self.base(level)
        return hb.BfvMultiply(out, ct1, ct2, self.n, self.mods, level, B, m_sk, self.t, batch, stream=stream)

    def relin(self, hb, out, ct1, ct2, level, batch=1, stream=None):
        B, m_sk = self.base(level)
        return hb.BfvMultiplyRelinearizeHybrid(out, ct1, ct2, self.n, level, self.L, self.K, self.alpha, self.mods, B,
                                               m_sk, self.t, self.handle, batch, stream=stream)

    def expected(self, ct1, ct2, level, batch=1):
        """(products, relinearized) of every pair"""
        B, m_sk = self.base(level)
        per = 2 * level * self.n
        d, r = [], []
        for c in range(batch):
            x = bx.bfv_multiply(self.port, ct1[c * per:(c + 1) * per], ct2[c * per:(c + 1) * per], self.n,
                                self.mods[:level], B, m_sk, self.t)
            d.append(x)
            r.append(bx.relinearize(self.port, x, self.n, level, self.L, self.K, self.alpha, self.mods, self.keys))
        return np.concatenate(d), np.concatenate(r)


def _run(hb, case, level, seed, batch=1, square=False):
    ct1 = case.ciphertexts(level, batch, seed)
    ct2 = ct1 if square else case.ciphertexts(level, batch, seed + 1000)
    a = dev(ct1)
    b = a if square else dev(ct2)
    n = case.n
    d = torch.full((batch * 3 * level * n,), -1, dtype=torch.int64, device="cuda")
    r = torch.full((batch * 2 * level * n,), -1, dtype=torch.int64, device="cuda")
    case.multiply(hb, d, a, b, level, batch)
    case.relin(hb, r, a, b, level, batch)
    torch.cuda.synchronize()
    assert torch.equal(a, dev(ct1)) and torch.equal(b, dev(ct2)), "the ciphertexts changed"
    exp_d, exp_r = case.expected(ct1, ct2, level, batch)
    _check(host(d), exp_d, f"BfvMultiply level {level}")
    _check(host(r), exp_r, f"BfvMultiplyRelinearizeHybrid level {level}")


def _primes(port, n, count, bits, skip=()):
    return [int(q) for q in port.generate_primes(count + len(skip), bits, True, n) if int(q) not in skip][:count]


@pytest.mark.parametrize("n", sorted(SEAL_BITS))
@pytest.mark.parametrize("t", [65537, 786433])
def test_seal_default_moduli(hb, port, n, t):
    """SEAL-shaped keys: the last modulus is the special prime, alpha = K = 1"""
    mods = seal_moduli(port, n)
    L = len(mods) - 1
    case = Case(hb, port, n, mods, L, 1, 1, t, seed=n % 97)
    for level in sorted({L, max(1, L // 2)}):
        _run(hb, case, level, level)


@pytest.mark.parametrize("L, K, alpha", [(6, 2, 2), (7, 3, 3)])
def test_hybrid_shapes_at_every_level(hb, port, L, K, alpha):
    n = 256
    case = Case(hb, port, n, _primes(port, n, L, 50) + _primes(port, n, K, 55), L, K, alpha, 65537, seed=L)
    for level in range(1, L + 1):
        _run(hb, case, level, level)


@pytest.mark.parametrize("logn", range(1, 18))
def test_every_degree(hb, port, logn):
    n = 1 << logn
    case = Case(hb, port, n, _primes(port, n, 3, 50) + _primes(port, n, 1, 55), 3, 1, 2, 257, seed=logn)
    _run(hb, case, 3, logn)


def test_sixty_four_moduli_in_q_and_b(hb, port):
    """l = 64 and k = 64: both conversions of the scaling take 64 sources, the tensor two parameter blocks"""
    n = 16
    mods = _primes(port, n, 65, 58)
    bsk = _primes(port, n, 65, 60)
    case = Case(hb, port, n, mods, 64, 1, 64, 65537, bases={64: (bsk[:64], bsk[64])})
    assert bx.bound_holds(n, 65537, mods[:64], bsk[:64], bsk[64])
    _run(hb, case, 64, 5)


@pytest.mark.parametrize("t", [2, 3, 65537, (1 << 61) - 1])
def test_worst_case_words_and_plain_moduli(hb, port, t):
    """the largest NTT primes below 2^61 in Q and Bsk, every ciphertext and key word q - 1, t up to 2^61 - 1"""
    n = 64
    top = [int(q) for q in port.generate_primes(12, 60, False, n)]
    assert min(top) > 1 << 60
    B, m_sk = top[4:10], top[10]
    case = Case(hb, port, n, top[:3] + [top[11]], 3, 1, 1, t, bases={3: (B, m_sk)}, fill="q-1")
    assert bx.bound_holds(n, t, top[:3], B, m_sk)
    _run(hb, case, 3, 0)
    case.fill = None
    _run(hb, case, 3, 4)


def test_largest_plain_modulus_the_bound_accepts(hb, port):
    n = 32
    mods = _primes(port, n, 3, 59)
    bsk = _primes(port, n, 3, 60)
    t = bx.largest_plain_modulus(n, mods[:2], bsk[:2], bsk[2])
    assert 2 <= t < 1 << 61
    case = Case(hb, port, n, mods, 2, 1, 1, t, bases={2: (bsk[:2], bsk[2])}, fill="q-1")
    _run(hb, case, 2, 0)


def test_squaring_and_batches(hb, port):
    n = 1 << 11
    case = Case(hb, port, n, _primes(port, n, 5, 50) + _primes(port, n, 2, 55), 5, 2, 2, 65537, seed=9)
    _run(hb, case, 5, 3, batch=3, square=True)
    _run(hb, case, 4, 4, batch=3)


# ------------------------------------------------------------------------------------------------ equalities
def _chain(hb, case, d, level):
    """BfvMultiply's d, then forward NTT of d2, KeySwitchHybrid into zeros, inverse NTT and the addition of (d0, d1)"""
    n, comp = case.n, level * case.n
    ntts = [hb.GetNTT(n, q) for q in case.mods[:level]]
    t = torch.empty(comp, dtype=torch.int64, device="cuda")
    hb.ComputeForwardMulti(ntts, t, d[2 * comp:].clone())
    ks = torch.zeros(2 * comp, dtype=torch.int64, device="cuda")
    hb.KeySwitchHybrid(ks, t, n, level, case.L, case.K, case.alpha, 2, case.mods, case.handle)
    hb.ComputeInverseMulti(ntts * 2, ks, ks)
    out = torch.empty(2 * comp, dtype=torch.int64, device="cuda")
    hb.EltwiseAddModMulti(out, ks, d[:2 * comp].clone(), n, case.mods[:level] * 2)
    return out


@pytest.mark.parametrize("n, L, K, alpha", [(1 << 12, 6, 2, 3), (1 << 15, 15, 1, 1)])
def test_relinearized_call_equals_the_chain(hb, port, n, L, K, alpha):
    case = Case(hb, port, n, _primes(port, n, L, 55) + _primes(port, n, K, 56), L, K, alpha, 65537)
    for level in (L, L // 2 + 1):
        comp = level * n
        ct1, ct2 = dev(case.ciphertexts(level, 1, 4)), dev(case.ciphertexts(level, 1, 5))
        d = torch.zeros(3 * comp, dtype=torch.int64, device="cuda")
        case.multiply(hb, d, ct1, ct2, level)
        fused = torch.zeros(2 * comp, dtype=torch.int64, device="cuda")
        case.relin(hb, fused, ct1, ct2, level)
        chain = _chain(hb, case, d, level)
        torch.cuda.synchronize()
        assert torch.equal(fused, chain), f"n = {n}, level {level}"


def test_alpha_one_k_one_equals_the_chain_with_key_switch_resident(hb, port):
    n, L = 1 << 12, 6
    case = Case(hb, port, n, _primes(port, n, L, 50) + _primes(port, n, 1, 55), L, 1, 1, 65537)
    P = case.mods[-1]
    for level in (L, 3):
        comp = level * n
        ct1, ct2 = dev(case.ciphertexts(level, 1, 6)), dev(case.ciphertexts(level, 1, 7))
        d = torch.zeros(3 * comp, dtype=torch.int64, device="cuda")
        case.multiply(hb, d, ct1, ct2, level)
        fused = torch.zeros(2 * comp, dtype=torch.int64, device="cuda")
        case.relin(hb, fused, ct1, ct2, level)
        ntts = [hb.GetNTT(n, q) for q in case.mods[:level]]
        t = torch.empty(comp, dtype=torch.int64, device="cuda")
        hb.ComputeForwardMulti(ntts, t, d[2 * comp:].clone())
        ks = torch.zeros(2 * comp, dtype=torch.int64, device="cuda")
        modswitch = [pow(P % q, -1, q) for q in case.mods[:level]]
        hb.KeySwitchResident(ks, t, n, level, L + 1, level + 1, 2, case.mods, case.handle, modswitch)
        hb.ComputeInverseMulti(ntts * 2, ks, ks)
        chain = torch.empty(2 * comp, dtype=torch.int64, device="cuda")
        hb.EltwiseAddModMulti(chain, ks, d[:2 * comp].clone(), n, case.mods[:level] * 2)
        torch.cuda.synchronize()
        assert torch.equal(fused, chain), f"level {level}"


# ------------------------------------------------------------------------------------------------ buffers
@pytest.fixture(scope="module")
def buffers_case(hb, port):
    n = 1 << 11
    case = Case(hb, port, n, _primes(port, n, 5, 50) + _primes(port, n, 2, 55), 5, 2, 3, 65537, seed=77)
    level, batch = 4, 3
    ct1, ct2 = case.ciphertexts(level, batch, 21), case.ciphertexts(level, batch, 22)
    exp = {sq: case.expected(ct1, ct1 if sq else ct2, level, batch) for sq in (False, True)}
    return case, level, batch, ct1, ct2, exp


@pytest.mark.parametrize("square", [False, True])
@pytest.mark.parametrize("which", [0, 1])
@pytest.mark.parametrize("entry", ["device", "host", "pinned", "managed", "host_split"])
def test_buffers(hb, buffers_case, entry, which, square):
    """batch 3 between sentinel words; which = 0 the product, 1 the relinearized product"""
    case, level, batch, ct1, ct2, exps = buffers_case
    exp = exps[square][which]
    size = exp.size
    call = case.multiply if which == 0 else case.relin

    def run(out, a, b, stream=None):
        call(hb, out, a, a if square else b, level, batch, stream=stream)

    try:
        if entry == "device":
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                buf = torch.full((size + 2,), SENTINEL - (1 << 64), dtype=torch.int64, device="cuda")
                a, b = dev(ct1), dev(ct2)
                run(buf[1:1 + size], a, b, stream=s)
            s.synchronize()
            got = host(buf)
        elif entry in ("managed", "pinned"):
            alloc, free = ((hb.managed_empty, hb.managed_free) if entry == "managed"
                           else (hb.pinned_empty, hb.pinned_free))
            a, b, buf = alloc(ct1.size), alloc(ct2.size), alloc(size + 2)
            try:
                a[:], b[:], buf[:] = ct1, ct2, SENTINEL
                run(buf[1:1 + size], a, b)
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
            run(buf[1:1 + size], a, b)
            assert (a == ct1).all() and (b == ct2).all(), "the ciphertexts changed"
            got = buf
    finally:
        hb.set_host_devices([])
    assert got[0] == SENTINEL and got[-1] == SENTINEL, "a word next to the output was written"
    _check(got[1:1 + size], exp, f"{entry} which {which} square {square}")


def test_host_batches_wrap_the_staging_slots(hb, port):
    """7 pairs through the 3 rotating staging slots, over one and two host devices"""
    n = 1 << 10
    case = Case(hb, port, n, _primes(port, n, 3, 50) + _primes(port, n, 1, 55), 3, 1, 1, 65537, seed=3)
    batch = 7
    ct1, ct2 = case.ciphertexts(3, batch, 31), case.ciphertexts(3, batch, 32)
    exp_d, exp_r = case.expected(ct1, ct2, 3, batch)
    for devices in ([], [0, 0]):
        try:
            hb.set_host_devices(devices)
            d = np.zeros(exp_d.size, dtype=U64)
            r = np.zeros(exp_r.size, dtype=U64)
            case.multiply(hb, d, ct1, ct2, 3, batch)
            case.relin(hb, r, ct1, ct2, 3, batch)
        finally:
            hb.set_host_devices([])
        _check(d, exp_d, f"products over {devices}")
        _check(r, exp_r, f"relinearized over {devices}")


@pytest.mark.parametrize("which", [0, 1])
def test_graph_replay(hb, buffers_case, which):
    case, level, batch, ct1, ct2, exps = buffers_case
    call = case.multiply if which == 0 else case.relin
    out = torch.zeros(exps[False][which].size, dtype=torch.int64, device="cuda")
    a, b = dev(ct1), dev(ct2)
    call(hb, out, a, b, level, batch)  # warm: tables and pool
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        call(hb, out, a, b, level, batch)
    out.fill_(0)
    graph.replay()
    torch.cuda.synchronize()
    _check(host(out), exps[False][which], "graph replay")
    n1, n2 = case.ciphertexts(level, batch, 23), case.ciphertexts(level, batch, 24)
    a.copy_(dev(n1))
    b.copy_(dev(n2))
    graph.replay()
    torch.cuda.synchronize()
    _check(host(out), case.expected(n1, n2, level, batch)[which], "graph replay, new data")


@pytest.mark.parametrize("which", [0, 1])
def test_held_stream(hb, buffers_case, which):
    """the inputs are written behind a bounded spin on the call's stream, and the result read behind the call"""
    case, level, batch, ct1, ct2, exps = buffers_case
    call = case.multiply if which == 0 else case.relin
    out = torch.zeros(exps[False][which].size, dtype=torch.int64, device="cuda")
    a, b = torch.zeros(ct1.size, dtype=torch.int64, device="cuda"), torch.zeros(ct2.size, dtype=torch.int64,
                                                                                device="cuda")
    src1, src2 = dev(ct1), dev(ct2)
    call(hb, out, src1, src2, level, batch)  # warm
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(50_000_000)
        a.copy_(src1)
        b.copy_(src2)
        out.fill_(0)
        call(hb, out, a, b, level, batch, stream=s)
        got = out.clone()
    s.synchronize()
    _check(host(got), exps[False][which], "held stream")


# ------------------------------------------------------------------------------------------------ launch counts
def _ntt_launches(hb, n, forward):
    ntt = hb.GetNTT(n, hb.GeneratePrimes(1, 50, True, n)[0])
    x = torch.zeros(n, dtype=torch.int64, device="cuda")
    fn = hb.ComputeForwardMulti if forward else hb.ComputeInverseMulti
    fn([ntt], x, x)
    torch.cuda.synchronize()
    before = hb.launch_count()
    fn([ntt], x, x)
    torch.cuda.synchronize()
    return hb.launch_count() - before


def bfv_launches(level, k, square, fwd, inv):
    """per pair: one extension launch per input ciphertext, the forward transforms of the lifted polynomials in
    blocks of 64, one tensor launch per block of 64 moduli, the inverse transforms of the tensor, one scaling launch"""
    M = level + k + 1
    inputs = 2 if square else 4
    return (1 if square else 2) + fwd * -(-inputs * M // 64) + -(-M // 64) + inv * -(-3 * M // 64) + 1


@pytest.mark.parametrize("L, K, alpha, level", [(6, 2, 2, 6), (30, 1, 1, 30), (20, 2, 5, 12)])
def test_launch_counts(hb, port, L, K, alpha, level):
    """the relinearized call adds the launches of KeySwitchHybrid less its first inverse transform; its mod-down
    transforms the products' data limbs back instead of the correction forward"""
    from test_gpu_hybrid_key_switch import expected_launches
    n = 1 << 12
    case = Case(hb, port, n, _primes(port, n, L, 45) + _primes(port, n, K, 46), L, K, alpha, 65537)
    k = len(case.base(level)[0])
    fwd, inv = _ntt_launches(hb, n, True), _ntt_launches(hb, n, False)
    ct1, ct2 = dev(case.ciphertexts(level, 2, 1)), dev(case.ciphertexts(level, 2, 2))
    d = torch.zeros(2 * 3 * level * n, dtype=torch.int64, device="cuda")
    r = torch.zeros(2 * 2 * level * n, dtype=torch.int64, device="cuda")
    blocks = -(-level // 64)
    ks = expected_launches(n, level, L, K, alpha, fwd, inv) - inv * blocks - fwd * blocks + inv * blocks
    runs = [("product", lambda: case.multiply(hb, d, ct1, ct2, level, 2), bfv_launches(level, k, False, fwd, inv)),
            ("square", lambda: case.multiply(hb, d, ct1, ct1, level, 2), bfv_launches(level, k, True, fwd, inv)),
            ("relinearized", lambda: case.relin(hb, r, ct1, ct2, level, 2),
             bfv_launches(level, k, False, fwd, inv) + ks)]
    for name, run, exp in runs:
        run()  # warm
        torch.cuda.synchronize()
        before = hb.launch_count()
        run()
        torch.cuda.synchronize()
        got = hb.launch_count() - before
        assert got == 2 * exp, (name, got, 2 * exp, fwd, inv)


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals(hb, port):
    n, L, K, alpha = 64, 4, 1, 2
    mods = _primes(port, n, L, 50) + _primes(port, n, K, 55)
    case = Case(hb, port, n, mods, L, K, alpha, 65537)
    B, m_sk = case.base(L)
    ct1, ct2 = dev(case.ciphertexts(L, 1, 2)), dev(case.ciphertexts(L, 1, 3))
    d = torch.zeros(3 * L * n, dtype=torch.int64, device="cuda")
    r = torch.zeros(2 * L * n, dtype=torch.int64, device="cuda")

    def refused(what, relin=None, out=None, a=ct1, b=ct2, nn=n, level=L, qmods=None, base=None, msk=None, t=65537,
                keys=case.handle, digit=alpha):
        qmods = qmods if qmods is not None else mods
        base = base if base is not None else B
        msk = msk if msk is not None else m_sk
        mp = np.ascontiguousarray(qmods, dtype=U64)
        bp = np.ascontiguousarray(base, dtype=U64)
        for rl in ((False, True) if relin is None else (relin,)):
            o = out if out is not None else (r if rl else d)
            before = o.clone()
            with pytest.raises(hb.HexlB200Error) as e:
                if rl:
                    hb._check(hb._lib.hexl_b200_bfv_multiply_relinearize_hybrid(
                        o.data_ptr(), a.data_ptr() if a is not None else None, b.data_ptr(), nn, level, L, K, digit,
                        mp.ctypes.data, bp.ctypes.data, bp.size, msk, t, keys._h if keys is not None else None, 1,
                        None))
                else:
                    hb._check(hb._lib.hexl_b200_bfv_multiply(
                        o.data_ptr(), a.data_ptr() if a is not None else None, b.data_ptr(), nn, mp.ctypes.data,
                        level, bp.ctypes.data, bp.size, msk, t, 1, None))
            assert e.value.code == INVALID_ARG, (what, rl, e.value)
            assert torch.equal(o, before), f"{what}: output written"

    refused("null ct1", a=None)
    refused("null keys", relin=True, keys=None)
    refused("n = 1", nn=1)
    refused("n not a power of two", nn=48)
    refused("n = 2^21", nn=1 << 21)
    refused("level 0", level=0)
    refused("level 65", relin=False, level=65, qmods=mods + _primes(port, n, 61, 40))
    refused("k = 0", base=np.zeros(0, dtype=U64))
    refused("k = 65", base=_primes(port, n, 65, 61))
    refused("t = 1", t=1)
    refused("t = 0", t=0)
    refused("t = 2^61", t=1 << 61)
    refused("a modulus of B >= 2^61", base=list(B[:-1]) + [int(port.generate_primes(1, 62, True, n)[0])])
    refused("m_sk >= 2^61", msk=int(port.generate_primes(1, 62, True, n)[0]))
    refused("m_sk not NTT-friendly", msk=(1 << 61) - 1)
    refused("a B modulus not NTT-friendly for n", base=list(B[:-1]) + [B[0] + 2])
    refused("m_sk equal to a modulus of Q", msk=mods[0])
    refused("a B modulus equal to another", base=list(B[:-1]) + [B[0]])
    refused("m_sk equal to a modulus of B", msk=B[0])
    refused("a handle of another digit size", relin=True, digit=1)
    big = torch.zeros(8 * L * n, dtype=torch.int64, device="cuda")
    refused("result overlaps ct1", out=big[L * n:4 * L * n], a=big[:2 * L * n], relin=False)
    refused("result overlaps ct2", out=big[4 * L * n:6 * L * n], b=big[5 * L * n:7 * L * n], relin=True)
    # the bound: the largest t it accepts runs, one more is refused
    tmax = bx.largest_plain_modulus(n, mods[:L], B, m_sk)
    tight = _primes(port, n, 4, 60, set(mods))
    tq = bx.largest_plain_modulus(n, mods[:L], tight[:3], tight[3])
    assert 2 <= tq < 1 << 61 <= tmax
    refused("t one past the bound", t=tq + 1, base=tight[:3], msk=tight[3])
    hb.BfvMultiply(d, ct1, ct2, n, mods, L, tight[:3], tight[3], tq)
    torch.cuda.synchronize()
    _check(host(d), bx.bfv_multiply(port, host(ct1), host(ct2), n, mods[:L], tight[:3], tight[3], tq),
           "the largest t the bound accepts")
    bad = case.ciphertexts(L, 1, 2)
    bad[(L + 1) * n + 3] = mods[1]
    hb.set_debug(True)
    try:
        refused("a ct1 word = q under debug", a=dev(bad))
        refused("a ct2 word = q under debug", b=dev(bad))
    finally:
        hb.set_debug(False)
    before = d.clone()
    case.multiply(hb, d, ct1, ct2, L, 0)
    before_r = r.clone()
    case.relin(hb, r, ct1, ct2, L, 0)
    torch.cuda.synchronize()
    assert torch.equal(d, before) and torch.equal(r, before_r), "batch = 0 wrote"


def test_cpp_caller_runs(hb, tmp_path):
    if not shutil.which("g++"):
        pytest.skip("g++ not present")
    exe = tmp_path / "bfv_caller"
    libdir = os.path.dirname(hb.LIB_PATH)
    subprocess.run(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "cpp", "bfv_caller.cpp"), "-o", str(exe),
                    "-L", libdir, "-lhexl_b200", f"-Wl,-rpath,{libdir}"], check=True)
    res = subprocess.run([str(exe), "run"], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
