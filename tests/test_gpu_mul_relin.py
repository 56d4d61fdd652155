"""MultiplyRelinearizeHybrid on the GPU.

Both rescale modes are compared bit for bit with the exact model of tests/mul_relin_exact.py over the (L, K, alpha)
shapes of the hybrid key-switch tests and their levels (a partial last digit and level 1 included), the three word
classes, every degree from 2 to 2^17, 70 data moduli in 64-modulus digits (two parameter blocks in the mod-up and the
mod-down), primes just below 2^61 with every ciphertext and key word q - 1 (20 digits: multiply-accumulate chunks of
the 128-bit bound), squaring, batch 3, and device, pageable, pinned, split-host and managed buffers.  Also pinned:
rescale = 0 equals DyadicMultiply followed by KeySwitchHybrid bit for bit (at the production shape N = 2^16, L = 30,
alpha = K = 10 too), and at digit size 1 with one special prime DyadicMultiply followed by KeySwitchResident; the inputs
are left unchanged; graph replay with new data; launch counts; the argument refusals; and a C++ caller.  tests/test_gpu_hybrid_rounds.py runs the call with both rescale modes at N = 2^16, (30, 10, 10),
where the merged rescale's mod-down converts into 27 + 2 targets, at budget-limited multi-round shapes, at every
level, over wrapping host batches, offset views and threads."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import hybrid_exact as hx
import mul_relin_exact as mr
from test_gpu_hybrid_key_switch import SENTINEL, _check, _levels, _ntt_launches, _primes, dev, expected_launches, host
from test_gpu_hybrid_rotation import _mod_down_launches, _mod_up_launches
from util import uniform_below

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U64 = np.uint64
INVALID_ARG = -1


@pytest.fixture(scope="module", autouse=True)
def _need_cuda(hb):
    if not torch.cuda.is_available() or hb.device_count() == 0:
        pytest.fail("gpu-marked test collected on a machine without CUDA")


class Case:
    """L data moduli then K special primes, one set of relinearization keys (key component count 2) and its handle"""

    def __init__(self, hb, port, L, K, alpha, n, data_bits=(50,), special_bits=(50,), fill=None, seed=1):
        self.L, self.K, self.alpha, self.n, self.fill = L, K, alpha, n, fill
        self.mods = _primes(port, n, L, data_bits, False) + _primes(port, n, K, special_bits, True)
        assert len(set(self.mods)) == L + K
        self.keys = hx.random_keys(self.mods, n, L, alpha, 2, seed, fill)
        self.handle = hb.KeySwitchKeys(self.keys, n, len(self.keys), L + K, 2)

    def ciphertexts(self, level, batch, seed):
        n, q = self.n, self.mods
        if self.fill == "q-1":
            return np.concatenate([np.full(n, q[i] - 1, dtype=U64) for _ in range(2 * batch) for i in range(level)])
        return np.concatenate([uniform_below(seed * 7919 + 64 * c + i, n, q[i]) for c in range(2 * batch)
                               for i in range(level)])

    def call(self, hb, out, ct1, ct2, level, rescale, batch=1, stream=None):
        return hb.MultiplyRelinearizeHybrid(out, ct1, ct2, self.n, level, self.L, self.K, self.alpha, self.mods,
                                            self.handle, rescale, batch, stream=stream)

    def expected(self, port, ct1, ct2, level, rescale, batch=1):
        per = 2 * level * self.n
        return np.concatenate([mr.multiply_relinearize(port, ct1[c * per:(c + 1) * per], ct2[c * per:(c + 1) * per],
                                                       self.n, level, self.L, self.K, self.alpha, self.mods,
                                                       self.keys, rescale) for c in range(batch)])


def _out(level, rescale, n, batch=1):
    return torch.full((batch * 2 * (level - int(rescale)) * n,), -1, dtype=torch.int64, device="cuda")


def _run(hb, port, case, level, seed, batch=1, square=False):
    """both rescale modes (rescale = 1 from level 2) against the model; the inputs must not change"""
    ct1 = case.ciphertexts(level, batch, seed)
    ct2 = ct1 if square else case.ciphertexts(level, batch, seed + 1000)
    a = dev(ct1)
    b = a if square else dev(ct2)
    for rescale in (False, True) if level >= 2 else (False,):
        out = _out(level, rescale, case.n, batch)
        case.call(hb, out, a, b, level, rescale, batch)
        torch.cuda.synchronize()
        assert torch.equal(a, dev(ct1)) and torch.equal(b, dev(ct2)), "the ciphertexts changed"
        _check(host(out), case.expected(port, ct1, ct2, level, rescale, batch), f"level {level} rescale {rescale}")


@pytest.mark.parametrize("L, K, alpha", [(4, 1, 1), (6, 2, 2), (7, 3, 3), (5, 2, 5), (8, 4, 2)])
def test_shapes_equal_the_model(hb, port, L, K, alpha):
    case = Case(hb, port, L, K, alpha, 256, seed=L * 100 + K * 10 + alpha)
    for level in _levels(L, alpha):
        _run(hb, port, case, level, level)


def test_word_classes(hb, port):
    """29-, 50- and 58-bit data primes in every digit, 45- and 60-bit special primes"""
    case = Case(hb, port, 6, 2, 3, 1 << 10, data_bits=(29, 50, 58), special_bits=(45, 60))
    for level in _levels(6, 3):
        _run(hb, port, case, level, 3)


@pytest.mark.parametrize("logn", range(1, 18))
def test_every_degree(hb, port, logn):
    case = Case(hb, port, 6, 2, 2, 1 << logn, seed=logn)
    _run(hb, port, case, 5, logn)


def test_seventy_moduli_in_64_modulus_digits(hb, port):
    """70 data moduli, alpha = 64, K = 2: B takes two mod-up rounds (the tensor terms in both) and the mod-down two
    blocks of targets, with and without the merged rescale"""
    case = Case(hb, port, 70, 2, 64, 16, data_bits=(55,), special_bits=(55,))
    for level in (70, 66, 5):
        _run(hb, port, case, level, level)


@pytest.mark.parametrize("L, K, alpha, level", [(20, 2, 1, 20), (64, 3, 64, 64), (64, 3, 64, 33)])
def test_worst_case_words_below_2_61(hb, port, L, K, alpha, level):
    """the largest NTT primes below 2^61, every ciphertext and key word q - 1.  (20, 2, 1): 20 digits, so the
    multiply-accumulate takes a chunk of 16 digits (the 128-bit bound) that stores with the tensor terms, and one of 4
    that adds"""
    case = Case(hb, port, L, K, alpha, 64, data_bits=(60,), special_bits=(60,), fill="q-1")
    assert min(case.mods) > 1 << 60
    _run(hb, port, case, level, 0)


def test_squaring(hb, port):
    case = Case(hb, port, 7, 3, 3, 1 << 11, seed=5)
    for level in (7, 5):
        _run(hb, port, case, level, 9, batch=2, square=True)


# ------------------------------------------------------------------------------------------------ equalities
@pytest.mark.parametrize("n, L, K, alpha", [(1 << 12, 9, 3, 4), (1 << 16, 30, 10, 10)])
def test_no_rescale_equals_dyadic_multiply_then_key_switch_hybrid(hb, port, n, L, K, alpha):
    case = Case(hb, port, L, K, alpha, n)
    for level in (L, L // 2 + 1):
        comp = level * n
        ct1, ct2 = dev(case.ciphertexts(level, 1, 4)), dev(case.ciphertexts(level, 1, 5))
        fused = torch.zeros(2 * comp, dtype=torch.int64, device="cuda")
        case.call(hb, fused, ct1, ct2, level, False)
        d = torch.ones(3 * comp, dtype=torch.int64, device="cuda")
        hb.DyadicMultiply(d, ct1, ct2, n, case.mods[:level], level)
        chain = d[:2 * comp].clone()
        hb.KeySwitchHybrid(chain, d[2 * comp:].clone(), n, level, L, K, alpha, 2, case.mods, case.handle)
        torch.cuda.synchronize()
        assert torch.equal(fused, chain), f"n = {n}, level {level}"


@pytest.mark.parametrize("n, L", [(1 << 12, 8), (1 << 16, 30)])
def test_alpha_one_k_one_equals_dyadic_multiply_then_key_switch_resident(hb, port, n, L):
    case = Case(hb, port, L, 1, 1, n)
    P = case.mods[-1]
    for level in (L, L // 2 + 1):
        comp = level * n
        ct1, ct2 = dev(case.ciphertexts(level, 1, 6)), dev(case.ciphertexts(level, 1, 7))
        fused = torch.zeros(2 * comp, dtype=torch.int64, device="cuda")
        case.call(hb, fused, ct1, ct2, level, False)
        d = torch.ones(3 * comp, dtype=torch.int64, device="cuda")
        hb.DyadicMultiply(d, ct1, ct2, n, case.mods[:level], level)
        chain = d[:2 * comp].clone()
        modswitch = [pow(P % q, -1, q) for q in case.mods[:level]]
        hb.KeySwitchResident(chain, d[2 * comp:].clone(), n, level, L + 1, level + 1, 2, case.mods, case.handle,
                             modswitch)
        torch.cuda.synchronize()
        assert torch.equal(fused, chain), f"n = {n}, level {level}"


# ------------------------------------------------------------------------------------------------ buffers
@pytest.fixture(scope="module")
def buffers_case(hb, port):
    case = Case(hb, port, 7, 3, 3, 1 << 11, seed=77)
    level, batch = 5, 3
    ct1, ct2 = case.ciphertexts(level, batch, 21), case.ciphertexts(level, batch, 22)
    exp = {(rs, sq): case.expected(port, ct1, ct1 if sq else ct2, level, rs, batch)
           for rs in (False, True) for sq in (False, True)}
    return case, level, batch, ct1, ct2, exp


@pytest.mark.parametrize("square", [False, True])
@pytest.mark.parametrize("rescale", [False, True])
@pytest.mark.parametrize("entry", ["device", "host", "pinned", "managed", "host_split"])
def test_buffers(hb, buffers_case, entry, rescale, square):
    """batch 3 between sentinel words"""
    case, level, batch, ct1, ct2, exps = buffers_case
    exp = exps[rescale, square]
    size = exp.size

    def run(out, a, b, stream=None):
        case.call(hb, out, a, a if square else b, level, rescale, batch, stream=stream)

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
    _check(got[1:1 + size], exp, f"{entry} rescale {rescale} square {square}")


@pytest.mark.parametrize("rescale", [False, True])
def test_graph_replay(hb, port, buffers_case, rescale):
    case, level, batch, ct1, ct2, exps = buffers_case
    out = torch.zeros(exps[rescale, False].size, dtype=torch.int64, device="cuda")
    a, b = dev(ct1), dev(ct2)
    case.call(hb, out, a, b, level, rescale, batch)  # warm: tables and pool
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        case.call(hb, out, a, b, level, rescale, batch)
    out.fill_(0)
    graph.replay()
    torch.cuda.synchronize()
    _check(host(out), exps[rescale, False], "graph replay")
    n1, n2 = case.ciphertexts(level, batch, 23), case.ciphertexts(level, batch, 24)
    a.copy_(dev(n1))
    b.copy_(dev(n2))
    graph.replay()
    torch.cuda.synchronize()
    _check(host(out), case.expected(port, n1, n2, level, rescale, batch), "graph replay, new data")


# ------------------------------------------------------------------------------------------------ launch counts
def relin_launches(n, level, K, alpha, rescale, fwd, inv):
    """per pair, moduli below 2^60: the mod-up of the hybrid switch (its first inverse transform multiplies on load),
    one multiply-accumulate launch per round (D <= 64 digits), and one mod-down from K + rescale special limbs into
    level - rescale data moduli"""
    return (_mod_up_launches(n, level, K, alpha, fwd, inv, 1)
            + _mod_down_launches(level - int(rescale), K + int(rescale), fwd, inv))


@pytest.mark.parametrize("L, K, alpha, level", [(6, 2, 2, 6), (30, 10, 10, 30), (70, 2, 64, 70), (70, 2, 64, 65),
                                                (12, 1, 1, 12)])
def test_launch_counts(hb, port, L, K, alpha, level):
    """(70, 2, 64, 65): the merged rescale leaves 64 targets, one block of the mod-down instead of two.  The key
    switch's own count is unchanged (expected_launches of the hybrid key-switch tests)."""
    n = 1 << 12
    case = Case(hb, port, L, K, alpha, n, data_bits=(45,), special_bits=(45,))
    ct1, ct2 = dev(case.ciphertexts(level, 2, 1)), dev(case.ciphertexts(level, 2, 2))
    fwd, inv = _ntt_launches(hb, n, True), _ntt_launches(hb, n, False)
    ks_out = torch.zeros(2 * 2 * level * n, dtype=torch.int64, device="cuda")
    runs = [("key switch", lambda: hb.KeySwitchHybrid(ks_out, ct1[:2 * level * n], n, level, L, K, alpha, 2, case.mods,
                                                      case.handle, 2),
             expected_launches(n, level, L, K, alpha, fwd, inv))]
    for rescale in (False, True):
        out = _out(level, rescale, n, 2)
        runs.append((f"rescale {rescale}", lambda out=out, rescale=rescale: case.call(hb, out, ct1, ct2, level,
                                                                                       rescale, 2),
                     relin_launches(n, level, K, alpha, rescale, fwd, inv)))
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
    case = Case(hb, port, 6, 2, 2, 64)
    n, L, K, alpha = case.n, 6, 2, 2
    other = Case(hb, port, 6, 2, 3, 64)  # keys for digit size 3: fewer digits than alpha = 2 needs
    kcc3 = hb.KeySwitchKeys(hx.random_keys(case.mods, n, L, alpha, 3, 4), n, 3, L + K, 3)
    ct1, ct2 = dev(case.ciphertexts(L, 1, 2)), dev(case.ciphertexts(L, 1, 3))
    res = torch.zeros(2 * L * n, dtype=torch.int64, device="cuda")

    def refused(what, out=res, a=ct1, b=ct2, level=L, p_size=K, digit=alpha, mods=None, keys=case.handle, rescale=0):
        mods = mods if mods is not None else case.mods
        before = out.clone()
        with pytest.raises(hb.HexlB200Error) as e:
            hb._check(hb._lib.hexl_b200_multiply_relinearize_hybrid(
                out.data_ptr(), a.data_ptr(), b.data_ptr(), n, level, L, p_size, digit,
                np.ascontiguousarray(mods, dtype=U64).ctypes.data, keys._h if keys is not None else None, rescale, 1,
                None))
        assert e.value.code == INVALID_ARG, (what, e.value)
        assert torch.equal(out, before), f"{what}: output written"

    try:
        hb.set_host_devices([0, 0])
        sharded = hb.KeySwitchKeys(case.keys, n, len(case.keys), L + K, 2, sharded_by_modulus=True)
    finally:
        hb.set_host_devices([])
    refused("null keys", keys=None)
    refused("a handle of another digit size", keys=other.handle)
    refused("a handle for key component count 3", keys=kcc3)
    refused("a sharded handle", keys=sharded)
    refused("level 0", level=0)
    refused("level above q_size", level=L + 1)
    refused("digit size 65", digit=65)
    refused("p_size 0", p_size=0)
    refused("a modulus >= 2^61", mods=case.mods[:-1] + [int(port.generate_primes(1, 62, True, n)[0])])
    refused("a repeated modulus", mods=case.mods[:-1] + [case.mods[0]])
    refused("rescale = 2", rescale=2)
    refused("rescale = -1", rescale=-1)
    refused("rescale at level 1", level=1, rescale=1)
    many = [int(q) for q in port.generate_primes(64, 45, True, n)]
    keys64 = hb.KeySwitchKeys(hx.random_keys(case.mods[:L] + many, n, L, alpha, 2, 8), n, 3, L + 64, 2)
    refused("rescale with 64 special primes", p_size=64, mods=case.mods[:L] + many, keys=keys64, rescale=1)
    big = torch.zeros(8 * L * n, dtype=torch.int64, device="cuda")
    refused("ct1 overlaps ct2", a=big[:2 * L * n], b=big[L * n:3 * L * n])
    refused("result overlaps ct1", out=big[L * n:3 * L * n], a=big[:2 * L * n], b=ct2)
    refused("result overlaps ct2", out=big[4 * L * n:6 * L * n], a=ct1, b=big[5 * L * n:7 * L * n])
    refused("result is the squared ciphertext", out=big[:2 * L * n], a=big[:2 * L * n], b=big[:2 * L * n])
    bad = case.ciphertexts(L, 1, 2)
    bad[(L + 1) * n + 3] = case.mods[1]  # component 1, limb 1
    hb.set_debug(True)
    try:
        refused("a ct1 word = q under debug", a=dev(bad))
        refused("a ct2 word = q under debug", b=dev(bad))
    finally:
        hb.set_debug(False)
    # 64 special primes without rescale are accepted
    out = torch.zeros(2 * L * n, dtype=torch.int64, device="cuda")
    hb.MultiplyRelinearizeHybrid(out, ct1, ct2, n, L, L, 64, alpha, case.mods[:L] + many, keys64)
    torch.cuda.synchronize()
    exp = mr.multiply_relinearize(port, host(ct1), host(ct2), n, L, L, 64, alpha, case.mods[:L] + many,
                                  hx.random_keys(case.mods[:L] + many, n, L, alpha, 2, 8), False)
    _check(host(out), exp, "64 special primes")
    before = res.clone()
    case.call(hb, res, ct1, ct2, L, True, 0)
    torch.cuda.synchronize()
    assert torch.equal(res, before), "batch = 0 wrote"


def test_cpp_caller_runs(hb, tmp_path):
    if not shutil.which("g++"):
        pytest.skip("g++ not present")
    exe = tmp_path / "mul_relin_caller"
    libdir = os.path.dirname(hb.LIB_PATH)
    subprocess.run(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "cpp", "mul_relin_caller.cpp"), "-o", str(exe),
                    "-L", libdir, "-lhexl_b200", f"-Wl,-rpath,{libdir}"], check=True)
    res = subprocess.run([str(exe), "run"], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
