"""ApplyGaloisKeySwitchHybridHoisted and LinearTransformHybrid on the GPU.

Both calls are compared bit for bit with the exact model of tests/hybrid_rotation_exact.py over the (L, K, alpha)
shapes of the hybrid key-switch tests and their levels (a partial last digit and level 1 included), the three word
classes, every degree from 2 to 2^17, 70 data moduli in 64-modulus digits (two parameter blocks, and enough elements
for several multiply-accumulate chunks and two permuted-sum chunks), primes just below 2^61 with every word q - 1 in
ciphertexts, keys and diagonals (digit chunks of the 128-bit bound as well), the elements 1, 3, 5^k and 2n - 1,
repeated elements and identity terms without keys, and device, pageable, pinned, split-host and managed buffers.
Also pinned: equality with ApplyGaloisKeySwitchHoisted at digit size 1 and one special prime, with
[c0, 0] + KeySwitchHybrid(c1) at g = 1, and between the two calls for one element with a unit diagonal; graph replay
with new data; launch counts; the argument refusals; and a C++ caller.  tests/test_gpu_hybrid_rounds.py runs both calls at production sizes whose mod-up takes several
rounds, at every level, over wrapping host batches, offset views and threads, with launch counts from
tests/composite_plan.py."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import hybrid_exact as hx
import hybrid_rotation_exact as hr
from test_gpu_hybrid_key_switch import SENTINEL, _check, _levels, _ntt_launches, _primes, _targets_per_launch, dev, host
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
    """L data moduli then K special primes, `sets` hybrid key sets (key component count 2) and their handles"""

    def __init__(self, hb, port, L, K, alpha, n, data_bits=(50,), special_bits=(50,), fill=None, seed=1, sets=3):
        self.L, self.K, self.alpha, self.n, self.fill = L, K, alpha, n, fill
        self.mods = _primes(port, n, L, data_bits, False) + _primes(port, n, K, special_bits, True)
        assert len(set(self.mods)) == L + K
        self.keys = [hx.random_keys(self.mods, n, L, alpha, 2, seed * 10 + k, fill) for k in range(sets)]
        self.handles = [hb.KeySwitchKeys(k, n, len(k), L + K, 2) for k in self.keys]

    def basis(self, level):
        return self.mods[:level] + self.mods[self.L:]

    def ciphertexts(self, level, batch, seed):
        n, q = self.n, self.mods
        if self.fill == "q-1":
            return np.concatenate([np.full(n, q[i] - 1, dtype=U64) for _ in range(2 * batch) for i in range(level)])
        return np.concatenate([uniform_below(seed * 7919 + 64 * c + i, n, q[i]) for c in range(2 * batch)
                               for i in range(level)])

    def diagonals(self, level, count, seed, fill=None):
        return hr.random_diagonals(self.basis(level), self.n, count, seed, fill or self.fill)

    # spec: [(g, key set or None)], None an identity term (linear transform only)
    def handles_of(self, spec):
        return [None if k is None else self.handles[k] for _, k in spec]

    def keys_of(self, spec):
        return [None if k is None else self.keys[k] for _, k in spec]

    def hoisted(self, hb, out, ct, level, spec, batch=1, stream=None):
        return hb.ApplyGaloisKeySwitchHybridHoisted(out, ct, self.n, level, self.L, self.K, self.alpha, self.mods,
                                                    self.handles_of(spec), [g for g, _ in spec], batch, stream=stream)

    def linear(self, hb, out, ct, diag, level, spec, batch=1, stream=None):
        return hb.LinearTransformHybrid(out, ct, self.n, level, self.L, self.K, self.alpha, self.mods,
                                        self.handles_of(spec), [g for g, _ in spec], diag, batch, stream=stream)

    def expected_hoisted(self, port, ct, level, spec, batch=1):
        per = 2 * level * self.n
        return np.concatenate([hr.hoisted_exact(port, ct[c * per:(c + 1) * per], self.n, level, self.L, self.K,
                                                self.alpha, self.mods, [g for g, _ in spec], self.keys_of(spec))
                               for c in range(batch)])

    def expected_linear(self, port, ct, diag, level, spec, batch=1):
        per = 2 * level * self.n
        return np.concatenate([hr.linear_transform_exact(port, ct[c * per:(c + 1) * per], self.n, level, self.L,
                                                         self.K, self.alpha, self.mods, [g for g, _ in spec],
                                                         self.keys_of(spec), diag) for c in range(batch)])


def _elements(n):
    """3, 5, 25, 2n - 1 (conjugation), 3 again and 1 with keys, each reduced mod 2n"""
    return [(3 % (2 * n), 0), (5 % (2 * n), 1), (2 * n - 1, 2), (25 % (2 * n), 0), (3 % (2 * n), 1), (1, 2)]


def _linear_spec(n):
    """the hoisted elements plus an identity term"""
    return _elements(n) + [(1, None)]


def _run_both(hb, port, case, level, spec, lspec, seed, batch=1):
    n = case.n
    ct = case.ciphertexts(level, batch, seed)
    src = dev(ct)
    out = torch.full((batch * len(spec) * 2 * level * n,), -1, dtype=torch.int64, device="cuda")
    case.hoisted(hb, out, src, level, spec, batch)
    diag = case.diagonals(level, len(lspec), seed)
    res = torch.full((batch * 2 * level * n,), -1, dtype=torch.int64, device="cuda")
    case.linear(hb, res, src, dev(diag), level, lspec, batch)
    torch.cuda.synchronize()
    assert torch.equal(src, dev(ct)), "the ciphertexts changed"
    _check(host(out), case.expected_hoisted(port, ct, level, spec, batch), f"hoisted at level {level}")
    _check(host(res), case.expected_linear(port, ct, diag, level, lspec, batch), f"linear transform at level {level}")


@pytest.mark.parametrize("L, K, alpha", [(4, 1, 1), (6, 2, 2), (7, 3, 3), (5, 2, 5), (8, 4, 2)])
def test_shapes_equal_the_model(hb, port, L, K, alpha):
    case = Case(hb, port, L, K, alpha, 256, seed=L * 100 + K * 10 + alpha)
    for level in _levels(L, alpha):
        _run_both(hb, port, case, level, _elements(256), _linear_spec(256), level)


def test_word_classes(hb, port):
    """29-, 50- and 58-bit data primes in every digit, 45- and 60-bit special primes"""
    case = Case(hb, port, 6, 2, 3, 1 << 10, data_bits=(29, 50, 58), special_bits=(45, 60))
    for level in _levels(6, 3):
        _run_both(hb, port, case, level, _elements(1 << 10), _linear_spec(1 << 10), 3)


@pytest.mark.parametrize("logn", range(1, 18))
def test_every_degree(hb, port, logn):
    n = 1 << logn
    case = Case(hb, port, 6, 2, 2, n, seed=logn, sets=2)
    spec = [(5 % (2 * n), 0), (2 * n - 1, 1)]
    _run_both(hb, port, case, 5, spec, spec + [(1, None)], logn)


def test_seventy_moduli_in_64_modulus_digits(hb, port):
    """70 data moduli, alpha = 64, K = 2: B takes two mod-up rounds and the mod-down two blocks; 70 elements give two
    permuted-sum chunks per block and, with two digits (32 elements per launch), three multiply-accumulate chunks"""
    n = 16
    case = Case(hb, port, 70, 2, 64, n, data_bits=(55,), special_bits=(55,), sets=4)
    elts = [pow(5, k, 2 * n) for k in range(1, 9)] + [2 * n - 1]
    lspec = [(elts[r % len(elts)], r % 4) for r in range(66)] + [(1, None)] * 4
    for level in (70, 5):
        _run_both(hb, port, case, level, [(3, 0), (2 * n - 1, 1), (5, 2)], lspec, level)


@pytest.mark.parametrize("L, K, alpha, level", [(20, 2, 1, 20), (64, 3, 64, 64), (64, 3, 64, 33)])
def test_worst_case_words_below_2_61(hb, port, L, K, alpha, level):
    """the largest NTT primes below 2^61, every ciphertext, key and diagonal word q - 1.  (20, 2, 1): 20 digits, so the
    multiply-accumulate takes chunks of 16 digits (the 128-bit bound) and 4 elements"""
    n = 64
    case = Case(hb, port, L, K, alpha, n, data_bits=(60,), special_bits=(60,), fill="q-1", sets=2)
    assert min(case.mods) > 1 << 60
    spec = [(3, 0), (5, 1), (2 * n - 1, 0), (3, 1), (25, 0), (1, 1)]
    _run_both(hb, port, case, level, spec, spec + [(1, None)], 0)


# ------------------------------------------------------------------------------------------------ equalities
@pytest.mark.parametrize("n, L", [(1 << 12, 8), (1 << 16, 30)])
def test_alpha_one_k_one_equals_apply_galois_key_switch_hoisted(hb, port, n, L):
    case = Case(hb, port, L, 1, 1, n, sets=1)
    spec = [(3, 0), (2 * n - 1, 0), (5, 0)]
    P = case.mods[-1]
    for level in (L, L // 2 + 1):
        ct = dev(case.ciphertexts(level, 2, 4))
        hybrid = torch.zeros(2 * len(spec) * 2 * level * n, dtype=torch.int64, device="cuda")
        seal = torch.ones_like(hybrid)
        case.hoisted(hb, hybrid, ct, level, spec, 2)
        modswitch = [pow(P % q, -1, q) for q in case.mods[:level]]
        hb.ApplyGaloisKeySwitchHoisted(seal, ct, n, level, L + 1, level + 1, 2, case.mods, case.handles_of(spec),
                                       modswitch, [g for g, _ in spec], 2)
        torch.cuda.synchronize()
        assert torch.equal(hybrid, seal), f"n = {n}, level {level}"


@pytest.mark.parametrize("L, K, alpha, level", [(6, 2, 2, 6), (7, 3, 3, 5), (30, 10, 10, 30)])
def test_identity_element_equals_the_hybrid_key_switch(hb, port, L, K, alpha, level):
    n = 1 << 12
    case = Case(hb, port, L, K, alpha, n, sets=1)
    ct = case.ciphertexts(level, 1, 8)
    comp = level * n
    out = torch.zeros(2 * comp, dtype=torch.int64, device="cuda")
    case.hoisted(hb, out, dev(ct), level, [(1, 0)])
    chain = dev(np.concatenate([ct[:comp], np.zeros(comp, dtype=U64)]))
    hb.KeySwitchHybrid(chain, dev(ct[comp:]), n, level, L, K, alpha, 2, case.mods, case.handles[0])
    torch.cuda.synchronize()
    assert torch.equal(out, chain)


@pytest.mark.parametrize("g", [1, 3, 5, (1 << 13) - 1])
def test_one_element_with_unit_diagonal_equals_the_hoisted_call(hb, port, g):
    n, L, K, alpha = 1 << 12, 9, 3, 4
    case = Case(hb, port, L, K, alpha, n, sets=1)
    for level in (9, 6):
        ct = dev(case.ciphertexts(level, 2, g))
        a = torch.zeros(2 * 2 * level * n, dtype=torch.int64, device="cuda")
        b = torch.ones_like(a)
        case.hoisted(hb, a, ct, level, [(g, 0)], 2)
        case.linear(hb, b, ct, dev(case.diagonals(level, 1, 0, fill="one")), level, [(g, 0)], 2)
        torch.cuda.synchronize()
        assert torch.equal(a, b), f"g = {g}, level {level}"


# ------------------------------------------------------------------------------------------------ buffers
@pytest.fixture(scope="module")
def buffers_case(hb, port):
    case = Case(hb, port, 7, 3, 3, 1 << 11, seed=77)
    level, batch = 5, 3
    spec, lspec = _elements(1 << 11)[:3], _linear_spec(1 << 11)[2:]
    ct = case.ciphertexts(level, batch, 21)
    diag = case.diagonals(level, len(lspec), 21)
    return (case, level, batch, spec, lspec, ct, diag, case.expected_hoisted(port, ct, level, spec, batch),
            case.expected_linear(port, ct, diag, level, lspec, batch))


@pytest.mark.parametrize("call", ["hoisted", "linear"])
@pytest.mark.parametrize("entry", ["device", "host", "pinned", "managed", "host_split"])
def test_buffers(hb, buffers_case, call, entry):
    """batch 3 between sentinel words"""
    case, level, batch, spec, lspec, ct, diag, exp_h, exp_l = buffers_case
    exp = exp_h if call == "hoisted" else exp_l
    size = exp.size

    def run(out, src, d, stream=None):
        if call == "hoisted":
            case.hoisted(hb, out, src, level, spec, batch, stream=stream)
        else:
            case.linear(hb, out, src, d, level, lspec, batch, stream=stream)

    try:
        if entry == "device":
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                buf = torch.full((size + 2,), SENTINEL - (1 << 64), dtype=torch.int64, device="cuda")
                src, d = dev(ct), dev(diag)
                run(buf[1:1 + size], src, d, stream=s)
            s.synchronize()
            got = host(buf)
        elif entry in ("managed", "pinned"):
            alloc, free = ((hb.managed_empty, hb.managed_free) if entry == "managed"
                           else (hb.pinned_empty, hb.pinned_free))
            src, d, buf = alloc(ct.size), alloc(diag.size), alloc(size + 2)
            try:
                src[:], d[:], buf[:] = ct, diag, SENTINEL
                run(buf[1:1 + size], src, d)
                got = buf.copy()
                assert (src == ct).all(), "the ciphertexts changed"
            finally:
                for a in (src, d, buf):
                    free(a)
        else:
            if entry == "host_split":
                hb.set_host_devices([0, 0])
            buf = np.full(size + 2, SENTINEL, dtype=U64)
            src = ct.copy()
            run(buf[1:1 + size], src, diag.copy())
            assert (src == ct).all(), "the ciphertexts changed"
            got = buf
    finally:
        hb.set_host_devices([])
    assert got[0] == SENTINEL and got[-1] == SENTINEL, "a word next to the output was written"
    _check(got[1:1 + size], exp, f"{call} {entry}")


@pytest.mark.parametrize("call", ["hoisted", "linear"])
def test_graph_replay(hb, port, buffers_case, call):
    case, level, batch, spec, lspec, ct, diag, exp_h, exp_l = buffers_case
    exp = exp_h if call == "hoisted" else exp_l
    out = torch.zeros(exp.size, dtype=torch.int64, device="cuda")
    src, d = dev(ct), dev(diag)

    def run():
        if call == "hoisted":
            case.hoisted(hb, out, src, level, spec, batch)
        else:
            case.linear(hb, out, src, d, level, lspec, batch)

    run()  # warm: tables and pool
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        run()
    out.fill_(0)
    graph.replay()
    torch.cuda.synchronize()
    _check(host(out), exp, "graph replay")
    ct2, diag2 = case.ciphertexts(level, batch, 22), case.diagonals(level, len(lspec), 22)
    src.copy_(dev(ct2))
    d.copy_(dev(diag2))
    graph.replay()
    torch.cuda.synchronize()
    exp2 = (case.expected_hoisted(port, ct2, level, spec, batch) if call == "hoisted"
            else case.expected_linear(port, ct2, diag2, level, lspec, batch))
    _check(host(out), exp2, "graph replay, new data")


# ------------------------------------------------------------------------------------------------ launch counts
def _mod_up_launches(n, level, K, alpha, fwd, inv, macs_per_round):
    """the target's inverse transform; per mod-up round, one base conversion per digit and block of targets, a
    forward transform and the round's multiply-accumulates"""
    groups = hx.digits(level, alpha)
    nb = level + K
    ichunk = min(max(1, (256 << 20) // (len(groups) * n * 8)), nb, 64)
    total = inv * -(-level // 64)
    for b0 in range(0, nb, ichunk):
        cnt = min(ichunk, nb - b0)
        total += sum(-(-cnt // _targets_per_launch(len(S))) for S in groups) + fwd + macs_per_round
    return total


def _mod_down_launches(level, K, fwd, inv):
    """the special limbs' inverse transform; per block of 64 data moduli the rounding base conversion, a forward
    transform and the finish"""
    return inv + sum(-(-min(64, level - i0) // _targets_per_launch(K)) + fwd + 1 for i0 in range(0, level, 64))


def hoisted_launches(n, level, K, alpha, elts, fwd, inv):
    """per ciphertext, moduli below 2^60 (one multiply-accumulate launch per element and round): one automorphism
    launch per element, the mod-up, and one mod-down per element"""
    return elts + _mod_up_launches(n, level, K, alpha, fwd, inv, elts) + elts * _mod_down_launches(level, K, fwd, inv)


def linear_launches(n, level, K, alpha, elts, keyed, fwd, inv):
    """per ciphertext, moduli below 2^60: one permuted-sum launch per chunk of 64 elements and block of 64 data moduli;
    when some element has keys, the mod-up with ceil(D / jc) x ceil(keyed / floor(64 / jc)) multiply-accumulate
    launches per round (jc = min(D, 64) digits per launch) and ONE mod-down"""
    total = -(-level // 64) * -(-elts // 64)
    if keyed == 0:
        return total
    D = len(hx.digits(level, alpha))
    jc = min(D, 64)
    macs = -(-D // jc) * -(-keyed // max(1, 64 // jc))
    return total + _mod_up_launches(n, level, K, alpha, fwd, inv, macs) + _mod_down_launches(level, K, fwd, inv)


@pytest.mark.parametrize("L, K, alpha, level", [(6, 2, 2, 6), (30, 10, 10, 30), (70, 2, 64, 70), (12, 1, 1, 12)])
@pytest.mark.parametrize("elts", [1, 4, 16])
def test_launch_counts(hb, port, L, K, alpha, level, elts):
    n = 1 << 12
    case = Case(hb, port, L, K, alpha, n, data_bits=(45,), special_bits=(45,), sets=2)
    spec = [(pow(5, r + 1, 2 * n), r % 2) for r in range(elts)]
    lspec = spec + [(1, None)]
    ct = dev(case.ciphertexts(level, 2, 1))
    out = torch.zeros(2 * elts * 2 * level * n, dtype=torch.int64, device="cuda")
    res = torch.zeros(2 * 2 * level * n, dtype=torch.int64, device="cuda")
    diag = dev(case.diagonals(level, len(lspec), 1))
    fwd, inv = _ntt_launches(hb, n, True), _ntt_launches(hb, n, False)
    for name, run, exp in (
            ("hoisted", lambda: case.hoisted(hb, out, ct, level, spec, 2),
             hoisted_launches(n, level, K, alpha, elts, fwd, inv)),
            ("linear", lambda: case.linear(hb, res, ct, diag, level, lspec, 2),
             linear_launches(n, level, K, alpha, elts + 1, elts, fwd, inv)),
            ("identity only", lambda: case.linear(hb, res, ct, diag, level, [(1, None)] * (elts + 1), 2),
             linear_launches(n, level, K, alpha, elts + 1, 0, fwd, inv))):
        run()  # warm
        torch.cuda.synchronize()
        before = hb.launch_count()
        run()
        torch.cuda.synchronize()
        got = hb.launch_count() - before
        assert got == 2 * exp, (name, got, 2 * exp, fwd, inv)


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals(hb, port):
    case = Case(hb, port, 6, 2, 2, 64, sets=2)
    n, L, K, alpha = case.n, 6, 2, 2
    other = Case(hb, port, 6, 2, 3, 64, sets=1)  # keys for digit size 3: fewer digits than alpha = 2 needs
    spec = [(3, 0), (5, 1)]
    ct = dev(case.ciphertexts(L, 1, 2))
    diag = dev(case.diagonals(L, 3, 2))
    outs = torch.zeros(2 * 2 * L * n, dtype=torch.int64, device="cuda")
    res = torch.zeros(2 * L * n, dtype=torch.int64, device="cuda")

    def refused(what, call, handles=None, elts=None, out=None, src=ct, d=diag, level=L, digit=alpha, mods=None):
        handles = handles if handles is not None else case.handles_of(spec)
        elts = elts if elts is not None else [g for g, _ in spec]
        mods = mods if mods is not None else case.mods
        out = out if out is not None else (outs if call == "hoisted" else res)
        before = out.clone()
        with pytest.raises(hb.HexlB200Error) as e:
            if call == "hoisted":
                hb.ApplyGaloisKeySwitchHybridHoisted(out, src, n, level, L, K, digit, mods, handles, elts)
            else:
                hb.LinearTransformHybrid(out, src, n, level, L, K, digit, mods, handles, elts, d)
        assert e.value.code == INVALID_ARG, (what, call, e.value)
        assert torch.equal(out, before), f"{what} ({call}): output written"

    try:
        hb.set_host_devices([0, 0])
        sharded = hb.KeySwitchKeys(case.keys[0], n, len(case.keys[0]), L + K, 2, sharded_by_modulus=True)
    finally:
        hb.set_host_devices([])
    big = torch.zeros(8 * L * n, dtype=torch.int64, device="cuda")
    for call in ("hoisted", "linear"):
        refused("a null key for g = 3", call, handles=[None, case.handles[1]])
        refused("a handle of another digit size", call, handles=[case.handles[0], other.handles[0]])
        refused("a sharded handle", call, handles=[case.handles[0], sharded])
        refused("an even element", call, elts=[3, 4])
        refused("an element of 2n", call, elts=[3, 2 * n + 1])
        refused("level 0", call, level=0)
        refused("digit size 65", call, digit=65)
        refused("a modulus >= 2^61", call, mods=case.mods[:-1] + [int(port.generate_primes(1, 62, True, n)[0])])
        refused("output overlaps the ciphertexts", call, out=big[:4 * L * n if call == "hoisted" else 2 * L * n],
                src=big[L * n:3 * L * n])
        bad = case.ciphertexts(L, 1, 2)
        bad[7] = case.mods[0]
        hb.set_debug(True)
        try:
            refused("a ciphertext word = q under debug", call, src=dev(bad))
        finally:
            hb.set_debug(False)
    refused("a null key for g = 1 in the hoisted call", "hoisted", handles=[None, case.handles[1]], elts=[1, 5])
    d_big = torch.zeros(4 * (L + K) * n, dtype=torch.int64, device="cuda")
    refused("result overlaps the diagonals", "linear", out=d_big[:2 * L * n], d=d_big[n:])
    bad = case.diagonals(L, 3, 2)
    bad[(L + 1) * n + 3] = case.mods[L + 1]  # diagonal 0, limb L + 1: under p_1
    hb.set_debug(True)
    try:
        refused("a diagonal word = its modulus under debug", "linear", d=dev(bad))
    finally:
        hb.set_debug(False)
    before_o, before_r = outs.clone(), res.clone()
    case.hoisted(hb, outs, ct, L, [], 1)
    case.hoisted(hb, outs, ct, L, spec, 0)
    case.linear(hb, res, ct, diag, L, [], 1)
    case.linear(hb, res, ct, diag, L, spec, 0)
    torch.cuda.synchronize()
    assert torch.equal(outs, before_o) and torch.equal(res, before_r), "num_elts = 0 or batch = 0 wrote"


def test_cpp_caller_runs(hb, tmp_path):
    if not shutil.which("g++"):
        pytest.skip("g++ not present")
    exe = tmp_path / "hybrid_rotation_caller"
    libdir = os.path.dirname(hb.LIB_PATH)
    subprocess.run(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "cpp", "hybrid_rotation_caller.cpp"), "-o", str(exe),
                    "-L", libdir, "-lhexl_b200", f"-Wl,-rpath,{libdir}"], check=True)
    res = subprocess.run([str(exe), "run"], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
