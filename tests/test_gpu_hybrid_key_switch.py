"""KeySwitchHybrid and FastBaseConvert on the GPU.

Every output is compared bit for bit with the exact model of tests/hybrid_exact.py: the shapes (L, K, alpha) the
definitions distinguish (one-modulus digits, a partial last digit, one digit, more special primes than a digit holds),
the three word classes of the transforms, 70 data moduli in one 64-modulus digit (two parameter blocks and a 64-term
base conversion), primes just below 2^61 with every word q - 1, levels L, a partial digit and 1, key component counts
1 to 3, and every degree from 2 to 2^17.  At alpha = 1 and K = 1 the call equals KeySwitchResident bit for bit.  Device,
pageable and pinned host, split host and managed buffers, graph replay, launch counts, decryption and the argument
refusals are pinned.  tests/test_gpu_hybrid_rounds.py runs the call at production sizes whose mod-up takes several
rounds, at every level, over wrapping host batches, offset views and threads; tests/test_gpu_base_convert_domain.py
runs FastBaseConvert across its whole domain against plain integers."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import hybrid_exact as hx
from util import uniform_below

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U64 = np.uint64
SENTINEL = 0xA5A5A5A5A5A5A5A5
INVALID_ARG = -1


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=U64).view(np.int64)).to("cuda")


def host(t):
    return t.cpu().numpy().view(U64)


@pytest.fixture(scope="module", autouse=True)
def _need_cuda(hb):
    if not torch.cuda.is_available() or hb.device_count() == 0:
        pytest.fail("gpu-marked test collected on a machine without CUDA")


def _check(got, exp, what):
    bad = int((np.asarray(got, dtype=U64) != exp).sum())
    assert bad == 0, f"{what}: {bad} of {exp.size} words differ"


class Case:
    """moduli (L data, then K special), keys and their handle"""

    def __init__(self, hb, port, L, K, alpha, n, kcc, data_bits=(50,), special_bits=(50,), fill=None, seed=1):
        self.L, self.K, self.alpha, self.n, self.kcc, self.fill = L, K, alpha, n, kcc, fill
        self.mods = _primes(port, n, L, data_bits, False) + _primes(port, n, K, special_bits, True)
        assert len(set(self.mods)) == L + K
        self.keys = hx.random_keys(self.mods, n, L, alpha, kcc, seed, fill)
        self.dnum = len(self.keys)
        self.handle = hb.KeySwitchKeys(self.keys, n, self.dnum, L + K, kcc)

    def inputs(self, level, batch, seed):
        """(result, target) of `batch` ciphertexts, canonical"""
        n, q = self.n, self.mods
        if self.fill == "q-1":
            res = np.concatenate([np.full(n, q[i] - 1, dtype=U64) for _ in range(batch * self.kcc)
                                  for i in range(level)])
            t = np.concatenate([np.full(n, q[i] - 1, dtype=U64) for _ in range(batch) for i in range(level)])
            return res, t
        res = np.concatenate([uniform_below(seed * 7919 + 64 * c + i, n, q[i]) for c in range(batch * self.kcc)
                              for i in range(level)])
        t = np.concatenate([uniform_below(seed * 104729 + 64 * c + i, n, q[i]) for c in range(batch)
                            for i in range(level)])
        return res, t

    def expected(self, port, level, res, t, batch):
        per_r, per_t = self.kcc * level * self.n, level * self.n
        return np.concatenate([hx.key_switch_hybrid(port, res[c * per_r:(c + 1) * per_r], t[c * per_t:(c + 1) * per_t],
                                                    self.n, level, self.L, self.K, self.alpha, self.kcc, self.mods,
                                                    self.keys) for c in range(batch)])

    def call(self, hb, result, target, level, batch=1, stream=None):
        return hb.KeySwitchHybrid(result, target, self.n, level, self.L, self.K, self.alpha, self.kcc, self.mods,
                                  self.handle, batch, stream=stream)


def _primes(port, n, count, bits, avoid_first):
    """count NTT primes cycling through the bit sizes; distinct from those of the same sizes drawn for the data
    moduli when avoid_first (the special primes take them from the other end of the range)"""
    out = []
    per = {b: (count + len(bits) - 1 - k) // len(bits) for k, b in enumerate(bits)}
    for b in bits:
        if per[b] == 0:
            continue
        if b >= 60:
            ps = port.generate_primes(per[b] + (128 if avoid_first else 0), b, False, n)
        else:
            ps = port.generate_primes(per[b] + (128 if avoid_first else 0), b, True, n)
        out += [int(q) for q in (ps[-per[b]:] if avoid_first else ps[:per[b]])]
    return out


def _levels(L, alpha):
    """L, a level that leaves a partial last digit (when there is one), and 1"""
    partial = next((l for l in range(L - 1, 0, -1) if l % alpha), None)
    return sorted({L, 1} | ({partial} if partial else set()), reverse=True)


def _run_device(case, hb, level, res, t, batch=1):
    out, src = dev(res), dev(t)
    case.call(hb, out, src, level, batch)
    torch.cuda.synchronize()
    assert torch.equal(src, dev(t)), "the target changed"
    return host(out)


@pytest.mark.parametrize("kcc", [1, 2, 3])
@pytest.mark.parametrize("L, K, alpha", [(4, 1, 1), (6, 2, 2), (7, 3, 3), (5, 2, 5), (8, 4, 2)])
def test_shapes_equal_the_model(hb, port, L, K, alpha, kcc):
    case = Case(hb, port, L, K, alpha, 256, kcc, seed=L * 100 + K * 10 + alpha)
    for level in _levels(L, alpha):
        res, t = case.inputs(level, 1, level)
        _check(_run_device(case, hb, level, res, t), case.expected(port, level, res, t, 1),
               f"({L}, {K}, {alpha}) kcc {kcc} level {level}")


def test_word_classes(hb, port):
    """29-, 50- and 58-bit data primes (the three word classes of the transforms) in every digit, 45- and 60-bit
    special primes, the larger above every data prime"""
    case = Case(hb, port, 6, 2, 3, 1 << 10, 2, data_bits=(29, 50, 58), special_bits=(45, 60))
    for level in _levels(6, 3):
        res, t = case.inputs(level, 1, 3)
        _check(_run_device(case, hb, level, res, t), case.expected(port, level, res, t, 1), f"level {level}")


def test_seventy_moduli_in_a_64_modulus_digit(hb, port):
    """70 data moduli, alpha = 64, K = 2: the 72 moduli of B take two mod-up rounds and the mod-down two blocks, and
    the first digit's base conversion sums 64 terms"""
    case = Case(hb, port, 70, 2, 64, 1 << 10, 2, data_bits=(55,), special_bits=(55,))
    for level in (70, 64, 1):
        res, t = case.inputs(level, 1, 5)
        _check(_run_device(case, hb, level, res, t), case.expected(port, level, res, t, 1), f"level {level}")


def test_worst_case_words_below_2_61(hb, port):
    """the largest NTT primes below 2^61, every input, result and key word q - 1: the 128-bit sums of the 64-term
    base conversion and of the multiply-accumulate at their largest"""
    case = Case(hb, port, 64, 3, 64, 64, 2, data_bits=(60,), special_bits=(60,), fill="q-1")
    assert min(case.mods) > 1 << 60
    for level in (64, 33):
        res, t = case.inputs(level, 1, 0)
        _check(_run_device(case, hb, level, res, t), case.expected(port, level, res, t, 1), f"level {level}")


@pytest.mark.parametrize("logn", range(1, 18))
def test_every_degree(hb, port, logn):
    case = Case(hb, port, 6, 2, 2, 1 << logn, 2, seed=logn)
    for level in (6, 3):
        res, t = case.inputs(level, 1, logn)
        _check(_run_device(case, hb, level, res, t), case.expected(port, level, res, t, 1), f"n = 2^{logn} level {level}")


def test_n16_thirty_moduli_ten_digit_size_ten_special(hb, port):
    case = Case(hb, port, 30, 10, 10, 1 << 16, 2)
    res, t = case.inputs(30, 1, 9)
    _check(_run_device(case, hb, 30, res, t), case.expected(port, 30, res, t, 1), "N = 2^16, (30, 10, 10)")


@pytest.mark.parametrize("n, L", [(1 << 12, 8), (1 << 16, 30)])
def test_alpha_one_k_one_equals_key_switch_resident(hb, port, n, L):
    case = Case(hb, port, L, 1, 1, n, 2)
    P = case.mods[-1]
    for level in (L, L // 2 + 1):
        res, t = case.inputs(level, 2, 4)
        hybrid, resident = dev(res), dev(res)
        case.call(hb, hybrid, dev(t), level, 2)
        modswitch = [pow(P % q, -1, q) for q in case.mods[:level]]
        hb.KeySwitchResident(resident, dev(t), n, level, L + 1, level + 1, 2, case.mods, case.handle, modswitch, 2)
        torch.cuda.synchronize()
        assert torch.equal(hybrid, resident), f"n = {n}, level {level}"


# ------------------------------------------------------------------------------------------------ base conversion
def _convert_model(port, x, n, src, dst, count):
    per = len(src) * n
    return np.concatenate([hx.fast_base_convert(port, x[p * per:(p + 1) * per], n, src, dst) for p in range(count)])


@pytest.mark.parametrize("shape, n", [(shape, n) for shape in ("from64_worst", "to70", "small")
                                      for n in (1, 3, 1 << 10)] + [("one_per_slot", 1 << 16)])
def test_fast_base_convert(hb, port, shape, n):
    """one_per_slot: a polynomial's result (33 x 2^16 words) is more than half of a 32 MiB staging chunk, so each
    host chunk is one polynomial, and 4 of them wrap around the 3 staging slots"""
    count = 4 if shape == "one_per_slot" else 3
    if shape == "from64_worst":
        mods = [int(q) for q in port.generate_primes(67, 60, False, 2)]
        src, dst = mods[:64], mods[64:]
        x = np.concatenate([np.full(n, q - 1, dtype=U64) for _ in range(count) for q in src])
    else:
        sizes = {"to70": (3, 70), "small": (2, 3), "one_per_slot": (2, 33)}[shape]
        mods = [int(q) for q in port.generate_primes(sum(sizes), 50, True, 2)]
        src, dst = mods[:sizes[0]], mods[sizes[0]:]
        x = np.concatenate([uniform_below(11 * p + i, n, q) for p in range(count) for i, q in enumerate(src)])
    exp = _convert_model(port, x, n, src, dst, count)
    out = torch.full((exp.size,), -1, dtype=torch.int64, device="cuda")
    hb.FastBaseConvert(out, dev(x), n, src, dst, count)
    torch.cuda.synchronize()
    _check(host(out), exp, f"{shape} n={n} device")
    # an unaligned view (8-byte offset) runs the word-at-a-time kernel
    buf = torch.full((exp.size + 2,), -1, dtype=torch.int64, device="cuda")
    xin = torch.zeros(x.size + 1, dtype=torch.int64, device="cuda")
    xin[1:] = dev(x)
    hb.FastBaseConvert(buf[1:1 + exp.size], xin[1:], n, src, dst, count)
    torch.cuda.synchronize()
    _check(host(buf[1:1 + exp.size]), exp, f"{shape} n={n} offset view")
    assert int(buf[0]) == -1 and int(buf[-1]) == -1, "a word next to the result was written"
    for devices in ([], [0, 0]):
        try:
            hb.set_host_devices(devices)
            got = np.full(exp.size, SENTINEL, dtype=U64)
            hb.FastBaseConvert(got, x.copy(), n, src, dst, count)
        finally:
            hb.set_host_devices([])
        _check(got, exp, f"{shape} n={n} host {devices}")


def test_fast_base_convert_refusals(hb, port):
    mods = [int(q) for q in port.generate_primes(4, 50, True, 2)]
    n = 8
    x = dev(np.zeros(2 * n, dtype=U64))
    out = torch.full((2 * n,), -1, dtype=torch.int64, device="cuda")

    def refused(what, src=mods[:2], dst=mods[2:], operand=x, result=out):
        with pytest.raises(hb.HexlB200Error) as e:
            hb.FastBaseConvert(result, operand, n, src, dst)
        assert e.value.code == INVALID_ARG, (what, e.value)

    refused("65 sources", src=[int(q) for q in port.generate_primes(65, 50, True, 2)],
            operand=dev(np.zeros(65 * n, dtype=U64)))
    refused("source modulus 1", src=[1, mods[0]])
    refused("target >= 2^61", dst=[(1 << 61) + 1, mods[2]])
    refused("sources not coprime", src=[mods[0], mods[0]])
    refused("result overlaps operand", result=x)
    refused("no targets", dst=[])
    hb.set_debug(True)
    try:
        refused("input = q under debug", operand=dev(np.full(2 * n, mods[0], dtype=U64)))
    finally:
        hb.set_debug(False)
    assert (host(out) == ~U64(0)).all(), "a refused call wrote"
    hb.FastBaseConvert(out, x, n, mods[:2], mods[2:], count=0)
    torch.cuda.synchronize()
    assert (host(out) == ~U64(0)).all(), "count = 0 wrote"


# ------------------------------------------------------------------------------------------------ buffers
@pytest.fixture(scope="module")
def buffers_case(hb, port):
    case = Case(hb, port, 7, 3, 3, 1 << 11, 2, seed=77)
    level = 5
    res, t = case.inputs(level, 3, 21)
    return case, level, res, t, case.expected(port, level, res, t, 3)


@pytest.mark.parametrize("entry", ["device", "host", "pinned", "managed", "host_split"])
def test_buffers(hb, buffers_case, entry):
    """batch 3 between sentinel words"""
    case, level, res, t, exp = buffers_case
    size = res.size
    try:
        if entry == "device":
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                buf = torch.full((size + 2,), SENTINEL - (1 << 64), dtype=torch.int64, device="cuda")
                buf[1:1 + size] = dev(res)
                src = dev(t)
                case.call(hb, buf[1:1 + size], src, level, 3, stream=s)
            s.synchronize()
            got = host(buf)
        elif entry == "managed":
            src, buf = hb.managed_empty(t.size), hb.managed_empty(size + 2)
            try:
                src[:] = t
                buf[:] = SENTINEL
                buf[1:1 + size] = res
                case.call(hb, buf[1:1 + size], src, level, 3)
                got = buf.copy()
            finally:
                hb.managed_free(src)
                hb.managed_free(buf)
        elif entry == "pinned":
            src, buf = hb.pinned_empty(t.size), hb.pinned_empty(size + 2)
            try:
                src[:] = t
                buf[:] = SENTINEL
                buf[1:1 + size] = res
                case.call(hb, buf[1:1 + size], src, level, 3)
                got = buf.copy()
            finally:
                hb.pinned_free(src)
                hb.pinned_free(buf)
        else:
            if entry == "host_split":
                hb.set_host_devices([0, 0])
            buf = np.full(size + 2, SENTINEL, dtype=U64)
            buf[1:1 + size] = res
            src = t.copy()
            case.call(hb, buf[1:1 + size], src, level, 3)
            assert (src == t).all(), "the target changed"
            got = buf
    finally:
        hb.set_host_devices([])
    assert got[0] == SENTINEL and got[-1] == SENTINEL, "a word next to result was written"
    _check(got[1:1 + size], exp, entry)


def test_graph_replay(hb, port, buffers_case):
    case, level, res, t, exp = buffers_case
    out, src = dev(res), dev(t)
    case.call(hb, out, src, level, 3)  # warm: tables and pool
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        case.call(hb, out, src, level, 3)
    out.copy_(dev(res))
    graph.replay()
    torch.cuda.synchronize()
    _check(host(out), exp, "graph replay")
    res2, t2 = case.inputs(level, 3, 22)
    out.copy_(dev(res2))
    src.copy_(dev(t2))
    graph.replay()
    torch.cuda.synchronize()
    _check(host(out), case.expected(port, level, res2, t2, 3), "graph replay, new data")


def _targets_per_launch(sources):
    """internal.h: base_conv_targets, the targets one base-conversion launch takes"""
    return (480 - 4 * sources) // (5 + sources)


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


def expected_launches(n, level, L, K, alpha, fwd, inv):
    """per ciphertext, moduli below 2^60 (one multiply-accumulate launch per round): the target's inverse transform;
    per mod-up round, one base conversion per digit and block of targets, a forward transform and the
    multiply-accumulate; the special limbs' inverse transform; per block of 64 data moduli the rounding base
    conversion, a forward transform and the finish"""
    groups = hx.digits(level, alpha)
    nb = level + K
    ichunk = min(max(1, (256 << 20) // (len(groups) * n * 8)), nb, 64)
    total = inv * -(-level // 64)
    for b0 in range(0, nb, ichunk):
        cnt = min(ichunk, nb - b0)
        total += sum(-(-cnt // _targets_per_launch(len(S))) for S in groups) + fwd + 1
    total += inv
    for i0 in range(0, level, 64):
        cnt = min(64, level - i0)
        total += -(-cnt // _targets_per_launch(K)) + fwd + 1
    return total


@pytest.mark.parametrize("L, K, alpha, level", [(6, 2, 2, 6), (30, 10, 10, 30), (70, 2, 64, 70), (70, 2, 64, 5),
                                                (12, 1, 1, 12)])
def test_launch_counts(hb, port, L, K, alpha, level):
    n = 1 << 12
    case = Case(hb, port, L, K, alpha, n, 2, data_bits=(45,), special_bits=(45,))
    res, t = case.inputs(level, 2, 1)
    out, src = dev(res), dev(t)
    case.call(hb, out, src, level, 2)  # warm
    torch.cuda.synchronize()
    before = hb.launch_count()
    case.call(hb, out, src, level, 2)
    torch.cuda.synchronize()
    got = hb.launch_count() - before
    fwd, inv = _ntt_launches(hb, n, True), _ntt_launches(hb, n, False)
    assert got == 2 * expected_launches(n, level, L, K, alpha, fwd, inv), (got, fwd, inv)


@pytest.mark.parametrize("L, K, alpha", [(6, 2, 2), (7, 3, 3), (5, 5, 5)])
def test_switched_ciphertext_decrypts(hb, port, L, K, alpha):
    """keys from a secret (hybrid_exact.hybrid_keys): u0 + u1 s - t s_new stays within the bound of
    tests/test_hybrid_exact.py at full and partial level, and the keys of another secret miss it by far"""
    from test_hybrid_exact import hybrid_case, noise_bound
    n = 1 << 12
    mods, s, s_new, keys = hybrid_case(port, L, K, alpha, n, 40 + L)
    handle = hb.KeySwitchKeys(keys, n, len(keys), L + K, 2)
    for level in sorted({L, L - 1}):
        t = np.concatenate([uniform_below(90 + i, n, q) for i, q in enumerate(mods[:level])])
        out = torch.zeros(2 * level * n, dtype=torch.int64, device="cuda")
        hb.KeySwitchHybrid(out, dev(t), n, level, L, K, alpha, 2, mods, handle)
        got = hx.noise(port, host(out), t, s, s_new, n, level, mods)
        bound = noise_bound(mods, L, K, alpha, level, n, 8)
        assert got <= bound, f"level {level}: noise {got} above {bound}"
        assert hx.noise(port, host(out), t, s, s, n, level, mods) > bound << 20


def test_refusals(hb, port):
    case = Case(hb, port, 6, 2, 2, 64, 2)
    n, L, K, alpha = case.n, 6, 2, 2
    res, t = case.inputs(L, 1, 2)
    # room for every shape tried below, so that each refusal comes from the library
    out = torch.zeros(3 * (L + 1) * n, dtype=torch.int64, device="cuda")
    out[:res.size] = dev(res)
    src = torch.zeros((L + 1) * n, dtype=torch.int64, device="cuda")
    src[:t.size] = dev(t)

    def refused(what, result=out, target=src, nn=n, level=L, q_size=L, p_size=K, digit=alpha, kcc=2, mods=None,
                keys=case.handle):
        before = result.clone()
        with pytest.raises(hb.HexlB200Error) as e:
            hb.KeySwitchHybrid(result, target, nn, level, q_size, p_size, digit, kcc,
                               case.mods if mods is None else mods, keys, 1)
        assert e.value.code == INVALID_ARG, (what, e.value)
        assert torch.equal(result, before), f"{what}: result written"

    refused("null keys", keys=None)
    refused("n not a power of two", nn=48)
    refused("n = 2^21", nn=1 << 21, result=torch.zeros(2 * L << 21, dtype=torch.int64, device="cuda"),
            target=torch.zeros(L << 21, dtype=torch.int64, device="cuda"))
    refused("level 0", level=0)
    refused("level above q_size", level=L + 1)
    refused("digit size 0", digit=0)
    refused("digit size 65", digit=65)
    refused("p_size 0", p_size=0, mods=case.mods[:L])
    refused("p_size 65", p_size=65, mods=case.mods + [case.mods[0]] * 63)
    refused("a modulus that is not NTT-friendly", mods=case.mods[:-1] + [(1 << 40) + 15])
    refused("a modulus >= 2^61", mods=case.mods[:-1] + [int(port.generate_primes(1, 62, True, n)[0])])
    refused("a repeated modulus", mods=case.mods[:-1] + [case.mods[0]])
    refused("a handle with fewer digits than the shape needs", digit=1)
    refused("a handle for another component count", kcc=3)
    refused("a handle for another number of special primes", p_size=1, mods=case.mods[:-1])
    try:
        hb.set_host_devices([0, 0])
        sharded = hb.KeySwitchKeys(case.keys, n, case.dnum, L + K, 2, sharded_by_modulus=True)
    finally:
        hb.set_host_devices([])
    refused("a sharded handle", keys=sharded)
    big = torch.zeros(4 * L * n, dtype=torch.int64, device="cuda")
    refused("result overlaps target", result=big[:2 * L * n], target=big[L * n:2 * L * n])
    bad = t.copy()
    bad[5] = case.mods[0]
    hb.set_debug(True)
    try:
        refused("target word = q under debug", target=dev(bad))
    finally:
        hb.set_debug(False)
    before = out.clone()
    hb.KeySwitchHybrid(out, src, n, L, L, K, alpha, 2, case.mods, case.handle, 0)
    torch.cuda.synchronize()
    assert torch.equal(out, before), "batch = 0 wrote"


def test_cpp_caller_runs(hb, tmp_path):
    if not shutil.which("g++"):
        pytest.skip("g++ not present")
    exe = tmp_path / "hybrid_caller"
    libdir = os.path.dirname(hb.LIB_PATH)
    subprocess.run(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "cpp", "hybrid_caller.cpp"), "-o", str(exe),
                    "-L", libdir, "-lhexl_b200", f"-Wl,-rpath,{libdir}"], check=True)
    res = subprocess.run([str(exe), "run"], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
