"""MultiplyRelinearizeSumHybrid on the GPU.

Both rescale modes are compared bit for bit with the exact model of tests/mul_relin_sum_exact.py, and the inputs must
be left unchanged, over the (L, K, alpha) shapes of the hybrid key-switch tests and their levels (a partial last digit
and level 1 included), the three word classes, every degree from 2 to 2^17, 70 data moduli in 64-modulus digits (two
blocks of limbs in the tensor-sum kernel, two mod-up rounds), 2, 3, 32, 33 and 65 pairs with every word q - 1 under the
largest NTT primes below 2^61 (across the 32-pair chunks of the 128-bit sums), repeated ciphertexts across pairs and
outputs, squares, and batch 3 with pairs shared between outputs.  Also pinned: one pair equals MultiplyRelinearizeHybrid
bit for bit; rescale = 0 equals DyadicMultiply of every pair, EltwiseAddModMulti and KeySwitchHybrid bit for bit (at
N = 2^16, L = 30, alpha = K = 10 with 4 pairs too); device, pageable, pinned, split-host and managed buffers; graph
replay with new data written into the same input buffers; launch counts; the call runs in order on a held stream;
every refusal; and a C++ caller."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import hybrid_exact as hx
import mul_relin_sum_exact as ms
from test_gpu_hybrid_key_switch import SENTINEL, _check, _levels, _ntt_launches, dev, host
from test_gpu_mul_relin import Case, relin_launches
from test_gpu_stream_order import Row, _finish, _stage, hold_cycles  # noqa: F401 (hold_cycles is a fixture)

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U64 = np.uint64
INVALID_ARG = -1
MIXED_POINTERS = -5


@pytest.fixture(scope="module", autouse=True)
def _need_cuda(hb):
    if not torch.cuda.is_available() or hb.device_count() == 0:
        pytest.fail("gpu-marked test collected on a machine without CUDA")


class SumCase(Case):
    """a Case of tests/test_gpu_mul_relin.py with the sum call; pairs are index lists into a pool of ciphertexts"""

    def pool(self, level, count, seed):
        return [self.ciphertexts(level, 1, seed + j) for j in range(count)]

    def call_sum(self, hb, out, ct1s, ct2s, level, rescale, batch=1, stream=None):
        return hb.MultiplyRelinearizeSumHybrid(out, ct1s, ct2s, self.n, level, self.L, self.K, self.alpha, self.mods,
                                               self.handle, rescale, batch, stream=stream)

    def expected_sum(self, port, ct1s, ct2s, level, rescale, batch=1):
        k = len(ct1s) // batch
        return np.concatenate([ms.multiply_relinearize_sum(port, ct1s[c * k:(c + 1) * k], ct2s[c * k:(c + 1) * k],
                                                           self.n, level, self.L, self.K, self.alpha, self.mods,
                                                           self.keys, rescale) for c in range(batch)])


def _out(level, rescale, n, batch=1):
    return torch.full((batch * 2 * (level - int(rescale)) * n,), -1, dtype=torch.int64, device="cuda")


def _distinct_pairs(pairs, batch):
    """pool indices: every entry its own ciphertext"""
    total = pairs * batch
    return list(range(total)), list(range(total, 2 * total)), 2 * total


def _shared_pairs(pairs, batch):
    """pool indices with repeats: pair r of every output shares ct1 with output 0, every third pair squares, and the
    ct2 pool is smaller than the pairs, so ciphertexts repeat within an output too"""
    i1, i2 = [], []
    m = max(2, pairs // 2)
    for c in range(batch):
        for r in range(pairs):
            a = r if c % 2 == 0 else pairs + r
            i1.append(a)
            i2.append(a if r % 3 == 2 else 2 * pairs + (r + c) % m)
    return i1, i2, 2 * pairs + m


def _run(hb, port, case, level, seed, pairs, batch=1, layout=_distinct_pairs):
    """both rescale modes (rescale = 1 from level 2) against the model; the inputs must not change"""
    i1, i2, count = layout(pairs, batch)
    pool = case.pool(level, count, seed)
    tens = [dev(ct) for ct in pool]
    ct1s, ct2s = [pool[i] for i in i1], [pool[i] for i in i2]
    for rescale in (False, True) if level >= 2 else (False,):
        out = _out(level, rescale, case.n, batch)
        case.call_sum(hb, out, [tens[i] for i in i1], [tens[i] for i in i2], level, rescale, batch)
        torch.cuda.synchronize()
        assert all(torch.equal(t, dev(ct)) for t, ct in zip(tens, pool)), "an input ciphertext changed"
        _check(host(out), case.expected_sum(port, ct1s, ct2s, level, rescale, batch),
               f"level {level} rescale {rescale} pairs {pairs}")


@pytest.mark.parametrize("L, K, alpha", [(4, 1, 1), (6, 2, 2), (7, 3, 3), (5, 2, 5), (8, 4, 2)])
def test_shapes_equal_the_model(hb, port, L, K, alpha):
    case = SumCase(hb, port, L, K, alpha, 256, seed=L * 100 + K * 10 + alpha)
    for level in _levels(L, alpha):
        _run(hb, port, case, level, level, 3)


def test_word_classes(hb, port):
    """29-, 50- and 58-bit data primes in every digit, 45- and 60-bit special primes"""
    case = SumCase(hb, port, 6, 2, 3, 1 << 10, data_bits=(29, 50, 58), special_bits=(45, 60))
    for level in _levels(6, 3):
        _run(hb, port, case, level, 3, 2)


@pytest.mark.parametrize("logn", range(1, 18))
def test_every_degree(hb, port, logn):
    case = SumCase(hb, port, 6, 2, 2, 1 << logn, seed=logn)
    _run(hb, port, case, 5, logn, 2)


def test_seventy_moduli_in_64_modulus_digits(hb, port):
    """70 data moduli, alpha = 64, K = 2: two blocks of limbs in the tensor-sum kernel, two mod-up rounds and two
    blocks of targets in the mod-down, with and without the merged rescale"""
    case = SumCase(hb, port, 70, 2, 64, 16, data_bits=(55,), special_bits=(55,))
    for level in (70, 66, 5):
        _run(hb, port, case, level, level, 2)


@pytest.mark.parametrize("pairs", [2, 3, 32, 33, 65])
def test_worst_case_words_below_2_61(hb, port, pairs):
    """the largest NTT primes below 2^61, every ciphertext and key word q - 1: each chunk of 32 pairs puts 64 products
    of (q - 1)^2 into d1's 128-bit sum, and 33 and 65 pairs add a chunk of one pair mod q"""
    case = SumCase(hb, port, 20, 2, 1, 64, data_bits=(60,), special_bits=(60,), fill="q-1")
    assert min(case.mods) > 1 << 60
    _run(hb, port, case, 20, 0, pairs)


def test_worst_case_words_at_64_moduli(hb, port):
    case = SumCase(hb, port, 64, 3, 64, 64, data_bits=(60,), special_bits=(60,), fill="q-1")
    _run(hb, port, case, 64, 0, 33)


@pytest.mark.parametrize("pairs", [2, 5])
def test_repeats_squares_and_shared_pairs(hb, port, pairs):
    """batch 3: outputs 0 and 2 share their ct1 entries, squares, and repeated ct2 entries within and across outputs"""
    case = SumCase(hb, port, 7, 3, 3, 1 << 11, seed=5)
    for level in (7, 5):
        _run(hb, port, case, level, 9, pairs, batch=3, layout=_shared_pairs)


# ------------------------------------------------------------------------------------------------ equalities
def test_one_pair_equals_multiply_relinearize(hb, port):
    case = SumCase(hb, port, 7, 3, 3, 1 << 12, seed=3)
    level, batch, per = 6, 2, 2 * 6 * (1 << 12)
    ct1, ct2 = dev(case.ciphertexts(level, batch, 1)), dev(case.ciphertexts(level, batch, 2))
    for rescale in (False, True):
        single, summed = _out(level, rescale, case.n, batch), _out(level, rescale, case.n, batch)
        case.call(hb, single, ct1, ct2, level, rescale, batch)
        case.call_sum(hb, summed, [ct1[c * per:(c + 1) * per] for c in range(batch)],
                      [ct2[c * per:(c + 1) * per] for c in range(batch)], level, rescale, batch)
        torch.cuda.synchronize()
        assert torch.equal(single, summed), f"rescale {rescale}"


@pytest.mark.parametrize("n, L, K, alpha, pairs", [(1 << 12, 9, 3, 4, 3), (1 << 16, 30, 10, 10, 4)])
def test_no_rescale_equals_the_chain(hb, port, n, L, K, alpha, pairs):
    """DyadicMultiply of every pair, the three components summed with EltwiseAddModMulti, then KeySwitchHybrid of the
    summed d2 into the summed (d0, d1)"""
    case = SumCase(hb, port, L, K, alpha, n)
    for level in (L, L // 2 + 1):
        comp = level * n
        ct1s = [dev(case.ciphertexts(level, 1, 10 + r)) for r in range(pairs)]
        ct2s = [dev(case.ciphertexts(level, 1, 20 + r)) for r in range(pairs)]
        fused = torch.zeros(2 * comp, dtype=torch.int64, device="cuda")
        case.call_sum(hb, fused, ct1s, ct2s, level, False)
        acc = torch.empty(3 * comp, dtype=torch.int64, device="cuda")
        d = torch.empty(3 * comp, dtype=torch.int64, device="cuda")
        hb.DyadicMultiply(acc, ct1s[0], ct2s[0], n, case.mods[:level], level)
        for r in range(1, pairs):
            hb.DyadicMultiply(d, ct1s[r], ct2s[r], n, case.mods[:level], level)
            hb.EltwiseAddModMulti(acc, acc, d, n, case.mods[:level] * 3)
        chain = acc[:2 * comp].clone()
        hb.KeySwitchHybrid(chain, acc[2 * comp:].clone(), n, level, L, K, alpha, 2, case.mods, case.handle)
        torch.cuda.synchronize()
        assert torch.equal(fused, chain), f"n = {n}, level {level}"


# ------------------------------------------------------------------------------------------------ buffers
@pytest.fixture(scope="module")
def buffers_case(hb, port):
    case = SumCase(hb, port, 7, 3, 3, 1 << 11, seed=77)
    level, batch, pairs = 5, 3, 2
    i1, i2, count = _shared_pairs(pairs, batch)
    pool = case.pool(level, count, 31)
    exp = {rs: case.expected_sum(port, [pool[i] for i in i1], [pool[i] for i in i2], level, rs, batch)
           for rs in (False, True)}
    return case, level, batch, i1, i2, pool, exp


@pytest.mark.parametrize("rescale", [False, True])
@pytest.mark.parametrize("entry", ["device", "host", "pinned", "managed", "host_split"])
def test_buffers(hb, buffers_case, entry, rescale):
    """batch 3 with shared pairs, the output between sentinel words"""
    case, level, batch, i1, i2, pool, exps = buffers_case
    exp = exps[rescale]
    size = exp.size

    def run(out, bufs, stream=None):
        case.call_sum(hb, out, [bufs[i] for i in i1], [bufs[i] for i in i2], level, rescale, batch, stream=stream)

    try:
        if entry == "device":
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                buf = torch.full((size + 2,), SENTINEL - (1 << 64), dtype=torch.int64, device="cuda")
                bufs = [dev(ct) for ct in pool]
                run(buf[1:1 + size], bufs, stream=s)
            s.synchronize()
            got = host(buf)
        elif entry in ("managed", "pinned"):
            alloc, free = ((hb.managed_empty, hb.managed_free) if entry == "managed"
                           else (hb.pinned_empty, hb.pinned_free))
            bufs, buf = [alloc(ct.size) for ct in pool], alloc(size + 2)
            try:
                for b, ct in zip(bufs, pool):
                    b[:] = ct
                buf[:] = SENTINEL
                run(buf[1:1 + size], bufs)
                got = buf.copy()
                assert all((b == ct).all() for b, ct in zip(bufs, pool)), "an input ciphertext changed"
            finally:
                for x in bufs + [buf]:
                    free(x)
        else:
            if entry == "host_split":
                hb.set_host_devices([0, 0])
            buf = np.full(size + 2, SENTINEL, dtype=U64)
            bufs = [ct.copy() for ct in pool]
            run(buf[1:1 + size], bufs)
            assert all((b == ct).all() for b, ct in zip(bufs, pool)), "an input ciphertext changed"
            got = buf
    finally:
        hb.set_host_devices([])
    assert got[0] == SENTINEL and got[-1] == SENTINEL, "a word next to the output was written"
    _check(got[1:1 + size], exp, f"{entry} rescale {rescale}")


@pytest.mark.parametrize("rescale", [False, True])
def test_graph_replay(hb, port, buffers_case, rescale):
    case, level, batch, i1, i2, pool, exps = buffers_case
    out = torch.zeros(exps[rescale].size, dtype=torch.int64, device="cuda")
    bufs = [dev(ct) for ct in pool]
    a, b = [bufs[i] for i in i1], [bufs[i] for i in i2]
    case.call_sum(hb, out, a, b, level, rescale, batch)  # warm: tables and pool
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        case.call_sum(hb, out, a, b, level, rescale, batch)
    out.fill_(0)
    graph.replay()
    torch.cuda.synchronize()
    _check(host(out), exps[rescale], "graph replay")
    fresh = case.pool(level, len(pool), 57)
    for t, ct in zip(bufs, fresh):
        t.copy_(dev(ct))
    graph.replay()
    torch.cuda.synchronize()
    _check(host(out), case.expected_sum(port, [fresh[i] for i in i1], [fresh[i] for i in i2], level, rescale, batch),
           "graph replay, new data")


# ------------------------------------------------------------------------------------------------ launch counts
def sum_launches(n, level, K, alpha, rescale, pairs, fwd, inv):
    """per output, moduli below 2^60: one pair is MultiplyRelinearizeHybrid's count; more add one tensor-sum launch per
    block of 64 data limbs and chunk of 32 pairs (the mod-up's first inverse transform launches alike without the
    multiply on load)"""
    extra = 0 if pairs == 1 else -(-level // 64) * -(-pairs // 32)
    return relin_launches(n, level, K, alpha, rescale, fwd, inv) + extra


@pytest.mark.parametrize("L, K, alpha, level, pairs", [(6, 2, 2, 6, 1), (6, 2, 2, 6, 2), (6, 2, 2, 5, 33),
                                                       (30, 10, 10, 30, 4), (70, 2, 64, 70, 33),
                                                       (70, 2, 64, 65, 65)])
def test_launch_counts(hb, port, L, K, alpha, level, pairs):
    n = 1 << 12
    case = SumCase(hb, port, L, K, alpha, n, data_bits=(45,), special_bits=(45,))
    a, b = dev(case.ciphertexts(level, 1, 1)), dev(case.ciphertexts(level, 1, 2))
    fwd, inv = _ntt_launches(hb, n, True), _ntt_launches(hb, n, False)
    batch = 2
    for rescale in (False, True):
        out = _out(level, rescale, n, batch)

        def run():
            case.call_sum(hb, out, [a] * (pairs * batch), [b, a] * (pairs * batch // 2) + [b] * (pairs * batch % 2),
                          level, rescale, batch)
        run()  # warm
        torch.cuda.synchronize()
        before = hb.launch_count()
        run()
        torch.cuda.synchronize()
        got = hb.launch_count() - before
        exp = batch * sum_launches(n, level, K, alpha, rescale, pairs, fwd, inv)
        assert got == exp, (rescale, got, exp, fwd, inv)


# ------------------------------------------------------------------------------------------------ stream order
def test_held_stream(hb, port, hold_cycles):
    """inputs written behind a hold are the ones read, the call does not wait, and the result is complete before the
    next work on the stream (tests/test_gpu_stream_order.py, for this call), plain and under the debug checks"""
    case = SumCase(hb, port, 6, 2, 2, 1 << 12, seed=11)
    level = 5
    pool = case.pool(level, 4, 61)
    names = ["x0", "x1", "x2", "x3"]
    i1, i2 = [0, 1, 2, 0], [1, 1, 3, 3]
    for rescale in (False, True):
        exp = case.expected_sum(port, [pool[i] for i in i1], [pool[i] for i in i2], level, rescale, 2)
        row = Row("mul_relin_sum", {**dict(zip(names, pool)), "r": np.full(exp.size, SENTINEL, dtype=U64)},
                  tuple(names), {"r": exp},
                  lambda hb, t, s, rescale=rescale: case.call_sum(hb, t["r"], [t[names[i]] for i in i1],
                                                                  [t[names[i]] for i in i2], level, rescale, 2,
                                                                  stream=s), tuple(names))
        t = {k: dev(v) for k, v in row.bufs.items()}  # warm
        row.call(hb, t, None)
        torch.cuda.synchronize()
        _check(host(t["r"]), exp, "warm-up")
        s = torch.cuda.Stream()
        t, _ = _stage(row, s, hold_cycles)
        row.call(hb, t, s)
        waited = s.query()
        got = _finish(row, t, s)
        assert not waited, f"rescale {rescale}: the call waited for its stream"
        _check(got["r"], exp, f"held stream, rescale {rescale}")
        # the debug checks may wait for the stream; they must see what was written behind the hold
        for mode in ("valid", "refuse"):
            s = torch.cuda.Stream()
            t, _ = _stage(row, s, hold_cycles, mode)
            hb.set_debug(True)
            try:
                if mode == "valid":
                    row.call(hb, t, s)
                else:
                    with pytest.raises(hb.HexlB200Error) as e:
                        row.call(hb, t, s)
            finally:
                hb.set_debug(False)
                s.synchronize()
            if mode == "refuse":
                assert e.value.code == INVALID_ARG and "exceeds" in str(e.value), e.value
                continue
            _check(_finish(row, t, s)["r"], exp, f"held stream under debug, rescale {rescale}")


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals(hb, port):
    case = SumCase(hb, port, 6, 2, 2, 64)
    n, L, K, alpha = case.n, 6, 2, 2
    per = 2 * L * n
    other = SumCase(hb, port, 6, 2, 3, 64)  # keys for digit size 3: fewer digits than alpha = 2 needs
    kcc3 = hb.KeySwitchKeys(hx.random_keys(case.mods, n, L, alpha, 3, 4), n, 3, L + K, 3)
    ct1, ct2 = dev(case.ciphertexts(L, 1, 2)), dev(case.ciphertexts(L, 1, 3))
    res = torch.zeros(per, dtype=torch.int64, device="cuda")
    Ptrs = hb._vp * 2

    def refused(what, code=INVALID_ARG, out=res, a=(ct1, ct2), b=(ct2, ct1), level=L, p_size=K, digit=alpha, mods=None,
                keys=case.handle, rescale=0, pairs=2, null_arrays=False):
        mods = mods if mods is not None else case.mods
        before = out.clone()
        pa = None if null_arrays else Ptrs(*[x.data_ptr() if x is not None else None for x in a])
        pb = None if null_arrays else Ptrs(*[x.data_ptr() if x is not None else None for x in b])
        with pytest.raises(hb.HexlB200Error) as e:
            hb._check(hb._lib.hexl_b200_multiply_relinearize_sum_hybrid(
                out.data_ptr(), pa, pb, pairs, n, level, L, p_size, digit,
                np.ascontiguousarray(mods, dtype=U64).ctypes.data, keys._h if keys is not None else None, rescale, 1,
                None))
        assert e.value.code == code, (what, e.value)
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
    refused("null arrays", null_arrays=True)
    refused("a null ct1 entry", a=(ct1, None))
    refused("a null ct2 entry", b=(None, ct1))
    big = torch.zeros(4 * per, dtype=torch.int64, device="cuda")
    refused("result overlaps a ct1 entry", out=big[per // 2:3 * per // 2], a=(ct1, big[:per]))
    refused("result overlaps a ct2 entry", out=big[2 * per:3 * per], b=(ct2, big[5 * per // 2:7 * per // 2]))
    refused("result is an input", out=big[:per], a=(big[:per], big[:per]), b=(big[:per], big[:per]))
    pinned = hb.pinned_empty(per)
    try:
        pinned[:] = host(ct2)
        with pytest.raises(hb.HexlB200Error) as e:
            hb._check(hb._lib.hexl_b200_multiply_relinearize_sum_hybrid(
                res.data_ptr(), Ptrs(ct1.data_ptr(), ct2.data_ptr()), Ptrs(ct2.data_ptr(), pinned.ctypes.data), 2, n,
                L, L, K, alpha, np.ascontiguousarray(case.mods, dtype=U64).ctypes.data, case.handle._h, 0, 1, None))
        assert e.value.code == MIXED_POINTERS, e.value
    finally:
        hb.pinned_free(pinned)
    bad = case.ciphertexts(L, 1, 2)
    bad[(L + 1) * n + 3] = case.mods[1]  # component 1, limb 1
    hb.set_debug(True)
    try:
        refused("a ct1 word = q under debug", a=(ct1, dev(bad)))
        refused("a ct2 word = q under debug", b=(dev(bad), ct1))
    finally:
        hb.set_debug(False)
    # nothing to do: no pairs, or no outputs
    before = res.clone()
    for pairs, batch in ((0, 1), (2, 0)):
        hb._check(hb._lib.hexl_b200_multiply_relinearize_sum_hybrid(
            res.data_ptr(), None if pairs == 0 else Ptrs(ct1.data_ptr(), ct2.data_ptr()),
            None if pairs == 0 else Ptrs(ct2.data_ptr(), ct1.data_ptr()), pairs, n, L, L, K, alpha,
            np.ascontiguousarray(case.mods, dtype=U64).ctypes.data, case.handle._h, 1, batch, None))
    torch.cuda.synchronize()
    assert torch.equal(res, before), "an empty call wrote"


def test_cpp_caller_runs(hb, tmp_path):
    if not shutil.which("g++"):
        pytest.skip("g++ not present")
    exe = tmp_path / "mul_relin_sum_caller"
    libdir = os.path.dirname(hb.LIB_PATH)
    subprocess.run(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "cpp", "mul_relin_sum_caller.cpp"), "-o", str(exe),
                    "-L", libdir, "-lhexl_b200", f"-Wl,-rpath,{libdir}"], check=True)
    res = subprocess.run([str(exe), "run"], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
