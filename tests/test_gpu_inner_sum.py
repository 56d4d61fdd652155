"""InnerSumHybrid on the GPU.

Compared bit for bit with the exact model of tests/inner_sum_exact.py, with rescale 0 and 1: over the (L, K, alpha)
shapes of the hybrid tests and their levels, every degree from 2 to 2^17, and primes just below 2^61 with every word
q - 1; over sum counts that are powers of two, 2^m - 1, 2^m + 1 and n / 2 at small n; over the conjugation 2n - 1
(order 2: identity doublings and shifts) and elements whose powers reach 1 before k.  Also pinned, against the existing
GPU calls at N = 2^12 and at N = 2^16, L = 30, alpha = K = 10: k = 1 is LinearTransformHybridBSGS with one identity
baby and giant (and a copy of ct without the rescale); k = 2 is ApplyGaloisKeySwitchHybridHoisted plus
EltwiseAddModMulti with ct, and LinearTransformHybrid over {1, g}; k = 3 and 4 are LinearTransformHybridBSGS with unit
diagonals.  Device, pageable, pinned, managed and split-host buffers; host batches that wrap the staging slots; graph
replay with new data; a stream held back while the inputs are written; launch counts against the plan of
tests/inner_sum_exact.py; the refusals, the missing-key message included; and a C++ caller."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import inner_sum_exact as ix
from test_gpu_hybrid_key_switch import SENTINEL, _check, _levels, dev, host
from test_gpu_hybrid_rotation import Case
from test_gpu_hybrid_rounds import _ntt

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U64 = np.uint64
INVALID_ARG = -1


@pytest.fixture(scope="module", autouse=True)
def _need_cuda(hb):
    if not torch.cuda.is_available() or hb.device_count() == 0:
        pytest.fail("gpu-marked test collected on a machine without CUDA")


def table(case, g, ks, extra=()):
    """the key table for every k in ks: each needed element with key set (index mod the case's sets), plus `extra`
    (element, set) entries that no sum needs, first so that a lookup has to skip them"""
    elts = sorted({e for k in ks for e in ix.needed_elements(g, k, case.n)})
    rows = list(extra) + [(e, r % len(case.keys)) for r, e in enumerate(elts)]
    return [e for e, _ in rows], [case.handles[s] for _, s in rows], {e: case.keys[s] for e, s in reversed(rows)}


def inner_sum(hb, case, out, ct, level, g, k, tab, rescale, batch=1, stream=None):
    elts, handles, _ = tab
    return hb.InnerSumHybrid(out, ct, case.n, level, case.L, case.K, case.alpha, case.mods, g, k, handles, elts,
                             rescale, batch, stream=stream)


def expected(port, case, ct, level, g, k, tab, rescale, batch=1):
    per = 2 * level * case.n
    return np.concatenate([ix.inner_sum_exact(port, ct[c * per:(c + 1) * per], case.n, level, case.L, case.K,
                                              case.alpha, case.mods, g, k, tab[2], rescale) for c in range(batch)])


def out_words(case, level, rescale, batch=1):
    return batch * 2 * (level - int(rescale)) * case.n


def _run(hb, port, case, level, g, ks, seed, rescales=(False, True), batch=1):
    ct = case.ciphertexts(level, batch, seed)
    src = dev(ct)
    tab = table(case, g, ks, extra=[(1, 0)])
    for k in ks:
        for rescale in rescales:
            if rescale and level < 2:
                continue
            out = torch.full((out_words(case, level, rescale, batch),), -1, dtype=torch.int64, device="cuda")
            inner_sum(hb, case, out, src, level, g, k, tab, rescale, batch)
            torch.cuda.synchronize()
            assert torch.equal(src, dev(ct)), "the ciphertexts changed"
            _check(host(out), expected(port, case, ct, level, g, k, tab, rescale, batch),
                   f"level {level} g {g} k {k} rescale {rescale}")


@pytest.mark.parametrize("L, K, alpha", [(4, 1, 1), (6, 2, 2), (7, 3, 3), (5, 2, 5), (8, 4, 2)])
def test_shapes_equal_the_model(hb, port, L, K, alpha):
    case = Case(hb, port, L, K, alpha, 256, seed=L * 100 + K * 10 + alpha)
    for level in _levels(L, alpha):
        _run(hb, port, case, level, 5, (1, 2, 3, 5, 8), level)


@pytest.mark.parametrize("logn", range(1, 18))
def test_every_degree(hb, port, logn):
    """k = 5 rotates by g at bit 0, g^2 at bit 1 and g again at bit 2; at n = 2 the only element of order 4 is 3"""
    n = 1 << logn
    case = Case(hb, port, 6, 2, 2, n, seed=logn, sets=2)
    g = 3 if n == 2 else 5
    _run(hb, port, case, 5, g, (5,), logn)


@pytest.mark.parametrize("n, ks", [(16, (4, 7, 8, 9, 15, 16, 17)), (32, (16, 31, 33)), (64, (32, 63, 65))])
def test_sum_counts(hb, port, n, ks):
    """powers of two, 2^m - 1 and 2^m + 1, and k = n / 2 (a sum over every slot of the row)"""
    case = Case(hb, port, 5, 2, 2, n, seed=n, sets=3)
    _run(hb, port, case, 4, 5, ks, n)


@pytest.mark.parametrize("n", [16, 256])
def test_small_orders(hb, port, n):
    """the conjugation 2n - 1: g^2 = 1, so identity doublings (component 1 doubles) and identity shifts after the first
    set bit; and 5^(n/8), of order 4 mod 2n, whose powers reach 1 before k"""
    case = Case(hb, port, 6, 2, 3, n, seed=3, sets=2)
    _run(hb, port, case, 6, 2 * n - 1, (2, 3, 5, 6, 7, 12), n)
    _run(hb, port, case, 5, pow(5, n // 8, 2 * n), (4, 5, 9, 13), n + 1)


@pytest.mark.parametrize("L, K, alpha, level", [(20, 2, 1, 20), (64, 3, 64, 33)])
def test_worst_case_words_below_2_61(hb, port, L, K, alpha, level):
    """the largest NTT primes below 2^61 and every ciphertext and key word q - 1; (20, 2, 1): digit chunks of 16 in the
    multiply-accumulates, and (64, 3, 64) a level across two blocks of moduli"""
    n = 64
    case = Case(hb, port, L, K, alpha, n, data_bits=(60,), special_bits=(60,), fill="q-1", sets=2)
    assert min(case.mods) > 1 << 60
    _run(hb, port, case, level, 5, (7,), 0)


def test_seventy_moduli(hb, port):
    """70 data moduli in 64-modulus digits: every step and the final mod-down take two blocks of moduli"""
    n = 16
    case = Case(hb, port, 70, 2, 64, n, data_bits=(55,), special_bits=(55,), sets=2)
    for level in (70, 65):
        _run(hb, port, case, level, 3, (6,), level)


# ------------------------------------------------------------------------------------------------ equalities
def _bsgs(hb, case, out, src, level, babies, giants, grid, rescale, tab):
    """LinearTransformHybridBSGS with the keys of tab: babies and giants are element lists, 1 the identity"""
    handles = dict(zip(tab[0], tab[1]))
    return hb.LinearTransformHybridBSGS(out, src, case.n, level, case.L, case.K, case.alpha, case.mods,
                                        [None if e == 1 else handles[e] for e in babies], babies,
                                        [None if e == 1 else handles[e] for e in giants], giants, grid, rescale)


@pytest.mark.parametrize("n, L, K, alpha", [(1 << 12, 9, 3, 4), (1 << 16, 30, 10, 10)])
def test_anchors_equal_the_existing_calls(hb, port, n, L, K, alpha):
    case = Case(hb, port, L, K, alpha, n, sets=2)
    g = 5
    g2 = g * g % (2 * n)
    tab = table(case, g, (2, 4))
    handles = dict(zip(tab[0], tab[1]))
    level = L if n == 1 << 12 else L - 1
    nb, comp = level + K, level * n
    ct = case.ciphertexts(level, 1, 9)
    src = dev(ct)
    ones = dev(case.diagonals(level, 2, 0, fill="one"))
    w = ones[:nb * n]
    for rescale in (False, True):
        words = out_words(case, level, rescale)
        a, b = (torch.full((words,), -1, dtype=torch.int64, device="cuda") for _ in range(2))
        inner_sum(hb, case, a, src, level, g, 1, tab, rescale)
        _bsgs(hb, case, b, src, level, [1], [1], [[w]], rescale, tab)
        torch.cuda.synchronize()
        assert torch.equal(a, b), f"k = 1, rescale {rescale}"
        if not rescale:
            assert torch.equal(a, src), "k = 1 is a copy"
        inner_sum(hb, case, a, src, level, g, 3, tab, rescale)
        _bsgs(hb, case, b, src, level, [1, g], [1, g], [[w, None], [w, w]], rescale, tab)
        torch.cuda.synchronize()
        assert torch.equal(a, b), f"k = 3, rescale {rescale}"
        inner_sum(hb, case, a, src, level, g, 4, tab, rescale)
        _bsgs(hb, case, b, src, level, [1, g], [1, g2], [[w, w], [w, w]], rescale, tab)
        torch.cuda.synchronize()
        assert torch.equal(a, b), f"k = 4, rescale {rescale}"
    a, b = (torch.full((2 * comp,), -1, dtype=torch.int64, device="cuda") for _ in range(2))
    inner_sum(hb, case, a, src, level, g, 2, tab, False)
    hb.ApplyGaloisKeySwitchHybridHoisted(b, src, n, level, L, K, alpha, case.mods, [handles[g]], [g])
    mods = case.mods[:level] * 2
    hb.EltwiseAddModMulti(b, b, src, n, mods)
    torch.cuda.synchronize()
    assert torch.equal(a, b), "k = 2: the hoisted rotation plus ct"
    hb.LinearTransformHybrid(b, src, n, level, L, K, alpha, case.mods, [None, handles[g]], [1, g], ones)
    torch.cuda.synchronize()
    assert torch.equal(a, b), "k = 2: the linear transform over {1, g}"


# ------------------------------------------------------------------------------------------------ buffers
@pytest.fixture(scope="module")
def buffers_case(hb, port):
    case = Case(hb, port, 7, 3, 3, 1 << 11, seed=77)
    level, batch, g, k = 5, 3, 5, 7
    ct = case.ciphertexts(level, batch, 21)
    tab = table(case, g, (k,))
    exp = {rs: expected(port, case, ct, level, g, k, tab, rs, batch) for rs in (False, True)}
    return case, level, batch, g, k, ct, tab, exp


@pytest.mark.parametrize("rescale", [False, True])
@pytest.mark.parametrize("entry", ["device", "host", "pinned", "managed", "host_split"])
def test_buffers(hb, buffers_case, entry, rescale):
    """batch 3 between sentinel words"""
    case, level, batch, g, k, ct, tab, exp = buffers_case
    size = exp[rescale].size

    def run(out, src, stream=None):
        inner_sum(hb, case, out, src, level, g, k, tab, rescale, batch, stream=stream)

    try:
        if entry == "device":
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                buf = torch.full((size + 2,), SENTINEL - (1 << 64), dtype=torch.int64, device="cuda")
                src = dev(ct)
                run(buf[1:1 + size], src, stream=s)
            s.synchronize()
            got = host(buf)
        elif entry in ("managed", "pinned"):
            alloc, free = ((hb.managed_empty, hb.managed_free) if entry == "managed"
                           else (hb.pinned_empty, hb.pinned_free))
            src, buf = alloc(ct.size), alloc(size + 2)
            try:
                src[:], buf[:] = ct, SENTINEL
                run(buf[1:1 + size], src)
                got = buf.copy()
                assert (src == ct).all(), "the ciphertexts changed"
            finally:
                free(src)
                free(buf)
        else:
            if entry == "host_split":
                hb.set_host_devices([0, 0])
            buf = np.full(size + 2, SENTINEL, dtype=U64)
            src = ct.copy()
            run(buf[1:1 + size], src)
            assert (src == ct).all(), "the ciphertexts changed"
            got = buf
    finally:
        hb.set_host_devices([])
    assert got[0] == SENTINEL and got[-1] == SENTINEL, "a word next to the output was written"
    _check(got[1:1 + size], exp[rescale], f"{entry} rescale {rescale}")


@pytest.mark.parametrize("devices", [[0], [0, 0, 0]])
def test_host_batch_wraps_the_staging_slots(hb, port, devices):
    """seven ciphertexts at N = 2^14: more than the staging slots of each device, so slots are reused"""
    case = Case(hb, port, 6, 2, 2, 1 << 14, seed=5, sets=2)
    level, batch, g, k = 6, 7, 5, 6
    ct = case.ciphertexts(level, batch, 31)
    tab = table(case, g, (k,))
    try:
        hb.set_host_devices(devices)
        for rescale in (False, True):
            out = np.full(out_words(case, level, rescale, batch), SENTINEL, dtype=U64)
            inner_sum(hb, case, out, ct, level, g, k, tab, rescale, batch)
            _check(out, expected(port, case, ct, level, g, k, tab, rescale, batch), f"{devices} rescale {rescale}")
    finally:
        hb.set_host_devices([])


@pytest.mark.parametrize("rescale", [False, True])
def test_graph_replay(hb, port, buffers_case, rescale):
    case, level, batch, g, k, ct, tab, exp = buffers_case
    out = torch.zeros(exp[rescale].size, dtype=torch.int64, device="cuda")
    src = dev(ct)

    def run():
        inner_sum(hb, case, out, src, level, g, k, tab, rescale, batch)

    run()  # warm: tables and pool
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        run()
    out.fill_(0)
    graph.replay()
    torch.cuda.synchronize()
    _check(host(out), exp[rescale], "graph replay")
    ct2 = case.ciphertexts(level, batch, 22)
    src.copy_(dev(ct2))
    graph.replay()
    torch.cuda.synchronize()
    _check(host(out), expected(port, case, ct2, level, g, k, tab, rescale, batch), "graph replay, new data")


def test_held_stream(hb, buffers_case):
    """the ciphertexts are written behind a bounded spin on a fresh stream: the call must not wait for the stream, must
    read what the stream wrote, and its result must be complete before the next work on the stream"""
    case, level, batch, g, k, ct, tab, exp = buffers_case
    for rescale in (False, True):
        src = torch.zeros(ct.size, dtype=torch.int64, device="cuda")
        out = torch.full((exp[rescale].size,), -1, dtype=torch.int64, device="cuda")
        real = dev(ct)
        inner_sum(hb, case, out, real, level, g, k, tab, rescale, batch)  # warm
        torch.cuda.synchronize()
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            torch.cuda._sleep(1 << 28)
            src.copy_(real)
        inner_sum(hb, case, out, src, level, g, k, tab, rescale, batch, stream=s)
        waited = s.query()
        with torch.cuda.stream(s):
            clone = out.clone()
            out.fill_(0)
            src.fill_(0)
        s.synchronize()
        assert not waited, "the call waited for its stream"
        _check(host(clone), exp[rescale], f"held stream, rescale {rescale}")


# ------------------------------------------------------------------------------------------------ launch counts
@pytest.mark.parametrize("L, K, alpha, level", [(6, 2, 2, 6), (30, 10, 10, 30), (70, 2, 64, 70), (12, 1, 1, 12)])
def test_launch_counts(hb, port, L, K, alpha, level):
    n = 1 << 12
    case = Case(hb, port, L, K, alpha, n, data_bits=(45,), special_bits=(45,), sets=2)
    ct = dev(case.ciphertexts(level, 2, 1))
    ntt = _ntt(hb, n)
    for g, ks in ((5, (1, 2, 3, 4, 7, 16, 21)), (2 * n - 1, (2, 5, 6))):
        tab = table(case, g, ks)
        for k in ks:
            for rescale in (False, True):
                out = torch.zeros(out_words(case, level, rescale, 2), dtype=torch.int64, device="cuda")
                inner_sum(hb, case, out, ct, level, g, k, tab, rescale, 2)  # warm
                torch.cuda.synchronize()
                before = hb.launch_count()
                inner_sum(hb, case, out, ct, level, g, k, tab, rescale, 2)
                torch.cuda.synchronize()
                got = hb.launch_count() - before
                exp = ix.inner_sum_launches(n, level, K, alpha, case.basis(level), ntt, g, k, rescale)
                assert got == 2 * exp, (g, k, rescale, got, 2 * exp)


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals(hb, port):
    case = Case(hb, port, 6, 2, 2, 64, sets=2)
    n, L, K, alpha = case.n, 6, 2, 2
    other = Case(hb, port, 6, 2, 3, 64, sets=1)  # keys for digit size 3: fewer digits than alpha = 2 needs
    g = 5
    tab = table(case, g, (7,))
    elts, handles = tab[0], tab[1]
    ct = dev(case.ciphertexts(L, 1, 2))
    res = torch.zeros(2 * L * n, dtype=torch.int64, device="cuda")

    def refused(what, out=res, src=ct, level=L, digit=alpha, mods=None, elt=g, k=7, hs=None, es=None, rescale=0,
                raw=False, message=None):
        hs = hs if hs is not None else handles
        es = es if es is not None else elts
        mods = mods if mods is not None else case.mods
        before = out.clone()
        with pytest.raises(hb.HexlB200Error) as e:
            if raw:  # through the C entry point: a rescale the wrapper would not pass, or null tables
                import ctypes as C
                vp = C.c_void_p
                m = np.ascontiguousarray(mods, dtype=U64)
                ke = np.ascontiguousarray(es, dtype=U64)
                keys = (vp * len(hs))(*[h._h for h in hs])
                hb._check(hb._lib.hexl_b200_inner_sum_hybrid(
                    out.data_ptr(), src.data_ptr(), n, level, L, K, digit, m.ctypes.data, elt, k,
                    None if raw == "null" else keys, None if raw == "null" else ke.ctypes.data, len(hs), rescale,
                    1, None))
            else:
                hb.InnerSumHybrid(out, src, n, level, L, K, digit, mods, elt, k, hs, es, rescale)
        assert e.value.code == INVALID_ARG, (what, e.value)
        if message:
            assert message in str(e.value), (what, str(e.value))
        assert torch.equal(out, before), f"{what}: output written"

    try:
        hb.set_host_devices([0, 0])
        sharded = hb.KeySwitchKeys(case.keys[0], n, len(case.keys[0]), L + K, 2, sharded_by_modulus=True)
    finally:
        hb.set_host_devices([])
    g2 = g * g % (2 * n)
    missing = [i for i, e in enumerate(elts) if e != g2]
    refused("a missing key", hs=[handles[i] for i in missing], es=[elts[i] for i in missing],
            message=f"no key for the Galois element {g2}")
    refused("an empty table", hs=[], es=[], message=f"no key for the Galois element {g}")
    refused("a null key", hs=[None if e == g else h for e, h in zip(elts, handles)])
    refused("a handle of another digit size", hs=[other.handles[0] if e == g else h for e, h in zip(elts, handles)])
    refused("a sharded handle", hs=[sharded if e == g else h for e, h in zip(elts, handles)])
    refused("an even element", elt=4)
    refused("an element of 2n + 1", elt=2 * n + 1)
    refused("level 0", level=0)
    refused("digit size 65", digit=65)
    refused("a modulus >= 2^61", mods=case.mods[:-1] + [int(port.generate_primes(1, 62, True, n)[0])])
    refused("rescale = 2", rescale=2, raw=True)
    refused("rescale = -1", rescale=-1, raw=True)
    refused("null tables with num_keys > 0", raw="null")
    refused("rescale at level 1", level=1, rescale=1)
    big = torch.zeros(8 * L * n, dtype=torch.int64, device="cuda")
    refused("result overlaps the ciphertexts", out=big[:2 * L * n], src=big[L * n:3 * L * n])
    bad = case.ciphertexts(L, 1, 2)
    bad[7] = case.mods[0]
    hb.set_debug(True)
    try:
        refused("a ciphertext word = q under debug", src=dev(bad))
    finally:
        hb.set_debug(False)
    wide = Case(hb, port, 2, 64, 2, 16, sets=1)  # p_size 64: the merged mod-down would convert from 65 moduli
    out = torch.zeros(2 * 16, dtype=torch.int64, device="cuda")
    with pytest.raises(hb.HexlB200Error) as e:
        hb.InnerSumHybrid(out, dev(wide.ciphertexts(2, 1, 1)), 16, 2, 2, 64, 2, wide.mods, 5, 1, [], [], 1)
    assert e.value.code == INVALID_ARG and not out.any(), "rescale with p_size 64"
    before = res.clone()
    hb.InnerSumHybrid(res, ct, n, L, L, K, alpha, case.mods, g, 0, [], [], 0)
    hb.InnerSumHybrid(res, ct, n, L, L, K, alpha, case.mods, g, 7, handles, elts, 0, batch=0)
    torch.cuda.synchronize()
    assert torch.equal(res, before), "sum_count = 0 or batch = 0 wrote"


def test_cpp_caller_runs(hb, tmp_path):
    if not shutil.which("g++"):
        pytest.skip("g++ not present")
    exe = tmp_path / "inner_sum_caller"
    libdir = os.path.dirname(hb.LIB_PATH)
    subprocess.run(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "cpp", "inner_sum_caller.cpp"), "-o", str(exe),
                    "-L", libdir, "-lhexl_b200", f"-Wl,-rpath,{libdir}"], check=True)
    res = subprocess.run([str(exe), "run"], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
