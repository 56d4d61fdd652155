"""DivideAndRoundQLast on the GPU against the model (tests/rescale_exact.py), bit for bit, in NTT and coefficient
form, through every entry point: device pointers on a non-default stream, host pointers (also larger than one staging
chunk, and split over set_host_devices), managed memory, in place and out of place.  Also: the device call equals the
same rescale chained from the library's existing calls, its launch count depends neither on the number of
polynomials nor on the number of moduli within a parameter block, it replays from a CUDA graph, and a C++ caller
links and runs through include/hexl/hexl.hpp."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import rescale_exact as rx

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U64 = np.uint64
SENTINEL = 0xA5A5A5A5A5A5A5A5
FORMS = [True, False]

# name -> (n, chain, limbs, count)
SHAPES = {
    "seal_n15": (1 << 15, "seal", 31, 4),   # SEAL-style chain: 60-bit first prime, 40-bit middles, 50-bit last
    "classes": (1 << 12, "classes", 4, 4),  # 58/29/50-bit moduli, 45-bit last
    "blocks70": (1 << 11, "blocks", 70, 2),  # more than one parameter block
    "tiny2": (2, "seal", 6, 3),
    "tiny4": (4, "seal", 6, 3),
    "tiny8": (8, "seal", 6, 3),
    "seal_n16": (1 << 16, "seal", 31, 2),        # DESIGN §6's shape
    "classes_n18": (1 << 18, "classes", 4, 2),  # from 2^18 on, the transforms take two column passes
    "seal_n20": (1 << 20, "seal", 6, 1),        # the largest degree accepted
}


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=U64).view(np.int64)).to("cuda")


def host(t):
    return t.cpu().numpy().view(U64)


@pytest.fixture(scope="module", autouse=True)
def _need_cuda(hb):
    if not torch.cuda.is_available() or hb.device_count() == 0:
        pytest.fail("gpu-marked test collected on a machine without CUDA")


_cache = {}


def _prepared(port, shape, ntt_form):
    """(n, moduli, count, operand, model result), computed once per shape and form"""
    key = (shape, ntt_form)
    if key not in _cache:
        n, name, limbs, count = SHAPES[shape] if isinstance(shape, str) else shape
        mods = rx.chain(port.generate_primes, n, name, limbs)
        x = rx.random_operand(len(mods) + n, n, mods, count)
        _cache[key] = n, mods, count, x, rx.rescale_exact(port, x, n, mods, count, ntt_form)
    return _cache[key]


def _check(got, exp, x, n, mods, count, limb_last_is, what):
    """limbs 0..L-1 equal the model; limb L is `limb_last_is` ("operand" or "sentinel")"""
    rns = len(mods)
    g = np.asarray(got).reshape(count, rns, n)
    e = exp.reshape(count, rns, n)
    wrong = int((g[:, :-1] != e[:, :-1]).sum())
    assert wrong == 0, f"{what}: {wrong} of {count * (rns - 1) * n} words differ from the model"
    want_last = x.reshape(count, rns, n)[:, -1] if limb_last_is == "operand" else U64(SENTINEL)
    assert (g[:, -1] == want_last).all(), f"{what}: limb L of result was written"


def _sentinel(size):
    return np.full(size, SENTINEL, dtype=U64)


@pytest.mark.parametrize("ntt_form", FORMS)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_device_pointers_on_a_stream(hb, port, shape, ntt_form):
    n, mods, count, x, exp = _prepared(port, shape, ntt_form)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        d_in = dev(x)
        d_out = dev(_sentinel(x.size))
        hb.DivideAndRoundQLast(d_out, d_in, n, mods, len(mods), count, ntt_form, stream=s)
    s.synchronize()
    _check(host(d_out), exp, x, n, mods, count, "sentinel", f"{shape} device out of place")
    assert (host(d_in) == x).all(), "the operand was modified"
    d = dev(x)
    hb.DivideAndRoundQLast(d, d, n, mods, len(mods), count, ntt_form)
    _check(host(d), exp, x, n, mods, count, "operand", f"{shape} device in place")


@pytest.mark.parametrize("ntt_form", FORMS)
@pytest.mark.parametrize("shape", ["seal_n15", "classes", "blocks70", "tiny4"])
def test_host_pointers(hb, port, shape, ntt_form):
    n, mods, count, x, exp = _prepared(port, shape, ntt_form)
    out = _sentinel(x.size)
    hb.DivideAndRoundQLast(out, x, n, mods, len(mods), count, ntt_form)
    _check(out, exp, x, n, mods, count, "sentinel", f"{shape} host out of place")
    inplace = x.copy()
    hb.DivideAndRoundQLast(inplace, inplace, n, mods, len(mods), count, ntt_form)
    _check(inplace, exp, x, n, mods, count, "operand", f"{shape} host in place")


@pytest.mark.parametrize("ntt_form", FORMS)
def test_host_polynomial_larger_than_a_staging_chunk(hb, port, ntt_form):
    """n = 2^17 with 33 limbs: 34.6 MB per polynomial, more than one 32 MiB staging buffer"""
    shape = (1 << 17, "seal", 33, 2)
    n, mods, count, x, exp = _prepared(port, shape, ntt_form)
    assert len(mods) * n * 8 > 32 << 20
    out = _sentinel(x.size)
    hb.DivideAndRoundQLast(out, x, n, mods, len(mods), count, ntt_form)
    _check(out, exp, x, n, mods, count, "sentinel", "n = 2^17 host")


@pytest.mark.parametrize("ntt_form", FORMS)
def test_managed_memory(hb, port, ntt_form):
    n, mods, count, x, exp = _prepared(port, "classes", ntt_form)
    buf = hb.managed_empty(x.size)
    try:
        buf[:] = x
        hb.DivideAndRoundQLast(buf, buf, n, mods, len(mods), count, ntt_form)
        _check(buf.copy(), exp, x, n, mods, count, "operand", "managed in place")
    finally:
        hb.managed_free(buf)


@pytest.mark.parametrize("ntt_form", FORMS)
def test_host_devices_split_by_polynomial(hb, port, ntt_form):
    n, mods, count, x, exp = _prepared(port, "classes", ntt_form)
    out = _sentinel(x.size)
    try:
        hb.set_host_devices([0, 0, 0])
        hb.DivideAndRoundQLast(out, x, n, mods, len(mods), count, ntt_form)
    finally:
        hb.set_host_devices([])
    _check(out, exp, x, n, mods, count, "sentinel", "set_host_devices([0, 0, 0])")


@pytest.mark.parametrize("ntt_form", FORMS)
@pytest.mark.parametrize("name,limbs", [("seal", 31), ("classes", 4)])
def test_equals_the_chain_of_existing_calls(hb, port, name, limbs, ntt_form):
    n, count = 1 << 12, 2
    mods = rx.chain(port.generate_primes, n, name, limbs)
    x = rx.random_operand(7, n, mods, count)
    ntts = [hb.GetNTT(n, q) for q in mods]
    chained = rx.rescale_chain(hb, dev(x), dev(x), n, mods, count, ntt_form, ntts)
    d = dev(x)
    hb.DivideAndRoundQLast(d, d, n, mods, len(mods), count, ntt_form)
    assert (host(d) == host(chained)).all()
    assert (host(d) == rx.rescale_exact(port, x, n, mods, count, ntt_form)).all()


@pytest.mark.parametrize("ntt_form", FORMS)
def test_launch_count_depends_on_neither_count_nor_moduli(hb, port, ntt_form):
    n = 1 << 12

    def launches(limbs, count):
        mods = rx.chain(port.generate_primes, n, "seal", limbs)
        d = dev(rx.random_operand(limbs, n, mods, count))
        hb.DivideAndRoundQLast(d, d, n, mods, limbs, count, ntt_form)   # warm: tables and pool
        torch.cuda.synchronize()
        before = hb.launch_count()
        hb.DivideAndRoundQLast(d, d, n, mods, limbs, count, ntt_form)
        torch.cuda.synchronize()
        return hb.launch_count() - before

    by_count = launches(6, 1), launches(6, 8)
    by_moduli = launches(3, 2), launches(60, 2)
    assert by_count[0] == by_count[1], by_count
    assert by_moduli[0] == by_moduli[1], by_moduli
    if not ntt_form:
        assert by_count[0] == 1   # one fused kernel per parameter block


@pytest.mark.parametrize("ntt_form", FORMS)
def test_graph_capture_and_replay(hb, port, ntt_form):
    n, mods, count, x, exp = _prepared(port, "classes", ntt_form)
    d_in = dev(x)
    d_out = dev(_sentinel(x.size))

    def call():
        hb.DivideAndRoundQLast(d_out, d_in, n, mods, len(mods), count, ntt_form)

    call()  # tables and pool are set up outside the capture
    torch.cuda.synchronize()
    d_out.copy_(dev(_sentinel(x.size)))
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        call()
    g.replay()
    torch.cuda.synchronize()
    _check(host(d_out), exp, x, n, mods, count, "sentinel", "graph replay")
    x2 = rx.random_operand(1234, n, mods, count)
    d_in.copy_(dev(x2))
    g.replay()
    torch.cuda.synchronize()
    _check(host(d_out), rx.rescale_exact(port, x2, n, mods, count, ntt_form), x2, n, mods, count, "sentinel",
           "graph replay, new data")


def test_cpp_caller_runs(hb, tmp_path):
    if not shutil.which("g++"):
        pytest.skip("g++ not present")
    exe = tmp_path / "rescale_caller"
    libdir = os.path.dirname(hb.LIB_PATH)
    subprocess.run(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "cpp", "rescale_caller.cpp"), "-o", str(exe),
                    "-L", libdir, "-lhexl_b200", f"-Wl,-rpath,{libdir}"], check=True)
    res = subprocess.run([str(exe), "run"], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
