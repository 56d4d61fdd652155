"""LinearTransformHybridBSGS on the GPU.

Compared bit for bit with the exact model of tests/bsgs_exact.py, with rescale 0 and 1: over the (L, K, alpha) shapes
of the hybrid tests and their levels, every degree from 2 to 2^17, more than 64 present babies in a row (two sum
chunks), 70 data moduli in 64-modulus digits (two blocks of B), and primes just below 2^61 with every word q - 1.
Grids are sparse and hold identity babies and giants (element 1 without a key) and repeated elements.  Also pinned,
against the existing GPU calls: one identity giant is LinearTransformHybrid over the babies, and one identity baby
with diagonals of ones is LinearTransformHybrid over the giants (with one giant, ApplyGaloisKeySwitchHybridHoisted),
at N = 2^12 and at N = 2^16, L = 30, alpha = K = 10, and at N = 2^16, L = 30, alpha = 1, where the mod-up takes
several rounds and eight babies' products are stored.  Device, pageable, pinned, managed and split-host buffers; graph
replay with new data; launch counts against the plan of tests/composite_plan.py (bsgs_launches); the refusals; and a
C++ caller.

tests/test_gpu_bsgs_rounds.py holds the production coverage: every HYBRID_SHAPES entry at each of its levels with both
rescale modes, tools/bsgs_bench.py's full 8 x 8 grid at N = 2^16, every level of two shapes, host batches that wrap
the staging slots, host calls of different slot sizes in sequence, threads, offset views and the aliasing the API
allows."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import bsgs_exact as bx
import composite_plan as plan
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


# spec: [(element, key set or None)] for the babies and for the giants; grid[j][i]: numpy diagonal or None
def bsgs(hb, case, out, ct, grid, level, bspec, gspec, rescale, batch=1, stream=None):
    return hb.LinearTransformHybridBSGS(out, ct, case.n, level, case.L, case.K, case.alpha, case.mods,
                                        case.handles_of(bspec), [g for g, _ in bspec], case.handles_of(gspec),
                                        [g for g, _ in gspec], grid, rescale, batch, stream=stream)


def expected(port, case, ct, grid, level, bspec, gspec, rescale, batch=1):
    per = 2 * level * case.n
    return np.concatenate([bx.bsgs_exact(port, ct[c * per:(c + 1) * per], case.n, level, case.L, case.K, case.alpha,
                                         case.mods, [g for g, _ in bspec], case.keys_of(bspec),
                                         [g for g, _ in gspec], case.keys_of(gspec), grid, rescale)
                           for c in range(batch)])


def dev_grid(grid):
    return [[None if w is None else dev(w) for w in row] for row in grid]


def out_words(case, level, rescale, batch=1):
    return batch * 2 * (level - int(rescale)) * case.n


def _specs(n):
    """babies 1 (identity), 3, 2n - 1, 5 and 3 again; giants 1 (identity), 9, 25 and 2n - 1"""
    bspec = [(1, None), (3 % (2 * n), 0), (2 * n - 1, 1), (5 % (2 * n), 2), (3 % (2 * n), 1)]
    gspec = [(1, None), (9 % (2 * n), 0), (25 % (2 * n), 1), (2 * n - 1, 2)]
    return bspec, gspec


# the identity giant over every baby but 3; giant 9 over the identity baby alone (no keyed baby); giant 25 over four
# babies; the last giant over none
PRESENT = {(0, 0), (0, 1), (0, 2), (0, 4), (1, 0), (2, 0), (2, 1), (2, 3), (2, 4)}


def _run(hb, port, case, level, bspec, gspec, present, seed, rescales=(False, True), batch=1, fill=None):
    ct = case.ciphertexts(level, batch, seed)
    grid = bx.grid_diagonals(case.basis(level), case.n, len(gspec), len(bspec), present, seed, fill or case.fill)
    src, dgrid = dev(ct), dev_grid(grid)
    for rescale in rescales:
        if rescale and level < 2:
            continue
        out = torch.full((out_words(case, level, rescale, batch),), -1, dtype=torch.int64, device="cuda")
        bsgs(hb, case, out, src, dgrid, level, bspec, gspec, rescale, batch)
        torch.cuda.synchronize()
        assert torch.equal(src, dev(ct)), "the ciphertexts changed"
        _check(host(out), expected(port, case, ct, grid, level, bspec, gspec, rescale, batch),
               f"level {level} rescale {rescale}")


@pytest.mark.parametrize("L, K, alpha", [(4, 1, 1), (6, 2, 2), (7, 3, 3), (5, 2, 5), (8, 4, 2)])
def test_shapes_equal_the_model(hb, port, L, K, alpha):
    case = Case(hb, port, L, K, alpha, 256, seed=L * 100 + K * 10 + alpha)
    bspec, gspec = _specs(256)
    for level in _levels(L, alpha):
        _run(hb, port, case, level, bspec, gspec, PRESENT, level)


@pytest.mark.parametrize("logn", range(1, 18))
def test_every_degree(hb, port, logn):
    n = 1 << logn
    case = Case(hb, port, 6, 2, 2, n, seed=logn, sets=2)
    bspec = [(1, None), (5 % (2 * n), 0)]
    gspec = [(2 * n - 1, 1), (1, None)]
    _run(hb, port, case, 5, bspec, gspec, {(0, 0), (0, 1), (1, 1)}, logn)


def test_more_than_64_present_babies_in_a_row(hb, port):
    """70 babies in each of two rows: two sum launches per block of moduli, the second adding into the first's x1/y1"""
    n = 16
    case = Case(hb, port, 5, 2, 2, n, sets=3)
    elts = [pow(5, k, 2 * n) for k in range(1, 8)] + [2 * n - 1]
    bspec = [(elts[i % len(elts)], i % 3) for i in range(66)] + [(1, None)] * 4
    gspec = [(3, 0), (1, None)]
    _run(hb, port, case, 4, bspec, gspec, None, 7)


def test_seventy_moduli_in_64_modulus_digits(hb, port):
    """70 data moduli, alpha = 64, K = 2: B takes two blocks of sums and two mod-up rounds"""
    n = 16
    case = Case(hb, port, 70, 2, 64, n, data_bits=(55,), special_bits=(55,), sets=3)
    bspec = [(1, None), (3, 0), (2 * n - 1, 1)]
    gspec = [(5, 2), (1, None), (9, 0)]
    present = {(0, 0), (0, 1), (1, 2), (2, 0), (2, 2)}
    for level in (70, 5):
        _run(hb, port, case, level, bspec, gspec, present, level)


@pytest.mark.parametrize("L, K, alpha, level", [(20, 2, 1, 20), (64, 3, 64, 33)])
def test_worst_case_words_below_2_61(hb, port, L, K, alpha, level):
    """the largest NTT primes below 2^61, every ciphertext, key and diagonal word q - 1, 64 present babies in a row:
    the sums' 128-bit bound at its largest; (20, 2, 1): digit chunks of 16 in the multiply-accumulates"""
    n = 64
    case = Case(hb, port, L, K, alpha, n, data_bits=(60,), special_bits=(60,), fill="q-1", sets=2)
    assert min(case.mods) > 1 << 60
    bspec = [((3, 5, 2 * n - 1, 25)[i % 4], i % 2) for i in range(62)] + [(1, None)] * 2
    gspec = [(1, None), (5, 1)]
    _run(hb, port, case, level, bspec, gspec, None, 0)


# ------------------------------------------------------------------------------------------------ equalities
@pytest.mark.parametrize("n, L, K, alpha", [(1 << 12, 9, 3, 4), (1 << 16, 30, 10, 10), (1 << 16, 30, 2, 1)])
def test_equalities_with_the_existing_calls(hb, port, n, L, K, alpha):
    """(a) one identity giant: LinearTransformHybrid over the babies, absent diagonals as zero ones; (b) one identity
    baby, diagonals of ones: LinearTransformHybrid over the giants with unit diagonals, and with one giant
    ApplyGaloisKeySwitchHybridHoisted.  The third shape stores eight babies' products over mod-up rounds of 17 + 14
    moduli at level 29."""
    case = Case(hb, port, L, K, alpha, n, sets=3)
    level = L if n == 1 << 12 else L - 1
    nb, comp = level + K, level * n
    src = dev(case.ciphertexts(level, 1, 5))
    bspec = [(pow(5, i + 1, 2 * n), i % 3) for i in range(8)] + [(1, None)]
    diags = torch.zeros(len(bspec) * nb * n, dtype=torch.int64, device="cuda")
    diags.copy_(dev(case.diagonals(level, len(bspec), 3)))
    absent = 2
    diags[absent * nb * n:(absent + 1) * nb * n] = 0
    grid = [[None if i == absent else diags[i * nb * n:(i + 1) * nb * n] for i in range(len(bspec))]]
    a, b = (torch.full((2 * comp,), -1, dtype=torch.int64, device="cuda") for _ in range(2))
    bsgs(hb, case, a, src, grid, level, bspec, [(1, None)], False)
    case.linear(hb, b, src, diags, level, bspec)
    torch.cuda.synchronize()
    assert torch.equal(a, b), "(a) one identity giant"
    gspec = [(2 * n - 1, 0), (1, None), (pow(3, 2, 2 * n), 1), (2 * n - 1, 2)]
    ones = dev(case.diagonals(level, len(gspec), 0, fill="one"))
    grid = [[ones[j * nb * n:(j + 1) * nb * n]] for j in range(len(gspec))]
    bsgs(hb, case, a, src, grid, level, [(1, None)], gspec, False)
    case.linear(hb, b, src, ones, level, gspec)
    torch.cuda.synchronize()
    assert torch.equal(a, b), "(b) one identity baby"
    bsgs(hb, case, a, src, grid[:1], level, [(1, None)], gspec[:1], False)
    case.hoisted(hb, b, src, level, gspec[:1])
    torch.cuda.synchronize()
    assert torch.equal(a, b), "(b) one identity baby, one giant"


# ------------------------------------------------------------------------------------------------ buffers
@pytest.fixture(scope="module")
def buffers_case(hb, port):
    case = Case(hb, port, 7, 3, 3, 1 << 11, seed=77)
    level, batch = 5, 3
    bspec, gspec = _specs(1 << 11)
    ct = case.ciphertexts(level, batch, 21)
    grid = bx.grid_diagonals(case.basis(level), case.n, len(gspec), len(bspec), PRESENT, 21)
    exp = {rs: expected(port, case, ct, grid, level, bspec, gspec, rs, batch) for rs in (False, True)}
    return case, level, batch, bspec, gspec, ct, grid, exp


@pytest.mark.parametrize("rescale", [False, True])
@pytest.mark.parametrize("entry", ["device", "host", "pinned", "managed", "host_split"])
def test_buffers(hb, buffers_case, entry, rescale):
    """batch 3 between sentinel words"""
    case, level, batch, bspec, gspec, ct, grid, exp = buffers_case
    size = exp[rescale].size

    def run(out, src, g, stream=None):
        bsgs(hb, case, out, src, g, level, bspec, gspec, rescale, batch, stream=stream)

    try:
        if entry == "device":
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                buf = torch.full((size + 2,), SENTINEL - (1 << 64), dtype=torch.int64, device="cuda")
                src, g = dev(ct), dev_grid(grid)
                run(buf[1:1 + size], src, g, stream=s)
            s.synchronize()
            got = host(buf)
        elif entry in ("managed", "pinned"):
            alloc, free = ((hb.managed_empty, hb.managed_free) if entry == "managed"
                           else (hb.pinned_empty, hb.pinned_free))
            src, buf = alloc(ct.size), alloc(size + 2)
            g = [[None if w is None else alloc(w.size) for w in row] for row in grid]
            try:
                src[:], buf[:] = ct, SENTINEL
                for row, drow in zip(grid, g):
                    for w, d in zip(row, drow):
                        if w is not None:
                            d[:] = w
                run(buf[1:1 + size], src, g)
                got = buf.copy()
                assert (src == ct).all(), "the ciphertexts changed"
            finally:
                for a in [src, buf] + [d for row in g for d in row if d is not None]:
                    free(a)
        else:
            if entry == "host_split":
                hb.set_host_devices([0, 0])
            buf = np.full(size + 2, SENTINEL, dtype=U64)
            src = ct.copy()
            run(buf[1:1 + size], src, [[None if w is None else w.copy() for w in row] for row in grid])
            assert (src == ct).all(), "the ciphertexts changed"
            got = buf
    finally:
        hb.set_host_devices([])
    assert got[0] == SENTINEL and got[-1] == SENTINEL, "a word next to the output was written"
    _check(got[1:1 + size], exp[rescale], f"{entry} rescale {rescale}")


@pytest.mark.parametrize("rescale", [False, True])
def test_graph_replay(hb, port, buffers_case, rescale):
    case, level, batch, bspec, gspec, ct, grid, exp = buffers_case
    out = torch.zeros(exp[rescale].size, dtype=torch.int64, device="cuda")
    src, g = dev(ct), dev_grid(grid)

    def run():
        bsgs(hb, case, out, src, g, level, bspec, gspec, rescale, batch)

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
    grid2 = bx.grid_diagonals(case.basis(level), case.n, len(gspec), len(bspec), PRESENT, 22)
    src.copy_(dev(ct2))
    for row, drow in zip(grid2, g):
        for w, d in zip(row, drow):
            if w is not None:
                d.copy_(dev(w))
    graph.replay()
    torch.cuda.synchronize()
    _check(host(out), expected(port, case, ct2, grid2, level, bspec, gspec, rescale, batch), "graph replay, new data")


# ------------------------------------------------------------------------------------------------ launch counts
@pytest.mark.parametrize("L, K, alpha, level", [(6, 2, 2, 6), (30, 10, 10, 30), (70, 2, 64, 70), (12, 1, 1, 12)])
def test_launch_counts(hb, port, L, K, alpha, level):
    n = 1 << 12
    case = Case(hb, port, L, K, alpha, n, data_bits=(45,), special_bits=(45,), sets=3)
    bspec, gspec = _specs(n)
    ct = dev(case.ciphertexts(level, 2, 1))
    ntt = _ntt(hb, n)
    many = [(pow(5, i + 1, 2 * n), i % 3) for i in range(66)]
    cases = [("sparse", bspec, gspec, PRESENT),
             ("identity rows only", bspec, [(1, None), (1, None)], {(0, 0), (1, 0)}),
             ("keyed giants over the identity baby", bspec, gspec, {(1, 0), (2, 0), (3, 0)}),
             ("66 babies", many, gspec[:2], {(j, i) for j in range(2) for i in range(66)})]
    for name, bs, gs, present in cases:
        grid = bx.grid_diagonals(case.basis(level), n, len(gs), len(bs), present, 1)
        g = dev_grid(grid)
        for rescale in (False, True):
            out = torch.zeros(out_words(case, level, rescale, 2), dtype=torch.int64, device="cuda")
            bsgs(hb, case, out, ct, g, level, bs, gs, rescale, 2)  # warm
            torch.cuda.synchronize()
            before = hb.launch_count()
            bsgs(hb, case, out, ct, g, level, bs, gs, rescale, 2)
            torch.cuda.synchronize()
            got = hb.launch_count() - before
            exp = plan.bsgs_launches(n, level, K, alpha, case.basis(level), ntt, [k is not None for _, k in bs],
                                     [k is not None for _, k in gs], present, rescale)
            assert got == 2 * exp, (name, rescale, got, 2 * exp)


# ------------------------------------------------------------------------------------------------ refusals
def test_refusals(hb, port):
    case = Case(hb, port, 6, 2, 2, 64, sets=2)
    n, L, K, alpha = case.n, 6, 2, 2
    other = Case(hb, port, 6, 2, 3, 64, sets=1)  # keys for digit size 3: fewer digits than alpha = 2 needs
    bspec, gspec = [(3, 0), (1, None)], [(5, 1), (1, None)]
    ct = dev(case.ciphertexts(L, 1, 2))
    grid = dev_grid(bx.grid_diagonals(case.basis(L), n, 2, 2, None, 2))
    res = torch.zeros(2 * L * n, dtype=torch.int64, device="cuda")
    bh, gh = case.handles_of(bspec), case.handles_of(gspec)

    def refused(what, babies=None, belts=None, giants=None, gelts=None, out=res, src=ct, g=grid, level=L,
                digit=alpha, mods=None, rescale=0, raw=False, null_table=False):
        babies = babies if babies is not None else bh
        giants = giants if giants is not None else gh
        belts = belts if belts is not None else [e for e, _ in bspec]
        gelts = gelts if gelts is not None else [e for e, _ in gspec]
        mods = mods if mods is not None else case.mods
        before = out.clone()
        with pytest.raises(hb.HexlB200Error) as e:
            if raw:  # through the C entry point: a rescale the wrapper would not pass, or a null diagonals array
                import ctypes as C
                vp = C.c_void_p
                table = None if null_table else (vp * 4)(*[d.data_ptr() for row in g for d in row])
                m = np.ascontiguousarray(mods, dtype=U64)
                be, ge = np.ascontiguousarray(belts, dtype=U64), np.ascontiguousarray(gelts, dtype=U64)
                bk = (vp * 2)(*[k._h if k is not None else None for k in babies])
                gk = (vp * 2)(*[k._h if k is not None else None for k in giants])
                hb._check(hb._lib.hexl_b200_linear_transform_hybrid_bsgs(
                    out.data_ptr(), src.data_ptr(), n, level, L, K, digit, m.ctypes.data, bk, be.ctypes.data, 2, gk,
                    ge.ctypes.data, 2, table, rescale, 1, None))
            else:
                hb.LinearTransformHybridBSGS(out, src, n, level, L, K, digit, mods, babies, belts, giants, gelts, g,
                                             rescale)
        assert e.value.code == INVALID_ARG, (what, e.value)
        assert torch.equal(out, before), f"{what}: output written"

    try:
        hb.set_host_devices([0, 0])
        sharded = hb.KeySwitchKeys(case.keys[0], n, len(case.keys[0]), L + K, 2, sharded_by_modulus=True)
    finally:
        hb.set_host_devices([])
    for side in ("baby", "giant"):
        def on(handles=None, elts=None):
            base_h, base_e = (bh, [e for e, _ in bspec]) if side == "baby" else (gh, [e for e, _ in gspec])
            h = handles if handles is not None else base_h
            e = elts if elts is not None else base_e
            return dict(babies=h, belts=e) if side == "baby" else dict(giants=h, gelts=e)
        refused(f"a null {side} key for g = 3", **on(handles=[None, None], elts=[3, 1]))
        refused(f"a {side} handle of another digit size", **on(handles=[other.handles[0], None]))
        refused(f"a sharded {side} handle", **on(handles=[sharded, None]))
        refused(f"an even {side} element", **on(elts=[4, 1]))
        refused(f"a {side} element of 2n", **on(elts=[2 * n + 1, 1]))
    refused("level 0", level=0)
    refused("digit size 65", digit=65)
    refused("a modulus >= 2^61", mods=case.mods[:-1] + [int(port.generate_primes(1, 62, True, n)[0])])
    refused("rescale = 2", rescale=2, raw=True)
    refused("rescale = -1", rescale=-1, raw=True)
    refused("rescale at level 1", level=1, rescale=1, g=dev_grid(bx.grid_diagonals(case.basis(1), n, 2, 2, None, 2)))
    refused("a null diagonals array", raw=True, null_table=True)
    big = torch.zeros(8 * L * n, dtype=torch.int64, device="cuda")
    refused("result overlaps the ciphertexts", out=big[:2 * L * n], src=big[L * n:3 * L * n])
    d_big = torch.zeros(4 * (L + K) * n, dtype=torch.int64, device="cuda")
    overlap = [[d_big[n:n + (L + K) * n], None], [None, None]]
    refused("result overlaps a diagonal", out=d_big[:2 * L * n], g=overlap)
    bad = case.ciphertexts(L, 1, 2)
    bad[7] = case.mods[0]
    badg = bx.grid_diagonals(case.basis(L), n, 2, 2, None, 2)
    badg[1][0] = badg[1][0].copy()
    badg[1][0][(L + 1) * n + 3] = case.mods[L + 1]  # limb L + 1: under p_1
    hb.set_debug(True)
    try:
        refused("a ciphertext word = q under debug", src=dev(bad))
        refused("a diagonal word = its modulus under debug", g=dev_grid(badg))
    finally:
        hb.set_debug(False)
    wide = Case(hb, port, 2, 64, 2, 16, sets=1)  # p_size 64: the merged mod-down would convert from 65 moduli
    out = torch.zeros(2 * 16, dtype=torch.int64, device="cuda")
    with pytest.raises(hb.HexlB200Error) as e:
        hb.LinearTransformHybridBSGS(out, dev(wide.ciphertexts(2, 1, 1)), 16, 2, 2, 64, 2, wide.mods, [None], [1],
                                     [None], [1], dev_grid(bx.grid_diagonals(wide.basis(2), 16, 1, 1, None, 1)), 1)
    assert e.value.code == INVALID_ARG and not out.any(), "rescale with p_size 64"
    before = res.clone()
    empty = [[None] * 2] * 2
    hb.LinearTransformHybridBSGS(res, ct, n, L, L, K, alpha, case.mods, [], [], gh, [5, 1], [], 0)
    hb.LinearTransformHybridBSGS(res, ct, n, L, L, K, alpha, case.mods, bh, [3, 1], [], [], [], 0)
    hb.LinearTransformHybridBSGS(res, ct, n, L, L, K, alpha, case.mods, bh, [3, 1], gh, [5, 1], empty, 0, batch=0)
    torch.cuda.synchronize()
    assert torch.equal(res, before), "num_baby = 0, num_giant = 0 or batch = 0 wrote"


def test_cpp_caller_runs(hb, tmp_path):
    if not shutil.which("g++"):
        pytest.skip("g++ not present")
    exe = tmp_path / "bsgs_caller"
    libdir = os.path.dirname(hb.LIB_PATH)
    subprocess.run(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "cpp", "bsgs_caller.cpp"), "-o", str(exe),
                    "-L", libdir, "-lhexl_b200", f"-Wl,-rpath,{libdir}"], check=True)
    res = subprocess.run([str(exe), "run"], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
