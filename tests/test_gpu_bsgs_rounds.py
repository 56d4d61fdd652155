"""LinearTransformHybridBSGS where its rounds and blocks repeat: at production sizes, on the benchmark's grid, at every
level, over host batches that wrap the staging slots, between host calls of other slot sizes, from several threads, on
offset views and on every diagonal aliasing the API allows.

Every output is compared bit for bit with the exact model (tests/bsgs_exact.py), every counted device call's launches
with the plan of tests/composite_plan.py (bsgs_launches), and every input must come back unchanged.  The grids are
composite_plan's BSGS_SPARSE, BSGS_SWEEP and BSGS_BENCH (test_composite_plan.py asserts what each holds):
    production      every HYBRID_SHAPES entry at each of its levels, rescale 0 and 1: the baby and giant mod-ups at
                    rounds 34 + 6 (budget_a2), the level-28 round mixing data limbs with special primes (budget_a3,
                    N = 2^17), the giants' accumulating multiply-accumulate in 16 + 8 digit chunks (mixed_chunks) and
                    the merged mod-down's 27 + 2 targets (bench_rescale), with the one-component mod-down of a keyed
                    giant over keyed babies at each
    benchmark grid  tools/bsgs_bench.py's 8 x 8 grid at N = 2^16, (L, K, alpha) = (30, 10, 10), level 30
    every level     levels 1..L of (30, 10, 10) and (13, 3, 4) at n = 2^8: the one-component mod-down crosses its
                    29 | 30 block, the mod-up 19 | 20 and the merged rescale 28 | 29
Two key sets alternate over the keyed terms, so a mix-up of baby and giant keys or of stored-product indices changes
the result.  Each shape's keys are freed when its tests end."""
import threading

import numpy as np
import pytest

import bsgs_exact as bx
import composite_plan as plan
import hybrid_exact as hx
from test_gpu_hybrid_key_switch import SENTINEL, dev, host
from test_gpu_hybrid_rounds import Shape, _check, _counted, _guarded, _ntt, _out, _placed

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

U64 = np.uint64
MIXED_POINTERS = -5   # HEXL_B200_ERR_MIXED_POINTERS


@pytest.fixture(scope="module", autouse=True)
def _need_cuda(hb):
    if not torch.cuda.is_available() or hb.device_count() == 0:
        pytest.fail("gpu-marked test collected on a machine without CUDA")


class Shape2(Shape):
    """Shape with a second key set: a spec lists (element, key set 0 or 1, or None for an identity term)"""

    def __init__(self, hb, port, n, L, K, alpha, data_bits=50, special_bits=50, seed=1):
        super().__init__(hb, port, n, L, K, alpha, data_bits, special_bits, seed)
        self.keys2 = hx.random_keys(self.mods, n, L, alpha, 2, seed + 7777)
        self.handle2 = hb.KeySwitchKeys(self.keys2, n, len(self.keys2), L + K, 2)

    def free(self):
        self.handle2 = self.keys2 = None
        super().free()

    def handles_of(self, spec):
        return [None if k is None else (self.handle, self.handle2)[k] for _, k in spec]

    def keys_of(self, spec):
        return [None if k is None else (self.keys, self.keys2)[k] for _, k in spec]

    def grid(self, level, nb, ng, present, seed):
        return bx.grid_diagonals(self.basis(level), self.n, ng, nb, present, seed)

    def bsgs(self, hb, out, ct, grid, level, bspec, gspec, rescale, batch=1, stream=None):
        hb.LinearTransformHybridBSGS(out, ct, self.n, level, self.L, self.K, self.alpha, self.mods,
                                     self.handles_of(bspec), [g for g, _ in bspec], self.handles_of(gspec),
                                     [g for g, _ in gspec], grid, rescale, batch, stream=stream)

    def exp_bsgs(self, port, ct, grid, level, bspec, gspec, rescale, batch=1):
        per = 2 * level * self.n
        return np.concatenate([bx.bsgs_exact(port, ct[c * per:(c + 1) * per], self.n, level, self.L, self.K,
                                             self.alpha, self.mods, [g for g, _ in bspec], self.keys_of(bspec),
                                             [g for g, _ in gspec], self.keys_of(gspec), grid, rescale)
                               for c in range(batch)])

    def bsgs_launches(self, level, ntt, bspec, gspec, present, rescale):
        return plan.bsgs_launches(self.n, level, self.K, self.alpha, self.basis(level), ntt,
                                  [k is not None for _, k in bspec], [k is not None for _, k in gspec], present,
                                  rescale)


def sparse_specs(n):
    """BSGS_SPARSE's terms: babies 1, 5, 3 (without a diagonal), 2n - 1, 25 and 5 again under the other key set;
    giants 1, 125, 5 and 2n - 1 (the absent row)"""
    two = 2 * n
    bspec = [(1, None), (5 % two, 0), (3 % two, 1), (two - 1, 1), (25 % two, 0), (5 % two, 1)]
    gspec = [(1, None), (125 % two, 1), (5 % two, 0), (two - 1, 1)]
    babies, giants, present = plan.BSGS_SPARSE
    assert [k is not None for _, k in bspec] == list(babies) and [k is not None for _, k in gspec] == list(giants)
    return bspec, gspec, present


def sweep_specs(n):
    """BSGS_SWEEP's terms: babies 1, 5 and 2n - 1; giants 1, 25 and 2n - 1 (under the other key set)"""
    bspec = [(1, None), (5 % (2 * n), 0), (2 * n - 1, 1)]
    gspec = [(1, None), (25 % (2 * n), 1), (2 * n - 1, 0)]
    babies, giants, present = plan.BSGS_SWEEP
    assert [k is not None for _, k in bspec] == list(babies) and [k is not None for _, k in gspec] == list(giants)
    return bspec, gspec, present


def _dev_grid(grid):
    return [[None if w is None else dev(w) for w in row] for row in grid]


def _same(dgrid, grid):
    return all(d is None or torch.equal(d, dev(w)) for drow, row in zip(dgrid, grid) for d, w in zip(drow, row))


def _device_run(hb, port, shape, level, specs, seed):
    """device buffers at one level, rescale 0 and (from level 2) 1, against the model and the plan; the inputs must
    come back unchanged"""
    bspec, gspec, present = specs
    n = shape.n
    ct = shape.limbs(level, 2, seed)
    grid = shape.grid(level, len(bspec), len(gspec), present, seed)
    d_ct, d_grid = dev(ct), _dev_grid(grid)
    ntt = _ntt(hb, n)
    for rescale in (False, True)[:1 + (level >= 2)]:
        where = f"n = {n}, ({shape.L}, {shape.K}, {shape.alpha}), level {level}, rescale {rescale}"
        out = _out(2 * (level - int(rescale)) * n)
        shape.bsgs(hb, out, d_ct, d_grid, level, bspec, gspec, rescale)
        _check(host(out), shape.exp_bsgs(port, ct, grid, level, bspec, gspec, rescale), where)
        got = _counted(hb, lambda: shape.bsgs(hb, out, d_ct, d_grid, level, bspec, gspec, rescale))
        assert got == shape.bsgs_launches(level, ntt, bspec, gspec, present, rescale), (where, got)
    torch.cuda.synchronize()
    assert torch.equal(d_ct, dev(ct)) and _same(d_grid, grid), f"an input changed, level {level}"


# ------------------------------------------------------------------------------------------------ production sizes
@pytest.fixture(scope="class")
def production(hb, port, request):
    logn, L, K, alpha, dbits, sbits, levels = plan.HYBRID_SHAPES[request.param]
    shape = Shape2(hb, port, 1 << logn, L, K, alpha, dbits, sbits, seed=logn * 100 + alpha)
    yield shape, levels
    shape.free()


@pytest.mark.parametrize("production", sorted(plan.HYBRID_SHAPES), indirect=True)
class TestProductionShapes:
    def test_sparse_grid_at_each_level(self, hb, port, production):
        shape, levels = production
        for level in levels:
            _device_run(hb, port, shape, level, sparse_specs(shape.n), seed=level)


def test_benchmark_grid(hb, port):
    """tools/bsgs_bench.py's grid: babies 5^i and giants 5^(8j), i, j < 8, the first of each an identity term, every
    diagonal present; seven stored babies' products and seven one-component mod-downs"""
    logn, L, K, alpha, dbits, sbits, level = plan.BSGS_BENCH_SHAPE
    n = 1 << logn
    shape = Shape2(hb, port, n, L, K, alpha, dbits, sbits, seed=31)
    try:
        bspec = [(pow(5, i, 2 * n), None if i == 0 else i % 2) for i in range(8)]
        gspec = [(pow(5, 8 * j, 2 * n), None if j == 0 else (j + 1) % 2) for j in range(8)]
        babies, giants, present = plan.BSGS_BENCH
        assert [k is not None for _, k in bspec] == list(babies) and [k is not None for _, k in gspec] == list(giants)
        _device_run(hb, port, shape, level, (bspec, gspec, present), seed=8)
    finally:
        shape.free()


# ------------------------------------------------------------------------------------------------ every level
@pytest.mark.parametrize("L, K, alpha", [(30, 10, 10), (13, 3, 4)])
def test_every_level(hb, port, L, K, alpha):
    n = 1 << 8
    shape = Shape2(hb, port, n, L, K, alpha, seed=L + K + alpha)
    try:
        for level in range(1, L + 1):
            _device_run(hb, port, shape, level, sweep_specs(n), seed=level)
    finally:
        shape.free()


# ------------------------------------------------------------------------------------------------ host batches
@pytest.fixture(scope="module")
def small(hb, port):
    """(7, 3, 3) at n = 2^11, level 5 (a partial last digit), batch 7 over the sparse grid: inputs and models"""
    shape = Shape2(hb, port, 1 << 11, 7, 3, 3, seed=11)
    level, batch = 5, 7
    specs = sparse_specs(shape.n)
    bspec, gspec, present = specs
    ct = shape.limbs(level, 2 * batch, 51)
    grid = shape.grid(level, len(bspec), len(gspec), present, 52)
    exp = {rs: shape.exp_bsgs(port, ct, grid, level, bspec, gspec, rs, batch) for rs in (False, True)}
    yield dict(shape=shape, level=level, batch=batch, specs=specs, ct=ct, grid=grid, exp=exp)
    shape.free()


def _host_bsgs(hb, shape, level, specs, ct, grid, rescale, batch, exp):
    """one host-buffer call between sentinel words, against exp; the ciphertexts and diagonals come back unchanged"""
    bspec, gspec, _ = specs
    buf = np.full(exp.size + 2, SENTINEL, dtype=U64)
    src = ct[:batch * 2 * level * shape.n].copy()
    hgrid = [[None if w is None else w.copy() for w in row] for row in grid]
    shape.bsgs(hb, buf[1:-1], src, hgrid, level, bspec, gspec, rescale, batch)
    assert (src == ct[:src.size]).all(), "the ciphertexts changed"
    assert all(w is None or (w == v).all() for row, hrow in zip(grid, hgrid) for v, w in zip(row, hrow)), \
        "a diagonal changed"
    assert buf[0] == SENTINEL and buf[-1] == SENTINEL, "a word next to the output was written"
    return buf[1:-1]


def _small_exp(small, rescale, first, count):
    per = 2 * (small["level"] - int(rescale)) * small["shape"].n
    return small["exp"][rescale][first * per:(first + count) * per]


@pytest.mark.parametrize("rescale", [False, True])
@pytest.mark.parametrize("devices", [[], [0, 0], [0, 0, 0]], ids=["one", "split2", "split3"])
def test_host_batch_of_seven(hb, small, devices, rescale):
    """batch 7: blocks of 7, 3 + 4 and 2 + 2 + 3 ciphertexts, so the 3 staging slots of a device wrap; with
    [0, 0, 0] the present diagonals are uploaded three times to one device"""
    exp = _small_exp(small, rescale, 0, small["batch"])
    try:
        hb.set_host_devices(devices)
        got = _host_bsgs(hb, small["shape"], small["level"], small["specs"], small["ct"], small["grid"], rescale,
                         small["batch"], exp)
    finally:
        hb.set_host_devices([])
    _check(got, exp, f"batch 7 over {devices or 'the default device'}, rescale {rescale}")


def test_host_calls_of_different_slot_sizes_in_sequence(hb, port, small):
    """one device, host buffers, batch 4: BSGS with the rescale (output slots smaller than input), hoisted G = 5, the
    linear transform (which uploads diagonals too), BSGS without the rescale over the sweep grid, and BSGS with the
    rescale again.  None may read what an earlier call left in the slots."""
    shape, level = small["shape"], small["level"]
    n, comp = shape.n, level * shape.n
    ct = small["ct"][:4 * 2 * comp]

    def bsgs_rescale():
        exp = _small_exp(small, True, 0, 4)
        _check(_host_bsgs(hb, shape, level, small["specs"], ct, small["grid"], True, 4, exp), exp, "BSGS, rescale")

    bsgs_rescale()
    elts5 = [5, 2 * n - 1, 25, 3, 9]
    buf = np.full(4 * 5 * 2 * comp + 2, SENTINEL, dtype=U64)
    shape.hoisted(hb, buf[1:-1], ct.copy(), level, elts5, 4)
    assert buf[0] == SENTINEL and buf[-1] == SENTINEL, "hoisted: a word next to the output was written"
    _check(buf[1:-1], shape.exp_hoisted(port, ct, level, elts5, 4), "hoisted G = 5")
    lelts = [25, 1, 3]
    diag = shape.diagonals(level, len(lelts), 61)
    buf = np.full(4 * 2 * comp + 2, SENTINEL, dtype=U64)
    shape.linear(hb, buf[1:-1], ct.copy(), diag.copy(), level, lelts, 4)
    assert buf[0] == SENTINEL and buf[-1] == SENTINEL, "linear: a word next to the output was written"
    _check(buf[1:-1], shape.exp_linear(port, ct, diag, level, lelts, 4), "LinearTransformHybrid")
    specs = sweep_specs(n)
    grid = shape.grid(level, len(specs[0]), len(specs[1]), specs[2], 62)
    exp = shape.exp_bsgs(port, ct, grid, level, specs[0], specs[1], False, 4)
    _check(_host_bsgs(hb, shape, level, specs, ct, grid, False, 4, exp), exp, "BSGS over the sweep grid")
    bsgs_rescale()


def test_threads_share_keys_pool_caches_and_slots(hb, small):
    """four host threads, each on its own stream, four iterations: BSGS device calls with and without the rescale
    queued, then one BSGS host call of batch 2 while they run; the threads share the key handles, the scratch pool,
    the NTT cache and the staging slots"""
    shape, level, (bspec, gspec, _) = small["shape"], small["level"], small["specs"]
    n, per = shape.n, 2 * level * shape.n
    errors = []

    def worker(t):
        try:
            s = torch.cuda.Stream()
            for i in range(4):
                c = (t + 2 * i) % small["batch"]
                with torch.cuda.stream(s):
                    src, g = dev(small["ct"][c * per:(c + 1) * per]), _dev_grid(small["grid"])
                    outs = {rs: _out(2 * (level - int(rs)) * n) for rs in (False, True)}
                    for rs, o in outs.items():
                        shape.bsgs(hb, o, src, g, level, bspec, gspec, rs, stream=s)
                rs = bool((t + i) % 2)
                first = (t + i) % (small["batch"] - 1)
                exp = _small_exp(small, rs, first, 2)
                got = _host_bsgs(hb, shape, level, small["specs"], small["ct"][first * per:], small["grid"], rs, 2,
                                 exp)
                _check(got, exp, f"thread {t} iteration {i}: host call")
                s.synchronize()
                for rs, o in outs.items():
                    _check(host(o), _small_exp(small, rs, c, 1), f"thread {t} iteration {i}: rescale {rs}")
        except BaseException as e:  # noqa: BLE001 - reported by the main thread
            errors.append(e)

    threads = [threading.Thread(target=worker, args=(t,)) for t in range(4)]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors


# ------------------------------------------------------------------------------------------------ offset views
_VIEW_CASES = {}


def _view_case(hb, port, n):
    """(6, 2, 2) at level 5 and degree n, a keyed giant over a keyed baby: inputs and both models, built once per
    degree"""
    if n not in _VIEW_CASES:
        shape = Shape2(hb, port, n, 6, 2, 2, seed=n % 1000 + 5)
        level = 5
        specs = ([(1, None), (5 % (2 * n), 0), (2 * n - 1, 1)], [(1, None), (3 % (2 * n), 1)],
                 {(0, 0), (0, 1), (1, 0), (1, 2)})
        ct = shape.limbs(level, 2, 71)
        grid = shape.grid(level, 3, 2, specs[2], 72)
        exp = {rs: shape.exp_bsgs(port, ct, grid, level, specs[0], specs[1], rs) for rs in (False, True)}
        _VIEW_CASES[n] = dict(shape=shape, level=level, specs=specs, ct=ct, grid=grid, exp=exp)
    return _VIEW_CASES[n]


@pytest.fixture(scope="module", autouse=True)
def _free_view_cases():
    yield
    for v in _VIEW_CASES.values():
        v["shape"].free()
    _VIEW_CASES.clear()


@pytest.mark.parametrize("where", ["ciphertexts", "result", "diagonals", "all", "alternate"])
@pytest.mark.parametrize("n", [8, 1 << 12, 1 << 16])
def test_offset_views(hb, port, n, where):
    """the ciphertexts, the result or the diagonals 8 bytes off 16-byte alignment, one at a time and all together,
    and a grid whose diagonals alternate aligned and offset; inputs come back unchanged, guard words untouched"""
    v = _view_case(hb, port, n)
    shape, level, (bspec, gspec, present) = v["shape"], v["level"], v["specs"]
    off_ct, off_out = where in ("ciphertexts", "all"), where in ("result", "all")
    placed_ct = _placed(v["ct"].size, off_ct, v["ct"])
    placed_grid, k = [], 0
    for row in v["grid"]:
        prow = []
        for w in row:
            if w is None:
                prow.append(None)
                continue
            off = where in ("diagonals", "all") or (where == "alternate" and k % 2 == 1)
            prow.append(_placed(w.size, off, w))
            k += 1
        placed_grid.append(prow)
    d_grid = [[None if p is None else p[1] for p in row] for row in placed_grid]
    ntt = _ntt(hb, n)
    for rescale in (False, True):
        exp = v["exp"][rescale]
        obuf, out, ostart = _placed(exp.size, off_out)
        shape.bsgs(hb, out, placed_ct[1], d_grid, level, bspec, gspec, rescale)
        torch.cuda.synchronize()
        _check(host(out), exp, f"n = {n}, {where} offset, rescale {rescale}")
        assert _guarded(obuf, ostart, exp.size), "a guard word next to the result was written"
        got = _counted(hb, lambda: shape.bsgs(hb, out, placed_ct[1], d_grid, level, bspec, gspec, rescale))
        assert got == shape.bsgs_launches(level, ntt, bspec, gspec, present, rescale), (where, rescale, got)
    inputs = [(placed_ct, v["ct"])] + [(p, w) for prow, row in zip(placed_grid, v["grid"])
                                       for p, w in zip(prow, row) if p is not None]
    for (buf, view, start), x in inputs:
        assert (host(view) == x).all() and _guarded(buf, start, x.size), "an input or its guard words changed"


# ------------------------------------------------------------------------------------------------ aliasing
@pytest.fixture(scope="module")
def alias_shape(hb, port):
    shape = Shape2(hb, port, 1 << 10, 6, 2, 2, seed=91)
    yield shape
    shape.free()


def _alias_case(shape, kind):
    """(ciphertext, grid, specs) of one allowed aliasing, as numpy arrays that share memory the way the call's
    buffers will"""
    n, level = shape.n, 5
    comp, dw = level * n, (level + shape.K) * n
    bspec = [(1, None), (5, 0), (2 * n - 1, 1)]
    gspec = [(1, None), (3, 1), (25, 0)]
    present = {(0, 0), (0, 1), (1, 1), (1, 2), (2, 0), (2, 2)}
    if kind == "one_handle":  # every keyed baby and giant under key set 0
        bspec, gspec = ([(g, None if k is None else 0) for g, k in spec] for spec in (bspec, gspec))
    ct = shape.limbs(level, 2, 81)
    grid = shape.grid(level, 3, 3, present, 82)
    if kind == "same_buffer":  # one diagonal at every present position
        w = grid[1][1]
        grid = [[None if x is None else w for x in row] for row in grid]
    elif kind == "one_buffer":  # every diagonal a view into one buffer
        pairs = sorted(present)
        whole = np.concatenate([grid[j][i] for j, i in pairs])
        for k, (j, i) in enumerate(pairs):
            grid[j][i] = whole[k * dw:(k + 1) * dw]
    elif kind == "overlaps_ct":  # diagonal (1, 2) starts at c1: its data limbs are c1's, its special limbs follow
        whole = np.concatenate([ct, grid[1][2][comp:]])
        ct, grid[1][2] = whole[:2 * comp], whole[comp:comp + dw]
    return level, ct, grid, (bspec, gspec, present)


def _shared_copies(ct, grid, copy):
    """ct and grid copied by copy(buffer) once per underlying buffer, the copies sharing memory exactly as the numpy
    arrays do"""
    bases = {}
    for a in [ct] + [w for row in grid for w in row if w is not None]:
        base = a if a.base is None else a.base
        bases.setdefault(id(base), (base, copy(base)))

    def view(a):
        base, c = bases[id(a if a.base is None else a.base)]
        off = (a.__array_interface__["data"][0] - base.__array_interface__["data"][0]) // 8
        return c[off:off + a.size]

    return view(ct), [[None if w is None else view(w) for w in row] for row in grid]


@pytest.mark.parametrize("path", ["device", "host"])
@pytest.mark.parametrize("kind", ["same_buffer", "one_buffer", "overlaps_ct", "one_handle"])
def test_allowed_aliasing(hb, port, alias_shape, kind, path):
    """one diagonal buffer at several grid positions, every diagonal a view into one buffer, a diagonal overlapping
    the ciphertexts, and one key handle as every baby and giant key"""
    shape = alias_shape
    level, ct, grid, specs = _alias_case(shape, kind)
    bspec, gspec, present = specs
    ntt = _ntt(hb, shape.n)
    for rescale in (False, True):
        exp = shape.exp_bsgs(port, ct, grid, level, bspec, gspec, rescale)
        if path == "device":
            d_ct, d_grid = _shared_copies(ct, grid, dev)
            out = _out(exp.size)
            shape.bsgs(hb, out, d_ct, d_grid, level, bspec, gspec, rescale)
            _check(host(out), exp, f"{kind}, device, rescale {rescale}")
            got = _counted(hb, lambda: shape.bsgs(hb, out, d_ct, d_grid, level, bspec, gspec, rescale))
            assert got == shape.bsgs_launches(level, ntt, bspec, gspec, present, rescale), (kind, rescale, got)
            assert torch.equal(d_ct, dev(ct)) and _same(d_grid, grid), f"{kind}: an input changed"
        else:
            h_ct, h_grid = _shared_copies(ct, grid, np.copy)
            buf = np.full(exp.size + 2, SENTINEL, dtype=U64)
            shape.bsgs(hb, buf[1:-1], h_ct, h_grid, level, bspec, gspec, rescale)
            assert buf[0] == SENTINEL and buf[-1] == SENTINEL, "a word next to the output was written"
            _check(buf[1:-1], exp, f"{kind}, host, rescale {rescale}")
            assert (h_ct == ct).all() and all(w is None or (w == v).all() for row, hrow in zip(grid, h_grid)
                                              for v, w in zip(row, hrow)), f"{kind}: an input changed"


def test_device_diagonal_with_host_ciphertexts_is_refused(hb, alias_shape):
    shape = alias_shape
    level, ct, grid, (bspec, gspec, _) = _alias_case(shape, "one_handle")
    mixed = [[w if (j, i) != (1, 1) or w is None else dev(w) for i, w in enumerate(row)] for j, row in enumerate(grid)]
    assert mixed[1][1] is not None
    out = np.full(2 * level * shape.n, SENTINEL, dtype=U64)
    with pytest.raises(hb.HexlB200Error) as e:
        shape.bsgs(hb, out, ct.copy(), mixed, level, bspec, gspec, False)
    assert e.value.code == MIXED_POINTERS, e.value
    assert (out == SENTINEL).all(), "the output was written"
