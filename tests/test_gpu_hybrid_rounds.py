"""The hybrid family where its rounds and blocks repeat: KeySwitchHybrid, ApplyGaloisKeySwitchHybridHoisted,
LinearTransformHybrid and MultiplyRelinearizeHybrid at production sizes, at every level, over host batches that wrap
the staging slots, on offset views and from several threads.

Every output is compared bit for bit with the exact models (tests/hybrid_exact.py, hybrid_rotation_exact.py,
mul_relin_exact.py), and every launch count with the plan of tests/composite_plan.py (hybrid_launches), so each test
shows that the rounds and blocks it names really ran:
    bench_rescale   N = 2^16, (L, K, alpha) = (30, 10, 10): the merged rescale's mod-down converts into 27 + 2 targets
    budget_a2       N = 2^16, (30, 10, 2): mod-up rounds 34 + 6 under the 256 MiB scratch budget, 34 + 5 at level 29
    budget_a3       N = 2^17, (30, 3, 3): rounds 25 + 8, and 25 + 6 at level 28, whose second round mixes data limbs
                    with special primes (key slots q_size + j, not their positions in B)
    mixed_chunks    N = 2^16, (24, 2, 1), special primes just below 2^61: rounds 21 + 5, the multiply-accumulate one
                    launch in the first round and 16 + 8 in the second
tests/test_composite_plan.py asserts on the CPU that each name still has that plan.  One key set (about 0.6 GB at the
budget shapes) serves every element, and is freed with its shape."""
import gc
import threading

import numpy as np
import pytest

import composite_plan as plan
import hybrid_exact as hx
import hybrid_rotation_exact as hr
import mul_relin_exact as mr
from test_gpu_hybrid_key_switch import SENTINEL, _check, _primes, dev, host
from util import uniform_below

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

U64 = np.uint64


@pytest.fixture(scope="module", autouse=True)
def _need_cuda(hb):
    if not torch.cuda.is_available() or hb.device_count() == 0:
        pytest.fail("gpu-marked test collected on a machine without CUDA")


class Shape:
    """L data moduli then K special primes and ONE hybrid key set (key component count 2) with its handle: every
    call and every Galois element of this file uses it, since distinct elements still give distinct products"""

    def __init__(self, hb, port, n, L, K, alpha, data_bits=50, special_bits=50, seed=1):
        self.n, self.L, self.K, self.alpha = n, L, K, alpha
        self.mods = _primes(port, n, L, (data_bits,), False) + _primes(port, n, K, (special_bits,), True)
        assert len(set(self.mods)) == L + K
        self.keys = hx.random_keys(self.mods, n, L, alpha, 2, seed)
        self.handle = hb.KeySwitchKeys(self.keys, n, len(self.keys), L + K, 2)

    def free(self):
        self.handle = self.keys = None
        gc.collect()

    def basis(self, level):
        return self.mods[:level] + self.mods[self.L:]

    def limbs(self, level, count, seed):
        """count polynomials of level canonical limbs"""
        return np.concatenate([uniform_below(seed * 7919 + 64 * c + i, self.n, self.mods[i]) for c in range(count)
                               for i in range(level)])

    def diagonals(self, level, count, seed):
        return hr.random_diagonals(self.basis(level), self.n, count, seed)

    # the four calls, on whatever buffers they get
    def switch(self, hb, out, t, level, batch=1, stream=None):
        hb.KeySwitchHybrid(out, t, self.n, level, self.L, self.K, self.alpha, 2, self.mods, self.handle, batch,
                           stream=stream)

    def hoisted(self, hb, out, ct, level, elts, batch=1, stream=None):
        hb.ApplyGaloisKeySwitchHybridHoisted(out, ct, self.n, level, self.L, self.K, self.alpha, self.mods,
                                             [self.handle] * len(elts), elts, batch, stream=stream)

    def linear(self, hb, out, ct, diag, level, elts, batch=1, stream=None):
        handles = [None if g == 1 else self.handle for g in elts]
        hb.LinearTransformHybrid(out, ct, self.n, level, self.L, self.K, self.alpha, self.mods, handles, elts, diag,
                                 batch, stream=stream)

    def mul(self, hb, out, ct1, ct2, level, rescale, batch=1, stream=None):
        hb.MultiplyRelinearizeHybrid(out, ct1, ct2, self.n, level, self.L, self.K, self.alpha, self.mods,
                                     self.handle, rescale, batch, stream=stream)

    # their models, per ciphertext of a batch
    def exp_switch(self, port, res, t, level, batch=1):
        pr, pt = 2 * level * self.n, level * self.n
        return np.concatenate([hx.key_switch_hybrid(port, res[c * pr:(c + 1) * pr], t[c * pt:(c + 1) * pt], self.n,
                                                    level, self.L, self.K, self.alpha, 2, self.mods, self.keys)
                               for c in range(batch)])

    def exp_hoisted(self, port, ct, level, elts, batch=1):
        per = 2 * level * self.n
        return np.concatenate([hr.hoisted_exact(port, ct[c * per:(c + 1) * per], self.n, level, self.L, self.K,
                                                self.alpha, self.mods, elts, [self.keys] * len(elts))
                               for c in range(batch)])

    def exp_linear(self, port, ct, diag, level, elts, batch=1):
        per = 2 * level * self.n
        keys = [None if g == 1 else self.keys for g in elts]
        return np.concatenate([hr.linear_transform_exact(port, ct[c * per:(c + 1) * per], self.n, level, self.L,
                                                         self.K, self.alpha, self.mods, elts, keys, diag)
                               for c in range(batch)])

    def exp_mul(self, port, ct1, ct2, level, rescale, batch=1):
        per = 2 * level * self.n
        return np.concatenate([mr.multiply_relinearize(port, ct1[c * per:(c + 1) * per], ct2[c * per:(c + 1) * per],
                                                       self.n, level, self.L, self.K, self.alpha, self.mods,
                                                       self.keys, rescale) for c in range(batch)])

    def launches(self, call, level, ntt, **kw):
        return plan.hybrid_launches(call, self.n, level, self.K, self.alpha, self.basis(level), ntt, **kw)


_NTT_LAUNCHES = {}


def _ntt(hb, n):
    """ntt(forward, units): the launches of one multi-modulus transform of `units` polynomials at degree n, measured
    once per (n, direction, units).  The measuring call passes at least two handles (a single one takes the
    single-modulus path, whose kernels differ at some degrees): c copies, c the least divisor of units in [2, 64].
    One unit (the mod-up of level 1) is measured as two: no kernel choice separates them."""
    def count(forward, units):
        key = (n, forward, units)
        if key not in _NTT_LAUNCHES:
            u = max(units, 2)
            c = next((d for d in range(2, 65) if u % d == 0), None)
            assert c is not None, f"{units} units have no divisor in [2, 64] to measure them as c copies by"
            h = hb.GetNTT(n, hb.GeneratePrimes(1, 50, True, n)[0])
            x = torch.zeros(u * n, dtype=torch.int64, device="cuda")
            fn = hb.ComputeForwardMulti if forward else hb.ComputeInverseMulti
            fn([h] * c, x, x)
            torch.cuda.synchronize()
            before = hb.launch_count()
            fn([h] * c, x, x)
            torch.cuda.synchronize()
            _NTT_LAUNCHES[key] = hb.launch_count() - before
        return _NTT_LAUNCHES[key]
    return count


def _counted(hb, run):
    """the launches of one more run(), after run() has warmed the tables and the pool"""
    torch.cuda.synchronize()
    before = hb.launch_count()
    run()
    torch.cuda.synchronize()
    return hb.launch_count() - before


def _out(words):
    return torch.full((words,), -1, dtype=torch.int64, device="cuda")


def _all_four(hb, port, shape, level, elts, lelts, seed, rescales=(False, True), count=True):
    """the four calls on device buffers at one level against their models, and (count) their launch counts against
    the plan; the inputs must come back unchanged"""
    n = shape.n
    comp = level * n
    ntt = _ntt(hb, n)
    ct, ct2 = shape.limbs(level, 2, seed), shape.limbs(level, 2, seed + 500)
    res = shape.limbs(level, 2, seed + 900)
    diag = shape.diagonals(level, len(lelts), seed)
    d_ct, d_ct2, d_diag = dev(ct), dev(ct2), dev(diag)
    where = f"n = {n}, ({shape.L}, {shape.K}, {shape.alpha}), level {level}"

    out = dev(res)
    shape.switch(hb, out, d_ct[comp:], level)
    _check(host(out), shape.exp_switch(port, res, ct[comp:], level), f"KeySwitchHybrid, {where}")
    if count:
        got = _counted(hb, lambda: shape.switch(hb, out, d_ct[comp:], level))
        assert got == shape.launches("switch", level, ntt), ("switch", where, got)

    out = _out(len(elts) * 2 * comp)
    shape.hoisted(hb, out, d_ct, level, elts)
    _check(host(out), shape.exp_hoisted(port, ct, level, elts), f"hoisted {elts}, {where}")
    if count:
        got = _counted(hb, lambda: shape.hoisted(hb, out, d_ct, level, elts))
        assert got == shape.launches("hoisted", level, ntt, elts=len(elts)), ("hoisted", where, got)

    out = _out(2 * comp)
    shape.linear(hb, out, d_ct, d_diag, level, lelts)
    _check(host(out), shape.exp_linear(port, ct, diag, level, lelts), f"linear transform {lelts}, {where}")
    if count:
        got = _counted(hb, lambda: shape.linear(hb, out, d_ct, d_diag, level, lelts))
        keyed = sum(g != 1 for g in lelts)
        assert got == shape.launches("linear", level, ntt, elts=len(lelts), keyed=keyed), ("linear", where, got)

    for rescale in rescales:
        if rescale and level < 2:
            continue
        out = _out(2 * (level - int(rescale)) * n)
        shape.mul(hb, out, d_ct, d_ct2, level, rescale)
        _check(host(out), shape.exp_mul(port, ct, ct2, level, rescale), f"mul_relin rescale {rescale}, {where}")
        if count:
            got = _counted(hb, lambda: shape.mul(hb, out, d_ct, d_ct2, level, rescale))
            assert got == shape.launches("mul_relin", level, ntt, rescale=rescale), ("mul_relin", rescale, where, got)
    torch.cuda.synchronize()
    assert torch.equal(d_ct, dev(ct)) and torch.equal(d_ct2, dev(ct2)) and torch.equal(d_diag, dev(diag)), \
        f"an input changed, {where}"


# ------------------------------------------------------------------------------------------------ production sizes
def _production(hb, port, name):
    logn, L, K, alpha, dbits, sbits, levels = plan.HYBRID_SHAPES[name]
    return Shape(hb, port, 1 << logn, L, K, alpha, dbits, sbits, seed=logn * 100 + alpha), levels


def _elts(n):
    """three elements for the hoisted call; the linear transform adds an identity term"""
    return [5, 25, 2 * n - 1], [5, 25, 2 * n - 1, 1]


@pytest.fixture(scope="class")
def production(hb, port, request):
    shape, levels = _production(hb, port, request.param)
    yield shape, levels
    shape.free()


@pytest.mark.parametrize("production", sorted(plan.HYBRID_SHAPES), indirect=True)
class TestProductionShapes:
    def test_all_four_calls_at_each_level(self, hb, port, production):
        shape, levels = production
        elts, lelts = _elts(shape.n)
        for level in levels:
            _all_four(hb, port, shape, level, elts, lelts, seed=level)

    def test_squaring(self, hb, port, production):
        """ct1 = ct2 in both rescale modes, at the first level of the shape"""
        shape, levels = production
        level, n = levels[0], shape.n
        ct = shape.limbs(level, 2, 77)
        d = dev(ct)
        for rescale in (False, True):
            out = _out(2 * (level - int(rescale)) * n)
            shape.mul(hb, out, d, d, level, rescale)
            _check(host(out), shape.exp_mul(port, ct, ct, level, rescale), f"squaring, rescale {rescale}")
        torch.cuda.synchronize()
        assert torch.equal(d, dev(ct))


# ------------------------------------------------------------------------------------------------ every level
@pytest.mark.parametrize("L, K, alpha", [(30, 10, 10), (13, 3, 4)])
def test_every_level(hb, port, L, K, alpha):
    """n = 2^8: every level 1..L crosses the block boundaries of the mod-up's and mod-down's base conversions (at
    (30, 10, 10): levels 19 | 20, 29 | 30 and, with the merged rescale, 28 | 29) and every partial last digit"""
    n = 1 << 8
    shape = Shape(hb, port, n, L, K, alpha, seed=L + K + alpha)
    for level in range(1, L + 1):
        _all_four(hb, port, shape, level, [5, 2 * n - 1], [5, 25, 1], seed=level)


# ------------------------------------------------------------------------------------------------ host batches
@pytest.fixture(scope="module")
def small(hb, port):
    """(7, 3, 3) at n = 2^11, level 5 (a partial last digit), batch 7: inputs and every model output"""
    shape = Shape(hb, port, 1 << 11, 7, 3, 3, seed=11)
    level, batch = 5, 7
    n = shape.n
    ct, ct2 = shape.limbs(level, 2 * batch, 31), shape.limbs(level, 2 * batch, 32)
    res = shape.limbs(level, 2 * batch, 33)
    elts, lelts = [5, 2 * n - 1, 25], [25, 1, 3]
    diag = shape.diagonals(level, len(lelts), 34)
    comp = level * n
    t = np.concatenate([ct[(2 * c + 1) * comp:(2 * c + 2) * comp] for c in range(batch)])
    exp = {"switch": shape.exp_switch(port, res, t, level, batch),
           "hoisted": shape.exp_hoisted(port, ct, level, elts, batch),
           "linear": shape.exp_linear(port, ct, diag, level, lelts, batch)}
    for rescale in (False, True):
        exp["mul", rescale, False] = shape.exp_mul(port, ct, ct2, level, rescale, batch)
        exp["mul", rescale, True] = shape.exp_mul(port, ct, ct, level, rescale, batch)
    return dict(shape=shape, level=level, batch=batch, ct=ct, ct2=ct2, res=res, t=t, elts=elts, lelts=lelts,
                diag=diag, exp=exp)


def _host_call(hb, s, call, batch, rescale=False, square=False):
    """one host-buffer call of `call` on batch ciphertexts of s between sentinel words; returns the output"""
    shape, level, n = s["shape"], s["level"], s["shape"].n
    comp = level * n
    if call == "switch":
        exp = s["exp"]["switch"][:batch * 2 * comp]
    elif call == "mul":
        exp = s["exp"]["mul", rescale, square][:batch * 2 * (level - int(rescale)) * n]
    else:
        exp = s["exp"][call][:batch * (len(s["elts"]) if call == "hoisted" else 1) * 2 * comp]
    buf = np.full(exp.size + 2, SENTINEL, dtype=U64)
    ct, ct2 = s["ct"][:batch * 2 * comp].copy(), s["ct2"][:batch * 2 * comp].copy()
    if call == "switch":
        buf[1:-1] = s["res"][:batch * 2 * comp]
        t = s["t"][:batch * comp].copy()
        shape.switch(hb, buf[1:-1], t, level, batch)
        assert (t == s["t"][:batch * comp]).all(), "the target changed"
    elif call == "hoisted":
        shape.hoisted(hb, buf[1:-1], ct, level, s["elts"], batch)
    elif call == "linear":
        diag = s["diag"].copy()
        shape.linear(hb, buf[1:-1], ct, diag, level, s["lelts"], batch)
        assert (diag == s["diag"]).all(), "the diagonals changed"
    else:
        shape.mul(hb, buf[1:-1], ct, ct if square else ct2, level, rescale, batch)
        assert (ct2 == s["ct2"][:batch * 2 * comp]).all(), "ct2 changed"
    assert (ct == s["ct"][:batch * 2 * comp]).all(), "the ciphertexts changed"
    assert buf[0] == SENTINEL and buf[-1] == SENTINEL, f"{call}: a word next to the output was written"
    return buf[1:-1], exp


@pytest.mark.parametrize("devices", [[], [0, 0], [0, 0, 0]], ids=["one", "split2", "split3"])
@pytest.mark.parametrize("call", ["switch", "hoisted", "linear", "mul", "mul_rescale", "square", "square_rescale"])
def test_host_batch_of_seven(hb, small, call, devices):
    """batch 7: blocks of 7, 3 + 4 and 2 + 2 + 3 ciphertexts, so the 3 staging slots of a device wrap"""
    kind = "mul" if call in ("mul", "mul_rescale", "square", "square_rescale") else call
    try:
        hb.set_host_devices(devices)
        got, exp = _host_call(hb, small, kind, small["batch"], rescale=call.endswith("rescale"),
                              square=call.startswith("square"))
    finally:
        hb.set_host_devices([])
    _check(got, exp, f"{call} over {devices or 'the default device'}")


def test_host_calls_of_different_slot_sizes_in_sequence(hb, port, small):
    """one device, host buffers, batch 4: hoisted G = 1, hoisted G = 5, mul_relin with rescale, the linear transform,
    KeySwitchHybrid and hoisted G = 1 again.  Each call sizes the staging slots for itself; none may read what an
    earlier one left in them."""
    shape, level = small["shape"], small["level"]
    n, comp = shape.n, level * shape.n
    ct = small["ct"][:4 * 2 * comp]

    def hoisted(elts):
        buf = np.full(4 * len(elts) * 2 * comp + 2, SENTINEL, dtype=U64)
        shape.hoisted(hb, buf[1:-1], ct.copy(), level, elts, 4)
        assert buf[0] == SENTINEL and buf[-1] == SENTINEL, "a word next to the output was written"
        return buf[1:-1]

    exp1 = small["exp"]["hoisted"].reshape(7, 3, -1)[:4, :1].ravel()  # 5 is the first of the fixture's elements
    _check(hoisted([5]), exp1, "hoisted G = 1")
    elts5 = [5, 2 * n - 1, 25, 3, 9]
    _check(hoisted(elts5), shape.exp_hoisted(port, ct, level, elts5, 4), "hoisted G = 5")
    for kind, kw in (("mul", dict(rescale=True)), ("linear", {}), ("switch", {})):
        got, exp = _host_call(hb, small, kind, 4, **kw)
        _check(got, exp, kind)
    _check(hoisted([5]), exp1, "hoisted G = 1 again")


def _small_slices(small, c):
    """ciphertext c of the fixture: (ct, ct2, res) and the expected outputs of the four device calls"""
    shape, level = small["shape"], small["level"]
    n, comp = shape.n, small["level"] * shape.n
    exp = small["exp"]
    rows = (2 * comp, 3 * 2 * comp, 2 * comp, 2 * (level - 1) * n)
    return ([x[c * 2 * comp:(c + 1) * 2 * comp] for x in (small["ct"], small["ct2"], small["res"])],
            [e[c * r:(c + 1) * r] for e, r in zip((exp["switch"], exp["hoisted"], exp["linear"],
                                                   exp["mul", True, False]), rows)])


def test_threads_share_keys_pool_caches_and_slots(hb, small):
    """four host threads, each on its own stream, four iterations: the four calls queued on device buffers, then one
    host-buffer call while they run; the threads share the key handle, the scratch pool, the NTT cache and the
    staging slots"""
    shape, level = small["shape"], small["level"]
    comp = level * shape.n
    errors = []

    def worker(t):
        try:
            s = torch.cuda.Stream()
            for i in range(4):
                c = (t + 2 * i) % small["batch"]
                (ct, ct2, res), exp = _small_slices(small, c)
                with torch.cuda.stream(s):
                    a, b, r, d = dev(ct), dev(ct2), dev(res), dev(small["diag"])
                    outs = [r, _out(exp[1].size), _out(exp[2].size), _out(exp[3].size)]
                    shape.switch(hb, r, a[comp:], level, stream=s)
                    shape.hoisted(hb, outs[1], a, level, small["elts"], stream=s)
                    shape.linear(hb, outs[2], a, d, level, small["lelts"], stream=s)
                    shape.mul(hb, outs[3], a, b, level, True, stream=s)
                got, want = _host_call(hb, small, ("hoisted", "mul", "linear", "switch")[(t + i) % 4], 2)
                _check(got, want, f"thread {t} iteration {i}: host call")
                s.synchronize()
                for name, o, e in zip(("switch", "hoisted", "linear", "mul_relin"), outs, exp):
                    _check(host(o), e, f"thread {t} iteration {i}: {name}")
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
    """(6, 2, 2) at level 5 and degree n: inputs and the models of the four calls, built once per degree"""
    if n not in _VIEW_CASES:
        shape = Shape(hb, port, n, 6, 2, 2, seed=n % 1000 + 3)
        level = 5
        comp = level * n
        ct, ct2, res = shape.limbs(level, 2, 41), shape.limbs(level, 2, 42), shape.limbs(level, 2, 43)
        elts, lelts = [5 % (2 * n), 2 * n - 1], [2 * n - 1, 1, 3]
        diag = shape.diagonals(level, len(lelts), 44)
        exp = {"switch": shape.exp_switch(port, res, ct[comp:], level),
               "hoisted": shape.exp_hoisted(port, ct, level, elts),
               "linear": shape.exp_linear(port, ct, diag, level, lelts),
               "mul": shape.exp_mul(port, ct, ct2, level, True)}
        _VIEW_CASES[n] = dict(shape=shape, level=level, ct=ct, ct2=ct2, res=res, elts=elts, lelts=lelts, diag=diag,
                              exp=exp)
    return _VIEW_CASES[n]


def _placed(words, offset, fill=None):
    """a device view of `words` words between guard words, 8 bytes off 16-byte alignment (offset) or aligned"""
    start = 1 if offset else 2
    buf = torch.full((words + 4,), SENTINEL - (1 << 64), dtype=torch.int64, device="cuda")
    if fill is not None:
        buf[start:start + words] = dev(fill)
    view = buf[start:start + words]
    assert (view.data_ptr() % 16 == 8) == offset
    return buf, view, start


def _guarded(buf, start, words):
    h = host(buf)
    return (h[:start] == SENTINEL).all() and (h[start + words:] == SENTINEL).all()


@pytest.mark.parametrize("where", ["input", "result", "both"])
@pytest.mark.parametrize("call", ["switch", "hoisted", "linear", "mul"])
@pytest.mark.parametrize("n", [8, 1 << 12, 1 << 16])
def test_offset_views(hb, port, n, call, where):
    """inputs (target, ciphertexts, ct1 and ct2, diagonals), the result or both 8 bytes off 16-byte alignment, so
    every kernel that reads or writes them takes its word-at-a-time path; inputs come back unchanged and the guard
    words untouched"""
    v = _view_case(hb, port, n)
    shape, level = v["shape"], v["level"]
    comp = level * n
    off_in, off_out = where in ("input", "both"), where in ("result", "both")
    exp = v["exp"][call]
    inputs = {"switch": [v["ct"][comp:]], "hoisted": [v["ct"]], "linear": [v["ct"], v["diag"]],
              "mul": [v["ct"], v["ct2"]]}[call]
    placed = [_placed(x.size, off_in, x) for x in inputs]
    obuf, out, ostart = _placed(exp.size, off_out, v["res"] if call == "switch" else None)
    ins = [p[1] for p in placed]
    if call == "switch":
        shape.switch(hb, out, ins[0], level)
    elif call == "hoisted":
        shape.hoisted(hb, out, ins[0], level, v["elts"])
    elif call == "linear":
        shape.linear(hb, out, ins[0], ins[1], level, v["lelts"])
    else:
        shape.mul(hb, out, ins[0], ins[1], level, True)
    torch.cuda.synchronize()
    _check(host(out), exp, f"{call}, n = {n}, {where} offset")
    assert _guarded(obuf, ostart, exp.size), "a guard word next to the result was written"
    for (buf, view, start), x in zip(placed, inputs):
        assert (host(view) == x).all() and _guarded(buf, start, x.size), "an input or its guard words changed"
