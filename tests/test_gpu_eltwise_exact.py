"""The element-wise kernels and DyadicMultiply on the GPU against exact modular arithmetic (tests/eltwise_exact.py), up
to each operation's own modulus limit:

    MultMod, MultModMulti, DyadicMultiply    q < 2^62 (MultMod: input_mod_factor * q < 2^63)
    AddModMulti, SubModMulti                 q < 2^62
    AddMod, SubMod (vector and scalar)       q < 2^63
    FMAMod                                   q < 2^61
    ReduceMod, CmpSubMod                     any q > 1
    Montgomery forms, r = 62                 odd q < 2^62

The moduli are the primes just below and just above each power of two where the word arithmetic changes, the 62-bit
primes at which a generalised Barrett product with one conditional subtraction is left unreduced, the largest modulus
each operation accepts, and composites.  The operands start with every pair of edge values (0, 1, q - 1, q - 2, the
top of the lazy input range), then a dense band within 2^20 of q, then uniform values.  Every case runs at 1, 7, 4099
and 2^16 + 1 words, through a view 8 bytes off a 16-byte boundary (the scalar instantiation), in place, and with host
pointers.  Canonical outputs are compared word for word; ReduceMod's lazy output must be congruent and below 2q."""
import numpy as np
import pytest

import eltwise_exact as ee

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

LENGTHS = (1, 7, 4099, (1 << 16) + 1)
N = LENGTHS[-1]
W = ee.BARRETT_62_BIT_WITNESSES

MULT_MODULI = [3] + ee.band_moduli((30, 32, 56, 60, 61)) + [ee.prime_below(1 << 62), *W, (1 << 62) - 1,
                                                             *ee.COMPOSITE_MODULI]
ADD_MODULI = [3] + ee.band_moduli((30, 32, 56, 60, 61, 62)) + [ee.prime_below(1 << 63), W[0], (1 << 63) - 1,
                                                                *ee.COMPOSITE_MODULI]
FMA_MODULI = [3] + ee.band_moduli((30, 32, 56, 60)) + [(1 << 61) - 1, *ee.COMPOSITE_MODULI]   # 2^61 - 1 is prime
REDUCE_MODULI = [3] + ee.band_moduli((30, 32, 56, 60, 61, 62, 63)) + [W[0], (1 << 63) + 5, ee.prime_below(1 << 64),
                                                                       (1 << 64) - 1, *ee.COMPOSITE_MODULI]


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64)).to("cuda")


def host(t):
    return t.cpu().numpy().view(np.uint64)


@pytest.fixture(scope="module", autouse=True)
def _need_cuda(hb):
    if not torch.cuda.is_available() or hb.device_count() == 0:
        pytest.fail("gpu-marked test collected on a machine without CUDA")


def _wide_edges(q):
    """64-bit inputs where a Barrett-64 quotient estimate is furthest off: around multiples of q near 2^64"""
    top = ((1 << 64) // q) * q
    return (top - 1, top, top + 1, (1 << 63) - 1, 1 << 63)


def _check(got, exp, q, lazy):
    return ee.wrong_lazy_words(got, exp, q) if lazy else ee.wrong_words(got, exp)


def _shapes(call, ins, exp, q=None, lazy=False, shapes=("lengths", "offset", "in place", "host")):
    """Run `call(result, *operands, n)` on every shape; operands are the words of `ins` (each at least N long), the
    expected words are exp[:n].  Returns one line per shape with wrong words."""
    bad = []

    def verdict(what, got, n):
        w = _check(got, exp[:n], q, lazy)
        if w:
            bad.append(f"{what}: {w} of {n} words wrong")

    if "lengths" in shapes:
        for n in LENGTHS:
            r = torch.empty(n, dtype=torch.int64, device="cuda")
            call(r, *[dev(x[:n]) for x in ins], n)
            verdict(f"device n={n}", host(r), n)
    if "offset" in shapes:   # views 8 bytes off a 16-byte boundary, with a guard word on either side
        bufs = [torch.zeros(N + 2, dtype=torch.int64, device="cuda") for _ in range(len(ins) + 1)]
        for b, x in zip(bufs[1:], ins):
            b[1:N + 1] = dev(x[:N])
        call(bufs[0][1:N + 1], *[b[1:N + 1] for b in bufs[1:]], N)
        got = host(bufs[0])
        verdict(f"offset view n={N}", got[1:N + 1], N)
        if got[0] or got[N + 1]:
            bad.append("offset view: guard word overwritten")
    if "in place" in shapes:
        d = [dev(x[:N]) for x in ins]
        call(d[0], *d, N)
        verdict(f"in place n={N}", host(d[0]), N)
    if "host" in shapes:
        r = np.zeros(N, dtype=np.uint64)
        call(r, *[np.ascontiguousarray(x[:N]) for x in ins], N)
        verdict(f"host pointers n={N}", r, N)
    torch.cuda.synchronize()
    return bad


def _report(bad, what):
    assert not bad, f"{what}:\n" + "\n".join(bad)


# ------------------------------------------------------------------------------------------------------- MultMod
@pytest.mark.parametrize("q", MULT_MODULI, ids=str)
def test_mult_mod(hb, q):
    bad = []
    for in_mf in (1, 2, 4):
        if in_mf * q >= 1 << 63:
            continue
        a, b = ee.operands(q, in_mf * q, 10 * in_mf, N)
        exp = ee.mult_mod(a, b, q)
        bad += [f"in_mf={in_mf} {s}" for s in _shapes(
            lambda r, x, y, n: hb.EltwiseMultMod(r, x, y, n, q, in_mf), (a, b), exp)]
    _report(bad, f"EltwiseMultMod q={q}")


def _rns_operands(moduli, in_mf, per_mod, seed):
    parts = [ee.operands(q, in_mf * q, seed + 100 * i, per_mod) for i, q in enumerate(moduli)]
    return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])


# a witness, a 60-bit prime and a 29-bit prime in one call; below 2^61 for input_mod_factor 4
MULTI_LISTS = {1: [W[0], ee.prime_below(1 << 60), ee.prime_below(1 << 29)],
               2: [W[1], ee.prime_below(1 << 60), ee.prime_below(1 << 29), W[2]],
               4: [(1 << 61) - 1, ee.prime_above(1 << 60), ee.prime_below(1 << 29)]}


@pytest.mark.parametrize("in_mf", sorted(MULTI_LISTS))
@pytest.mark.parametrize("per_mod", [4096, 4099])   # 128-bit and scalar instantiations
def test_mult_mod_multi(hb, in_mf, per_mod):
    moduli = MULTI_LISTS[in_mf]
    assert all(in_mf * q < 1 << 63 for q in moduli)
    a, b = _rns_operands(moduli, in_mf, per_mod, in_mf)
    exp = np.concatenate([ee.mult_mod(a[i * per_mod:(i + 1) * per_mod], b[i * per_mod:(i + 1) * per_mod], q)
                          for i, q in enumerate(moduli)])
    total = per_mod * len(moduli)
    bad = []

    def verdict(what, got):
        for i, q in enumerate(moduli):
            w = ee.wrong_words(got[i * per_mod:(i + 1) * per_mod], exp[i * per_mod:(i + 1) * per_mod])
            if w:
                bad.append(f"{what}, q={q}: {w} of {per_mod} words wrong")

    r = torch.empty(total, dtype=torch.int64, device="cuda")
    hb.EltwiseMultModMulti(r, dev(a), dev(b), per_mod, moduli, in_mf)
    verdict("device", host(r))
    da = dev(a)
    hb.EltwiseMultModMulti(da, da, dev(b), per_mod, moduli, in_mf)
    verdict("in place", host(da))
    bufs = [torch.zeros(total + 1, dtype=torch.int64, device="cuda") for _ in range(3)]
    bufs[1][1:], bufs[2][1:] = dev(a), dev(b)
    hb.EltwiseMultModMulti(bufs[0][1:], bufs[1][1:], bufs[2][1:], per_mod, moduli, in_mf)
    verdict("offset view", host(bufs[0])[1:])
    h = np.zeros(total, dtype=np.uint64)
    hb.EltwiseMultModMulti(h, a, b, per_mod, moduli, in_mf)
    verdict("host pointers", h)
    _report(bad, f"EltwiseMultModMulti in_mf={in_mf} moduli={moduli}")


# the largest prime below 2^62 and the largest modulus accepted (2^62 - 1, composite), a 60-bit, a 29-bit prime and 3
ADDSUB_MULTI_MODULI = [ee.prime_below(1 << 62), (1 << 62) - 1, ee.prime_below(1 << 60), ee.prime_below(1 << 29), 3]


@pytest.mark.parametrize("op", ["add", "sub"])
@pytest.mark.parametrize("per_mod", [4096, 4099])   # 128-bit and scalar instantiations
def test_add_sub_mod_multi(hb, op, per_mod):
    """every edge pair of each modulus (a sum of exactly q, a difference of exactly 0 or -1) in one call"""
    moduli = ADDSUB_MULTI_MODULI
    fn, model = (hb.EltwiseAddModMulti, ee.add_mod) if op == "add" else (hb.EltwiseSubModMulti, ee.sub_mod)
    a, b = _rns_operands(moduli, 1, per_mod, 80 + per_mod % 7)
    exp = np.concatenate([model(a[i * per_mod:(i + 1) * per_mod], b[i * per_mod:(i + 1) * per_mod], q)
                          for i, q in enumerate(moduli)])
    total = per_mod * len(moduli)
    bad = []

    def verdict(what, got):
        for i, q in enumerate(moduli):
            w = ee.wrong_words(got[i * per_mod:(i + 1) * per_mod], exp[i * per_mod:(i + 1) * per_mod])
            if w:
                bad.append(f"{what}, q={q}: {w} of {per_mod} words wrong")

    r = torch.empty(total, dtype=torch.int64, device="cuda")
    fn(r, dev(a), dev(b), per_mod, moduli)
    verdict("device", host(r))
    da = dev(a)
    fn(da, da, dev(b), per_mod, moduli)
    verdict("in place", host(da))
    bufs = [torch.zeros(total + 2, dtype=torch.int64, device="cuda") for _ in range(3)]
    bufs[1][1:-1], bufs[2][1:-1] = dev(a), dev(b)
    fn(bufs[0][1:-1], bufs[1][1:-1], bufs[2][1:-1], per_mod, moduli)
    got = host(bufs[0])
    verdict("offset view", got[1:-1])
    if got[0] or got[-1]:
        bad.append("offset view: guard word overwritten")
    h = np.zeros(total, dtype=np.uint64)
    fn(h, a, b, per_mod, moduli)
    verdict("host pointers", h)
    _report(bad, f"Eltwise{op.capitalize()}ModMulti moduli={moduli}")


# ------------------------------------------------------------------------------------------------ DyadicMultiply
DYADIC_LISTS = {"witnesses": [*W, ee.prime_below(1 << 62), ee.prime_below(1 << 60), ee.prime_below(1 << 29)],
                "below_2_61": [(1 << 61) - 1, ee.prime_above(1 << 60), ee.prime_below(1 << 30), ee.COMPOSITE_MODULI[1]],
                # more moduli than one parameter block: kernel launches and host staging chunks of 64 and 6 moduli
                "seventy": [ee.prime_below((1 << 62) - (i << 55)) for i in range(70)]}


@pytest.mark.parametrize("n", [4096, 4099])
@pytest.mark.parametrize("name", sorted(DYADIC_LISTS))
def test_dyadic_multiply(hb, name, n):
    """all three terms of every modulus, the middle one a sum of two products; result aliasing operand1"""
    moduli = DYADIC_LISTS[name]
    m = len(moduli)
    parts = [[ee.operands(q, q, 1000 * k + 10 * i, n) for i, q in enumerate(moduli)] for k in range(2)]
    # x0 = first operand of part 0, x1 = its second; y0 / y1 from part 1: every term meets the dense band
    op1 = np.concatenate([p[0] for p in parts[0]] + [p[1] for p in parts[0]])
    op2 = np.concatenate([p[1] for p in parts[1]] + [p[0] for p in parts[1]])
    exp = ee.dyadic_multiply(op1, op2, n, moduli)
    bad = []

    def verdict(what, got):
        got = np.asarray(got).reshape(3, m, n)
        for t, term in enumerate(("x0*y0", "x0*y1 + x1*y0", "x1*y1")):
            for i, q in enumerate(moduli):
                w = ee.wrong_words(got[t, i], exp.reshape(3, m, n)[t, i])
                if w:
                    bad.append(f"{what}, {term}, q={q}: {w} of {n} words wrong")

    out = torch.zeros(3 * m * n, dtype=torch.int64, device="cuda")
    hb.DyadicMultiply(out, dev(op1), dev(op2), n, moduli)
    verdict("device", host(out))
    alias = torch.zeros(3 * m * n, dtype=torch.int64, device="cuda")
    alias[:2 * m * n] = dev(op1)
    hb.DyadicMultiply(alias, alias, dev(op2), n, moduli)
    verdict("result aliasing operand1", host(alias))
    bufs = [torch.zeros(k * m * n + 1, dtype=torch.int64, device="cuda") for k in (3, 2, 2)]
    bufs[1][1:], bufs[2][1:] = dev(op1), dev(op2)
    hb.DyadicMultiply(bufs[0][1:], bufs[1][1:], bufs[2][1:], n, moduli)
    verdict("offset view", host(bufs[0])[1:])
    h = np.zeros(3 * m * n, dtype=np.uint64)
    hb.DyadicMultiply(h, op1, op2, n, moduli)
    verdict("host pointers", h)
    _report(bad, f"DyadicMultiply {name}")


# ------------------------------------------------------------------------------------------------ FMAMod
@pytest.mark.parametrize("q", FMA_MODULI, ids=str)
def test_fma_mod(hb, q):
    bad = []
    for in_mf in (1, 2, 4, 8):
        a, c = ee.operands(q, in_mf * q, 20 * in_mf, N)
        top = in_mf * q - 1
        scalars = [top, in_mf * q - 2, q - 1, 0, 1, int(ee.uniform_below(in_mf, 1, in_mf * q)[0])]
        for s in scalars:
            shapes = ("lengths", "offset", "in place", "host") if s == top else ("lengths",)
            exp = ee.fma_mod(a, s, c, q)
            bad += [f"in_mf={in_mf} arg2={s} {x}" for x in _shapes(
                lambda r, x, y, n: hb.EltwiseFMAMod(r, x, s, y, n, q, in_mf), (a, c), exp, shapes=shapes)]
            exp = ee.fma_mod(a, s, None, q)
            bad += [f"in_mf={in_mf} arg2={s} no arg3 {x}" for x in _shapes(
                lambda r, x, n: hb.EltwiseFMAMod(r, x, s, None, n, q, in_mf), (a,), exp, shapes=shapes)]
    _report(bad, f"EltwiseFMAMod q={q}")


# ------------------------------------------------------------------------------------------------ AddMod / SubMod
@pytest.mark.parametrize("q", ADD_MODULI, ids=str)
def test_add_sub_mod(hb, q):
    a, b = ee.operands(q, q, 30, N)
    bad = []
    for name, fn, model in (("add", hb.EltwiseAddMod, ee.add_mod), ("sub", hb.EltwiseSubMod, ee.sub_mod)):
        bad += [f"{name} vector {s}" for s in _shapes(lambda r, x, y, n: fn(r, x, y, n, q), (a, b), model(a, b, q))]
        for s in (q - 1, q - 2, 0, 1, int(b[-1])):
            shapes = ("lengths", "offset", "in place", "host") if s == q - 1 else ("lengths",)
            bad += [f"{name} scalar {s} {x}" for x in _shapes(
                lambda r, x, n: fn(r, x, s, n, q), (a,), model(a, s, q), shapes=shapes)]
    _report(bad, f"EltwiseAddMod / EltwiseSubMod q={q}")


# ------------------------------------------------------------------------------------------------ ReduceMod
@pytest.mark.parametrize("q", REDUCE_MODULI, ids=str)
def test_reduce_mod(hb, q):
    """every input_mod_factor / output_mod_factor pair; input_mod_factor q means any 64-bit word"""
    bad = []
    for in_mf in (q, 2, 4):
        bound = min(q * q if in_mf == q else in_mf * q, 1 << 64)
        x, _ = ee.operands(q, bound, 40 + in_mf % 7, N, edges=_wide_edges(q))
        exp = ee.reduce_mod(x, q)
        for out_mf in (1, 2):
            bad += [f"in_mf={'q' if in_mf == q else in_mf} out_mf={out_mf} {s}" for s in _shapes(
                lambda r, a, n: hb.EltwiseReduceMod(r, a, n, q, in_mf, out_mf), (x,), exp, q, lazy=out_mf == 2)]
    _report(bad, f"EltwiseReduceMod q={q}")


# ------------------------------------------------------------------------------------------------ CmpAdd / CmpSubMod
@pytest.mark.parametrize("q", REDUCE_MODULI, ids=str)
def test_cmp_sub_mod(hb, q):
    x, _ = ee.operands(q, 1 << 64, 50, N, edges=_wide_edges(q))
    bad = []
    for cmp in range(8):
        for bound, diff in ((q, q - 1), (q - 1, 1), (int(x[-1]), max(1, q >> 1))):
            if diff == 0 or diff >= q:
                continue
            shapes = ("lengths", "offset", "in place", "host") if (bound, diff) == (q, q - 1) else ("lengths",)
            exp = ee.cmp_sub_mod(x, q, cmp, bound, diff)
            bad += [f"cmp={cmp} bound={bound} diff={diff} {s}" for s in _shapes(
                lambda r, a, n: hb.EltwiseCmpSubMod(r, a, n, q, cmp, bound, diff), (x,), exp, shapes=shapes)]
    _report(bad, f"EltwiseCmpSubMod q={q}")


def test_cmp_add(hb):
    """the sum wraps mod 2^64 where the comparison holds"""
    x, _ = ee.operands(1 << 63, 1 << 64, 60, N, edges=((1 << 64) - 1, (1 << 64) - 2, 1 << 62))
    bad = []
    for cmp in range(8):
        for bound, diff in ((1 << 63, (1 << 64) - 1), (0, 1), ((1 << 64) - 1, 1 << 63), (int(x[-1]), 12345)):
            shapes = ("lengths", "offset", "in place", "host") if bound == 1 << 63 else ("lengths",)
            exp = ee.cmp_add(x, cmp, bound, diff)
            bad += [f"cmp={cmp} bound={bound} diff={diff} {s}" for s in _shapes(
                lambda r, a, n: hb.EltwiseCmpAdd(r, a, n, cmp, bound, diff), (x,), exp, shapes=shapes)]
    _report(bad, "EltwiseCmpAdd")


# ------------------------------------------------------------------------------------------------ Montgomery, r = 62
@pytest.mark.parametrize("q", [ee.prime_below(1 << 62), W[0], (1 << 62) - 1, ee.prime_above(1 << 61)], ids=str)
def test_montgomery_r62(hb, q):
    r = 62
    ninv = ee.neg_inv_mod(q, r)
    a, b = ee.operands(q, q, 70, N)
    r2 = pow(1 << r, 2, q)
    bad = [f"mont mult {s}" for s in _shapes(
        lambda res, x, y, n: hb.EltwiseMontReduceMod(res, x, y, n, q, r, ninv), (a, b), ee.mont_mult(a, b, q, r))]
    bad += [f"form in {s}" for s in _shapes(
        lambda res, x, n: hb.EltwiseMontgomeryFormIn(res, x, r2, n, q, r, ninv), (a,), ee.mont_in(a, q, r))]
    bad += [f"form out {s}" for s in _shapes(
        lambda res, x, n: hb.EltwiseMontgomeryFormOut(res, x, n, q, r, ninv), (a,), ee.mont_out(a, q, r))]
    _report(bad, f"Montgomery r=62 q={q}")
