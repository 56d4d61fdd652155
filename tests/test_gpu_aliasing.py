"""Every buffer aliasing the API allows, against the exact models.

The header lets `result` alias an input, and `PolyMultiplyMulti`'s `result` be a, b or a separate buffer; one buffer
may also be passed as both operands, which is how a caller squares (SEAL's square_inplace is DyadicMultiply with
op1 == op2 == result).  A kernel or a composite that reads an operand after it has written `result`, or transforms one
operand in place before it reads the other, is right in every other test and wrong here.  So each entry point runs
under each aliasing of its result and operands, written as buffer labels (result, operand, operand): "aab" is
result = op1, "raa" is op1 = op2 with a separate result, "aaa" all three one buffer.

    AddMod, SubMod, MultMod (in_mf 1, 2, 4), FMAMod, MontReduceMod   r=op1, r=op2, op1=op2, r=op1=op2
    AddModMulti, SubModMulti, MultModMulti, DyadicMultiply          the same four
    PolyMultiplyMulti                                                separate, r=a, r=b, a=b, r=a=b

through device buffers on a non-default stream (16-byte aligned, between guard words), an 8-byte-offset view (the
scalar instantiation of the element-wise kernels), managed buffers and pageable host buffers.  The element-wise
operands start with every pair of edge values (tests/eltwise_exact.py); AddMod, MultMod and FMAMod also run at 2^22 + 3
words on device buffers, more than one pass of the grid, so threads take a second unrolled tile and then the remainder
loop.  PolyMultiplyMulti runs at every kernel shape its transforms launch: one thread per polynomial (N = 2, 8), row
kernels whose CTAs span moduli (N = 16, 2^9 with one polynomial per modulus), one row kernel (2^13), a column pass
then rows (2^14, 2^16), the pipelined forward of 64 or more polynomials (2^17), two column passes (2^18), and 70
moduli, whose product is multiplied on load from the second parameter block.  Its operands hold polynomials at q - 1,
zeros and ones mixed with q - 1, and uniform values; the unfused chain runs in a subprocess.

Canonical outputs must equal the model word for word; an operand that is not the result must come back unchanged."""
import os
import subprocess
import sys

import numpy as np
import pytest

import eltwise_exact as ee
import ntt_exact as nx
from test_gpu_north_star import PIPE_SPREAD, _multi_mode
from util import uniform_below

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

U64 = np.uint64
N = (1 << 16) + 1
LONG = (1 << 22) + 3   # above the 8 x 132 CTAs x 256 threads x 4 pairs x 2 words = 2.16 M words of one grid pass
W = ee.BARRETT_62_BIT_WITNESSES
SENTINEL = 0x5A5A5A5A5A5A5A5A
KINDS = ("device", "offset", "managed", "host")

# labels of (result, operands): "r" is a result buffer that no operand shares
TWO_OPERAND = {"r=op1": "aab", "r=op2": "bab", "op1=op2": "raa", "r=op1=op2": "aaa"}
PRODUCT = {"separate": "rab", "r=a": "aab", "r=b": "bab", "a=b": "raa", "r=a=b": "aaa"}


@pytest.fixture(scope="module", autouse=True)
def _need_cuda(hb):
    if not torch.cuda.is_available() or hb.device_count() == 0:
        pytest.fail("gpu-marked test collected on a machine without CUDA")


@pytest.fixture(scope="module")
def stream():
    return torch.cuda.Stream()


def _call_aliased(hb, kind, call, roles, values, result_size, stream):
    """Allocate one buffer per distinct label of `roles`, operands holding `values[label]` and the rest SENTINEL, run
    call(*buffers in role order, stream) and return ({label: words before}, {label: words after}, guard errors)."""
    labels = list(dict.fromkeys(roles))
    before = {}
    for lab in labels:
        size = max(result_size if lab == roles[0] else 0, values[lab].size if lab in values else 0)
        before[lab] = np.full(size, SENTINEL, dtype=U64)
        if lab in values:
            before[lab][:values[lab].size] = values[lab]
    if kind == "host":
        bufs = {lab: before[lab].copy() for lab in labels}
        call(*[bufs[lab] for lab in roles], None)
        return before, bufs, []
    if kind == "managed":   # a call without a stream returns with the result complete
        bufs = {lab: hb.managed_empty(before[lab].size) for lab in labels}
        try:
            for lab in labels:
                bufs[lab][:] = before[lab]
            call(*[bufs[lab] for lab in roles], None)
            return before, {lab: bufs[lab].copy() for lab in labels}, []
        finally:
            for b in bufs.values():
                hb.managed_free(b)
    # device buffers on `stream`, between guard words: 2 words keep the view 16-byte aligned, 1 puts it 8 bytes off
    pad = 1 if kind == "offset" else 2
    full, views = {}, {}
    with torch.cuda.stream(stream):
        for lab in labels:
            size = before[lab].size
            full[lab] = torch.zeros(size + 2 * pad, dtype=torch.int64, device="cuda")
            views[lab] = full[lab][pad:pad + size]
            views[lab].copy_(torch.from_numpy(before[lab].view(np.int64)))
        call(*[views[lab] for lab in roles], stream)
    stream.synchronize()
    after, bad = {}, []
    for lab in labels:
        got = full[lab].cpu().numpy().view(U64)
        if got[:pad].any() or got[-pad:].any():
            bad.append(f"guard words of buffer {lab} overwritten")
        after[lab] = got[pad:-pad]
    return before, after, bad


def _aliasings(hb, call, aliasings, values, result_size, expected, stream, kinds=KINDS):
    """Run `call` under every aliasing and pointer kind.  expected(operand labels) -> [(slice of the result, words)].
    Returns one line per wrong result or modified operand."""
    bad = []
    for name, roles in aliasings.items():
        exp = expected(tuple(roles[1:]))
        for kind in kinds:
            before, after, guards = _call_aliased(hb, kind, call, roles, values, result_size, stream)
            bad += [f"{name} {kind}: {g}" for g in guards]
            got = after[roles[0]]
            w = sum(ee.wrong_words(got[sl], e) for sl, e in exp)
            if w:
                bad.append(f"{name} {kind}: {w} of {sum(e.size for _, e in exp)} compared result words wrong")
            for lab in after:
                if lab != roles[0] and (after[lab] != before[lab]).any():
                    bad.append(f"{name} {kind}: operand {lab} modified "
                               f"({int((after[lab] != before[lab]).sum())} words)")
    return bad


def _cached(model, values):
    """expected() of a model over whole buffers: model(*operands), computed once per distinct operand labels"""
    memo = {}

    def expected(ops):
        if ops not in memo:
            e = model(*[values[lab] for lab in ops])
            memo[ops] = [(slice(0, e.size), e)]
        return memo[ops]
    return expected


def _report(bad, what):
    assert not bad, f"{what}:\n" + "\n".join(bad)


def _elementwise(hb, call, model, a, b, n, stream, kinds=KINDS):
    """a two-operand element-wise call(result, x, y, n, stream) on the first n words of a and b"""
    values = {"a": a[:n], "b": b[:n]}
    return _aliasings(hb, lambda r, x, y, s: call(r, x, y, n, s), TWO_OPERAND, values, n, _cached(model, values),
                      stream, kinds)


# ------------------------------------------------------------------------------------------------ element-wise
ADD_MODULI = [ee.prime_below(1 << 63), (1 << 63) - 1, ee.prime_below(1 << 30)]
MULT_MODULI = [W[0], ee.prime_below(1 << 61), ee.prime_below(1 << 30)]   # a 62-bit witness takes the WIDE product
FMA_MODULI = [(1 << 61) - 1, ee.prime_below(1 << 30)]
MONT_MODULI = [ee.prime_below(1 << 62), W[0]]


@pytest.mark.parametrize("q", ADD_MODULI, ids=str)
def test_add_sub_mod(hb, stream, q):
    a, b = ee.operands(q, q, 31, N)
    bad = [f"add {x}" for x in _elementwise(
        hb, lambda r, x, y, n, s: hb.EltwiseAddMod(r, x, y, n, q, stream=s), lambda x, y: ee.add_mod(x, y, q),
        a, b, N, stream)]
    bad += [f"sub {x}" for x in _elementwise(
        hb, lambda r, x, y, n, s: hb.EltwiseSubMod(r, x, y, n, q, stream=s), lambda x, y: ee.sub_mod(x, y, q),
        a, b, N, stream)]
    _report(bad, f"EltwiseAddMod / EltwiseSubMod q={q}")


@pytest.mark.parametrize("q", MULT_MODULI, ids=str)
def test_mult_mod(hb, stream, q):
    bad = []
    for in_mf in (1, 2, 4):
        if in_mf * q >= 1 << 63:
            continue
        a, b = ee.operands(q, in_mf * q, 11 * in_mf, N)
        bad += [f"in_mf={in_mf} {x}" for x in _elementwise(
            hb, lambda r, x, y, n, s: hb.EltwiseMultMod(r, x, y, n, q, in_mf, stream=s),
            lambda x, y: ee.mult_mod(x, y, q), a, b, N, stream)]
    _report(bad, f"EltwiseMultMod q={q}")


@pytest.mark.parametrize("q", FMA_MODULI, ids=str)
def test_fma_mod(hb, stream, q):
    """arg1 and arg3 are the vector operands; arg2 the scalar at the top of the input range"""
    bad = []
    for in_mf in (1, 8):
        top = in_mf * q - 1
        a, c = ee.operands(q, in_mf * q, 21 * in_mf, N)
        bad += [f"in_mf={in_mf} {x}" for x in _elementwise(
            hb, lambda r, x, y, n, s: hb.EltwiseFMAMod(r, x, top, y, n, q, in_mf, stream=s),
            lambda x, y: ee.fma_mod(x, top, y, q), a, c, N, stream)]
    _report(bad, f"EltwiseFMAMod q={q}")


@pytest.mark.parametrize("q", MONT_MODULI, ids=str)
def test_mont_reduce_mod(hb, stream, q):
    r = 62
    ninv = ee.neg_inv_mod(q, r)
    a, b = ee.operands(q, q, 71, N)
    _report(_elementwise(hb, lambda res, x, y, n, s: hb.EltwiseMontReduceMod(res, x, y, n, q, r, ninv, stream=s),
                         lambda x, y: ee.mont_mult(x, y, q, r), a, b, N, stream),
            f"EltwiseMontReduceMod r=62 q={q}")


def test_long_lengths(hb, checker, stream):
    """2^22 + 3 words on device buffers: a second unrolled tile, the remainder loop and the odd tail.  A prime below
    2^60, where tests/test_eltwise_exact.py pins the checker to the exact model."""
    q = ee.prime_below(1 << 60)
    bad = []
    a, b = ee.operands(q, q, 41, LONG)
    bad += [f"add {x}" for x in _elementwise(
        hb, lambda r, x, y, n, s: hb.EltwiseAddMod(r, x, y, n, q, stream=s), lambda x, y: checker.add_mod(x, y, q),
        a, b, LONG, stream, kinds=("device",))]
    for in_mf in (1, 4):
        a, b = ee.operands(q, in_mf * q, 43 + in_mf, LONG)
        bad += [f"mult in_mf={in_mf} {x}" for x in _elementwise(
            hb, lambda r, x, y, n, s: hb.EltwiseMultMod(r, x, y, n, q, in_mf, stream=s),
            lambda x, y: checker.mult_mod(x, y, q, in_mf), a, b, LONG, stream, kinds=("device",))]
    in_mf = 8
    top = in_mf * q - 1
    a, c = ee.operands(q, in_mf * q, 47, LONG)
    bad += [f"fma in_mf={in_mf} {x}" for x in _elementwise(
        hb, lambda r, x, y, n, s: hb.EltwiseFMAMod(r, x, top, y, n, q, in_mf, stream=s),
        lambda x, y: checker.fma_mod(x, top, y, q, in_mf), a, c, LONG, stream, kinds=("device",))]
    _report(bad, f"element-wise at {LONG} words, q={q}")


# ------------------------------------------------------------------------------------------ RNS element-wise
MULTI_LISTS = {1: [W[0], ee.prime_below(1 << 60), ee.prime_below(1 << 29)],
               2: [W[1], ee.prime_below(1 << 60), ee.prime_below(1 << 29)],
               4: [(1 << 61) - 1, ee.prime_above(1 << 60), ee.prime_below(1 << 29)]}
ADDSUB_MULTI_MODULI = [ee.prime_below(1 << 62), (1 << 62) - 1, ee.prime_below(1 << 29), 3]


def _rns(model, moduli, per_mod):
    def run(x, y):
        return np.concatenate([model(x[i * per_mod:(i + 1) * per_mod], y[i * per_mod:(i + 1) * per_mod], q)
                               for i, q in enumerate(moduli)])
    return run


@pytest.mark.parametrize("per_mod", [4096, 4099])   # 128-bit and scalar instantiations
@pytest.mark.parametrize("op", ["add", "sub", "mult1", "mult2", "mult4"])
def test_multi(hb, stream, op, per_mod):
    if op.startswith("mult"):
        in_mf = int(op[-1])
        moduli = MULTI_LISTS[in_mf]
        call = lambda r, x, y, s: hb.EltwiseMultModMulti(r, x, y, per_mod, moduli, in_mf, stream=s)  # noqa: E731
        model = lambda x, y, q: ee.mult_mod(x, y, q)  # noqa: E731
    else:
        in_mf = 1
        moduli = ADDSUB_MULTI_MODULI
        fn, model = (hb.EltwiseAddModMulti, ee.add_mod) if op == "add" else (hb.EltwiseSubModMulti, ee.sub_mod)
        call = lambda r, x, y, s: fn(r, x, y, per_mod, moduli, stream=s)  # noqa: E731
    parts = [ee.operands(q, in_mf * q, 90 + 10 * i + in_mf, per_mod) for i, q in enumerate(moduli)]
    values = {"a": np.concatenate([p[0] for p in parts]), "b": np.concatenate([p[1] for p in parts])}
    total = per_mod * len(moduli)
    _report(_aliasings(hb, call, TWO_OPERAND, values, total, _cached(_rns(model, moduli, per_mod), values), stream),
            f"Eltwise{op}ModMulti per_mod={per_mod} moduli={moduli}")


# ------------------------------------------------------------------------------------------------ DyadicMultiply
DYADIC_CASES = {
    "witnesses_4096": (4096, [*W, ee.prime_below(1 << 62), ee.prime_below(1 << 60), ee.prime_below(1 << 29)]),
    "below_2_61_4099": (4099, [(1 << 61) - 1, ee.prime_above(1 << 60), ee.prime_below(1 << 30),
                               ee.COMPOSITE_MODULI[1]]),
    # two parameter blocks, the 62-bit product only in the second; the API does not require primes
    "70_moduli_256": (256, [ee.prime_below(1 << 60) - 2 * k * 1000003 for k in range(69)] + [W[0]]),
}


@pytest.mark.parametrize("case", sorted(DYADIC_CASES))
def test_dyadic_multiply(hb, stream, case):
    """operands of 2 x moduli x n words, result of 3: with result = op2 and op1 = op2 (squaring) the third term lands
    past the operands' end of the shared buffer"""
    n, moduli = DYADIC_CASES[case]
    m = len(moduli)
    parts = [[ee.operands(q, q, 1000 * k + 10 * i, n) for i, q in enumerate(moduli)] for k in range(2)]
    values = {"a": np.concatenate([p[0] for p in parts[0]] + [p[1] for p in parts[0]]),
              "b": np.concatenate([p[1] for p in parts[1]] + [p[0] for p in parts[1]])}
    _report(_aliasings(hb, lambda r, x, y, s: hb.DyadicMultiply(r, x, y, n, moduli, stream=s), TWO_OPERAND, values,
                       3 * m * n, _cached(lambda x, y: ee.dyadic_multiply(x, y, n, moduli), values), stream),
            f"DyadicMultiply {case}")


# --------------------------------------------------------------------------------------------- PolyMultiplyMulti
# (log2 N, polynomials per modulus); None: the fewest that make 64 polynomials, so the forward is the pipelined kernel
PRODUCT_SHAPES = [(1, 3), (3, 3), (4, 1), (9, 1), (13, 2), (14, 2), (16, 1), (17, None), (18, 1)]
PRODUCT_KINDS = ("device", "managed", "host")


def _product_operands(mods, n, group, seed):
    """polynomial u of modulus i is of kind (i + u) % 3: a and b all at q - 1; a alternating q - 1 with uniform values
    and b half zeros, half ones; or both uniform"""
    a, b = [], []
    for i, q in enumerate(mods):
        for u in range(group):
            x = uniform_below(seed + 2 * (i * group + u), n, q)
            y = uniform_below(seed + 2 * (i * group + u) + 1, n, q)
            kind = (i + u) % 3
            if kind == 0:
                x[:], y[:] = q - 1, q - 1
            elif kind == 1:
                x[::2] = q - 1
                y[:n // 2], y[n // 2:] = 0, 1
            a.append(x)
            b.append(y)
    return np.concatenate(a), np.concatenate(b)


def _product_expected(checker, values, n, mods, group, units):
    """the checker's FwdNTT -> MultMod -> InvNTT of polynomials `units`: a times b, or a squared when a = b"""
    fwd = {(lab, u): checker.ntt_forward(values[lab][u * n:(u + 1) * n], n, mods[u // group])
           for lab in "ab" for u in units}
    memo = {}

    def expected(ops):
        if ops not in memo:
            memo[ops] = []
            for u in units:
                q = mods[u // group]
                e = checker.ntt_inverse(checker.mult_mod(fwd[(ops[0], u)], fwd[(ops[1], u)], q), n, q)
                memo[ops].append((slice(u * n, (u + 1) * n), e))
        return memo[ops]
    return expected


def _product(hb, checker, stream, mods, n, group, units, what):
    ntts = [hb.NTT(n, q) for q in mods]
    a, b = _product_operands(mods, n, group, 7 * n + len(mods))
    values = {"a": a, "b": b}
    bad = _aliasings(hb, lambda r, x, y, s: hb.PolyMultiplyMulti(ntts, r, x, y, group, stream=s), PRODUCT, values,
                     a.size, _product_expected(checker, values, n, mods, group, units), stream, PRODUCT_KINDS)
    _report(bad, what)


@pytest.mark.parametrize("logn,group", PRODUCT_SHAPES, ids=[f"n=2^{s[0]}" for s in PRODUCT_SHAPES])
@pytest.mark.parametrize("name", ["fast_edges", "wide_small"])
def test_poly_multiply_aliasing(hb, checker, stream, name, logn, group):
    """wide_small holds moduli below 2^30, whose host-pointer products take the unfused chain, beside larger ones"""
    n = 1 << logn
    mods = nx.moduli(hb.GeneratePrimes, dict(nx.MODULUS_LISTS)[name])
    assert _multi_mode(mods) == {"fast_edges": "fast", "wide_small": "wide"}[name]
    if group is None:
        group = -(-64 // len(mods))
    units = len(mods) * group
    sample = sorted(set(PIPE_SPREAD) | {units - 1}) if logn == 17 else range(units)
    _product(hb, checker, stream, mods, n, group, sample, f"PolyMultiplyMulti {name} n=2^{logn} group={group}")


def test_poly_multiply_aliasing_70_moduli(hb, checker, stream):
    """moduli 64 to 69 run in a second launch, whose inverse multiplies on load from an offset into the scratch"""
    n, group = 1 << 8, 2
    mods = hb.GeneratePrimes(66, 50, True, n) + hb.GeneratePrimes(4, 29, False, n)
    assert len(set(mods)) == 70
    _product(hb, checker, stream, mods, n, group, range(70 * group), "PolyMultiplyMulti 70 moduli n=2^8")


def test_unfused_poly_multiply_aliasing():
    """HEXL_B200_NO_PRODUCT_FUSION=1 selects the chain of lazy transforms, MultMod kernel and inverse (read once per
    process), so the product tests above run again in a process of their own"""
    here = os.path.abspath(__file__)
    res = subprocess.run([sys.executable, "-m", "pytest", here, "-m", "gpu", "-q", "-p", "no:cacheprovider", "-k",
                          "poly_multiply_aliasing and not unfused"],
                         env={**os.environ, "HEXL_B200_NO_PRODUCT_FUSION": "1"}, capture_output=True, text=True,
                         timeout=900)
    assert res.returncode == 0 and " passed" in res.stdout, res.stdout[-4000:] + res.stderr[-2000:]
