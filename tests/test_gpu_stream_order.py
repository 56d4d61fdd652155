"""Every device-pointer entry point runs in order on the caller's stream.

include/hexl_b200.h promises that a call on device (or managed) pointers is enqueued on `stream` and returns without
synchronising.  A caller produces its inputs on a stream, calls the library on that stream and consumes the result
there, with no device-wide synchronisation in between.  Each test here holds a fresh non-blocking stream back with a
bounded spin kernel, writes the real inputs behind the hold, calls, and reads the result behind the call, all queued on
that stream:

* a call that reads an input before the caller's writes land sees the stale content (zeros here, or out-of-range
  words under the debug checks) and computes another result;
* a call that writes after later work on the stream has read the result leaves the clone with the sentinel the output
  held before.

Both fail deterministically, without repetition.  The table has a row for every device-capable compute entry point,
each with inputs and the output of the model the rest of the suite trusts (the checker's NTT and element-wise
operations, ks_exact, galois_exact, rescale_exact, hoist_exact, hybrid_exact, hybrid_rotation_exact, bsgs_exact,
mul_relin_exact).  Every row also runs on two held streams at once with other inputs on the same handles and keys,
and as a CUDA graph captured on a warm handle and replayed behind a hold.  NTT, an element-wise operation and
KeySwitchHybrid run on managed buffers, with the legacy stream held (the call returns with the result complete) and
with a held stream (the call stays asynchronous).  Under hexl_b200_set_debug(1) the range checks must see the inputs
written behind the hold: valid words written there pass when the stale ones were out of range, and out-of-range words
written there are refused when the stale ones were valid.  A debug call inside a capture is refused and the capture
stays usable.  Key handles uploaded from device tensors written behind a hold hold the written keys."""
from __future__ import annotations

import contextlib
from dataclasses import dataclass
from typing import Callable

import numpy as np
import pytest

import bsgs_exact as bx
import galois_exact as gx
import hoist_exact as hox
import hybrid_exact as hx
import hybrid_rotation_exact as hr
import ks_exact
import mul_relin_exact as mr
import rescale_exact as rx
from eltwise_exact import dyadic_multiply, mont_in, mont_mult, mont_out, neg_inv_mod
from util import uniform_below

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

U64 = np.uint64
N = 1 << 12
SENTINEL = -0x5A5A5A5A5A5A5A5B   # 0xA5A5A5A5A5A5A5A5 as int64: what an output holds before the call
OVERWRITE = 0x3C3C3C3C3C3C3C3C   # what every buffer gets after the result is cloned
HOLD_SECONDS = 0.2
L, K, ALPHA, LEVEL = 6, 2, 2, 5  # the hybrid rows


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=U64).view(np.int64)).to("cuda")


def host(t):
    return t.cpu().numpy().view(U64)


@pytest.fixture(scope="module", autouse=True)
def _need_cuda(hb):
    if not torch.cuda.is_available() or hb.device_count() == 0:
        pytest.fail("gpu-marked test collected on a machine without CUDA")
    yield
    hb.set_debug(False)


@pytest.fixture(scope="module")
def hold_cycles():
    """Spin cycles for a HOLD_SECONDS hold: torch.cuda._sleep counts device clock cycles, timed here against CUDA
    events, and bounded so a slow clock reading cannot make a long hold"""
    probe = 1 << 22
    torch.cuda._sleep(probe)                 # first launch outside the timing
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    torch.cuda._sleep(probe)
    end.record()
    end.synchronize()
    per_second = probe / max(start.elapsed_time(end) / 1e3, 1e-6)
    return int(min(max(per_second * HOLD_SECONDS, 1 << 24), 1 << 30))


def hold(cycles):
    """a bounded spin on the current stream"""
    torch.cuda._sleep(cycles)


@dataclass
class Row:
    """One entry point.  bufs: the content of every buffer the call touches when it is called (inputs real, outputs
    SENTINEL unless the call accumulates into them); reads: the buffers it reads; expected: the model's content of
    the buffers it writes; checked: the reads the debug range checks cover; call(hb, t, stream) calls it on the
    tensors t."""
    name: str
    bufs: dict
    reads: tuple
    expected: dict
    call: Callable
    checked: tuple = ()


def _out(words):
    return np.full(words, SENTINEL & ((1 << 64) - 1), dtype=U64)


def _mods(hb, count=3):
    return [int(q) for q in hb.GeneratePrimes(count, 50, True, N)]


def _poly(seed, mods, per=1):
    """per polynomials under each modulus of mods in turn, canonical"""
    return np.concatenate([uniform_below(seed * 977 + 31 * i + p, N, q) for i, q in enumerate(mods)
                           for p in range(per)])


# ------------------------------------------------------------------------------------------------ the table
def _ntt_rows(hb, port, seed):
    q = _mods(hb, 1)[0]
    mods = _mods(hb)
    x = _poly(seed, [q], 2)
    ntt = hb.GetNTT(N, q)                    # the process-wide handles: both tables share them
    ntts = [hb.GetNTT(N, m) for m in mods]
    xm = _poly(seed + 1, mods)
    ym = _poly(seed + 2, mods)
    fwd = np.concatenate([port.ntt_forward(x[p * N:(p + 1) * N], N, q) for p in range(2)])
    inv = np.concatenate([port.ntt_inverse(x[p * N:(p + 1) * N], N, q) for p in range(2)])
    per = [slice(i * N, (i + 1) * N) for i in range(len(mods))]
    fwd_m = np.concatenate([port.ntt_forward(xm[s], N, m) for s, m in zip(per, mods)])
    inv_m = np.concatenate([port.ntt_inverse(xm[s], N, m) for s, m in zip(per, mods)])
    prod = np.concatenate([port.ntt_inverse(port.mult_mod(port.ntt_forward(xm[s], N, m), port.ntt_forward(ym[s], N, m),
                                                          m), N, m) for s, m in zip(per, mods)])
    return [
        Row("ntt_forward", {"x": x, "r": _out(x.size)}, ("x",), {"r": fwd},
            lambda hb, t, s: ntt.ComputeForward(t["r"], t["x"], 1, 1, stream=s), ("x",)),
        Row("ntt_inverse", {"x": x, "r": _out(x.size)}, ("x",), {"r": inv},
            lambda hb, t, s: ntt.ComputeInverse(t["r"], t["x"], 1, 1, stream=s), ("x",)),
        Row("ntt_forward_multi", {"x": xm, "r": _out(xm.size)}, ("x",), {"r": fwd_m},
            lambda hb, t, s: hb.ComputeForwardMulti(ntts, t["r"], t["x"], stream=s), ("x",)),
        Row("ntt_inverse_multi", {"x": xm, "r": _out(xm.size)}, ("x",), {"r": inv_m},
            lambda hb, t, s: hb.ComputeInverseMulti(ntts, t["r"], t["x"], stream=s), ("x",)),
        Row("poly_multiply_multi", {"a": xm, "b": ym, "r": _out(xm.size)}, ("a", "b"), {"r": prod},
            lambda hb, t, s: hb.PolyMultiplyMulti(ntts, t["r"], t["a"], t["b"], stream=s), ("a", "b")),
    ]


def _eltwise_rows(hb, port, seed):
    q = _mods(hb, 1)[0]
    mods = _mods(hb)
    n = 2 * N
    a, b = uniform_below(seed * 11 + 1, n, q), uniform_below(seed * 11 + 2, n, q)
    wide = uniform_below(seed * 11 + 3, n, 1 << 64)
    am, bm = _poly(seed + 3, mods), _poly(seed + 4, mods)
    scalar, bound, diff = 12345 + seed, q // 2, 977
    r_bits = 62
    nim = neg_inv_mod(q, r_bits)
    r2 = pow(1 << r_bits, 2, q)
    per = [slice(i * N, (i + 1) * N) for i in range(len(mods))]

    def multi(fn):
        return np.concatenate([fn(am[s], bm[s], m) for s, m in zip(per, mods)])

    def two(name, exp, call, checked=("a", "b")):
        return Row(name, {"a": a, "b": b, "r": _out(n)}, ("a", "b"), {"r": exp}, call, checked)

    def one(name, src, exp, call, checked=("a",)):
        return Row(name, {"a": src, "r": _out(n)}, ("a",), {"r": exp}, call, checked)

    def rns(name, exp, call):
        return Row(name, {"a": am, "b": bm, "r": _out(am.size)}, ("a", "b"), {"r": exp}, call, ("a", "b"))

    dm1, dm2 = _poly(seed + 5, mods, 1), _poly(seed + 6, mods, 1)
    d1 = np.concatenate([dm1, _poly(seed + 7, mods)])
    d2 = np.concatenate([dm2, _poly(seed + 8, mods)])
    return [
        two("eltwise_add_mod", port.add_mod(a, b, q),
            lambda hb, t, s: hb.EltwiseAddMod(t["r"], t["a"], t["b"], n, q, stream=s)),
        two("eltwise_sub_mod", port.sub_mod(a, b, q),
            lambda hb, t, s: hb.EltwiseSubMod(t["r"], t["a"], t["b"], n, q, stream=s)),
        two("eltwise_mult_mod", port.mult_mod(a, b, q),
            lambda hb, t, s: hb.EltwiseMultMod(t["r"], t["a"], t["b"], n, q, 1, stream=s)),
        two("eltwise_fma_mod", port.fma_mod(a, scalar, b, q),
            lambda hb, t, s: hb.EltwiseFMAMod(t["r"], t["a"], scalar, t["b"], n, q, 1, stream=s), ("a", "b")),
        one("eltwise_reduce_mod", wide, port.reduce_mod(wide, q, q, 1),
            lambda hb, t, s: hb.EltwiseReduceMod(t["r"], t["a"], n, q, q, 1, stream=s), ()),
        one("eltwise_cmp_add", a, port.cmp_add(a, hb.CMPINT.LT, bound, diff),
            lambda hb, t, s: hb.EltwiseCmpAdd(t["r"], t["a"], n, hb.CMPINT.LT, bound, diff, stream=s), ()),
        one("eltwise_cmp_sub_mod", a, port.cmp_sub_mod(a, q, hb.CMPINT.NLT, bound, diff),
            lambda hb, t, s: hb.EltwiseCmpSubMod(t["r"], t["a"], n, q, hb.CMPINT.NLT, bound, diff, stream=s), ()),
        rns("eltwise_mult_mod_multi", multi(port.mult_mod),
            lambda hb, t, s: hb.EltwiseMultModMulti(t["r"], t["a"], t["b"], N, mods, stream=s)),
        rns("eltwise_add_mod_multi", multi(port.add_mod),
            lambda hb, t, s: hb.EltwiseAddModMulti(t["r"], t["a"], t["b"], N, mods, stream=s)),
        rns("eltwise_sub_mod_multi", multi(port.sub_mod),
            lambda hb, t, s: hb.EltwiseSubModMulti(t["r"], t["a"], t["b"], N, mods, stream=s)),
        two("eltwise_mont_reduce_mod", mont_mult(a, b, q, r_bits),
            lambda hb, t, s: hb.EltwiseMontReduceMod(t["r"], t["a"], t["b"], n, q, r_bits, nim, stream=s)),
        one("eltwise_montgomery_form_in", a, mont_in(a, q, r_bits),
            lambda hb, t, s: hb.EltwiseMontgomeryFormIn(t["r"], t["a"], r2, n, q, r_bits, nim, stream=s)),
        one("eltwise_montgomery_form_out", a, mont_out(a, q, r_bits),
            lambda hb, t, s: hb.EltwiseMontgomeryFormOut(t["r"], t["a"], n, q, r_bits, nim, stream=s)),
        Row("dyadic_multiply", {"a": d1, "b": d2, "r": _out(3 * len(mods) * N)}, ("a", "b"),
            {"r": dyadic_multiply(d1, d2, N, mods)},
            lambda hb, t, s: hb.DyadicMultiply(t["r"], t["a"], t["b"], N, mods, stream=s)),
    ]


def _key_switch_rows(hb, port, seed, shared):
    case = shared["ks_case"]
    res, tt = ks_exact.ciphertext(case, seed)
    res2, tt2 = ks_exact.ciphertext(case, seed + 50)
    keys = {f"k{j}": k for j, k in enumerate(case.keys)}
    handle = shared["ks_handle"]
    d = case.decomp
    exp = ks_exact.expected(port, case, res, tt)
    exp2 = ks_exact.expected(port, case, res2, tt2)

    def key_switch(hb, t, s):
        hb.KeySwitch(t["res"], t["t"], *case.shape, [t[f"k{j}"] for j in range(d)], case.modswitch, stream=s)

    rows = [
        Row("key_switch", {"res": res, "t": tt, **keys}, ("res", "t", *keys), {"res": exp}, key_switch),
        Row("key_switch_resident", {"res": np.concatenate([res, res2]), "t": np.concatenate([tt, tt2])}, ("res", "t"),
            {"res": np.concatenate([exp, exp2])},
            lambda hb, t, s: hb.KeySwitchResident(t["res"], t["t"], *case.shape, handle, case.modswitch, 2,
                                                  stream=s)),
    ]
    # rescale, both forms, in place (limb L keeps the operand's word, as the model leaves it)
    rmods = shared["ks_case"].mods[:4]
    x = np.concatenate([_poly(seed + 9, rmods), _poly(seed + 10, rmods)])
    for form in (1, 0):
        rows.append(Row(f"divide_and_round_q_last_ntt{form}", {"x": x}, ("x",),
                        {"x": rx.rescale_exact(port, x, N, rmods, 2, bool(form))},
                        lambda hb, t, s, form=form: hb.DivideAndRoundQLast(t["x"], t["x"], N, rmods, 4, 2, bool(form),
                                                                           stream=s), ("x",)))
    # the automorphism, both forms, in place and out of place
    g = 5
    for form in (1, 0):
        exp_g = gx.sigma_ntt(x, N, g) if form else gx.sigma_coef(x, N, g, rmods, 2)
        rows.append(Row(f"apply_galois_ntt{form}_in_place", {"x": x}, ("x",), {"x": exp_g},
                        lambda hb, t, s, form=form: hb.ApplyGalois(t["x"], t["x"], N, rmods, 4, 2, g, bool(form),
                                                                   stream=s), ("x",)))
        rows.append(Row(f"apply_galois_ntt{form}", {"x": x, "r": _out(x.size)}, ("x",), {"r": exp_g},
                        lambda hb, t, s, form=form: hb.ApplyGalois(t["r"], t["x"], N, rmods, 4, 2, g, bool(form),
                                                                   stream=s), ("x",)))
    # rotations with the KeySwitch keys (key_component_count 2)
    ct = np.concatenate([_poly(seed + 11, case.mods[:d]), _poly(seed + 12, case.mods[:d])])
    rows.append(Row("apply_galois_key_switch", {"ct": ct}, ("ct",), {"ct": gx.rotation_exact(port, case, ct, g, 1)},
                    lambda hb, t, s: hb.ApplyGaloisKeySwitch(t["ct"], *case.shape, handle, case.modswitch, g, 1,
                                                             stream=s), ("ct",)))
    elts = [g, 2 * N - 1]
    hoisted = hox.hoisted_exact(port, ct, N, d, case.kms, case.mods, elts, [case.keys] * 2, case.modswitch)
    rows.append(Row("apply_galois_key_switch_hoisted", {"ct": ct, "r": _out(2 * ct.size)}, ("ct",), {"r": hoisted},
                    lambda hb, t, s: hb.ApplyGaloisKeySwitchHoisted(t["r"], t["ct"], *case.shape, [handle] * 2,
                                                                    case.modswitch, elts, 1, stream=s), ("ct",)))
    # fast base conversion, coefficient form: 3 sources to the other 2 moduli of the case
    src, dst = case.mods[:3], case.mods[3:5]
    y = np.concatenate([_poly(seed + 13, src), _poly(seed + 14, src)])
    conv = np.concatenate([hx.fast_base_convert(port, y[p * 3 * N:(p + 1) * 3 * N], N, src, dst) for p in range(2)])
    rows.append(Row("fast_base_convert", {"x": y, "r": _out(2 * 2 * N)}, ("x",), {"r": conv},
                    lambda hb, t, s: hb.FastBaseConvert(t["r"], t["x"], N, src, dst, 2, stream=s), ("x",)))
    return rows


def _hybrid_rows(hb, port, seed, shared):
    mods, keys, handles = shared["hy_mods"], shared["hy_keys"], shared["hy_handles"]
    basis, _ = hr._basis(mods, LEVEL, L, K)
    comp = LEVEL * N
    res = np.concatenate([_poly(seed + 20, mods[:LEVEL]), _poly(seed + 21, mods[:LEVEL])])
    tgt = _poly(seed + 22, mods[:LEVEL])
    ct = np.concatenate([_poly(seed + 23, mods[:LEVEL]), _poly(seed + 24, mods[:LEVEL])])
    ct2 = np.concatenate([_poly(seed + 25, mods[:LEVEL]), _poly(seed + 26, mods[:LEVEL])])
    ks = hx.key_switch_hybrid(port, res, tgt, N, LEVEL, L, K, ALPHA, 2, mods, keys["relin"])
    rows = [Row("key_switch_hybrid", {"res": res, "t": tgt}, ("res", "t"), {"res": ks},
                lambda hb, t, s: hb.KeySwitchHybrid(t["res"], t["t"], N, LEVEL, L, K, ALPHA, 2, mods,
                                                    handles["relin"], 1, stream=s), ("t",))]
    elts = [5, 25]
    hoisted = hr.hoisted_exact(port, ct, N, LEVEL, L, K, ALPHA, mods, elts, [keys[5], keys[25]])
    rows.append(Row("hybrid_hoisted", {"ct": ct, "r": _out(2 * ct.size)}, ("ct",), {"r": hoisted},
                    lambda hb, t, s: hb.ApplyGaloisKeySwitchHybridHoisted(t["r"], t["ct"], N, LEVEL, L, K, ALPHA, mods,
                                                                          [handles[5], handles[25]], elts, 1,
                                                                          stream=s), ("ct",)))
    lt_elts = [1, 5]
    diag = hr.random_diagonals(basis, N, 2, seed + 27)
    lt = hr.linear_transform_exact(port, ct, N, LEVEL, L, K, ALPHA, mods, lt_elts, [None, keys[5]], diag)
    rows.append(Row("linear_transform_hybrid", {"ct": ct, "w": diag, "r": _out(2 * comp)}, ("ct", "w"), {"r": lt},
                    lambda hb, t, s: hb.LinearTransformHybrid(t["r"], t["ct"], N, LEVEL, L, K, ALPHA, mods,
                                                              [None, handles[5]], lt_elts, t["w"], 1, stream=s),
                    ("ct", "w")))
    babies, giants = [1, 5], [1, 25]
    grid = bx.grid_diagonals(basis, N, 2, 2, None, seed + 28)
    wbufs = {f"w{j}{i}": grid[j][i] for j in range(2) for i in range(2)}
    for rescale in (0, 1):
        exp = bx.bsgs_exact(port, ct, N, LEVEL, L, K, ALPHA, mods, babies, [None, keys[5]], giants, [None, keys[25]],
                            grid, bool(rescale))
        rows.append(Row(f"bsgs_rescale{rescale}", {"ct": ct, **wbufs, "r": _out(2 * (LEVEL - rescale) * N)},
                        ("ct", *wbufs), {"r": exp},
                        lambda hb, t, s, rescale=rescale: hb.LinearTransformHybridBSGS(
                            t["r"], t["ct"], N, LEVEL, L, K, ALPHA, mods, [None, handles[5]], babies,
                            [None, handles[25]], giants, [[t["w00"], t["w01"]], [t["w10"], t["w11"]]], bool(rescale),
                            1, stream=s), ("ct", *wbufs)))
    for rescale in (0, 1):
        exp = mr.multiply_relinearize(port, ct, ct2, N, LEVEL, L, K, ALPHA, mods, keys["relin"], bool(rescale))
        rows.append(Row(f"mul_relin_rescale{rescale}", {"a": ct, "b": ct2, "r": _out(2 * (LEVEL - rescale) * N)},
                        ("a", "b"), {"r": exp},
                        lambda hb, t, s, rescale=rescale: hb.MultiplyRelinearizeHybrid(
                            t["r"], t["a"], t["b"], N, LEVEL, L, K, ALPHA, mods, handles["relin"], bool(rescale), 1,
                            stream=s), ("a", "b")))
    sq = mr.multiply_relinearize(port, ct, ct, N, LEVEL, L, K, ALPHA, mods, keys["relin"], True)
    rows.append(Row("mul_relin_square", {"a": ct, "r": _out(2 * (LEVEL - 1) * N)}, ("a",), {"r": sq},
                    lambda hb, t, s: hb.MultiplyRelinearizeHybrid(t["r"], t["a"], t["a"], N, LEVEL, L, K, ALPHA, mods,
                                                                  handles["relin"], True, 1, stream=s), ("a",)))
    return rows


@pytest.fixture(scope="module")
def shared(hb, port):
    """moduli, keys and key handles every row of one table shares"""
    case = ks_exact.make_case(port, "uniform", N)
    primes = [int(q) for q in port.generate_primes(K + 128, 50, True, N)]
    hy_mods = primes[:L] + primes[-K:]      # L data primes, then K special primes from the far end: all distinct
    hy_keys = {name: hx.random_keys(hy_mods, N, L, ALPHA, 2, 7 + i) for i, name in enumerate(("relin", 5, 25))}
    return {"ks_case": case, "ks_handle": hb.KeySwitchKeys(case.keys, N, case.decomp, case.kms, case.kcc),
            "hy_mods": hy_mods, "hy_keys": hy_keys,
            "hy_handles": {k: hb.KeySwitchKeys(v, N, len(v), L + K, 2) for k, v in hy_keys.items()}}


def _table(hb, port, shared, seed):
    return (_ntt_rows(hb, port, seed) + _eltwise_rows(hb, port, seed) + _key_switch_rows(hb, port, seed, shared)
            + _hybrid_rows(hb, port, seed, shared))


@pytest.fixture(scope="module")
def table(hb, port, shared):
    """the rows, each called once on the default stream first: handles, tables, pools and kernel attributes are warm
    before any hold, and every row equals its model"""
    rows = {r.name: r for r in _table(hb, port, shared, 1)}
    for row in rows.values():
        t = {k: dev(v) for k, v in row.bufs.items()}
        row.call(hb, t, None)
        torch.cuda.synchronize()
        for k, exp in row.expected.items():
            _check(host(t[k]), exp, f"{row.name} (warm-up)")
    return rows


@pytest.fixture(scope="module")
def table2(hb, port, shared, table):
    """the same rows on other inputs, for the two-stream test"""
    return {r.name: r for r in _table(hb, port, shared, 2)}


ROW_NAMES = (
    ["ntt_forward", "ntt_inverse", "ntt_forward_multi", "ntt_inverse_multi", "poly_multiply_multi"]
    + ["eltwise_add_mod", "eltwise_sub_mod", "eltwise_mult_mod", "eltwise_fma_mod", "eltwise_reduce_mod",
       "eltwise_cmp_add", "eltwise_cmp_sub_mod", "eltwise_mult_mod_multi", "eltwise_add_mod_multi",
       "eltwise_sub_mod_multi", "eltwise_mont_reduce_mod", "eltwise_montgomery_form_in",
       "eltwise_montgomery_form_out", "dyadic_multiply"]
    + ["key_switch", "key_switch_resident", "divide_and_round_q_last_ntt1", "divide_and_round_q_last_ntt0",
       "apply_galois_ntt1_in_place", "apply_galois_ntt1", "apply_galois_ntt0_in_place", "apply_galois_ntt0",
       "apply_galois_key_switch", "apply_galois_key_switch_hoisted", "fast_base_convert"]
    + ["key_switch_hybrid", "hybrid_hoisted", "linear_transform_hybrid", "bsgs_rescale0", "bsgs_rescale1",
       "mul_relin_rescale0", "mul_relin_rescale1", "mul_relin_square"])
DEBUG_ROWS = [r for r in ROW_NAMES if r not in ("eltwise_reduce_mod", "eltwise_cmp_add", "eltwise_cmp_sub_mod",
                                                 "dyadic_multiply", "key_switch", "key_switch_resident")]


def _check(got, exp, what):
    bad = int((np.asarray(got, dtype=U64) != np.asarray(exp, dtype=U64)).sum())
    assert bad == 0, f"{what}: {bad} of {np.asarray(exp).size} words differ"


def _stale(row, mode):
    """what the read buffers hold before the hold ends: zeros, or under the debug modes out-of-range words in the
    checked buffers ("valid": the real words are valid) or the real words ("refuse": the real words are not)"""
    out = {}
    for k in row.reads:
        if mode == "valid" and k in row.checked:
            out[k] = np.full(row.bufs[k].size, (1 << 64) - 1, dtype=U64)
        elif mode == "refuse":
            out[k] = row.bufs[k]
        else:
            out[k] = np.zeros_like(row.bufs[k])
    return out


def _real(row, mode):
    """what is written behind the hold: the row's inputs, with one word out of range to refuse (the first of the
    first checked buffer: a check that reads its first limb early and the others late still misses it)"""
    out = {k: row.bufs[k] for k in row.reads}
    if mode == "refuse":
        bad = row.bufs[row.checked[0]].copy()
        bad[0] = U64((1 << 64) - 1)
        out[row.checked[0]] = bad
    return out


def _upload(row, mode=None):
    """the row's buffers holding the stale content, and the real inputs in buffers of their own"""
    stale = _stale(row, mode)
    t = {k: dev(stale.get(k, v)) for k, v in row.bufs.items()}
    return t, {k: dev(v) for k, v in _real(row, mode).items()}


def _hold_and_copy(t, src, s, cycles):
    """s held, then the real inputs copied behind the hold (the uploads are complete before this is called)"""
    with torch.cuda.stream(s):
        hold(cycles)
        for k, v in src.items():
            t[k].copy_(v)


def _stage(row, s, cycles, mode=None):
    """_upload, wait for it, then _hold_and_copy on s"""
    t, src = _upload(row, mode)
    torch.cuda.synchronize()
    _hold_and_copy(t, src, s, cycles)
    return t, src


def _finish(row, t, s):
    """clone the outputs behind the call on s, overwrite every buffer, wait for s only; the clones on the host"""
    with torch.cuda.stream(s):
        clones = {k: t[k].clone() for k in row.expected}
        for v in t.values():
            v.fill_(OVERWRITE)
    s.synchronize()
    return {k: host(v) for k, v in clones.items()}


@pytest.mark.parametrize("name", ROW_NAMES)
def test_held_stream(hb, table, hold_cycles, name):
    """inputs written behind a hold are the ones read, the call does not wait, and the result is complete before the
    next work on the stream"""
    row = table[name]
    s = torch.cuda.Stream()
    t, src = _stage(row, s, hold_cycles)
    row.call(hb, t, s)
    waited = s.query()
    got = _finish(row, t, s)
    assert not waited, f"{name}: the call waited for its stream"
    for k, exp in row.expected.items():
        _check(got[k], exp, name)


@pytest.mark.parametrize("name", ROW_NAMES)
def test_two_held_streams(hb, table, table2, hold_cycles, name):
    """two held streams call the same handles and keys on different inputs, both calls queued while both streams are
    still held, so the two calls run on the device at the same time: neither sees the other's scratch or tables"""
    rows = (table[name], table2[name])
    streams = (torch.cuda.Stream(), torch.cuda.Stream())
    staged = [_upload(r) for r in rows]
    torch.cuda.synchronize()                 # the uploads only: no hold is queued yet
    for s, (t, src) in zip(streams, staged):
        _hold_and_copy(t, src, s, hold_cycles)
    for r, s, (t, _) in zip(rows, streams, staged):
        r.call(hb, t, s)
    held = [not s.query() for s in streams]
    got = [_finish(r, t, s) for r, s, (t, _) in zip(rows, streams, staged)]
    assert all(held), f"{name}: a stream was no longer held when both calls were queued ({held})"
    for i, (r, g) in enumerate(zip(rows, got)):
        for k, exp in r.expected.items():
            _check(g[k], exp, f"{name} on stream {i + 1}")


@pytest.mark.parametrize("name", ROW_NAMES)
def test_graph_replay_behind_a_hold(hb, table, hold_cycles, name):
    """captured once on warm handles (on stale buffers), replayed on a held stream after the real inputs land"""
    row = table[name]
    t = {k: dev(v) for k, v in _stale(row, None).items()}
    for k, v in row.bufs.items():
        t.setdefault(k, dev(v))
    src = {k: dev(v) for k, v in _real(row, None).items()}
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        row.call(hb, t, None)
    for k, v in row.bufs.items():        # the capture ran nothing: restore the outputs' sentinel
        if k not in row.reads:
            t[k].copy_(dev(v))
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        hold(hold_cycles)
        for k, v in src.items():
            t[k].copy_(v)
        g.replay()
    got = _finish(row, t, s)
    for k, exp in row.expected.items():
        _check(got[k], exp, f"{name} (graph)")


@pytest.mark.parametrize("name", DEBUG_ROWS)
@pytest.mark.parametrize("mode", ["valid", "refuse"])
def test_debug_checks_read_on_the_stream(hb, table, hold_cycles, name, mode):
    """hexl_b200_set_debug(1): the range checks see what was written behind the hold.  valid: the stale words are out
    of range, the written ones valid, and the call passes with the model's result.  refuse: the stale words are valid,
    the written ones not, and the call is refused.  The checks may wait for the stream, so nothing is asserted about
    s.query() here."""
    row = table[name]
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
        assert e.value.code == -1 and "exceeds" in str(e.value), e.value
        return
    got = _finish(row, t, s)
    for k, exp in row.expected.items():
        _check(got[k], exp, f"{name} (debug)")


@pytest.mark.parametrize("name", ["ntt_forward", "eltwise_add_mod", "key_switch_hybrid", "fast_base_convert"])
def test_debug_call_inside_a_capture_is_refused(hb, table, name):
    """a range check cannot wait for a stream that is being captured: the call is refused with a message naming the
    capture, nothing is queued, and the capture stays valid (the same call without debug checks is captured and
    replays to the model's result)"""
    row = table[name]
    t = {k: dev(v) for k, v in row.bufs.items()}
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        g.capture_begin()
        try:
            hb.set_debug(True)
            try:
                with pytest.raises(hb.HexlB200Error) as e:
                    row.call(hb, t, None)
            finally:
                hb.set_debug(False)
            row.call(hb, t, None)
        except BaseException:
            with contextlib.suppress(Exception):
                g.capture_end()          # end the capture whatever happened: later work must not be captured
            raise
        g.capture_end()
    assert e.value.code == -1 and "captured" in str(e.value), e.value
    g.replay()
    torch.cuda.synchronize()
    for k, exp in row.expected.items():
        _check(host(t[k]), exp, f"{name} (captured after the refusal)")


@pytest.mark.parametrize("name", ["ntt_forward", "eltwise_add_mod", "key_switch_hybrid"])
def test_managed_buffers(hb, table, hold_cycles, name):
    """managed buffers: with stream None the call returns with the result complete even while the legacy stream is
    held (the host reads it without a sync); with a held stream the call stays asynchronous"""
    row = table[name]
    arrays = {k: hb.managed_empty(v.size) for k, v in row.bufs.items()}
    try:
        for k, v in row.bufs.items():
            arrays[k][:] = v
        torch.cuda.synchronize()
        with torch.cuda.stream(torch.cuda.default_stream()):
            hold(hold_cycles)
        row.call(hb, arrays, None)
        for k, exp in row.expected.items():
            _check(arrays[k], exp, f"{name} (managed, stream None)")
        torch.cuda.synchronize()
        for k, v in row.bufs.items():
            arrays[k][:] = v
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            hold(hold_cycles)
        row.call(hb, arrays, s)
        waited = s.query()
        s.synchronize()
        assert not waited, f"{name}: the managed call on a stream waited for it"
        for k, exp in row.expected.items():
            _check(arrays[k], exp, f"{name} (managed, held stream)")
    finally:
        torch.cuda.synchronize()
        for a in arrays.values():
            hb.managed_free(a)


@pytest.mark.parametrize("kind", ["plain", "hybrid", "sharded"])
def test_key_upload_from_tensors_written_behind_a_hold(hb, port, shared, hold_cycles, kind):
    """key tensors written on a held non-blocking stream and handed to KeySwitchKeys at once, with no caller sync:
    the handle holds the written keys, so the next switch equals the model under them"""
    if kind == "hybrid":
        mods, keys = shared["hy_mods"], shared["hy_keys"]["relin"]
        shape = (N, len(keys), L + K, 2)
    else:
        case = shared["ks_case"]
        keys, shape = case.keys, (N, case.decomp, case.kms, case.kcc)
    t = [torch.zeros(k.size, dtype=torch.int64, device="cuda") for k in keys]
    src = [dev(k) for k in keys]
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        hold(hold_cycles)
        for d, v in zip(t, src):
            d.copy_(v)
    try:
        if kind == "sharded":                # two shards on device 0
            hb.set_host_devices([0, 0])
        handle = hb.KeySwitchKeys(t, *shape, sharded_by_modulus=kind == "sharded")
        if kind == "hybrid":
            res = np.concatenate([_poly(40, mods[:LEVEL]), _poly(41, mods[:LEVEL])])
            tgt = _poly(42, mods[:LEVEL])
            exp = hx.key_switch_hybrid(port, res, tgt, N, LEVEL, L, K, ALPHA, 2, mods, keys)
            got = dev(res)
            hb.KeySwitchHybrid(got, dev(tgt), N, LEVEL, L, K, ALPHA, 2, mods, handle, 1)
        else:
            res, tt = ks_exact.ciphertext(case, 43)
            exp = ks_exact.expected(port, case, res, tt)
            # a sharded handle takes host buffers
            got = res.copy() if kind == "sharded" else dev(res)
            hb.KeySwitchResident(got, tt if kind == "sharded" else dev(tt), *case.shape, handle, case.modswitch)
        torch.cuda.synchronize()
    finally:
        hb.set_host_devices([])
        s.synchronize()
    _check(got if kind == "sharded" else host(got), exp, kind)
