"""The evaluator calls where their scratch rounds repeat: MultiplyRelinearizeSumHybrid, InnerSumHybrid, BfvMultiply,
BfvMultiplyRelinearizeHybrid, BgvModSwitch, BgvKeySwitchHybrid, BgvApplyGaloisKeySwitchHybridHoisted and
BgvMultiplyRelinearizeHybrid at production sizes, at every level of each shape.

Every output is compared bit for bit with the exact models (tests/mul_relin_sum_exact.py, inner_sum_exact.py,
bfv_exact.py, bgv_exact.py), every counted device call's launches with the plan of tests/composite_plan.py, and every
input must come back unchanged:
    HYBRID_SHAPES   each entry at each of its levels (test_composite_plan.py asserts what each name holds): the
                    mod-ups at rounds 34 + 6 (budget_a2), the level-28 round mixing data limbs with special primes
                    (budget_a3, N = 2^17), the multiply-accumulate in 16 + 8 digit launches (mixed_chunks), the BGV
                    mod-downs in t-corrected blocks (27 + 3 from 10 sources, 25 + 4 merged) and the BFV switch's
                    coefficient-form mod-up and mod-down; the sum of 2 and of 33 products (two tensor-sum chunks), the
                    inner sum of 7 rotations (bit 1 runs the doubling and the shift in one mod-up, their products a
                    pstride apart in every round) and of 16
    RESCALE_SHAPES  BgvModSwitch in both forms, out of place between guard words and in place: chunks of 16 + 16 + 3
                    polynomials at N = 2^16, and 31 + 2 at N = 2^14 with two parameter blocks of moduli each
    BEHZ_TILES      BFV at n = 2^12 with l = k = 64: every 32-slot tile full, 64 sources in both conversions of the
                    scaling, the tensor in blocks of 64 + 64 + 1 moduli
    host batch      4 ciphertexts of budget_a2 at level 30 through the 3 staging slots (one ciphertext each)
The models run in a thread pool while the GPU calls run: the C restatement releases the interpreter lock.  One key set
per shape (about 0.6 GB at the budget shapes) serves every call and element, and is freed with its shape."""
import gc
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import bfv_exact as bfx
import bgv_exact as bgx
import composite_plan as plan
import inner_sum_exact as ix
import mul_relin_sum_exact as mrs
import rescale_exact as rx
from test_gpu_hybrid_key_switch import SENTINEL, dev, host
from test_gpu_hybrid_rounds import Shape, _check, _counted, _ntt, _out

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

U64 = np.uint64
TAU = 65537               # BGV's plain modulus; 2^61 - 1 too at mixed_chunks
T_BFV = 65537
GUARD = 64                # words on each side of an output


@pytest.fixture(scope="module", autouse=True)
def _need_cuda(hb):
    if not torch.cuda.is_available() or hb.device_count() == 0:
        pytest.fail("gpu-marked test collected on a machine without CUDA")


def _pool():
    return ThreadPoolExecutor(max_workers=max(1, min(8, os.cpu_count() or 1)))


def behz_bases(port, n, Q, t, avoid):
    """(B, m_sk) by SEAL's rule (bfv_exact.seal_bases), drawn disjoint from Q and from `avoid` (the special primes,
    which at mixed_chunks are 60-bit primes like SEAL's B)"""
    k = bfx.seal_base_b_size(Q, t)
    avoid = set(avoid) | set(Q)
    primes = [int(p) for p in port.generate_primes(k + 1 + len(avoid), 60, True, n) if int(p) not in avoid][:k + 1]
    B, m_sk = primes[:k], primes[k]
    assert not (set(B) | {m_sk}) & avoid and bfx.bound_holds(n, t, Q, B, m_sk)
    return B, m_sk


class Evaluator(Shape):
    """Shape with the evaluator calls; ciphertexts are canonical limbs (NTT form for CKKS and BGV, coefficient form for
    BFV: the calls do not look at the difference)"""

    def bases(self, port, level):
        return behz_bases(port, self.n, self.mods[:level], T_BFV, self.mods[self.L:])

    # the calls
    def mul_sum(self, hb, out, ct1s, ct2s, level, rescale, batch=1):
        hb.MultiplyRelinearizeSumHybrid(out, ct1s, ct2s, self.n, level, self.L, self.K, self.alpha, self.mods,
                                        self.handle, rescale, batch)

    def inner_sum(self, hb, out, ct, level, g, k, rescale):
        elts = ix.needed_elements(g, k, self.n)
        hb.InnerSumHybrid(out, ct, self.n, level, self.L, self.K, self.alpha, self.mods, g, k,
                          [self.handle] * len(elts), elts, rescale)

    def bgv_switch(self, hb, out, t, level, tau):
        hb.BgvKeySwitchHybrid(out, t, self.n, level, self.L, self.K, self.alpha, 2, self.mods, tau, self.handle)

    def bgv_hoisted(self, hb, out, ct, level, elts, tau):
        hb.BgvApplyGaloisKeySwitchHybridHoisted(out, ct, self.n, level, self.L, self.K, self.alpha, self.mods, tau,
                                                [self.handle] * len(elts), elts)

    def bgv_mul(self, hb, out, a, b, level, tau, ms, batch=1):
        hb.BgvMultiplyRelinearizeHybrid(out, a, b, self.n, level, self.L, self.K, self.alpha, self.mods, tau,
                                        self.handle, ms, batch)

    def bfv_mul(self, hb, out, a, b, level, bases, batch=1):
        hb.BfvMultiply(out, a, b, self.n, self.mods, level, bases[0], bases[1], T_BFV, batch)

    def bfv_relin(self, hb, out, a, b, level, bases, batch=1):
        hb.BfvMultiplyRelinearizeHybrid(out, a, b, self.n, level, self.L, self.K, self.alpha, self.mods, bases[0],
                                        bases[1], T_BFV, self.handle, batch)

    # the models of one ciphertext or pair
    def exp_inner_sum(self, port, ct, level, g, k, rescale):
        keys = {e: self.keys for e in ix.needed_elements(g, k, self.n)}
        return ix.inner_sum_exact(port, ct, self.n, level, self.L, self.K, self.alpha, self.mods, g, k, keys, rescale)

    def exp_bgv_mul(self, port, a, b, level, tau, ms):
        return bgx.multiply_relinearize(port, a, b, self.n, level, self.L, self.K, self.alpha, self.mods, self.keys,
                                        tau, ms)

    def exp_bfv(self, port, a, b, level, bases):
        """(BfvMultiply's d, BfvMultiplyRelinearizeHybrid's output)"""
        d = bfx.bfv_multiply(port, a, b, self.n, self.mods[:level], bases[0], bases[1], T_BFV)
        return d, bfx.relinearize(port, d, self.n, level, self.L, self.K, self.alpha, self.mods, self.keys)


class Runs:
    """Calls on device buffers and their models: add() submits the model to the pool at once; check() then runs each
    call into a fresh output (or a copy of `init`, for the calls that add into it), compares it with its model, and
    counts the launches of a second run against `launches`"""

    def __init__(self, pool):
        self.pool, self.items = pool, []

    def add(self, what, words, call, model, launches, init=None):
        self.items.append((what, words, call, self.pool.submit(model), launches, init))

    def check(self, hb):
        for what, words, call, fut, launches, init in self.items:
            out = _out(words) if init is None else dev(init)
            call(out)
            got = host(out)
            count = _counted(hb, lambda: call(out))
            del out
            _check(got, fut.result(), what)
            assert count == launches, (what, count, launches)
        self.items.clear()


def _run_level(hb, port, shape, level, seed, taus, first):
    """every call of the file at one level; `first`: the level where k = 16 and the squared BFV pair run too"""
    n, comp = shape.n, level * shape.n
    ntt = _ntt(hb, n)
    where = f"n = {n}, ({shape.L}, {shape.K}, {shape.alpha}), level {level}"
    pool_ct = [shape.limbs(level, 2, seed + j) for j in range(5)]
    d_pool = [dev(c) for c in pool_ct]
    t = shape.limbs(level, 1, seed + 50)
    res = shape.limbs(level, 2, seed + 60)
    d_t = dev(t)
    rescales = (False, True) if level >= 2 else (False,)
    with _pool() as pool:
        runs = Runs(pool)
        # MultiplyRelinearizeSumHybrid: pair 0 squared; with 33 pairs, pair 32 (the second chunk's) differs from pair 0
        for k in (2, 33):
            idx = [(0, 0)] + [(r % 5, (r // 5 + r) % 5) for r in range(1, k)]
            ct1s, ct2s = [pool_ct[i] for i, _ in idx], [pool_ct[j] for _, j in idx]
            d1s, d2s = [d_pool[i] for i, _ in idx], [d_pool[j] for _, j in idx]
            tensor = pool.submit(mrs.tensor_sum, port, ct1s, ct2s, n, level, shape.mods)
            for rs in rescales:
                runs.add(f"MultiplyRelinearizeSumHybrid k = {k} rescale {rs}, {where}", 2 * (level - rs) * n,
                         lambda out, d1s=d1s, d2s=d2s, rs=rs: shape.mul_sum(hb, out, d1s, d2s, level, rs),
                         lambda tensor=tensor, rs=rs: mrs.relinearize(port, tensor.result(), n, level, shape.L,
                                                                      shape.K, shape.alpha, shape.mods, shape.keys, rs),
                         shape.launches("mul_relin_sum", level, ntt, rescale=rs, pairs=k))
        # InnerSumHybrid, g = 5
        for k in (7, 16) if first else (7,):
            for rs in rescales:
                runs.add(f"InnerSumHybrid k = {k} rescale {rs}, {where}", 2 * (level - rs) * n,
                         lambda out, k=k, rs=rs: shape.inner_sum(hb, out, d_pool[0], level, 5, k, rs),
                         lambda k=k, rs=rs: shape.exp_inner_sum(port, pool_ct[0], level, 5, k, rs),
                         ix.inner_sum_launches(n, level, shape.K, shape.alpha, shape.basis(level), ntt, 5, k, rs))
        # the BGV calls
        elts = [5, 2 * n - 1]
        for tau in taus:
            runs.add(f"BgvKeySwitchHybrid tau {tau}, {where}", 2 * comp,
                     lambda out, tau=tau: shape.bgv_switch(hb, out, d_t, level, tau),
                     lambda tau=tau: bgx.key_switch(port, res, t, n, level, shape.L, shape.K, shape.alpha, 2,
                                                    shape.mods, shape.keys, tau),
                     shape.launches("switch", level, ntt, tau=True), init=res)
            runs.add(f"BgvApplyGaloisKeySwitchHybridHoisted {elts} tau {tau}, {where}", len(elts) * 2 * comp,
                     lambda out, tau=tau: shape.bgv_hoisted(hb, out, d_pool[1], level, elts, tau),
                     lambda tau=tau: bgx.hoisted(port, pool_ct[1], n, level, shape.L, shape.K, shape.alpha,
                                                 shape.mods, elts, [shape.keys] * len(elts), tau),
                     shape.launches("hoisted", level, ntt, elts=len(elts), tau=True))
            for ms in rescales:
                runs.add(f"BgvMultiplyRelinearizeHybrid tau {tau} mod switch {ms}, {where}", 2 * (level - ms) * n,
                         lambda out, tau=tau, ms=ms: shape.bgv_mul(hb, out, d_pool[1], d_pool[2], level, tau, ms),
                         lambda tau=tau, ms=ms: shape.exp_bgv_mul(port, pool_ct[1], pool_ct[2], level, tau, ms),
                         shape.launches("mul_relin", level, ntt, rescale=ms, tau=True))
        # the BFV calls, t = 65537, one squared pair at the first level
        bases = shape.bases(port, level)
        M = level + len(bases[0]) + 1
        for i, j in ((3, 4), (3, 3)) if first else ((3, 4),):
            square = i == j
            model = pool.submit(shape.exp_bfv, port, pool_ct[i], pool_ct[j], level, bases)
            runs.add(f"BfvMultiply square {square}, {where}", 3 * comp,
                     lambda out, i=i, j=j: shape.bfv_mul(hb, out, d_pool[i], d_pool[j], level, bases),
                     lambda model=model: model.result()[0], plan.bfv_launches(M, square, ntt))
            runs.add(f"BfvMultiplyRelinearizeHybrid square {square}, {where}", 2 * comp,
                     lambda out, i=i, j=j: shape.bfv_relin(hb, out, d_pool[i], d_pool[j], level, bases),
                     lambda model=model: model.result()[1],
                     shape.launches("bfv_relin", level, ntt, M=M, square=square))
        runs.check(hb)
    torch.cuda.synchronize()
    assert all(torch.equal(d, dev(c)) for d, c in zip(d_pool, pool_ct)) and torch.equal(d_t, dev(t)), \
        f"an input changed, {where}"


# ------------------------------------------------------------------------------------------------ production sizes
@pytest.fixture(scope="class")
def production(hb, port, request):
    logn, L, K, alpha, dbits, sbits, levels = plan.HYBRID_SHAPES[request.param]
    shape = Evaluator(hb, port, 1 << logn, L, K, alpha, dbits, sbits, seed=logn * 100 + alpha)
    yield request.param, shape, levels
    shape.free()


@pytest.mark.parametrize("production", sorted(plan.HYBRID_SHAPES), indirect=True)
class TestProductionShapes:
    def test_every_call_at_each_level(self, hb, port, production):
        name, shape, levels = production
        taus = (TAU, (1 << 61) - 1) if name == "mixed_chunks" else (TAU,)
        for level in levels:
            _run_level(hb, port, shape, level, seed=level, taus=taus, first=level == levels[0])


# ------------------------------------------------------------------------------------------------ BgvModSwitch
def _mod_switch_model(port, pool, x, n, mods, count, ntt_form):
    """bgv_exact.mod_switch, one future per polynomial"""
    per = len(mods) * n
    futs = [pool.submit(bgx.mod_switch, port, x[p * per:(p + 1) * per], n, mods, 1, ntt_form, TAU)
            for p in range(count)]
    return np.concatenate([f.result() for f in futs])


@pytest.mark.parametrize("ntt_form", [True, False], ids=["ntt", "coef"])
@pytest.mark.parametrize("shape", sorted(plan.RESCALE_SHAPES))
def test_mod_switch_chunks(hb, port, shape, ntt_form):
    """out of place between guard words (limb L of every polynomial left as it was), then in place (limb L keeps the
    operand's); both launch counts against bgv_mod_switch_launches"""
    n, name, limbs, count = plan.RESCALE_SHAPES[shape]
    mods = rx.chain(port.generate_primes, n, name, limbs)
    assert all(np.gcd(q, TAU) == 1 for q in mods)
    x = rx.random_operand(limbs + n + 7, n, mods, count)
    with _pool() as pool:
        exp = _mod_switch_model(port, pool, x, n, mods, count, ntt_form).reshape(count, limbs, n)
    launches = plan.bgv_mod_switch_launches(n, limbs, count, ntt_form, _ntt(hb, n))
    d_in = dev(x)
    buf = torch.full((x.size + 2 * GUARD,), SENTINEL - (1 << 64), dtype=torch.int64, device="cuda")
    out = buf[GUARD:GUARD + x.size]

    def call(o, i):
        hb.BgvModSwitch(o, i, n, mods, limbs, TAU, count, ntt_form)

    call(out, d_in)  # warm: tables and pool
    out.fill_(SENTINEL - (1 << 64))
    got = _counted(hb, lambda: call(out, d_in))
    b = host(buf)
    assert (b[:GUARD] == U64(SENTINEL)).all() and (b[-GUARD:] == U64(SENTINEL)).all(), \
        f"{shape}: a guard word next to the result was written"
    g = b[GUARD:GUARD + x.size].reshape(count, limbs, n)
    bad = [p for p in range(count) if (g[p, :-1] != exp[p, :-1]).any()]
    assert not bad, f"{shape} ntt {ntt_form} out of place: polynomials {bad} differ from the model"
    assert (g[:, -1] == U64(SENTINEL)).all(), f"{shape}: limb L of the result was written"
    assert got == launches, (shape, ntt_form, "out of place", got, launches)
    del buf, out
    assert torch.equal(d_in, dev(x)), f"{shape}: the operand changed"
    got = _counted(hb, lambda: call(d_in, d_in))
    g = host(d_in).reshape(count, limbs, n)
    bad = [p for p in range(count) if (g[p] != exp[p]).any()]
    assert not bad, f"{shape} ntt {ntt_form} in place: polynomials {bad} differ from the model"
    assert got == launches, (shape, ntt_form, "in place", got, launches)


# ------------------------------------------------------------------------------------------------ BEHZ full tiles
def test_behz_full_tiles(hb, port):
    """l = k = 64 at n = 2^12: M = 129 moduli, both conversions of the scaling from 64 sources; a product and a
    square, plain and relinearized (64 data moduli in two 32-modulus digits, two special primes)"""
    logn, l, k = plan.BEHZ_TILES
    n = 1 << logn
    shape = Evaluator(hb, port, n, l, 2, 32, data_bits=58, special_bits=55, seed=129)
    try:
        bsk = [int(p) for p in port.generate_primes(k + 1, 60, True, n)]
        assert not set(bsk) & set(shape.mods)
        bases = (bsk[:k], bsk[k])
        assert bfx.bound_holds(n, T_BFV, shape.mods[:l], *bases)
        ntt = _ntt(hb, n)
        M = l + k + 1
        cts = [shape.limbs(l, 2, 300 + j) for j in range(2)]
        d_cts = [dev(c) for c in cts]
        with _pool() as pool:
            runs = Runs(pool)
            for i, j in ((0, 1), (0, 0)):
                square = i == j
                model = pool.submit(shape.exp_bfv, port, cts[i], cts[j], l, bases)
                runs.add(f"BfvMultiply l = k = 64, square {square}", 3 * l * n,
                         lambda out, i=i, j=j: shape.bfv_mul(hb, out, d_cts[i], d_cts[j], l, bases),
                         lambda model=model: model.result()[0], plan.bfv_launches(M, square, ntt))
                runs.add(f"BfvMultiplyRelinearizeHybrid l = k = 64, square {square}", 2 * l * n,
                         lambda out, i=i, j=j: shape.bfv_relin(hb, out, d_cts[i], d_cts[j], l, bases),
                         lambda model=model: model.result()[1],
                         shape.launches("bfv_relin", l, ntt, M=M, square=square))
            runs.check(hb)
        torch.cuda.synchronize()
        assert all(torch.equal(d, dev(c)) for d, c in zip(d_cts, cts)), "an input changed"
    finally:
        shape.free()


# ------------------------------------------------------------------------------------------------ host batch
def test_host_batch_wraps_the_slots_at_production_size(hb, port):
    """4 ciphertexts of budget_a2 at level 30 in host buffers between sentinel words: one per staging slot, so the
    fourth reuses the first slot's buffers"""
    name, level, batch = plan.EVALUATOR_HOST_BATCH
    logn, L, K, alpha, dbits, sbits, _ = plan.HYBRID_SHAPES[name]
    shape = Evaluator(hb, port, 1 << logn, L, K, alpha, dbits, sbits, seed=logn * 100 + alpha)
    try:
        n = shape.n
        per = 2 * level * n
        ct1, ct2 = shape.limbs(level, 2 * batch, 401), shape.limbs(level, 2 * batch, 402)
        bases = shape.bases(port, level)
        with _pool() as pool:
            bfv = [pool.submit(shape.exp_bfv, port, ct1[c * per:(c + 1) * per], ct2[c * per:(c + 1) * per], level,
                               bases) for c in range(batch)]
            bgv = [pool.submit(shape.exp_bgv_mul, port, ct1[c * per:(c + 1) * per], ct2[c * per:(c + 1) * per],
                               level, TAU, True) for c in range(batch)]
            runs = {"BfvMultiplyRelinearizeHybrid": (batch * per, lambda o, a, b: shape.bfv_relin(hb, o, a, b, level,
                                                                                                bases, batch)),
                    "BgvMultiplyRelinearizeHybrid": (batch * 2 * (level - 1) * n,
                                                     lambda o, a, b: shape.bgv_mul(hb, o, a, b, level, TAU, True,
                                                                                   batch))}
            got = {}
            for what, (words, call) in runs.items():
                buf = np.full(words + 2, SENTINEL, dtype=U64)
                a, b = ct1.copy(), ct2.copy()
                call(buf[1:-1], a, b)
                assert buf[0] == SENTINEL and buf[-1] == SENTINEL, f"{what}: a word next to the output was written"
                assert (a == ct1).all() and (b == ct2).all(), f"{what}: the ciphertexts changed"
                got[what] = buf[1:-1]
            _check(got["BfvMultiplyRelinearizeHybrid"], np.concatenate([f.result()[1] for f in bfv]),
                   f"BfvMultiplyRelinearizeHybrid, host batch {batch}")
            _check(got["BgvMultiplyRelinearizeHybrid"], np.concatenate([f.result() for f in bgv]),
                   f"BgvMultiplyRelinearizeHybrid, host batch {batch}")
    finally:
        shape.free()
        gc.collect()
