"""The RNS composites at production sizes, where one device call runs its scratch rounds more than once
(the rounds are restated in tests/composite_plan.py, which tests/test_composite_plan.py checks against the host sources):

    DivideAndRoundQLast, NTT form    polynomials per round: seal chain at N = 2^16, 31 limbs, 35 polynomials in rounds
                                     of 16, 16 and 3; 70 limbs at 2^14, 33 polynomials in rounds of 31 and 2, each round
                                     with two parameter blocks
    DivideAndRoundQLast, coef. form  the same shapes (no rounds: the production size of the fused kernel)
    ApplyGalois in place             N = 2^16, 31 limbs, 35 polynomials copied into scratch in rounds of 16, 16 and 3
    KeySwitch, KeySwitchResident,    N = 2^16 with 30 digits and N = 2^17 with 29, primes just below 2^61: step 2 runs
    ApplyGaloisKeySwitch             over moduli in rounds of 17 and 14 (8, 8, 8 and 6), and each round's
                                     multiply-accumulate in launches of 16 digits and the rest

Every comparison with the exact models is bit for bit, and every call's launch count shows that the planned number of
rounds ran."""
import numpy as np
import pytest

import composite_plan as plan
import galois_exact as gx
import ks_exact
import rescale_exact as rx
from test_gpu_galois import galois_elt, operand
from util import uniform_below

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

U64 = np.uint64
SENTINEL = 0xA5A5A5A5A5A5A5A5
GUARD = 64  # words: 512 bytes on each side of result
FORMS = [True, False]


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=U64).view(np.int64)).to("cuda")


def host(t):
    return t.cpu().numpy().view(U64)


@pytest.fixture(scope="module", autouse=True)
def _need_cuda(hb):
    if not torch.cuda.is_available() or hb.device_count() == 0:
        pytest.fail("gpu-marked test collected on a machine without CUDA")


def _guarded(size):
    buf = torch.full((size + 2 * GUARD,), SENTINEL - (1 << 64), dtype=torch.int64, device="cuda")
    return buf, buf[GUARD:GUARD + size]


def _guards_intact(buf):
    b = host(buf)
    return (b[:GUARD] == U64(SENTINEL)).all() and (b[-GUARD:] == U64(SENTINEL)).all()


def _launches(hb, fn):
    torch.cuda.synchronize()
    before = hb.launch_count()
    fn()
    torch.cuda.synchronize()
    return hb.launch_count() - before


def _wrong(got, exp):
    return int((np.asarray(got) != exp).sum())


# ---------------------------------------------------------------- DivideAndRoundQLast
@pytest.fixture(scope="module", params=sorted(plan.RESCALE_SHAPES))
def rescale_case(request, port):
    """(name, n, moduli, count, operand, {ntt_form: model result}): one shape at a time"""
    n, name, limbs, count = plan.RESCALE_SHAPES[request.param]
    mods = rx.chain(port.generate_primes, n, name, limbs)
    x = rx.random_operand(limbs + n + 1, n, mods, count)
    return request.param, n, mods, count, x, {}


def _rescale_model(port, case, ntt_form):
    _, n, mods, count, x, models = case
    if ntt_form not in models:
        models.clear()   # one form's model at a time: each is as large as the operand
        models[ntt_form] = rx.rescale_exact(port, x, n, mods, count, ntt_form)
    return models[ntt_form]


def _check_rescale(got, exp, x, n, rns, count, limb_last, what):
    g = np.asarray(got).reshape(count, rns, n)
    e = exp.reshape(count, rns, n)
    bad = [p for p in range(count) if (g[p, :-1] != e[p, :-1]).any()]
    assert not bad, f"{what}: polynomials {bad} differ from the model"
    want = x.reshape(count, rns, n)[:, -1] if limb_last == "operand" else U64(SENTINEL)
    assert (g[:, -1] == want).all(), f"{what}: limb L of result was written"


@pytest.mark.parametrize("ntt_form", FORMS, ids=["ntt", "coef"])
def test_rescale_rounds_equal_model(hb, port, rescale_case, ntt_form):
    shape, n, mods, count, x, _ = rescale_case
    rns = len(mods)
    exp = _rescale_model(port, rescale_case, ntt_form)
    rounds = plan.rescale_rounds(n, rns, count) if ntt_form else [count]
    unit = rns * n
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        d_in = dev(x)
        buf, d_out = _guarded(x.size)
    s.synchronize()

    def call(out, inp, polys):
        hb.DivideAndRoundQLast(out, inp, n, mods, rns, polys, ntt_form, stream=s)

    call(d_out, d_in, count)   # warm: tables and pool
    # one-round calls, then the whole call out of place
    one = {r: _launches(hb, lambda r=r: call(d_out[:r * unit], d_in[:r * unit], r)) for r in sorted(set(rounds))}
    with torch.cuda.stream(s):
        d_out.fill_(SENTINEL - (1 << 64))
    s.synchronize()
    whole = _launches(hb, lambda: call(d_out, d_in, count))
    _check_rescale(host(d_out), exp, x, n, rns, count, "sentinel", f"{shape} out of place")
    assert _guards_intact(buf), f"{shape}: a word next to result was written"
    assert (host(d_in) == x).all(), f"{shape}: the operand was modified"
    del buf, d_out
    assert len(set(one.values())) == 1, f"{shape}: one-round calls launch {one}"
    if ntt_form:
        assert whole == len(rounds) * one[rounds[0]], f"{shape}: {whole} launches, rounds {rounds} of {one}"
    else:
        assert whole == one[count] == (rns - 1 + plan.PARAM_BLOCK - 1) // plan.PARAM_BLOCK, (whole, one)
    # in place
    inplace = _launches(hb, lambda: call(d_in, d_in, count))
    assert inplace == whole, (inplace, whole)
    _check_rescale(host(d_in), exp, x, n, rns, count, "operand", f"{shape} in place")


# ---------------------------------------------------------------- ApplyGalois in place
_galois = {}


def _galois_operand(port):
    if "x" not in _galois:
        n, name, limbs, count = plan.GALOIS_SHAPE
        mods = rx.chain(port.generate_primes, n, name, limbs)
        _galois["x"] = n, mods, count, operand(limbs + 16, n, mods, count)
    return _galois["x"]


@pytest.mark.parametrize("ntt_form", FORMS, ids=["ntt", "coef"])
@pytest.mark.parametrize("gname", ["3", "2n-1", "random"])
def test_apply_galois_in_place_rounds_equal_model(hb, port, gname, ntt_form):
    n, mods, count, x = _galois_operand(port)
    rns, g = len(mods), galois_elt(n, gname)
    rounds = plan.galois_inplace_rounds(n, rns, count)
    exp = gx.sigma_ntt(x, n, g) if ntt_form else gx.sigma_coef(x, n, g, mods, count)
    d_in = dev(x)
    out = torch.empty_like(d_in)
    hb.ApplyGalois(out, d_in, n, mods, rns, count, g, ntt_form)   # warm; out of place is one round's permutation
    one = _launches(hb, lambda: hb.ApplyGalois(out, d_in, n, mods, rns, count, g, ntt_form))
    assert _wrong(host(out), exp) == 0, f"g={g} out of place"
    del out
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        buf, d_io = _guarded(x.size)
        d_io.copy_(d_in)
    s.synchronize()
    del d_in
    inplace = _launches(hb, lambda: hb.ApplyGalois(d_io, d_io, n, mods, rns, count, g, ntt_form, stream=s))
    got = host(d_io).reshape(count, rns * n)
    bad = [p for p in range(count) if (got[p] != exp.reshape(count, rns * n)[p]).any()]
    assert not bad, f"g={g} in place: polynomials {bad} differ from the model (rounds {rounds})"
    assert _guards_intact(buf), "a word next to the in-place buffer was written"
    assert inplace == len(rounds) * one, f"{inplace} launches in place, rounds {rounds} of {one}"


# ---------------------------------------------------------------- KeySwitch at the CKKS shape
class _KsCase:
    """moduli, random keys and two ciphertexts (r_c, t_c) with their exact key switches; everything the GPU calls need
    lives on the device once"""

    def __init__(self, port, logn, decomp):
        n = self.n = 1 << logn
        self.decomp = decomp
        self.mods = [int(q) for q in port.generate_primes(decomp + 1, 60, False, n)]
        kms = decomp + 1
        self.shape = (n, decomp, kms, kms, 2, self.mods)
        self.keys = [np.concatenate([uniform_below(7919 * logn + 1000 * j + 100 * k + i, n, self.mods[i])
                                     for k in range(2) for i in range(kms)]) for j in range(decomp)]
        self.modswitch = [port.inverse_mod(self.mods[-1] % q, q) for q in self.mods[:decomp]]
        self.cts = [ks_exact.ciphertext(self, seed) for seed in (1, 2)]
        # key_switch_exact(r, t) = r + key_switch_exact(0, t), word for word (r canonical): the switch of each t once
        self.switched = [ks_exact.key_switch_exact(port, np.zeros_like(r), t, *self.shape, self.keys, self.modswitch)
                         for r, t in self.cts]

    # ks_exact.ciphertext reads these
    kcc = 2
    digit_factor = 1

    def plus(self, port, r, switched):
        """r + the switched part, limb by limb (component k, limb i under q_i)"""
        n = self.n
        out = np.empty_like(r)
        for k in range(2):
            for i, q in enumerate(self.mods[:self.decomp]):
                sl = slice((k * self.decomp + i) * n, (k * self.decomp + i + 1) * n)
                out[sl] = port.add_mod(r[sl], switched[sl], q)
        return out


@pytest.fixture(scope="module", params=sorted(plan.KS_SHAPES))
def ks_case(request, port):
    logn, decomp = plan.KS_SHAPES[request.param]
    case = _KsCase(port, logn, decomp)
    r, t = case.cts[0]
    # the linearity the expectations rely on, checked on one whole ciphertext
    assert (case.plus(port, r, case.switched[0]) ==
            ks_exact.key_switch_exact(port, r, t, *case.shape, case.keys, case.modswitch)).all()
    yield case
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def test_key_switch_rounds_equal_exact_model(hb, port, ks_case):
    c = ks_case
    (r0, t0), _ = c.cts
    d_keys = [dev(k) for k in c.keys]
    d, d_t = dev(r0), dev(t0)
    hb.KeySwitch(dev(r0), d_t, *c.shape, d_keys, c.modswitch)   # warm: tables and pool
    launches = _launches(hb, lambda: hb.KeySwitch(d, d_t, *c.shape, d_keys, c.modswitch))
    wrong = _wrong(host(d), c.plus(port, r0, c.switched[0]))
    assert wrong == 0, f"n={c.n} decomp={c.decomp}: {wrong} words differ from the exact key switch"
    # the same call with moduli below 2^60, where one launch sums every digit of a round; above 2^60 a round takes
    # two, so the difference is the number of rounds (the transforms are WIDE either way; the values are not checked)
    mods60 = [int(q) for q in port.generate_primes(c.decomp + 1, 59, False, c.n)]
    assert plan.ks_mac_launches(c.decomp, max(mods60)) == [c.decomp]
    mac = plan.ks_mac_launches(c.decomp, max(c.mods))
    ms60 = [port.inverse_mod(mods60[-1] % q, q) for q in mods60[:c.decomp]]
    shape60 = c.shape[:-1] + (mods60,)
    hb.KeySwitch(d, d_t, *shape60, d_keys, ms60)   # warm: tables
    below = _launches(hb, lambda: hb.KeySwitch(d, d_t, *shape60, d_keys, ms60))
    rounds = plan.key_switch_rounds(c.n, c.decomp, c.decomp + 1)
    assert launches - below == len(rounds) * (len(mac) - 1), (launches, below, rounds, mac)


@pytest.mark.parametrize("where", ["device", "host"])
def test_key_switch_resident_rounds_equal_exact_model(hb, port, ks_case, where):
    c = ks_case
    handle = hb.KeySwitchKeys(c.keys, c.n, c.decomp, c.decomp + 1, 2)
    r = np.concatenate([ct[0] for ct in c.cts])
    t = np.concatenate([ct[1] for ct in c.cts])
    exp = np.concatenate([c.plus(port, ct[0], sw) for ct, sw in zip(c.cts, c.switched)])
    if where == "device":
        d = dev(r)
        hb.KeySwitchResident(d, dev(t), *c.shape, handle, c.modswitch, 2)
        got = host(d)
    else:
        got = r.copy()
        hb.KeySwitchResident(got, t, *c.shape, handle, c.modswitch, 2)
    wrong = _wrong(got, exp)
    assert wrong == 0, f"n={c.n} {where} batch 2: {wrong} words differ from the exact key switch"


@pytest.mark.parametrize("g", [3, "2n-1"])
def test_apply_galois_key_switch_rounds_equal_exact_rotation(hb, port, ks_case, g):
    """ciphertext (c0, c1) with c1 = sigma_g^-1(t): the key switch of [sigma(c0), 0] and sigma(c1) = t is
    [sigma(c0), 0] plus the switch of t"""
    c = ks_case
    n, comp = c.n, c.decomp * c.n
    g = 2 * n - 1 if g == "2n-1" else g
    g_inv = pow(g, -1, 2 * n)
    cts, exp = [], []
    for j, (_, t) in enumerate(c.cts):
        c0 = np.concatenate([uniform_below(31 * j + i, n, q) for i, q in enumerate(c.mods[:c.decomp])])
        c1 = gx.sigma_ntt(t, n, g_inv)
        assert (gx.sigma_ntt(c1, n, g) == t).all()
        cts.append(np.concatenate([c0, c1]))
        exp.append(c.plus(port, np.concatenate([gx.sigma_ntt(c0, n, g), np.zeros(comp, dtype=U64)]), c.switched[j]))
    handle = hb.KeySwitchKeys(c.keys, n, c.decomp, c.decomp + 1, 2)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        d = dev(np.concatenate(cts))
        hb.ApplyGaloisKeySwitch(d, *c.shape, handle, c.modswitch, g, 2, stream=s)
    s.synchronize()
    wrong = _wrong(host(d), np.concatenate(exp))
    assert wrong == 0, f"n={n} g={g} batch 2: {wrong} words differ from the exact rotation"
