"""DivideAndRoundQLast on the GPU across the domain it accepts, against the integer definition.

    chains       wide (primes just below 2^61, the limit), small (q_L < 2^30: its inverse runs the 32-bit kernels),
                 classes and seal, at n = 2, 4, 8, 16, 32, 2^8, 2^11, 2^12 and 2^17, in both forms, on device and
                 host pointers
    inputs       the rounding edges of rescale_exact.edge_values (X = 0, X = Q - 1, X mod q_L in {h - 1, h, h + 1}),
                 limbs at q_i - 1 with X mod q_L = h + 1, and a uniform polynomial
    coef. form   n = 1, 3 and 4099; q_i in {2, 3}; an even q_L; composite moduli; moduli that share factors with each
                 other (the per-limb formula is the reference there); 70 limbs with q_L the smallest and the largest
    refusals     the arguments the call must reject with HEXL_B200_ERR_INVALID_ARG, without writing anything

The coefficient form is compared with rescale_integer (CRT lift, divide and round) up to n = 2^12 and with
rescale_exact (pinned to it by tests/test_rescale_exact.py) at 2^17.  The NTT-form operand is the forward transform
(the C restatement) of the same coefficient-form polynomials, and its expected result is the forward transform of the
coefficient form's."""
import numpy as np
import pytest

import rescale_exact as rx

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

U64 = np.uint64
SENTINEL = 0xA5A5A5A5A5A5A5A5
CHAINS = ("wide", "small", "classes", "seal")
# 2, 4 and 8: the NTT form's transforms run one thread per polynomial; 16 to 2^11: one row kernel with several
# polynomials per CTA; 2^12 and up: row and column passes
LOGNS = (1, 2, 3, 4, 5, 8, 11, 12, 17)
INTEGER_MAX_N = 1 << 12   # above this, rescale_exact stands in for the Python-integer definition


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=U64).view(np.int64)).to("cuda")


def host(t):
    return t.cpu().numpy().view(U64)


@pytest.fixture(scope="module", autouse=True)
def _need_cuda(hb):
    if not torch.cuda.is_available() or hb.device_count() == 0:
        pytest.fail("gpu-marked test collected on a machine without CUDA")


def edge_operand(mods, n, seed):
    """coefficient form, [count][rns][n]: the edge rows, a row of limbs q_i - 1 with limb L = h + 1, a uniform row"""
    rows = rx.limbs_of(rx.edge_values(mods, n, seed), mods).reshape(-1, len(mods), n)
    top = np.array([[q - 1] * n for q in mods[:-1]] + [[(mods[-1] >> 1) + 1] * n], dtype=U64)[None]
    rand = rx.random_operand(seed + 1, n, mods, 1).reshape(1, len(mods), n)
    return np.concatenate([rows, top, rand])


def forward_limbs(port, x, n, mods, count):
    """the forward transform of every limb"""
    x = np.asarray(x, dtype=U64).reshape(count, len(mods), n)
    return np.stack([np.stack([port.ntt_forward(np.ascontiguousarray(x[p, i]), n, q) for i, q in enumerate(mods)])
                     for p in range(count)]).reshape(-1)


_cache = {}


def _prepared(port, name, logn, ntt_form):
    """(n, moduli, count, operand, expected), one chain and degree at a time"""
    key = (name, logn, ntt_form)
    if key not in _cache:
        _cache.clear()
        n = 1 << logn
        mods = rx.chain(port.generate_primes, n, name)
        coef = edge_operand(mods, n, 17 * logn + len(name))
        count = coef.shape[0]
        coef = coef.reshape(-1)
        if n <= INTEGER_MAX_N:
            exp = rx.rescale_integer(coef, n, mods, count)
        else:
            exp = rx.rescale_exact(port, coef, n, mods, count, ntt_form=False)
        if ntt_form:
            op = forward_limbs(port, coef, n, mods, count)
            exp = forward_limbs(port, exp, n, mods, count).reshape(count, len(mods), n)
            exp[:, -1] = op.reshape(count, len(mods), n)[:, -1]
            coef, exp = op, exp.reshape(-1)
        _cache[key] = n, mods, count, coef, exp
    return _cache[key]


def _check(got, exp, x, n, mods, count, limb_last, what):
    rns = len(mods)
    g, e = np.asarray(got).reshape(count, rns, n), exp.reshape(count, rns, n)
    bad = [(p, i) for p in range(count) for i in range(rns - 1) if (g[p, i] != e[p, i]).any()]
    assert not bad, f"{what}: (polynomial, limb) {bad[:8]} differ from the integer definition"
    want = x.reshape(count, rns, n)[:, -1] if limb_last == "operand" else U64(SENTINEL)
    assert (g[:, -1] == want).all(), f"{what}: limb L of result was written"


def _run(hb, where, x, n, mods, count, ntt_form):
    """out of place into a sentinel-filled result, and in place"""
    rns = len(mods)
    if where == "device":
        s = torch.cuda.Stream()
        with torch.cuda.stream(s):
            d_in, d_out = dev(x), dev(np.full(x.size, SENTINEL, dtype=U64))
            hb.DivideAndRoundQLast(d_out, d_in, n, mods, rns, count, ntt_form, stream=s)
            hb.DivideAndRoundQLast(d_in, d_in, n, mods, rns, count, ntt_form, stream=s)
        s.synchronize()
        return host(d_out), host(d_in)
    out = np.full(x.size, SENTINEL, dtype=U64)
    hb.DivideAndRoundQLast(out, x, n, mods, rns, count, ntt_form)
    io = x.copy()
    hb.DivideAndRoundQLast(io, io, n, mods, rns, count, ntt_form)
    return out, io


@pytest.mark.parametrize("where", ["device", "host"])
@pytest.mark.parametrize("ntt_form", [True, False], ids=["ntt", "coef"])
@pytest.mark.parametrize("logn", LOGNS)
@pytest.mark.parametrize("name", CHAINS)
def test_chains_and_rounding_edges(hb, port, name, logn, ntt_form, where):
    n, mods, count, x, exp = _prepared(port, name, logn, ntt_form)
    out, io = _run(hb, where, x, n, mods, count, ntt_form)
    what = f"{name} n={n} {'ntt' if ntt_form else 'coef'} {where}"
    _check(out, exp, x, n, mods, count, "sentinel", what + " out of place")
    _check(io, exp, x, n, mods, count, "operand", what + " in place")


# ---------------------------------------------------------------- the rest of the coefficient form's domain
def _blocks(port, last):
    """70 limbs (two parameter blocks) with the smallest or the largest modulus last"""
    mods = rx.chain(port.generate_primes, 16, "blocks")
    q = min(mods) if last == "smallest" else max(mods)
    return [m for m in mods if m != q] + [q]


P59 = 576460752303423433   # the largest prime below 2^59
P61 = (1 << 61) - 1        # prime
# name -> (n, moduli, or a function of port that returns them)
DOMAIN = {
    "n=1": (1, lambda port: rx.chain(port.generate_primes, 16, "wide")),
    "n=3": (3, lambda port: rx.chain(port.generate_primes, 16, "classes")),
    "n=4099": (4099, lambda port: rx.chain(port.generate_primes, 16, "seal")),
    "q_i=2,3": (4099, [2, 3, P61]),
    "q_L=3": (64, [P61, 2, 3]),
    "q_L=2^40": (64, [P61, 1000003, 3, 1 << 40]),
    "q_L=2p": (64, [P61, 1000003, 2 * P59]),
    "composite": (64, [3 * 5 * 7 * 11 * 13 * 17 * 19 * 23, 29 * 31 * 37 * 41 * 43 * 47, 53 * 59 * 61 * 67 * 71]),
    "shared_factors": (64, [15, 21, 35, 3 * P59, P61]),
    "70_limbs_q_L_smallest": (64, lambda port: _blocks(port, "smallest")),
    "70_limbs_q_L_largest": (64, lambda port: _blocks(port, "largest")),
}


def _pairwise_coprime(mods):
    return all(np.gcd(int(a), int(b)) == 1 for i, a in enumerate(mods) for b in mods[i + 1:])


def test_domain_moduli_are_what_their_names_say(port):
    assert P59 < 1 << 59 and P61 < 1 << 61
    for name, (n, mods) in DOMAIN.items():
        mods = mods(port) if callable(mods) else mods
        assert all(1 < q < 1 << 61 for q in mods), name
        assert all(np.gcd(int(q), int(mods[-1])) == 1 for q in mods[:-1]), name
        assert _pairwise_coprime(mods) == (name != "shared_factors"), name
    assert DOMAIN["q_L=2p"][1][-1] % 2 == 0 and DOMAIN["q_L=2^40"][1][-1] % 2 == 0
    assert min(_blocks(port, "smallest")) == _blocks(port, "smallest")[-1]
    assert max(_blocks(port, "largest")) == _blocks(port, "largest")[-1]


@pytest.mark.parametrize("where", ["device", "host"])
@pytest.mark.parametrize("name", list(DOMAIN))
def test_coefficient_form_domain(hb, port, name, where):
    """the integer definition where the moduli are pairwise coprime, the per-limb formula where they are not"""
    n, mods = DOMAIN[name]
    mods = mods(port) if callable(mods) else mods
    x = edge_operand(mods, n, 7 + n)
    count = x.shape[0]
    x = x.reshape(-1)
    reference = rx.rescale_integer if _pairwise_coprime(mods) else rx.rescale_per_limb
    exp = reference(x, n, mods, count)
    out, io = _run(hb, where, x, n, mods, count, False)
    _check(out, exp, x, n, mods, count, "sentinel", f"{name} {where} out of place")
    _check(io, exp, x, n, mods, count, "operand", f"{name} {where} in place")


# ---------------------------------------------------------------- refusals
def test_refusals_write_nothing(hb, port):
    """the cases tests/test_rescale_exact.py does not hold, on device buffers: each call raises
    HEXL_B200_ERR_INVALID_ARG and leaves result as it was"""
    seal = rx.chain(port.generate_primes, 16, "seal")
    refused = {
        "q_i = 2^61": (16, [1 << 61, 3, 5], False),
        "q_L = 2^61": (16, [3, 5, 1 << 61], False),
        "q_i = 2^61 in NTT form": (16, [1 << 61] + seal[1:], True),
        "q_i even, q_L = 2^40": (16, [P61, 6, 1 << 40], False),
        "q_i sharing a large prime with q_L": (16, [P61, 3 * P59, 5 * P59], False),
        "n = 3 in NTT form": (3, seal, True),
        "n = 4099 in NTT form": (4099, seal, True),
        "n = 2^20 + 2^19 in NTT form": ((1 << 20) + (1 << 19), [97, 193], True),
    }
    for what, (n, mods, ntt_form) in refused.items():
        size = 2 * len(mods) * n
        d_in = dev(np.ones(size, dtype=U64))
        d_out = dev(np.full(size, SENTINEL, dtype=U64))
        with pytest.raises(hb.HexlB200Error) as e:
            hb.DivideAndRoundQLast(d_out, d_in, n, mods, len(mods), 2, ntt_form)
        torch.cuda.synchronize()
        assert e.value.code == -1, (what, str(e.value))
        assert (host(d_out) == U64(SENTINEL)).all(), f"{what}: result was written"
