"""ApplyGaloisKeySwitch and ApplyGaloisKeySwitchHoisted across every degree, key shape, Galois element, host batch and
pointer kind they accept.

The rotations share the key switch's decomposition, but three parts are their own: the permuted multiply-accumulate
(ks_mac_kernel<true>, which reads digit slot pi_g(l) through galois.cuh:ntt_source), the per-element loops of the
hoisted call, and the host paths of key_switch_host_batch.  Every output is compared bit for bit with an exact model:
ApplyGaloisKeySwitch with galois_exact.rotation_exact (the exact key switch of [sigma(c0), 0] with sigma(c1)), the
hoisted call with hoist_exact.hoisted_exact.

    key shapes  one_digit, small_special, wrap_keys, slots2 and wrap17 (tests/ks_exact.py), through device, host and
                [0, 0]-split host buffers (the hoisted call also managed), batches 1 and 3
    degrees     uniform and one_digit at every n = 2^k, k = 1..20 (ntt_source on up to 20-bit indices, the transforms'
                one and two column passes), seal_chain and word_classes at 2^14, 2^16 and 2^17; below 2^17 every element
                of E(n) = {1, 3, 5, 25, 5^-1, n - 1, n + 1, 2n - 3, 2n - 1} mod 2n, from 2^17 on 5 and 2n - 1
    production  the benchmark's C5 shape (2^15, 29 digits of 50 bits) at real elements, and the hoisted call at 2^16 with
                30 digits just below 2^61, whose moduli run in rounds of 17 and 14 with two multiply-accumulate
                launches each
    elements    one hoisted call over all of E(n); 5 twice with different keys; 16 elements in one call
    host        batches of 7 (more than the 3 staging slots) over one, two and three listed devices, and a sequence of
                host calls of different slot sizes on one device, so the slot buffers are reused and reallocated
    pointers    8-byte-offset device views between guard words (the automorphism's word-at-a-time kernel), managed
                buffers for ApplyGaloisKeySwitch
    threads     four host threads with streams of their own, sharing the key handles, the scratch pool and the
                staging slots
"""
import threading

import numpy as np
import pytest

import composite_plan as plan
import galois_exact as gx
import hoist_exact as hx
import ks_exact
from util import uniform_below

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

U64 = np.uint64
SENTINEL = 0xA5A5A5A5A5A5A5A5
GUARD = 16  # words on each side of a guarded buffer
HOST_DEVICES = {"host": [], "host_split": [0, 0], "host_split3": [0, 0, 0]}


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=U64).view(np.int64)).to("cuda")


def host(t):
    return t.cpu().numpy().view(U64)


@pytest.fixture(scope="module", autouse=True)
def _need_cuda(hb):
    if not torch.cuda.is_available() or hb.device_count() == 0:
        pytest.fail("gpu-marked test collected on a machine without CUDA")


def elements(n):
    """E(n): 1, 3, the CKKS generator 5, 5^2, 5^-1, n - 1, n + 1, 2n - 3 and 2n - 1, reduced mod 2n, odd values only,
    without repeats"""
    two_n = 2 * n
    out = []
    for v in (1, 3, 5, 25, pow(5, -1, two_n), n - 1, n + 1, 2 * n - 3, 2 * n - 1):
        v %= two_n
        if v % 2 == 1 and v not in out:
            out.append(v)
    return out


def _check(got, exp, what):
    bad = int((np.asarray(got) != exp).sum())
    assert bad == 0, f"{what}: {bad} of {exp.size} words differ from the exact model"


class _Prepared:
    """One case's ciphertexts and its exact outputs, each computed once per ciphertext.  Element list position r of a
    hoisted call uses the keys rolled by rolls[r] (the digits rotated), so every element can have keys of its own."""

    def __init__(self, port, case, count):
        self.port, self.case, self.count = port, case, count
        self.per = 2 * case.decomp * case.n
        self.ct = hx.ciphertexts(case, count, 11)
        self._rot, self._hoist = {}, {}

    def cts(self, cs):
        return np.concatenate([self.ct[c * self.per:(c + 1) * self.per] for c in cs])

    def keys(self, roll):
        k = self.case.keys
        return k[roll % len(k):] + k[:roll % len(k)]

    def rotation(self, g, cs):
        for c in cs:
            if (g, c) not in self._rot:
                self._rot[g, c] = gx.rotation_exact(self.port, self.case, self.cts([c]), g, 1)
        return np.concatenate([self._rot[g, c] for c in cs])

    def hoisted(self, elts, rolls, cs):
        key = (tuple(elts), tuple(rolls))
        case = self.case
        for c in cs:
            if (key, c) not in self._hoist:
                self._hoist[key, c] = hx.hoisted_exact(self.port, self.cts([c]), case.n, case.decomp, case.kms,
                                                       case.mods, elts, [self.keys(r) for r in rolls], case.modswitch)
        return np.concatenate([self._hoist[key, c] for c in cs])


_cache = {}


def _prepared(port, name, logn=None, count=3):
    """the ks_exact case `name` at 2^logn (None: its default degree), kept for the whole module; the cases at 2^19 and
    2^20 (a few hundred MB of keys each) one at a time"""
    key = (name, logn, count)
    if key not in _cache:
        if logn and logn >= 19:
            for k in [k for k in _cache if k[1] and k[1] >= 19]:
                del _cache[k]
        _cache[key] = _Prepared(port, ks_exact.make_case(port, name, None if logn is None else 1 << logn), count)
    return _cache[key]


def _handle(hb, p, roll=0):
    c = p.case
    return hb.KeySwitchKeys(p.keys(roll), c.n, c.decomp, c.kms, c.kcc)


def _rotate(hb, p, g, cs, entry):
    """ApplyGaloisKeySwitch of the ciphertexts cs (one call) through one entry point"""
    case, src = p.case, p.cts(cs)
    try:
        hb.set_host_devices(HOST_DEVICES.get(entry, []))
        handle = _handle(hb, p)
        if entry == "device":
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                d = dev(src)
                hb.ApplyGaloisKeySwitch(d, *case.shape, handle, case.modswitch, g, len(cs), stream=s)
            s.synchronize()
            return host(d)
        if entry == "managed":
            buf = hb.managed_empty(src.size)
            try:
                buf[:] = src
                hb.ApplyGaloisKeySwitch(buf, *case.shape, handle, case.modswitch, g, len(cs))
                return buf.copy()
            finally:
                hb.managed_free(buf)
        got = src.copy()
        hb.ApplyGaloisKeySwitch(got, *case.shape, handle, case.modswitch, g, len(cs))
        return got
    finally:
        hb.set_host_devices([])


def _hoist(hb, p, elts, rolls, cs, entry):
    """ApplyGaloisKeySwitchHoisted of the ciphertexts cs by elts (one call) through one entry point; the input must
    come back unchanged"""
    case, src = p.case, p.cts(cs)
    n_out = len(cs) * len(elts) * p.per
    try:
        hb.set_host_devices(HOST_DEVICES.get(entry, []))
        handles = [_handle(hb, p, r) for r in rolls]
        if entry == "device":
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                d = dev(src)
                out = torch.full((n_out,), -1, dtype=torch.int64, device="cuda")
                hb.ApplyGaloisKeySwitchHoisted(out, d, *case.shape, handles, case.modswitch, elts, len(cs), stream=s)
            s.synchronize()
            assert (host(d) == src).all(), "the input changed"
            return host(out)
        if entry == "managed":
            d, out = hb.managed_empty(src.size), hb.managed_empty(n_out)
            try:
                d[:] = src
                out[:] = SENTINEL
                hb.ApplyGaloisKeySwitchHoisted(out, d, *case.shape, handles, case.modswitch, elts, len(cs))
                assert (d == src).all(), "the input changed"
                return out.copy()
            finally:
                hb.managed_free(d)
                hb.managed_free(out)
        d = src.copy()
        out = np.full(n_out, SENTINEL, dtype=U64)
        hb.ApplyGaloisKeySwitchHoisted(out, d, *case.shape, handles, case.modswitch, elts, len(cs))
        assert (d == src).all(), "the input changed"
        return out
    finally:
        hb.set_host_devices([])


# ---------------------------------------------------------------- key shapes
KEY_SHAPES = ("one_digit", "small_special", "wrap_keys", "slots2", "wrap17")


@pytest.mark.parametrize("entry", ["device", "host", "host_split"])
@pytest.mark.parametrize("name", KEY_SHAPES)
def test_rotation_key_shapes(hb, port, name, entry):
    """one digit (rns 2), a 29-bit special prime below every digit, 29 digits of q - 1 keys below 2^61 (the checkers'
    accumulator wraps), three unused key slots with kcc 2, and 17 digits below 2^61 (16 + 1 digits per launch)"""
    p = _prepared(port, name)
    for batch in (1, 3):
        _check(_rotate(hb, p, 5, range(batch), entry), p.rotation(5, range(batch)), f"{name} {entry} batch {batch}")


@pytest.mark.parametrize("entry", ["device", "host", "host_split", "managed"])
@pytest.mark.parametrize("name", KEY_SHAPES)
def test_hoisted_key_shapes(hb, port, name, entry):
    p = _prepared(port, name)
    n = p.case.n
    elts, rolls = [5, 2 * n - 1, pow(5, -1, 2 * n)], [0, 1, 2]
    for batch in (1, 3):
        _check(_hoist(hb, p, elts, rolls, range(batch), entry), p.hoisted(elts, rolls, range(batch)),
               f"{name} {entry} batch {batch}")


# ---------------------------------------------------------------- degrees
DEGREES = ([(name, logn) for name in ("uniform", "one_digit") for logn in range(1, 21)]
           + [(name, logn) for name in ("seal_chain", "word_classes") for logn in (14, 16, 17)])
DEGREE_CASES = [(name, logn, entry) for name, logn in DEGREES for entry in ("device", "host")]


@pytest.mark.parametrize("name,logn,entry", DEGREE_CASES,
                         ids=[f"{name}_n{logn}-{entry}" for name, logn, entry in DEGREE_CASES])
def test_rotations_at_every_degree(hb, port, name, logn, entry):
    """below 2^17 ApplyGaloisKeySwitch at every element of E(n) and one hoisted call over all of them; from 2^17 on the
    elements 5 and 2n - 1, so that the model stays affordable"""
    p = _prepared(port, name, logn, count=1)
    n = p.case.n
    elts = elements(n) if n < 1 << 17 else [5, 2 * n - 1]
    for g in elts:
        _check(_rotate(hb, p, g, [0], entry), p.rotation(g, [0]), f"{name} n={n} g={g} {entry}")
    rolls = list(range(len(elts)))
    _check(_hoist(hb, p, elts, rolls, [0], entry), p.hoisted(elts, rolls, [0]),
           f"{name} n={n} hoisted over {elts} {entry}")


def _ckks_case(port, logn, decomp, bits, below_top):
    """decomp digits + the special prime of `bits`-bit primes, random keys (the shapes of the benchmark and of
    composite_plan.KS_SHAPES)"""
    n = 1 << logn
    mods = [int(q) for q in port.generate_primes(decomp + 1, bits, below_top, n)]
    keys = [np.concatenate([uniform_below(1000 * j + 100 * k + i, n, mods[i]) for k in range(2)
                            for i in range(decomp + 1)]) for j in range(decomp)]
    modswitch = [port.inverse_mod(mods[-1] % q, q) for q in mods[:decomp]]
    return ks_exact.Case(n, decomp, decomp + 1, 2, mods, keys, modswitch, 1, ks_exact.can_wrap(mods, decomp))


def test_c5_shape_at_real_elements(hb, port):
    """N = 2^15, 29 digits + the special prime of 50 bits: ApplyGaloisKeySwitch at g = 5, the hoisted call at four
    elements other than 1, each with keys of its own"""
    p = _Prepared(port, _ckks_case(port, 15, 29, 50, True), 1)
    n = p.case.n
    _check(_rotate(hb, p, 5, [0], "device"), p.rotation(5, [0]), "C5 g=5")
    elts, rolls = [5, 25, pow(5, -1, 2 * n), 2 * n - 1], [0, 1, 2, 3]
    _check(_hoist(hb, p, elts, rolls, [0], "device"), p.hoisted(elts, rolls, [0]), f"C5 hoisted over {elts}")


def test_hoisted_products_survive_rounds_of_two_launches(hb, port):
    """composite_plan.KS_SHAPES["ckks_n16"]: 2^16 with 30 digits just below 2^61, moduli in rounds of 17 and 14, each
    round's multiply-accumulate in launches of 16 and 14 digits; both elements' products must survive all of them"""
    logn, decomp = plan.KS_SHAPES["ckks_n16"]
    case = _ckks_case(port, logn, decomp, 60, False)
    assert plan.key_switch_rounds(case.n, decomp, decomp + 1) == [17, 14]
    assert plan.ks_mac_launches(decomp, max(case.mods)) == [16, 14]
    p = _Prepared(port, case, 1)
    elts = [5, 2 * case.n - 1]
    _check(_hoist(hb, p, elts, [0, 0], [0], "device"), p.hoisted(elts, [0, 0], [0]), "ckks_n16 hoisted")


# ---------------------------------------------------------------- elements
def test_same_element_twice_with_different_keys(hb, port):
    p = _prepared(port, "uniform")
    elts, rolls = [5, 3, 5], [0, 1, 2]
    got = _hoist(hb, p, elts, rolls, [0], "device").reshape(3, p.per)
    exp = p.hoisted(elts, rolls, [0]).reshape(3, p.per)
    _check(got, exp, "5 twice")
    assert (exp[0] != exp[2]).any(), "the two keys give the same rotation"
    assert (got[0] != got[2]).any(), "both rotations by 5 used one key"


def test_sixteen_elements_in_one_call(hb, port):
    """G = 16 at 2^12: fifteen powers of 5 and 2n - 1, keys rolled over the 4 digits"""
    p = _prepared(port, "uniform")
    n = p.case.n
    elts = [pow(5, k, 2 * n) for k in range(1, 16)] + [2 * n - 1]
    assert len(set(elts)) == 16
    rolls = list(range(16))
    for entry in ("device", "host"):
        _check(_hoist(hb, p, elts, rolls, [0, 1], entry), p.hoisted(elts, rolls, [0, 1]), f"G = 16 {entry}")


# ---------------------------------------------------------------- host batches
@pytest.mark.parametrize("entry", ["host", "host_split", "host_split3"])
@pytest.mark.parametrize("call", ["rotation", "hoisted"])
def test_host_batch_of_seven(hb, port, call, entry):
    """7 ciphertexts cycle through the 3 staging slots more than twice; over two and three listed devices the blocks
    are 3 + 4 and 2 + 2 + 3, each starting again at slot 0"""
    p = _prepared(port, "uniform", count=7)
    n = p.case.n
    if call == "rotation":
        g = pow(5, -1, 2 * n)
        _check(_rotate(hb, p, g, range(7), entry), p.rotation(g, range(7)), f"rotation batch 7 {entry}")
    else:
        elts, rolls = [5, 2 * n - 1], [0, 1]
        _check(_hoist(hb, p, elts, rolls, range(7), entry), p.hoisted(elts, rolls, range(7)),
               f"hoisted batch 7 {entry}")


def test_host_calls_of_different_slot_sizes_in_sequence(hb, port):
    """On one device: hoisted with 1 and then 5 elements (the result slots grow fivefold), a rotation, a resident key
    switch and hoisted with 1 element again, batch 3 each, so every slot is used by every call"""
    p = _prepared(port, "uniform")
    n, case = p.case.n, p.case
    five = [5, 25, pow(5, -1, 2 * n), n + 1, 2 * n - 1]
    _check(_hoist(hb, p, [5], [0], range(3), "host"), p.hoisted([5], [0], range(3)), "hoisted G = 1")
    _check(_hoist(hb, p, five, range(5), range(3), "host"), p.hoisted(five, range(5), range(3)), "hoisted G = 5")
    _check(_rotate(hb, p, 3, range(3), "host"), p.rotation(3, range(3)), "rotation")
    cts = [ks_exact.ciphertext(case, seed) for seed in (1, 2, 3)]
    got = np.concatenate([r for r, _ in cts])
    hb.KeySwitchResident(got, np.concatenate([t for _, t in cts]), *case.shape, _handle(hb, p), case.modswitch, 3)
    _check(got, np.concatenate([ks_exact.expected(port, case, r, t) for r, t in cts]), "KeySwitchResident")
    _check(_hoist(hb, p, [2 * n - 1], [1], range(3), "host"), p.hoisted([2 * n - 1], [1], range(3)),
           "hoisted G = 1 again")


# ---------------------------------------------------------------- pointer kinds
def _guarded(values, offset):
    """a device buffer holding `values` `offset` words past a 16-byte boundary, between GUARD sentinel words"""
    buf = np.full(values.size + 2 * GUARD + offset, SENTINEL, dtype=U64)
    buf[GUARD + offset:GUARD + offset + values.size] = values
    d = dev(buf)
    return d, d[GUARD + offset:GUARD + offset + values.size]


def _guards_intact(buf, size, offset):
    b = host(buf)
    return (b[:GUARD + offset] == U64(SENTINEL)).all() and (b[GUARD + offset + size:] == U64(SENTINEL)).all()


@pytest.mark.parametrize("logn", [3, 12, 16])
def test_rotation_on_an_offset_view(hb, port, logn):
    """the ciphertexts 8 bytes off 16-byte alignment: the automorphism moves them a word at a time"""
    p = _prepared(port, "uniform", logn)
    case, g = p.case, 5
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        buf, view = _guarded(p.cts(range(2)), 1)
        assert view.data_ptr() % 16 == 8
        hb.ApplyGaloisKeySwitch(view, *case.shape, _handle(hb, p), case.modswitch, g, 2, stream=s)
    s.synchronize()
    _check(host(view), p.rotation(g, range(2)), f"n={case.n} offset view")
    assert _guards_intact(buf, view.numel(), 1), "a word next to the ciphertexts was written"


@pytest.mark.parametrize("offsets", [(1, 0), (0, 1), (1, 1)], ids=["input", "results", "both"])
@pytest.mark.parametrize("logn", [3, 12, 16])
def test_hoisted_on_offset_views(hb, port, logn, offsets):
    """the input, the results or both 8 bytes off 16-byte alignment; the input must come back unchanged"""
    p = _prepared(port, "uniform", logn)
    case, n = p.case, p.case.n
    elts, rolls = [5, 2 * n - 1], [0, 1]
    src = p.cts(range(2))
    handles = [_handle(hb, p, r) for r in rolls]
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        in_buf, d_in = _guarded(src, offsets[0])
        out_buf, d_out = _guarded(np.full(2 * len(elts) * p.per, SENTINEL, dtype=U64), offsets[1])
        hb.ApplyGaloisKeySwitchHoisted(d_out, d_in, *case.shape, handles, case.modswitch, elts, 2, stream=s)
    s.synchronize()
    _check(host(d_out), p.hoisted(elts, rolls, range(2)), f"n={n} offsets {offsets}")
    assert (host(d_in) == src).all(), "the input changed"
    assert _guards_intact(in_buf, src.size, offsets[0]), "a word next to the input was written"
    assert _guards_intact(out_buf, d_out.numel(), offsets[1]), "a word next to the results was written"


def test_rotation_on_managed_buffers(hb, port):
    p = _prepared(port, "uniform")
    _check(_rotate(hb, p, 5, range(3), "managed"), p.rotation(5, range(3)), "managed batch 3")


# ---------------------------------------------------------------- concurrent callers
def test_concurrent_callers_share_keys_scratch_and_staging(hb, port):
    """Four host threads, each with a stream of its own, each 4 times: a hoisted call and a rotation on device buffers
    queued on its stream, then one of the two on host buffers (the staging slots) while they run.  They share the key
    handles and the scratch pool; ctypes drops the GIL for every call, so the calls overlap."""
    p = _prepared(port, "uniform", count=4)
    case, n = p.case, p.case.n
    elts, rolls, g = [5, 2 * n - 1], [0, 1], pow(5, -1, 2 * n)
    handles = [_handle(hb, p, r) for r in rolls]
    rot = {c: p.rotation(g, [c]) for c in range(4)}
    hoist = {c: p.hoisted(elts, rolls, [c]) for c in range(4)}
    errors = []

    def worker(tid):
        try:
            s = torch.cuda.Stream()
            for it in range(4):
                c = (tid + it) % 4
                with torch.cuda.stream(s):
                    src = dev(p.cts([c]))
                    out = torch.empty(len(elts) * p.per, dtype=torch.int64, device="cuda")
                    hb.ApplyGaloisKeySwitchHoisted(out, src, *case.shape, handles, case.modswitch, elts, 1, stream=s)
                    d = dev(p.cts([c]))
                    hb.ApplyGaloisKeySwitch(d, *case.shape, handles[0], case.modswitch, g, 1, stream=s)
                if it % 2 == tid % 2:
                    h_out = np.zeros(len(elts) * p.per, dtype=U64)
                    hb.ApplyGaloisKeySwitchHoisted(h_out, p.cts([c]), *case.shape, handles, case.modswitch, elts)
                    h_exp = hoist[c]
                else:
                    h_out = p.cts([c])
                    hb.ApplyGaloisKeySwitch(h_out, *case.shape, handles[0], case.modswitch, g)
                    h_exp = rot[c]
                s.synchronize()
                for what, got, exp in (("hoisted device", host(out), hoist[c]), ("rotation device", host(d), rot[c]),
                                       ("host", h_out, h_exp)):
                    bad = int((got != exp).sum())
                    if bad:
                        errors.append(f"thread {tid} iteration {it} {what}: {bad} words differ")
        except Exception as exc:  # noqa: BLE001 - reported by the main thread
            errors.append(f"thread {tid}: {exc!r}")

    threads = [threading.Thread(target=worker, args=(t,)) for t in range(4)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
