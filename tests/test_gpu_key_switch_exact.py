"""KeySwitch on the GPU against the exact model (tests/ks_exact.py), through every entry point:

    device      hexl_b200_key_switch with device pointers
    host        hexl_b200_key_switch with host pointers (keys uploaded per call, staging streams)
    resident    hexl_b200_key_switch_resident, batch 2, host and device buffers
    sharded     a handle sharded by modulus over three shards on device 0
    sharded_one the same over a single shard: with wrap_blocks' 71 moduli, the shard's multiply-accumulate rounds and
                mod-down blocks each run two parameter blocks
    sharded_rns+2  the same with rns_modulus_size + 2 devices listed, at N = 2 and 4; the upload cuts the list to
                   rns_modulus_size shards of one modulus each

on the shapes the older tests never reach: moduli just below 2^61 with more digits than a 128-bit sum of lazy
products can hold (where the reference's own accumulator wraps, so only the exact model knows the answer), more digits
than one parameter block, a SEAL-style chain whose first digit prime is larger than the special prime, and moduli of
all three word classes in one switch.  The last two also run at the degrees CKKS uses, N = 2^14, 2^16 and 2^17 (SEAL's
largest), and a uniform chain at 2^18, where the transforms inside the switch take two column passes.

The shape arguments run across what the API accepts: key_component_count 1 and 3 (the older cases all have 2), one
digit, three unused key slots, a 29-bit special prime smaller than every digit, and 17 digits just below 2^61 with three
components (two multiply-accumulate launches).  uniform, kcc3 and one_digit run through every entry point at N = 2, 4
and 8 (the multi-modulus transforms are one thread per polynomial, with their own gather and mirrored stores),
N = 16 to 2^11 (one row kernel whose CTAs span several moduli and digits), and through device and host pointers at
2^19 and 2^20 (two column passes of different radices).  Every comparison is bit for bit."""
import numpy as np
import pytest

import ks_exact

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

GPU_CASES = ("wrap_keys", "wrap_blocks", "seal_chain", "word_classes", "kcc1", "kcc3", "one_digit", "slots",
             "small_special", "kcc3_wrap")
ENTRY_POINTS = ("device", "host", "resident", "sharded")
SMALL_LOGNS = (1, 2, 3, 4, 5, 8, 11)
# (case, log2 n) beyond each case's default degree: device and host pointers at each, every entry point at 2^17 and at
# the small degrees, and rns + 2 listed devices (cut to one shard per modulus) at N = 2 and 4
DEGREES = ([(name, logn) for logn in (14, 16, 17) for name in ("seal_chain", "word_classes")] + [("uniform", 18)]
           + [(name, logn) for logn in SMALL_LOGNS + (19, 20) for name in ("uniform", "kcc3", "one_digit")])


def _entries(logn):
    if logn in (1, 2):
        return ENTRY_POINTS + ("sharded_rns+2",)
    return ENTRY_POINTS if logn == 17 or logn in SMALL_LOGNS else ("device", "host")


CASES = ([(name, None, entry) for name in GPU_CASES for entry in ENTRY_POINTS + ("sharded_one",)]
         + [(name, logn, entry) for name, logn in DEGREES for entry in _entries(logn)])


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64)).to("cuda")


def host(t):
    return t.cpu().numpy().view(np.uint64)


@pytest.fixture(scope="module", autouse=True)
def _need_cuda(hb):
    if not torch.cuda.is_available() or hb.device_count() == 0:
        pytest.fail("gpu-marked test collected on a machine without CUDA")


_cache = {}


def _prepared(port, checker, name, logn, count=2):
    """(case, [(result, t_target)] x count, [exact result] x count), each computed once per case and degree; the cases
    at 2^19 and 2^20 (a few hundred MB each) are kept one at a time"""
    key = (name, logn)
    if key not in _cache:
        if logn and logn >= 19:
            for k in [k for k in _cache if k[1] and k[1] >= 19]:
                del _cache[k]
        _cache[key] = ks_exact.make_case(port, name, None if logn is None else 1 << logn), [], []
    case, cts, exp = _cache[key]
    while len(cts) < count:
        r, t = ks_exact.ciphertext(case, len(cts) + 1)
        cts.append((r, t))
        exp.append(ks_exact.expected(port, case, r, t))
        if len(cts) == 1 and not case.wraps:   # where the checker's accumulator cannot wrap, it must agree with the model
            assert (checker.key_switch(r.copy(), t, *case.shape, case.keys, case.modswitch) == exp[0]).all(), name
    return case, cts[:count], exp[:count]


def _check(got, exp, what):
    wrong = int((np.asarray(got) != exp).sum())
    assert wrong == 0, f"{what}: {wrong} of {exp.size} words differ from the exact key switch"


@pytest.mark.parametrize("name,logn,entry", CASES,
                         ids=[f"{name}{'' if logn is None else f'_n{logn}'}-{entry}" for name, logn, entry in CASES])
def test_key_switch_equals_exact_model(hb, port, checker, name, logn, entry):
    case, cts, exp = _prepared(port, checker, name, logn)
    name = f"{name} n={case.n}"
    (r0, t0), (r1, t1) = cts
    if entry == "device":
        d = dev(r0)
        hb.KeySwitch(d, dev(t0), *case.shape, [dev(k) for k in case.keys], case.modswitch)
        _check(host(d), exp[0], f"{name} device")
    elif entry == "host":
        got = r0.copy()
        hb.KeySwitch(got, t0, *case.shape, case.keys, case.modswitch)
        _check(got, exp[0], f"{name} host")
    elif entry == "resident":
        handle = hb.KeySwitchKeys(case.keys, case.n, case.decomp, case.kms, case.kcc)
        both_r, both_t = np.concatenate([r0, r1]), np.concatenate([t0, t1])
        got = both_r.copy()
        hb.KeySwitchResident(got, both_t, *case.shape, handle, case.modswitch, 2)
        _check(got, np.concatenate(exp), f"{name} resident host batch 2")
        d = dev(both_r)
        hb.KeySwitchResident(d, dev(both_t), *case.shape, handle, case.modswitch, 2)
        _check(host(d), np.concatenate(exp), f"{name} resident device batch 2")
    else:
        shards = {"sharded": 3, "sharded_one": 1}.get(entry, case.rns + 2)
        try:
            hb.set_host_devices([0] * shards)
            handle = hb.KeySwitchKeys(case.keys, case.n, case.decomp, case.kms, case.kcc, sharded_by_modulus=True)
        finally:
            hb.set_host_devices([])
        got = np.concatenate([r0, r1])
        hb.KeySwitchResident(got, np.concatenate([t0, t1]), *case.shape, handle, case.modswitch, 2)
        _check(got, np.concatenate(exp), f"{name} {entry} ({shards} shards) batch 2")


@pytest.mark.parametrize("devices", [[0, 0], [0, 0, 0, 0]], ids=["2_blocks", "4_blocks"])
@pytest.mark.parametrize("name", ["kcc1", "uniform", "kcc3"])
def test_resident_host_batch_split_over_host_devices(hb, port, checker, name, devices):
    """A host batch of 3 ciphertexts under set_host_devices, with the keys uploaded after the split: the batch is cut
    into one block of ciphertexts per listed device (with four devices, one block per ciphertext and one device
    left over), each staged through its own rotating slots."""
    case, cts, exp = _prepared(port, checker, name, None, 3)
    try:
        hb.set_host_devices(devices)
        handle = hb.KeySwitchKeys(case.keys, case.n, case.decomp, case.kms, case.kcc)
        got = np.concatenate([r for r, _ in cts])
        hb.KeySwitchResident(got, np.concatenate([t for _, t in cts]), *case.shape, handle, case.modswitch, 3)
    finally:
        hb.set_host_devices([])
    _check(got, np.concatenate(exp), f"{name} kcc={case.kcc} resident host batch 3 over {devices}")
