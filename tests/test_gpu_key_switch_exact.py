"""KeySwitch on the GPU against the exact model (tests/ks_exact.py), through every entry point:

    device      hexl_b200_key_switch with device pointers
    host        hexl_b200_key_switch with host pointers (keys uploaded per call, staging streams)
    resident    hexl_b200_key_switch_resident, batch 2, host and device buffers
    sharded     a handle sharded by modulus over three shards on device 0 (its own multiply-accumulate loop)

on the shapes the older tests never reach: moduli just below 2^61 with more digits than a 128-bit sum of lazy
products can hold (where the reference's own accumulator wraps, so only the exact model knows the answer), more digits
than one parameter block, a SEAL-style chain whose first digit prime is larger than the special prime, and moduli of
all three word classes in one switch.  The last two also run at the degrees CKKS uses, N = 2^14, 2^16 and 2^17 (SEAL's
largest), and a uniform chain at 2^18, where the transforms inside the switch take two column passes.  Every
comparison is bit for bit."""
import numpy as np
import pytest

import ks_exact

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

GPU_CASES = ("wrap_keys", "wrap_blocks", "seal_chain", "word_classes")
ENTRY_POINTS = ("device", "host", "resident", "sharded")
# (case, log2 n) beyond each case's default degree: device and host pointers at each, every entry point at 2^17
DEGREES = [(name, logn) for logn in (14, 16, 17) for name in ("seal_chain", "word_classes")] + [("uniform", 18)]
CASES = ([(name, None, entry) for name in GPU_CASES for entry in ENTRY_POINTS]
         + [(name, logn, entry) for name, logn in DEGREES
            for entry in (ENTRY_POINTS if logn == 17 else ("device", "host"))])


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64)).to("cuda")


def host(t):
    return t.cpu().numpy().view(np.uint64)


@pytest.fixture(scope="module", autouse=True)
def _need_cuda(hb):
    if not torch.cuda.is_available() or hb.device_count() == 0:
        pytest.fail("gpu-marked test collected on a machine without CUDA")


_cache = {}


def _prepared(port, checker, name, logn):
    """(case, [(result, t_target)] x 2, [exact result] x 2), computed once per case and degree"""
    if (name, logn) not in _cache:
        case = ks_exact.make_case(port, name, None if logn is None else 1 << logn)
        cts = [ks_exact.ciphertext(case, seed) for seed in (1, 2)]
        exp = [ks_exact.expected(port, case, r, t) for r, t in cts]
        if not case.wraps:   # where the checker's accumulator cannot wrap, it must agree with the model
            r, t = cts[0]
            assert (checker.key_switch(r.copy(), t, *case.shape, case.keys, case.modswitch) == exp[0]).all(), name
        _cache[name, logn] = case, cts, exp
    return _cache[name, logn]


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
        try:
            hb.set_host_devices([0, 0, 0])
            handle = hb.KeySwitchKeys(case.keys, case.n, case.decomp, case.kms, case.kcc, sharded_by_modulus=True)
        finally:
            hb.set_host_devices([])
        got = np.concatenate([r0, r1])
        hb.KeySwitchResident(got, np.concatenate([t0, t1]), *case.shape, handle, case.modswitch, 2)
        _check(got, np.concatenate(exp), f"{name} sharded batch 2")
