"""ApplyGaloisKeySwitchHoisted on the GPU.

Every output is compared bit for bit with the hoisted model (tests/hoist_exact.py): digits transformed once, then
permuted per element inside the multiply-accumulate.  The cases are those of the rotation tests, including wrap_blocks
(70 digits: two parameter blocks, and multiply-accumulates chunked below 2^61), through device, pinned host, split
host and managed buffers, at the small degrees, and at N = 2^16 with 31 digits, where the moduli run in two rounds and
every element's products must survive from one round to the next.  At g = 1 the call equals ApplyGaloisKeySwitch bit
for bit, and an element's output does not depend on the other elements of the list.  Rotated ciphertexts decrypt to
sigma_g of the message.  Graph replay, launch counts and argument refusals are pinned."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import composite_plan as plan
import galois_exact as gx
import hoist_exact as hx
import ks_exact
from util import uniform_below

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U64 = np.uint64
SENTINEL = 0xA5A5A5A5A5A5A5A5
INVALID_ARG = -1
CASES = ("uniform", "seal_chain", "word_classes", "wrap_blocks")


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=U64).view(np.int64)).to("cuda")


def host(t):
    return t.cpu().numpy().view(U64)


@pytest.fixture(scope="module", autouse=True)
def _need_cuda(hb):
    if not torch.cuda.is_available() or hb.device_count() == 0:
        pytest.fail("gpu-marked test collected on a machine without CUDA")


def _check(got, exp, what):
    bad = int((got != exp).sum())
    assert bad == 0, f"{what}: {bad} of {exp.size} words differ"


def _rolled_keys(case, r):
    """element r's keys: the case's keys with the digits rotated by r, so every element has keys of its own"""
    return case.keys[r % case.decomp:] + case.keys[:r % case.decomp]


_cache = {}


def _prepared(port, name, n=None):
    """(case, elements, per-element keys, 3 ciphertexts, expected rotations [c][r])"""
    if (name, n) not in _cache:
        case = ks_exact.make_case(port, name, n)
        elts = [3, 2 * case.n - 1, 3]
        keys = [_rolled_keys(case, r) for r in range(len(elts))]
        ct = hx.ciphertexts(case, 3, 11)
        per = 2 * case.decomp * case.n
        exp = np.concatenate([hx.hoisted_exact(port, ct[c * per:(c + 1) * per], case.n, case.decomp, case.kms,
                                               case.mods, elts, keys, case.modswitch) for c in range(3)])
        _cache[name, n] = case, elts, keys, ct, exp
    return _cache[name, n]


def _run(hb, case, elts, keys, ct, batch, entry):
    per = 2 * case.decomp * case.n
    n_out = batch * len(elts) * per
    try:
        if entry == "host_split":
            hb.set_host_devices([0, 0])
        handles = [hb.KeySwitchKeys(k, case.n, case.decomp, case.kms, case.kcc) for k in keys]
        if entry == "device":
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                src = dev(ct[:batch * per])
                out = torch.full((n_out,), -1, dtype=torch.int64, device="cuda")
                hb.ApplyGaloisKeySwitchHoisted(out, src, *case.shape, handles, case.modswitch, elts, batch, stream=s)
            s.synchronize()
            assert torch.equal(src, dev(ct[:batch * per])), "the input changed"
            return host(out)
        if entry == "managed":
            src, out = hb.managed_empty(batch * per), hb.managed_empty(n_out)
            try:
                src[:] = ct[:batch * per]
                out[:] = SENTINEL
                hb.ApplyGaloisKeySwitchHoisted(out, src, *case.shape, handles, case.modswitch, elts, batch)
                assert (src == ct[:batch * per]).all(), "the input changed"
                return out.copy()
            finally:
                hb.managed_free(src)
                hb.managed_free(out)
        src = ct[:batch * per].copy()
        out = np.full(n_out, SENTINEL, dtype=U64)
        hb.ApplyGaloisKeySwitchHoisted(out, src, *case.shape, handles, case.modswitch, elts, batch)
        assert (src == ct[:batch * per]).all(), "the input changed"
        return out
    finally:
        hb.set_host_devices([])


@pytest.mark.parametrize("entry", ["device", "host", "host_split", "managed"])
@pytest.mark.parametrize("name", CASES)
def test_hoisted_rotations_equal_the_model(hb, port, name, entry):
    case, elts, keys, ct, exp = _prepared(port, name)
    for batch in (1, 3):
        got = _run(hb, case, elts, keys, ct, batch, entry)
        _check(got, exp[:got.size], f"{name} {entry} batch {batch}")


@pytest.mark.parametrize("entry", ["device", "host"])
@pytest.mark.parametrize("logn", [1, 2, 3, 6, 10])
def test_hoisted_rotations_at_small_degrees(hb, port, logn, entry):
    """N = 2 (where 3 = 2n - 1), 4 and 8 run the tiny transform kernels and the permutation moves whole 16-byte pairs;
    64 and 2^10 the row kernels"""
    case, elts, keys, ct, exp = _prepared(port, "uniform", 1 << logn)
    for batch in (1, 3):
        got = _run(hb, case, elts, keys, ct, batch, entry)
        _check(got, exp[:got.size], f"n={case.n} {entry} batch {batch}")


def _c5_case(port):
    """N = 2^15, 29 digits + the special prime, 50-bit primes, random keys"""
    n, decomp = 1 << 15, 29
    mods = [int(q) for q in port.generate_primes(decomp + 1, 50, True, n)]
    keys = [np.concatenate([uniform_below(1000 * j + i, n, mods[i]) for _ in range(2) for i in range(decomp + 1)])
            for j in range(decomp)]
    modswitch = [port.inverse_mod(mods[-1] % q, q) for q in mods[:decomp]]
    return ks_exact.Case(n, decomp, decomp + 1, 2, mods, keys, modswitch, 1, False)


def test_identity_element_equals_apply_galois_key_switch(hb, port):
    case = _c5_case(port)
    handle = hb.KeySwitchKeys(case.keys, case.n, case.decomp, case.kms, case.kcc)
    ct = dev(hx.ciphertexts(case, 2, 3))
    out = torch.empty(2 * ct.numel(), dtype=torch.int64, device="cuda")
    hb.ApplyGaloisKeySwitchHoisted(out, ct, *case.shape, [handle, handle], case.modswitch, [1, 1], 2)
    hb.ApplyGaloisKeySwitch(ct, *case.shape, handle, case.modswitch, 1, 2)
    per = ct.numel() // 2
    for c in range(2):
        for r in range(2):
            got = out[(2 * c + r) * per:(2 * c + r + 1) * per]
            assert torch.equal(got, ct[c * per:(c + 1) * per]), (c, r)


def test_each_output_is_independent_of_the_other_elements(hb, port):
    case = ks_exact.make_case(port, "seal_chain")
    n, per = case.n, 2 * case.decomp * case.n
    elts = [3, 1, 2 * n - 1, 5]
    handles = {g: hb.KeySwitchKeys(_rolled_keys(case, r), n, case.decomp, case.kms, case.kcc)
               for r, g in enumerate(elts)}
    ct = dev(hx.ciphertexts(case, 2, 7))

    def rotations(sub):
        out = torch.empty(2 * len(sub) * per, dtype=torch.int64, device="cuda")
        hb.ApplyGaloisKeySwitchHoisted(out, ct, *case.shape, [handles[g] for g in sub], case.modswitch, sub, 2)
        return {(c, g): out[(c * len(sub) + r) * per:(c * len(sub) + r + 1) * per] for c in range(2)
                for r, g in enumerate(sub)}

    full = rotations(elts)
    for sub in ([5, 3], [2 * n - 1], [1, 5, 3, 2 * n - 1]):
        for (c, g), v in rotations(sub).items():
            assert torch.equal(v, full[c, g]), (sub, c, g)


def test_per_element_products_survive_repeated_rounds(hb, port):
    """N = 2^16 with 31 digits: the digits' transforms run in two rounds of 16 moduli, and each element's products
    from the first round must still be there when the second adds its moduli"""
    n, decomp = 1 << 16, 31
    assert plan.key_switch_rounds(n, decomp, decomp + 1) == [16, 16]
    mods = [int(q) for q in port.generate_primes(decomp + 1, 50, True, n)]
    keys = [np.concatenate([uniform_below(7000 * j + i, n, mods[i]) for _ in range(2) for i in range(decomp + 1)])
            for j in range(decomp)]
    modswitch = [port.inverse_mod(mods[-1] % q, q) for q in mods[:decomp]]
    case = ks_exact.Case(n, decomp, decomp + 1, 2, mods, keys, modswitch, 1, False)
    elts = [3, 2 * n - 1]
    ct = hx.ciphertexts(case, 1, 13)
    exp = hx.hoisted_exact(port, ct, n, decomp, case.kms, mods, elts, [keys, keys], modswitch)
    handle = hb.KeySwitchKeys(keys, n, decomp, case.kms, 2)
    out = torch.empty(exp.size, dtype=torch.int64, device="cuda")
    hb.ApplyGaloisKeySwitchHoisted(out, dev(ct), *case.shape, [handle, handle], modswitch, elts, 1)
    _check(host(out), exp, "N = 2^16, 31 digits")


def _crt_centred(residues, mods):
    Q = 1
    for q in mods:
        Q *= q
    basis = [(Q // q) * pow(Q // q, -1, q) for q in mods]
    out = []
    for l in range(residues.shape[1]):
        X = sum(int(residues[i, l]) * basis[i] for i in range(len(mods))) % Q
        out.append(X - Q if X > Q // 2 else X)
    return out


def test_hoisted_rotations_decrypt_to_the_rotated_message(hb, port):
    """As test_gpu_galois.py::test_rotated_ciphertext_decrypts_to_the_rotated_message, for three elements in one call:
    the signed digit lift is below q_j in magnitude, so the same bound B = decomp n B_e q_max / P + n + 1 holds.  With
    the keys of two elements swapped, their outputs miss it by many orders of magnitude."""
    n, decomp, bound_e = 1 << 12, 4, 8
    mods = [int(q) for q in port.generate_primes(decomp + 1, 49, True, n)]
    P, q_mods = mods[-1], mods[:decomp]
    elts = [3, 2 * n - 1, 25]
    s = [int(v) - 1 for v in uniform_below(1, n, 3)]
    handles = []
    for r, g in enumerate(elts):
        keys, modswitch = gx.galois_keys(port, s, g, n, mods, decomp, 77 + r, bound_e)
        handles.append(hb.KeySwitchKeys(keys, n, decomp, len(mods), 2))
    me = [int(v) - (1 << 30) for v in uniform_below(2, n, 1 << 31)]
    s_ntt = [port.ntt_forward(np.array([c % q for c in s], dtype=U64), n, q) for q in q_mods]
    c1 = [uniform_below(3 + i, n, q) for i, q in enumerate(q_mods)]
    c0 = [port.sub_mod(port.ntt_forward(np.array([c % q for c in me], dtype=U64), n, q),
                       port.mult_mod(c1[i], s_ntt[i], q), q) for i, q in enumerate(q_mods)]
    ct = np.concatenate(c0 + c1)
    bound = decomp * n * bound_e * max(q_mods) // P + n + 1

    def noises(hs):
        out = torch.empty(len(elts) * ct.size, dtype=torch.int64, device="cuda")
        hb.ApplyGaloisKeySwitchHoisted(out, dev(ct), n, decomp, len(mods), decomp + 1, 2, mods, hs, modswitch, elts)
        res = host(out).reshape(len(elts), 2, decomp, n)
        got = []
        for r, g in enumerate(elts):
            sme = gx.sigma_int(me, n, g)
            d = np.stack([port.sub_mod(port.ntt_inverse(port.add_mod(res[r, 0, i],
                                                                     port.mult_mod(res[r, 1, i], s_ntt[i], q), q),
                                                        n, q),
                                       np.array([c % q for c in sme], dtype=U64), q) for i, q in enumerate(q_mods)])
            got.append(max(abs(v) for v in _crt_centred(d, q_mods)))
        return got

    right = noises(handles)
    assert all(v < bound for v in right), f"noise {right} is not below the bound {bound}"
    swapped = noises([handles[1], handles[0], handles[2]])
    assert swapped[2] < bound
    assert swapped[0] > bound << 40 and swapped[1] > bound << 40, f"swapped keys decrypted: {swapped} (bound {bound})"


def test_graph_replay(hb, port):
    case, elts, keys, ct, exp = _prepared(port, "uniform")
    handles = [hb.KeySwitchKeys(k, case.n, case.decomp, case.kms, case.kcc) for k in keys]
    src = dev(ct)
    out = torch.empty(exp.size, dtype=torch.int64, device="cuda")
    hb.ApplyGaloisKeySwitchHoisted(out, src, *case.shape, handles, case.modswitch, elts, 3)  # warm: tables and pool
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        hb.ApplyGaloisKeySwitchHoisted(out, src, *case.shape, handles, case.modswitch, elts, 3)
    out.fill_(-1)
    graph.replay()
    torch.cuda.synchronize()
    _check(host(out), exp, "graph replay")
    ct2 = hx.ciphertexts(case, 3, 23)
    per = 2 * case.decomp * case.n
    exp2 = np.concatenate([hx.hoisted_exact(port, ct2[c * per:(c + 1) * per], case.n, case.decomp, case.kms,
                                            case.mods, elts, keys, case.modswitch) for c in range(3)])
    src.copy_(dev(ct2))
    graph.replay()
    torch.cuda.synchronize()
    _check(host(out), exp2, "graph replay, new data")


@pytest.mark.parametrize("decomp", [3, 8, 70])
def test_launch_counts(hb, port, decomp):
    """G = 1: the launches of ApplyGaloisKeySwitch.  Each further element adds the same number, which leaves out the
    digits' inverse transform and one forward transform per round of moduli"""
    n = 1 << 12
    mods = [int(q) for q in port.generate_primes(decomp + 1, 49, True, n)]
    keys = [uniform_below(j, 2 * (decomp + 1) * n, min(mods)) for j in range(decomp)]
    ms = [1] * decomp
    shape = (n, decomp, decomp + 1, decomp + 1, 2, mods)
    handle = hb.KeySwitchKeys(keys, n, decomp, decomp + 1, 2)
    comp = decomp * n
    ct = dev(np.zeros(2 * comp, dtype=U64))

    def launches(fn):
        fn()  # warm
        torch.cuda.synchronize()
        before = hb.launch_count()
        fn()
        torch.cuda.synchronize()
        return hb.launch_count() - before

    def hoisted(g):
        out = torch.empty(g * 2 * comp, dtype=torch.int64, device="cuda")
        return launches(lambda: hb.ApplyGaloisKeySwitchHoisted(out, ct, *shape, [handle] * g, ms, [3] * g))

    rot = launches(lambda: hb.ApplyGaloisKeySwitch(ct, *shape, handle, ms, 3))
    counts = [hoisted(g) for g in (1, 2, 3, 4)]
    assert counts[0] == rot, (counts, rot)
    inc = {b - a for a, b in zip(counts, counts[1:])}
    assert len(inc) == 1, counts
    rounds = len(plan.key_switch_rounds(n, decomp, decomp + 1))
    assert rot - inc.pop() >= 1 + rounds, (counts, rot, rounds)


def test_refusals(hb, port):
    case = ks_exact.make_case(port, "uniform")
    n, per = case.n, 2 * case.decomp * case.n
    handle = hb.KeySwitchKeys(case.keys, n, case.decomp, case.kms, case.kcc)
    ct = dev(hx.ciphertexts(case, 1, 5))
    out = torch.full((2 * per,), -1, dtype=torch.int64, device="cuda")

    def refused(what, results=out, src=ct, shape=case.shape, handles=(handle, handle), elts=(3, 5)):
        before = results.clone()
        with pytest.raises(hb.HexlB200Error) as e:
            hb.ApplyGaloisKeySwitchHoisted(results, src, *shape, list(handles), case.modswitch, list(elts), 1)
        assert e.value.code == INVALID_ARG, (what, e.value)
        assert torch.equal(results, before), f"{what}: results written"

    n_, d, kms, rns, kcc, mods = case.shape
    kcc3 = hb.KeySwitchKeys([np.concatenate([k, k[:kms * n]]) for k in case.keys], n, d, kms, 3)
    refused(what="kcc 3", shape=(n_, d, kms, rns, 3, mods), handles=(kcc3, kcc3),
            results=torch.full((6 * d * n,), -1, dtype=torch.int64, device="cuda"), src=dev(np.zeros(3 * d * n)))
    try:
        hb.set_host_devices([0, 0])
        sharded = hb.KeySwitchKeys(case.keys, n, d, kms, kcc, sharded_by_modulus=True)
    finally:
        hb.set_host_devices([])
    refused(what="sharded handle", handles=(handle, sharded))
    other = ks_exact.make_case(port, "uniform", n // 2)
    small = hb.KeySwitchKeys(other.keys, n // 2, other.decomp, other.kms, other.kcc)
    refused(what="handle of another degree", handles=(handle, small))
    for elts in ((3, 4), (2 * n, 3), (3, 0), (3, 2 * n + 1)):
        refused(what=f"element list {elts}", elts=elts)
    refused(what="null key", handles=(handle, None))
    refused(what="results overlap the input", results=out, src=out[per // 2:per // 2 + per])
    bad = hx.ciphertexts(case, 1, 5)
    bad[3] = case.mods[0]
    hb.set_debug(True)
    try:
        refused(what="input word = q under debug", src=dev(bad))
    finally:
        hb.set_debug(False)
    hb.ApplyGaloisKeySwitchHoisted(out, ct, *case.shape, [], case.modswitch, [], 1)
    torch.cuda.synchronize()
    assert (host(out) == ~U64(0)).all(), "num_elts = 0 wrote results"


def test_cpp_caller_runs(hb, tmp_path):
    if not shutil.which("g++"):
        pytest.skip("g++ not present")
    exe = tmp_path / "hoisted_caller"
    libdir = os.path.dirname(hb.LIB_PATH)
    subprocess.run(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "cpp", "hoisted_caller.cpp"), "-o", str(exe),
                    "-L", libdir, "-lhexl_b200", f"-Wl,-rpath,{libdir}"], check=True)
    res = subprocess.run([str(exe), "run"], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
