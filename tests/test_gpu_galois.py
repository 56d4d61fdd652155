"""ApplyGalois and ApplyGaloisKeySwitch on the GPU.

ApplyGalois is compared bit for bit with the model (tests/galois_exact.py) in both forms at every degree the library
takes a step of, with SEAL-shaped moduli chains, 70 moduli (two parameter blocks), inputs at 0 and q - 1, and through
every entry point: device pointers on a stream (out of place with guards around result, and in place), host pointers
(also larger than a staging chunk, and split over set_host_devices), managed memory and CUDA graph replay.  It is
cross-checked with the library's own transforms and products, and its launch counts are pinned.

ApplyGaloisKeySwitch is compared with the exact key switch (tests/ks_exact.py) of r = [sigma(c0), 0] and
t = sigma(c1), with the chain of existing calls, and by decryption: ciphertexts under a secret s, rotated with Galois
keys for sigma_g(s), decrypt to sigma_g of the message."""
import os
import shutil
import subprocess

import numpy as np
import pytest

import galois_exact as gx
import ks_exact
import rescale_exact as rx
from util import uniform_below

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U64 = np.uint64
SENTINEL = 0xA5A5A5A5A5A5A5A5
GUARD = 64  # words: 512 bytes on each side of result
FORMS = [True, False]
LOG_DEGREES = [1, 2, 3, 8, 11, 13, 14, 15, 16, 17, 18, 19, 20]
G_NAMES = ["1", "3", "2n-1", "random"]


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=U64).view(np.int64)).to("cuda")


def host(t):
    return t.cpu().numpy().view(U64)


@pytest.fixture(scope="module", autouse=True)
def _need_cuda(hb):
    if not torch.cuda.is_available() or hb.device_count() == 0:
        pytest.fail("gpu-marked test collected on a machine without CUDA")


def galois_elt(n, name):
    return {"1": 1, "3": 3 % (2 * n), "2n-1": 2 * n - 1,
            "random": int(uniform_below(n + 7, 1, n)[0]) * 2 + 1}[name]


def operand(seed, n, mods, count):
    """uniform limbs with every 5th coefficient 0 and every 7th q - 1, so both signs meet both edges"""
    x = rx.random_operand(seed, n, mods, count).reshape(count, len(mods), n)
    q = np.array(mods, dtype=U64)[None, :, None]
    x[:, :, ::5] = 0
    x[:, :, 3::7] = np.broadcast_to(q - U64(1), x[:, :, 3::7].shape)
    return x.reshape(-1)


_cache = {}


def _prepared(port, logn, chain="seal", limbs=None, count=3):
    """(n, moduli, operand): 31 limbs up to 2^16, 6 above (the buffers stay within a few hundred MB)"""
    n = 1 << logn
    limbs = limbs or (31 if logn <= 16 else 6)
    key = (logn, chain, limbs, count)
    if key not in _cache:
        mods = rx.chain(port.generate_primes, n, chain, limbs)
        _cache[key] = n, mods, operand(logn + limbs, n, mods, count)
    return _cache[key]


def model(x, n, mods, count, g, ntt_form):
    return gx.sigma_ntt(x, n, g) if ntt_form else gx.sigma_coef(x, n, g, mods, count)


def _check(got, exp, what):
    wrong = int((np.asarray(got) != exp).sum())
    assert wrong == 0, f"{what}: {wrong} of {exp.size} words differ from the model"


@pytest.mark.parametrize("ntt_form", FORMS, ids=["ntt", "coef"])
@pytest.mark.parametrize("gname", G_NAMES)
@pytest.mark.parametrize("logn", LOG_DEGREES)
def test_apply_galois_equals_model(hb, port, logn, gname, ntt_form):
    n, mods, x = _prepared(port, logn)
    g, rns, count = galois_elt(n, gname), len(mods), 3
    exp = model(x, n, mods, count, g, ntt_form)
    d_in = dev(x)
    d_out = torch.empty_like(d_in)
    hb.ApplyGalois(d_out, d_in, n, mods, rns, count, g, ntt_form)
    _check(host(d_out), exp, f"n={n} g={g} count 3")
    one = torch.empty(rns * n, dtype=torch.int64, device="cuda")
    hb.ApplyGalois(one, d_in, n, mods, rns, 1, g, ntt_form)
    _check(host(one), exp[:rns * n], f"n={n} g={g} count 1")


@pytest.mark.parametrize("ntt_form", FORMS, ids=["ntt", "coef"])
@pytest.mark.parametrize("g", [3, "2n-1"])
def test_seventy_moduli_two_parameter_blocks(hb, port, g, ntt_form):
    n, mods, x = _prepared(port, 11, "blocks", 70, 2)
    g = 2 * n - 1 if g == "2n-1" else g
    d = dev(x)
    out = torch.empty_like(d)
    hb.ApplyGalois(out, d, n, mods, 70, 2, g, ntt_form)
    _check(host(out), model(x, n, mods, 2, g, ntt_form), f"70 moduli g={g}")


def _guarded(size, offset=0):
    buf = torch.from_numpy(np.full(size + 2 * GUARD + offset, SENTINEL, dtype=U64).view(np.int64)).cuda()
    return buf, buf[GUARD + offset:GUARD + offset + size]


def _guards_intact(buf, size, offset=0):
    b = host(buf)
    return (b[:GUARD + offset] == U64(SENTINEL)).all() and (b[GUARD + offset + size:] == U64(SENTINEL)).all()


@pytest.mark.parametrize("ntt_form", FORMS, ids=["ntt", "coef"])
@pytest.mark.parametrize("logn", [3, 11, 14, 15, 17])
@pytest.mark.parametrize("offset", [0, 1], ids=["aligned", "8-byte-offset"])
def test_device_pointers_on_a_stream(hb, port, logn, ntt_form, offset):
    """out of place (operand unchanged, 512-byte guards on both sides of result) and in place, on a non-default
    stream; offset 1 puts result one word off 16-byte alignment, which takes the word-at-a-time kernels"""
    n, mods, x = _prepared(port, logn)
    rns, count, g = len(mods), 3, 2 * n - 3 if n > 2 else 1
    exp = model(x, n, mods, count, g, ntt_form)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        d_in = dev(x)
        buf, d_out = _guarded(x.size, offset)
        hb.ApplyGalois(d_out, d_in, n, mods, rns, count, g, ntt_form, stream=s)
        inbuf, d_io = _guarded(x.size, offset)
        d_io.copy_(d_in)
        hb.ApplyGalois(d_io, d_io, n, mods, rns, count, g, ntt_form, stream=s)
    s.synchronize()
    _check(host(d_out), exp, f"n={n} out of place")
    assert (host(d_in) == x).all(), "the operand was modified"
    assert _guards_intact(buf, x.size, offset), "a word next to result was written"
    _check(host(d_io), exp, f"n={n} in place")
    assert _guards_intact(inbuf, x.size, offset), "a word next to the in-place buffer was written"


@pytest.mark.parametrize("ntt_form", FORMS, ids=["ntt", "coef"])
def test_host_pointers(hb, port, ntt_form):
    n, mods, x = _prepared(port, 12)
    rns, count, g = len(mods), 3, 5
    exp = model(x, n, mods, count, g, ntt_form)
    out = np.full(x.size, SENTINEL, dtype=U64)
    hb.ApplyGalois(out, x, n, mods, rns, count, g, ntt_form)
    _check(out, exp, "host out of place")
    inplace = x.copy()
    hb.ApplyGalois(inplace, inplace, n, mods, rns, count, g, ntt_form)
    _check(inplace, exp, "host in place")


@pytest.mark.parametrize("ntt_form", FORMS, ids=["ntt", "coef"])
def test_host_polynomial_larger_than_a_staging_chunk(hb, port, ntt_form):
    """n = 2^17 with 33 limbs: 34.6 MB per polynomial, more than one 32 MiB staging buffer"""
    n, mods, x = _prepared(port, 17, "seal", 33, 2)
    assert len(mods) * n * 8 > 32 << 20
    g = 2 * n - 1
    out = np.full(x.size, SENTINEL, dtype=U64)
    hb.ApplyGalois(out, x, n, mods, len(mods), 2, g, ntt_form)
    _check(out, model(x, n, mods, 2, g, ntt_form), "n = 2^17 host")


@pytest.mark.parametrize("ntt_form", FORMS, ids=["ntt", "coef"])
def test_managed_memory(hb, port, ntt_form):
    n, mods, x = _prepared(port, 12)
    buf = hb.managed_empty(x.size)
    try:
        buf[:] = x
        hb.ApplyGalois(buf, buf, n, mods, len(mods), 3, 3, ntt_form)
        _check(buf.copy(), model(x, n, mods, 3, 3, ntt_form), "managed in place")
    finally:
        hb.managed_free(buf)


@pytest.mark.parametrize("ntt_form", FORMS, ids=["ntt", "coef"])
def test_host_devices_split_by_polynomial(hb, port, ntt_form):
    n, mods, x = _prepared(port, 12)
    out = np.full(x.size, SENTINEL, dtype=U64)
    try:
        hb.set_host_devices([0, 0, 0])
        hb.ApplyGalois(out, x, n, mods, len(mods), 3, 7, ntt_form)
    finally:
        hb.set_host_devices([])
    _check(out, model(x, n, mods, 3, 7, ntt_form), "set_host_devices([0, 0, 0])")


@pytest.mark.parametrize("ntt_form", FORMS, ids=["ntt", "coef"])
@pytest.mark.parametrize("logn", [12, 16])
def test_graph_capture_and_replay(hb, port, logn, ntt_form):
    n, mods, x = _prepared(port, logn)
    rns, count, g = len(mods), 3, 3
    d_in = dev(x)
    d_out = torch.empty_like(d_in)
    d_io = d_in.clone()

    def call():
        hb.ApplyGalois(d_out, d_in, n, mods, rns, count, g, ntt_form)
        hb.ApplyGalois(d_io, d_io, n, mods, rns, count, g, ntt_form)

    call()  # the pool is warm before the capture
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        call()
    x2 = operand(99, n, mods, count)
    d_in.copy_(dev(x2))
    d_io.copy_(dev(x2))
    graph.replay()
    torch.cuda.synchronize()
    exp = model(x2, n, mods, count, g, ntt_form)
    _check(host(d_out), exp, "graph replay, out of place")
    _check(host(d_io), exp, "graph replay, in place")


# ---------------------------------------------------------------- cross-checks with the library's own calls
@pytest.mark.parametrize("logn", LOG_DEGREES)
def test_forms_commute_with_the_library_transforms(hb, port, logn):
    """ComputeForwardMulti(sigma_coef(a)) == sigma_ntt(ComputeForwardMulti(a)), one polynomial of every limb"""
    n, mods, x = _prepared(port, logn)
    rns, g = len(mods), galois_elt(n, "random")
    ntts = [hb.GetNTT(n, q) for q in mods]
    a = dev(x[:rns * n])
    coef, fwd_of_coef, fwd, ntt = (torch.empty_like(a) for _ in range(4))
    hb.ApplyGalois(coef, a, n, mods, rns, 1, g, False)
    hb.ComputeForwardMulti(ntts, fwd_of_coef, coef, 1, 1, 1)
    hb.ComputeForwardMulti(ntts, fwd, a, 1, 1, 1)
    hb.ApplyGalois(ntt, fwd, n, mods, rns, 1, g, True)
    assert torch.equal(fwd_of_coef, ntt), f"n={n} g={g}"


def test_sigma_is_a_ring_map_under_the_library_product(hb, port):
    n, mods, x = _prepared(port, 14)
    rns, g = len(mods), 2 * n - 5
    ntts = [hb.GetNTT(n, q) for q in mods]
    a, b = dev(x[:rns * n]), dev(x[rns * n:2 * rns * n])
    sa, sb, prod_of_sigma, prod, sigma_of_prod = (torch.empty_like(a) for _ in range(5))
    hb.ApplyGalois(sa, a, n, mods, rns, 1, g, False)
    hb.ApplyGalois(sb, b, n, mods, rns, 1, g, False)
    hb.PolyMultiplyMulti(ntts, prod_of_sigma, sa, sb, 1)
    hb.PolyMultiplyMulti(ntts, prod, a, b, 1)
    hb.ApplyGalois(sigma_of_prod, prod, n, mods, rns, 1, g, False)
    assert torch.equal(prod_of_sigma, sigma_of_prod)


@pytest.mark.parametrize("logn", [11, 15])
def test_launch_counts(hb, port, logn):
    """NTT form out of place: one launch whatever the count and the limbs; coefficient form: one per 64 moduli"""
    n = 1 << logn

    def launches(limbs, count, ntt_form):
        mods = rx.chain(port.generate_primes, n, "blocks" if limbs == 70 else "seal", limbs)
        d = dev(rx.random_operand(limbs, n, mods, count))
        out = torch.empty_like(d)
        torch.cuda.synchronize()
        before = hb.launch_count()
        hb.ApplyGalois(out, d, n, mods, limbs, count, 3, ntt_form)
        torch.cuda.synchronize()
        return hb.launch_count() - before

    for limbs in (6, 70):
        for count in (1, 3):
            assert launches(limbs, count, True) == 1, (limbs, count)
            assert launches(limbs, count, False) == (limbs + 63) // 64, (limbs, count)


def test_cpp_caller_runs(hb, tmp_path):
    if not shutil.which("g++"):
        pytest.skip("g++ not present")
    exe = tmp_path / "galois_caller"
    libdir = os.path.dirname(hb.LIB_PATH)
    subprocess.run(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"),
                    os.path.join(ROOT, "tests", "cpp", "galois_caller.cpp"), "-o", str(exe),
                    "-L", libdir, "-lhexl_b200", f"-Wl,-rpath,{libdir}"], check=True)
    res = subprocess.run([str(exe), "run"], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr


# ---------------------------------------------------------------- ApplyGaloisKeySwitch
KS_CASES = ("uniform", "seal_chain", "word_classes", "wrap_blocks")
_ks_cache = {}


def _ciphertexts(case, batch, seed):
    """batch ciphertexts of two canonical components of decomp limbs"""
    n, d = case.n, case.decomp
    return np.concatenate([uniform_below(seed * 7919 + 100 * c + i, n, case.mods[i])
                           for c in range(2 * batch) for i in range(d)])


def _ks_prepared(port, name, g, n=None):
    if (name, g, n) not in _ks_cache:
        case = ks_exact.make_case(port, name, n)
        gg = 2 * case.n - 1 if g == "2n-1" else g
        ct = _ciphertexts(case, 3, 11)
        _ks_cache[name, g, n] = case, gg, ct, gx.rotation_exact(port, case, ct, gg, 3)
    return _ks_cache[name, g, n]


@pytest.mark.parametrize("entry", ["device", "host", "host_split"])
@pytest.mark.parametrize("g", [3, "2n-1"])
@pytest.mark.parametrize("name", KS_CASES)
def test_apply_galois_key_switch_equals_exact_rotation(hb, port, name, g, entry):
    _check_rotations(hb, name, *_ks_prepared(port, name, g), entry)


@pytest.mark.parametrize("entry", ["device", "host"])
@pytest.mark.parametrize("g", [3, "2n-1"])
@pytest.mark.parametrize("logn", [1, 2, 3, 6, 10])
def test_apply_galois_key_switch_at_small_degrees(hb, port, logn, g, entry):
    """uniform at N = 2 (where 3 = 2n - 1), 4 and 8, where the automorphism moves one or two 16-byte pairs per
    polynomial and the transforms of the switch run one thread per polynomial, and at 64 and 2^10 (row kernels)"""
    _check_rotations(hb, f"uniform n={1 << logn}", *_ks_prepared(port, "uniform", g, 1 << logn), entry)


def _check_rotations(hb, name, case, g, ct, exp, entry):
    """batch 1 and 3 through one entry point, against the exact rotation"""
    per = 2 * case.decomp * case.n
    for batch in (1, 3):
        if entry == "device":
            handle = hb.KeySwitchKeys(case.keys, case.n, case.decomp, case.kms, case.kcc)
            s = torch.cuda.Stream()
            with torch.cuda.stream(s):
                d = dev(ct[:batch * per])
                hb.ApplyGaloisKeySwitch(d, *case.shape, handle, case.modswitch, g, batch, stream=s)
            s.synchronize()
            got = host(d)
        else:
            try:
                if entry == "host_split":
                    hb.set_host_devices([0, 0])
                handle = hb.KeySwitchKeys(case.keys, case.n, case.decomp, case.kms, case.kcc)
                got = ct[:batch * per].copy()
                hb.ApplyGaloisKeySwitch(got, *case.shape, handle, case.modswitch, g, batch)
            finally:
                hb.set_host_devices([])
        _check(got, exp[:batch * per], f"{name} g={g} {entry} batch {batch}")


def test_apply_galois_key_switch_equals_the_chain_of_existing_calls(hb, port):
    case, g, ct, _ = _ks_prepared(port, "seal_chain", 3)
    handle = hb.KeySwitchKeys(case.keys, case.n, case.decomp, case.kms, case.kcc)
    comp, batch = case.decomp * case.n, 3
    d = dev(ct)
    hb.ApplyGaloisKeySwitch(d, *case.shape, handle, case.modswitch, g, batch)
    perm = torch.empty_like(d)
    hb.ApplyGalois(perm, dev(ct), case.n, case.mods, case.decomp, 2 * batch, g, True)
    p = perm.view(batch, 2, comp)
    r = torch.zeros_like(p)
    r[:, 0] = p[:, 0]
    t = p[:, 1].contiguous()
    hb.KeySwitchResident(r.view(-1), t.view(-1), *case.shape, handle, case.modswitch, batch)
    assert torch.equal(d, r.view(-1))


def test_apply_galois_key_switch_graph_replay(hb, port):
    case, g, ct, exp = _ks_prepared(port, "uniform", 3)
    handle = hb.KeySwitchKeys(case.keys, case.n, case.decomp, case.kms, case.kcc)
    d = dev(ct)
    hb.ApplyGaloisKeySwitch(d, *case.shape, handle, case.modswitch, g, 3)  # warm: tables and pool
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        hb.ApplyGaloisKeySwitch(d, *case.shape, handle, case.modswitch, g, 3)
    d.copy_(dev(ct))
    graph.replay()
    torch.cuda.synchronize()
    _check(host(d), exp, "graph replay")
    ct2 = _ciphertexts(case, 3, 23)
    d.copy_(dev(ct2))
    graph.replay()
    torch.cuda.synchronize()
    _check(host(d), gx.rotation_exact(port, case, ct2, g, 3), "graph replay, new data")


def test_apply_galois_key_switch_refuses_sharded_keys(hb, port):
    case = ks_exact.make_case(port, "uniform")
    try:
        hb.set_host_devices([0, 0])
        handle = hb.KeySwitchKeys(case.keys, case.n, case.decomp, case.kms, case.kcc, sharded_by_modulus=True)
    finally:
        hb.set_host_devices([])
    ct = _ciphertexts(case, 1, 5)
    with pytest.raises(hb.HexlB200Error) as e:
        hb.ApplyGaloisKeySwitch(ct, *case.shape, handle, case.modswitch, 3)
    assert e.value.code == -1 and "sharded" in str(e.value)


@pytest.mark.parametrize("decomp", [3, 8])
def test_launches_per_ciphertext_are_the_key_switch_plus_one(hb, port, decomp):
    n = 1 << 12
    mods = [int(q) for q in port.generate_primes(decomp + 1, 49, True, n)]
    keys = [uniform_below(j, 2 * (decomp + 1) * n, min(mods)) for j in range(decomp)]
    ms = [1] * decomp
    shape = (n, decomp, decomp + 1, decomp + 1, 2, mods)
    handle = hb.KeySwitchKeys(keys, n, decomp, decomp + 1, 2)
    comp = decomp * n

    def launches(fn):
        fn()  # warm
        torch.cuda.synchronize()
        before = hb.launch_count()
        fn()
        torch.cuda.synchronize()
        return hb.launch_count() - before

    for batch in (1, 3):
        ct = dev(np.zeros(batch * 2 * comp, dtype=U64))
        t = dev(np.zeros(batch * comp, dtype=U64))
        rot = launches(lambda: hb.ApplyGaloisKeySwitch(ct, *shape, handle, ms, 3, batch))
        ks = launches(lambda: hb.KeySwitchResident(ct, t, *shape, handle, ms, batch))
        assert rot % batch == 0 and ks % batch == 0, (rot, ks, batch)
        assert rot // batch == ks // batch + 1, (decomp, batch, rot, ks)


# ---------------------------------------------------------------- decryption
def _crt_centred(residues, mods):
    """centred CRT lift of per-limb residues ([limb][n]) -> Python ints"""
    Q = 1
    for q in mods:
        Q *= q
    basis = [(Q // q) * pow(Q // q, -1, q) for q in mods]
    out = []
    for l in range(residues.shape[1]):
        X = sum(int(residues[i, l]) * basis[i] for i in range(len(mods))) % Q
        out.append(X - Q if X > Q // 2 else X)
    return out


@pytest.mark.parametrize("g", [3, "2n-1"])
def test_rotated_ciphertext_decrypts_to_the_rotated_message(hb, port, g):
    """Keys for g from a ternary secret s (galois_exact.galois_keys); c = (-c1 s + m + e, c1) in NTT form.  After the
    rotation, c0' + c1' s - sigma_g(m + e) has a centred CRT lift below

        B = decomp n B_e q_max / P + n + 1,

    because the key switch adds sum_j d_j e_j (digits d_j < q_j, |e_j| <= B_e, n terms per coefficient) divided by P,
    plus a rounding error of at most 1/2 per coefficient in each component, the one of c1' multiplied by the ternary s
    (at most n/2).  With a key for a different g the same check fails by many orders of magnitude."""
    n, decomp, bound_e = 1 << 12, 4, 8
    mods = [int(q) for q in port.generate_primes(decomp + 1, 49, True, n)]
    P, q_mods = mods[-1], mods[:decomp]
    g = 2 * n - 1 if g == "2n-1" else g
    s = [int(v) - 1 for v in uniform_below(1, n, 3)]
    keys, modswitch = gx.galois_keys(port, s, g, n, mods, decomp, 77, bound_e)
    handle = hb.KeySwitchKeys(keys, n, decomp, len(mods), 2)
    me = [int(v) - (1 << 30) for v in uniform_below(2, n, 1 << 31)]  # message plus encryption error
    s_ntt = [port.ntt_forward(np.array([c % q for c in s], dtype=U64), n, q) for q in q_mods]
    c1 = [uniform_below(3 + i, n, q) for i, q in enumerate(q_mods)]
    c0 = [port.sub_mod(port.ntt_forward(np.array([c % q for c in me], dtype=U64), n, q),
                       port.mult_mod(c1[i], s_ntt[i], q), q) for i, q in enumerate(q_mods)]
    ct = np.concatenate(c0 + c1)
    sme = gx.sigma_int(me, n, g)
    bound = decomp * n * bound_e * max(q_mods) // P + n + 1

    def noise(galois_elt):
        d = dev(ct)
        hb.ApplyGaloisKeySwitch(d, n, decomp, len(mods), decomp + 1, 2, mods, handle, modswitch, galois_elt)
        r = host(d).reshape(2, decomp, n)
        res = np.stack([port.sub_mod(port.ntt_inverse(port.add_mod(r[0, i], port.mult_mod(r[1, i], s_ntt[i], q), q),
                                                      n, q),
                                     np.array([c % q for c in sme], dtype=U64), q) for i, q in enumerate(q_mods)])
        return max(abs(v) for v in _crt_centred(res, q_mods))

    right = noise(g)
    assert right < bound, f"noise {right} is not below the bound {bound}"
    wrong = noise(5 if g != 5 else 7)
    assert wrong > bound << 40, f"a key for another element decrypted with noise {wrong} (bound {bound})"
