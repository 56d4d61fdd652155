"""Parity at the exact shapes BASELINE.json's north_star names (configs[3] and configs[4]) and of
the product's own multi-GPU mechanism (hexl_b200_set_host_devices), through the C ABI.

    C4  FwdNTT -> EltwiseMultMod -> InvNTT, N = 2^17, 16 moduli = GeneratePrimes(16, 60, true, 2^17)
    C5  CKKS KeySwitch, N = 2^15, 30 RNS moduli (decomp_modulus_size 29 + the special prime)
        hexl/experimental/seal/key-switch-internal.cpp:25-201

The checker is the compiled reference when oracle/_ref travelled with the repo, else the C
restatement; every comparison is bit for bit.
"""
import numpy as np
import pytest

from util import uniform_below

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


def dev(a, device="cuda"):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64)).to(device)


def host(t):
    return t.cpu().numpy().view(np.uint64)


@pytest.fixture(scope="module", autouse=True)
def _need_cuda(hb):
    if not torch.cuda.is_available() or hb.device_count() == 0:
        pytest.fail("gpu-marked test collected on a machine without CUDA")


def _c4_case(hb, checker, group):
    n = 1 << 17
    mods = hb.GeneratePrimes(16, 60, True, n)
    assert len(set(mods)) == 16 and all((1 << 60) < q < (1 << 61) for q in mods)
    ntts = [hb.NTT(n, q) for q in mods]
    sz = n * group
    a = np.concatenate([uniform_below(41 * i + 1, sz, q) for i, q in enumerate(mods)])
    b = np.concatenate([uniform_below(41 * i + 2, sz, q) for i, q in enumerate(mods)])
    conv = np.concatenate([
        checker.ntt_inverse(checker.mult_mod(checker.ntt_forward(a[i * sz:(i + 1) * sz], n, q),
                                             checker.ntt_forward(b[i * sz:(i + 1) * sz], n, q), q), n, q)
        for i, q in enumerate(mods)])
    return n, mods, ntts, a, b, conv


def test_c4_poly_multiply_16_moduli_n17(hb, checker):
    """north_star configs[3]: the whole product pipeline as one call, device and host pointers, and as
    the three separate calls a caller of the reference would make (multi-modulus launches)."""
    group = 2
    n, mods, ntts, a, b, conv = _c4_case(hb, checker, group)
    da, db = dev(a), dev(b)
    o = torch.zeros_like(da)
    hb.PolyMultiplyMulti(ntts, o, da, db, group)
    assert (host(o) == conv).all()
    assert (host(da) == a).all() and (host(db) == b).all()
    # the unfused sequence: lazy forward transforms feed EltwiseMultMod(in_mf 4), as in dyadic-multiply / key-switch
    fa, fb = torch.zeros_like(da), torch.zeros_like(da)
    hb.ComputeForwardMulti(ntts, fa, da, 1, 4, batch_per_modulus=group)
    hb.ComputeForwardMulti(ntts, fb, db, 1, 4, batch_per_modulus=group)
    hb.EltwiseMultModMulti(fa, fa, fb, n * group, mods, 4)
    hb.ComputeInverseMulti(ntts, fa, fa, 1, 1, batch_per_modulus=group)
    assert (host(fa) == conv).all()
    # host pointers (an unmodified caller): pageable numpy buffers
    h = np.zeros_like(a)
    hb.PolyMultiplyMulti(ntts, h, a, b, group)
    assert (h == conv).all()
    # per-modulus calls through the single-modulus entry points give the same bits
    q = mods[5]
    lo, hi = 5 * n * group, 6 * n * group
    t = hb.NTT(n, q)
    x, y = dev(a[lo:hi]), dev(b[lo:hi])
    t.ComputeForward(x, x, 1, 4)
    t.ComputeForward(y, y, 1, 4)
    hb.EltwiseMultMod(x, x, y, n * group, q, 4)
    t.ComputeInverse(x, x, 1, 1)
    assert (host(x) == conv[lo:hi]).all()


# The multi-modulus forward transform at N = 2^17 of 64 or more units is the pipelined kernel, one launch; below 64 units
# it is the split, a column pass and a row pass.  C4 in bench.py (16 moduli x 32 polynomials) takes the pipelined kernel;
# these cases run it at 64 units under one modulus set per arithmetic mode: (name, mode, [(count, bits, first)], group).
PIPE_SETS = [("c4_60bit", "wide", [(16, 60, True)], 4),
             ("50_55bit", "fast", [(4, 50, True), (4, 55, True)], 8),
             ("below_2_62", "generic", [(8, 61, False)], 8)]
PIPE_SPREAD = [0, 1, 7, 8, 30, 31, 32, 45, 62, 63]  # units compared with the checker


def _multi_mode(mods):
    """the arithmetic mode launch_ntt_multi picks for a list of moduli"""
    if min(mods) >= 1 << 32 and max(mods) < 1 << 56:
        return "fast"
    return "wide" if max(mods) < 1 << 61 else "generic"


@pytest.mark.parametrize("name,mode,primes,group", PIPE_SETS, ids=[s[0] for s in PIPE_SETS])
def test_multi_forward_n17_pipelined(hb, checker, name, mode, primes, group):
    """ComputeForwardMulti (canonical and lazy outputs) and PolyMultiplyMulti, whose forward transforms take the same
    kernel; PolyMultiplyMulti needs q < 2^61, so not under the GENERIC set."""
    n = 1 << 17
    mods = [q for count, bits, first in primes for q in hb.GeneratePrimes(count, bits, first, n)]
    assert len(set(mods)) == len(mods) and len(mods) * group == 64 and _multi_mode(mods) == mode
    ntts = [hb.NTT(n, q).Prepare() for q in mods]
    sz = n * group
    a = np.concatenate([uniform_below(43 * i + 1, sz, q) for i, q in enumerate(mods)])
    b = np.concatenate([uniform_below(43 * i + 2, sz, q) for i, q in enumerate(mods)])
    da, db = dev(a), dev(b)
    o = torch.zeros_like(da)
    launches = hb.launch_count()
    hb.ComputeForwardMulti(ntts, o, da, 1, 1, batch_per_modulus=group)
    assert hb.launch_count() - launches == 1
    got = host(o)
    exp_f = {u: checker.ntt_forward(a[u * n:(u + 1) * n], n, mods[u // group]) for u in PIPE_SPREAD}
    for u in PIPE_SPREAD:
        assert (got[u * n:(u + 1) * n] == exp_f[u]).all(), ("fwd", name, u)
    hb.ComputeForwardMulti(ntts, o, da, 1, 4, batch_per_modulus=group)
    got = host(o)
    for u in PIPE_SPREAD:
        q = np.uint64(mods[u // group])
        g = got[u * n:(u + 1) * n]
        assert (g % q == exp_f[u]).all() and (g < np.uint64(4) * q).all(), ("fwd lazy", name, u)
    if mode == "generic":
        return
    hb.PolyMultiplyMulti(ntts, o, da, db, group)
    got = host(o)
    for u in PIPE_SPREAD:
        q = mods[u // group]
        fb = checker.ntt_forward(b[u * n:(u + 1) * n], n, q)
        exp = checker.ntt_inverse(checker.mult_mod(exp_f[u], fb, q), n, q)
        assert (got[u * n:(u + 1) * n] == exp).all(), ("poly multiply", name, u)


def _c5_case(hb, n, decomp, bits, kcc=2):
    kms = rns = decomp + 1
    mods = hb.GeneratePrimes(kms, bits, True, n)
    t_target = np.concatenate([uniform_below(30 + j, n, mods[j]) for j in range(decomp)])
    keys = [np.concatenate([uniform_below(1000 * j + 37 * k + i, n, mods[i]) for k in range(kcc) for i in range(kms)])
            for j in range(decomp)]
    result = np.concatenate([uniform_below(5000 + 100 * k + i, n, mods[i]) for k in range(kcc) for i in range(decomp)])
    modswitch = [hb.InverseMod(mods[-1] % mods[i], mods[i]) for i in range(decomp)]
    return kms, rns, kcc, mods, t_target, keys, result, modswitch


def test_c5_key_switch_30_moduli_n15(hb, checker):
    """north_star configs[4]: N = 2^15, L = 30 (29 digits + special prime), 50-bit primes."""
    n, decomp = 1 << 15, 29
    kms, rns, kcc, mods, t_target, keys, result, modswitch = _c5_case(hb, n, decomp, 50)
    exp = checker.key_switch(result.copy(), t_target, n, decomp, kms, rns, kcc, mods, keys, modswitch)
    dres = dev(result)
    hb.KeySwitch(dres, dev(t_target), n, decomp, kms, rns, kcc, mods, [dev(x) for x in keys], modswitch)
    assert (host(dres) == exp).all()
    # host pointers
    res = result.copy()
    hb.KeySwitch(res, t_target, n, decomp, kms, rns, kcc, mods, keys, modswitch)
    assert (res == exp).all()


def test_c5_key_switch_60_bit_moduli(hb, checker):
    """the same shape class with 60-bit primes (WIDE-mode transforms inside the composite), fewer digits"""
    n, decomp = 1 << 15, 9
    kms, rns, kcc, mods, t_target, keys, result, modswitch = _c5_case(hb, n, decomp, 60)
    exp = checker.key_switch(result.copy(), t_target, n, decomp, kms, rns, kcc, mods, keys, modswitch)
    dres = dev(result)
    hb.KeySwitch(dres, dev(t_target), n, decomp, kms, rns, kcc, mods, [dev(x) for x in keys], modswitch)
    assert (host(dres) == exp).all()


# ------------------------------------------------ hexl_b200_set_host_devices: the host-side batch split
def _host_split_cases(hb, checker):
    """(name, run(), expected) for batched host-pointer calls whose unit counts do not divide evenly"""
    n = 1 << 12
    q = hb.GeneratePrimes(1, 55, True, n)[0]
    t = hb.NTT(n, q)
    batch = 37
    x = uniform_below(77, n * batch, q)
    yield "ntt_forward", (lambda: t.ComputeForward(np.zeros_like(x), x, 1, 1)), checker.ntt_forward(x, n, q)
    yield "ntt_inverse", (lambda: t.ComputeInverse(np.zeros_like(x), x, 1, 1)), checker.ntt_inverse(x, n, q)
    big = 3 * (4 << 20) + 12345  # elements: several 32 MiB staging chunks per device
    q2 = hb.GeneratePrimes(1, 60, True, 1)[0]
    a, b = uniform_below(5, big, q2), uniform_below(6, big, q2)
    yield "mult_mod", (lambda: hb.EltwiseMultMod(np.zeros_like(a), a, b, big, q2, 1)), checker.mult_mod(a, b, q2, 1)
    yield "fma_mod", (lambda: hb.EltwiseFMAMod(np.zeros_like(a), a, 12345, b, big, q2, 1)), checker.fma_mod(a, 12345, b, q2, 1)
    yield "reduce_mod", (lambda: hb.EltwiseReduceMod(np.zeros_like(a), a, big, q2 >> 3, q2 >> 3, 1)), a % np.uint64(q2 >> 3)


def test_set_host_devices_single_and_repeated_device(hb, checker):
    """Runs on any box: the split over [0] and over [0, 0] (two blocks on one GPU, sharing its staging
    streams) must give the single-device bits."""
    try:
        for devices in ([0], [0, 0], [0, 0, 0]):
            hb.set_host_devices(devices)
            for name, run, exp in _host_split_cases(hb, checker):
                assert (run() == exp).all(), (devices, name)
    finally:
        hb.set_host_devices([])
    with pytest.raises(hb.HexlB200Error):
        hb.set_host_devices([hb.device_count()])  # out of range


def test_set_host_devices_across_gpus(hb, checker):
    """Two or more GPUs: contiguous blocks of whole units per device, bit-identical to one device;
    the per-device twiddle tables are uploaded on first use on each device."""
    ndev = hb.device_count()
    if ndev < 2:
        pytest.skip("needs at least 2 GPUs")
    try:
        for devices in (list(range(ndev)), [1, 0], list(range(ndev))[::-1]):
            hb.set_host_devices(devices)
            for name, run, exp in _host_split_cases(hb, checker):
                assert (run() == exp).all(), (devices, name)
        # composites take the same split (RNS moduli / ciphertext components are independent units)
        n, mods, ntts, a, b, conv = _c4_case(hb, checker, 1)
        hb.set_host_devices(list(range(ndev)))
        h = np.zeros_like(a)
        hb.PolyMultiplyMulti(ntts, h, a, b, 1)
        assert (h == conv).all()
    finally:
        hb.set_host_devices([])
    # device pointers on a GPU other than the current one: tables follow the data
    n = 1 << 13
    q = hb.GeneratePrimes(1, 50, True, n)[0]
    t = hb.NTT(n, q)
    x = uniform_below(9, n * 3, q)
    with torch.cuda.device(1):
        d = dev(x, "cuda:1")
        t.ComputeForward(d, d, 1, 1)
        torch.cuda.synchronize()
    assert (host(d) == checker.ntt_forward(x, n, q)).all()


# ------------------------------------- composite host paths: chunked, multi-stream staging and resident keys
def test_composite_host_paths_span_many_staging_chunks(hb, checker):
    """Host-pointer RNS calls larger than one 32 MiB staging chunk, with chunk boundaries inside a modulus:
    forward/inverse multi-modulus transforms, the element-wise RNS ops, the product pipeline and DyadicMultiply."""
    n, group = 1 << 14, 96                       # 12 MiB per modulus: a 32 MiB chunk ends inside modulus 2
    mods = [hb.GeneratePrimes(1, b, True, n)[0] for b in (50, 55, 29, 60, 45)]
    ntts = [hb.NTT(n, q) for q in mods]
    sz = n * group
    a = np.concatenate([uniform_below(11 * i + 1, sz, q) for i, q in enumerate(mods)])
    b = np.concatenate([uniform_below(11 * i + 2, sz, q) for i, q in enumerate(mods)])
    exp_f = np.concatenate([checker.ntt_forward(a[i * sz:(i + 1) * sz], n, q) for i, q in enumerate(mods)])
    h = np.zeros_like(a)
    hb.ComputeForwardMulti(ntts, h, a, 1, 1, batch_per_modulus=group)
    assert (h == exp_f).all()
    hb.ComputeInverseMulti(ntts, h, h, 1, 1, batch_per_modulus=group)       # in place
    assert (h == a).all()
    prod = np.concatenate([checker.mult_mod(a[i * sz:(i + 1) * sz], b[i * sz:(i + 1) * sz], q) for i, q in enumerate(mods)])
    hb.EltwiseMultModMulti(h, a, b, sz, mods)
    assert (h == prod).all()
    for fn, ref in ((hb.EltwiseAddModMulti, checker.add_mod), (hb.EltwiseSubModMulti, checker.sub_mod)):
        exp = np.concatenate([ref(a[i * sz:(i + 1) * sz], b[i * sz:(i + 1) * sz], q) for i, q in enumerate(mods)])
        fn(h, a, b, sz, mods)
        assert (h == exp).all()
    fast = [q for q in mods if q < (1 << 61)]
    conv = np.concatenate([
        checker.ntt_inverse(checker.mult_mod(checker.ntt_forward(a[i * sz:(i + 1) * sz], n, q),
                                             checker.ntt_forward(b[i * sz:(i + 1) * sz], n, q), q), n, q)
        for i, q in enumerate(fast)])
    k = len(fast) * sz
    aa, bb = a[:k].copy(), b[:k].copy()
    hb.PolyMultiplyMulti(ntts[:len(fast)], h[:k], aa, bb, group)
    assert (h[:k] == conv).all() and (aa == a[:k]).all() and (bb == b[:k]).all()
    hb.PolyMultiplyMulti(ntts[:len(fast)], bb, aa, bb, group)                  # result aliases b
    assert (bb == conv).all()
    # DyadicMultiply: 70 moduli (more than one parameter block and several staging rounds)
    dn = 1 << 13
    dm = hb.GeneratePrimes(70, 50, True, dn)
    x = np.concatenate([uniform_below(10 + i, dn, q) for _ in range(2) for i, q in enumerate(dm)])
    y = np.concatenate([uniform_below(300 + i, dn, q) for _ in range(2) for i, q in enumerate(dm)])
    out = np.zeros(3 * dn * len(dm), dtype=np.uint64)
    hb.DyadicMultiply(out, x, y, dn, dm)
    assert (out == checker.dyadic_multiply(x, y, dn, dm)).all()


def test_key_switch_resident_keys_and_batches(hb, checker):
    """hexl_b200_keys_upload + hexl_b200_key_switch_resident: several ciphertexts per call against keys uploaded
    once, host buffers (pipelined over the staging streams) and device buffers, against the reference per ciphertext;
    and refusals, one of them part-way through a host batch."""
    n, decomp, batch = 1 << 13, 7, 5
    kms, rns, kcc, mods, _, keys, _, modswitch = _c5_case(hb, n, decomp, 50)
    t_all = np.concatenate([np.concatenate([uniform_below(900 * c + j, n, mods[j]) for j in range(decomp)])
                            for c in range(batch)])
    r_all = np.concatenate([np.concatenate([uniform_below(7000 * c + 10 * k + i, n, mods[i]) for k in range(kcc)
                                            for i in range(decomp)]) for c in range(batch)])
    res_sz, t_sz = kcc * decomp * n, decomp * n
    exp = np.concatenate([checker.key_switch(r_all[c * res_sz:(c + 1) * res_sz].copy(), t_all[c * t_sz:(c + 1) * t_sz], n,
                                             decomp, kms, rns, kcc, mods, keys, modswitch) for c in range(batch)])
    handle = hb.KeySwitchKeys(keys, n, decomp, kms, kcc)                       # from host buffers
    got = r_all.copy()
    hb.KeySwitchResident(got, t_all, n, decomp, kms, rns, kcc, mods, handle, modswitch, batch)
    assert (got == exp).all()
    d = dev(r_all)
    hb.KeySwitchResident(d, dev(t_all), n, decomp, kms, rns, kcc, mods, handle, modswitch, batch)
    assert (host(d) == exp).all()
    handle2 = hb.KeySwitchKeys([dev(k) for k in keys], n, decomp, kms, kcc)    # from device buffers
    got = r_all[:res_sz].copy()
    hb.KeySwitchResident(got, t_all[:t_sz], n, decomp, kms, rns, kcc, mods, handle2, modswitch)
    assert (got == exp[:res_sz]).all()
    with pytest.raises(hb.HexlB200Error):                                     # shape mismatch is refused
        hb.KeySwitchResident(got, t_all[:t_sz], n // 2, decomp, kms, rns, kcc, mods, handle2, modswitch)
    # a digit modulus >= 2^61 is refused inside the switch of the first ciphertext, after its copies are queued, on a
    # batch split over two blocks: result stays as it was, and the next call is right
    try:
        hb.set_host_devices([0, 0])
        h_split = hb.KeySwitchKeys(keys, n, decomp, kms, kcc)
        got = r_all.copy()
        with pytest.raises(hb.HexlB200Error) as e:
            hb.KeySwitchResident(got, t_all, n, decomp, kms, rns, kcc, [(1 << 61) + 1] + list(mods[1:]), h_split,
                                 modswitch, batch)
        assert e.value.code == -1 and "KeySwitch: Require moduli < 2^61 (slot 0)" in str(e.value), e.value
        assert (got == r_all).all(), "a refused call wrote"
        hb.KeySwitchResident(got, t_all, n, decomp, kms, rns, kcc, mods, h_split, modswitch, batch)
        assert (got == exp).all()
    finally:
        hb.set_host_devices([])
    ndev = hb.device_count()
    if ndev >= 2:                                                             # keys on every device, batch split
        try:
            hb.set_host_devices(list(range(ndev)))
            h3 = hb.KeySwitchKeys(keys, n, decomp, kms, kcc)
            got = r_all.copy()
            hb.KeySwitchResident(got, t_all, n, decomp, kms, rns, kcc, mods, h3, modswitch, batch)
            assert (got == exp).all()
        finally:
            hb.set_host_devices([])


def test_cold_handle_inside_a_capture_is_refused_and_prepare_fixes_it(hb, checker):
    """The first transform of a handle on a device uploads its tables synchronously, which a stream capture
    forbids: the call reports that instead of killing the capture; NTT.Prepare() warms the handle."""
    n = 1 << 11
    q = hb.GeneratePrimes(1, 47, True, n)[0]
    x = uniform_below(4, n, q)
    d, o = dev(x), dev(np.zeros_like(x))
    cold = hb.NTT(n, q)
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        g = torch.cuda.CUDAGraph()
        g.capture_begin()
        with pytest.raises(hb.HexlB200Error):
            cold.ComputeForward(o, d, 1, 1)
        cold_ok = hb.NTT(n, q)
        g.capture_end()
    warm = hb.NTT(n, q).Prepare()
    g2 = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g2):
        warm.ComputeForward(o, d, 1, 1)
    g2.replay()
    torch.cuda.synchronize()
    assert (host(o) == checker.ntt_forward(x, n, q)).all()


def test_key_switch_sharded_by_modulus(hb, checker):
    """hexl_b200_keys_upload_sharded: the RNS moduli of ONE key switch spread over several shards (one per listed
    device; listing device 0 several times puts several shards on one GPU, so the exchange logic -- digit all-gather,
    special-prime broadcast, cross-stream events -- runs on any box), bit for bit against the reference; uneven splits,
    a shard that owns only the special prime, more shards than moduli, key_modulus_size > rns_modulus_size."""
    ndev = hb.device_count()
    layouts = [[0], [0, 0], [0, 0, 0], [0] * 9]
    if ndev >= 2:
        layouts += [list(range(ndev)), [1, 0, 1]]
    for n, decomp, extra_slots in ((1 << 12, 7, 0), (1 << 13, 2, 0), (1 << 12, 5, 2)):
        kcc = 2
        rns = decomp + 1
        kms = rns + extra_slots
        mods = hb.GeneratePrimes(kms, 50, True, n)
        if extra_slots:   # unused middle slots: the special prime is the LAST modulus (key-switch-internal.cpp:62-63)
            mods = mods[:decomp] + mods[rns:] + [mods[decomp]]
        t_target = np.concatenate([uniform_below(30 + j, n, mods[j]) for j in range(decomp)])
        keys = [np.concatenate([uniform_below(1000 * j + 37 * k + i, n, mods[i]) for k in range(kcc) for i in range(kms)])
                for j in range(decomp)]
        result = np.concatenate([uniform_below(5000 + 100 * k + i, n, mods[i]) for k in range(kcc) for i in range(decomp)])
        modswitch = [hb.InverseMod(mods[-1] % mods[i], mods[i]) for i in range(decomp)]
        exp = checker.key_switch(result.copy(), t_target, n, decomp, kms, rns, kcc, mods, keys, modswitch)
        for devices in layouts:
            try:
                hb.set_host_devices(devices)
                handle = hb.KeySwitchKeys(keys, n, decomp, kms, kcc, sharded_by_modulus=True)
            finally:
                hb.set_host_devices([])
            got = np.concatenate([result, result])
            hb.KeySwitchResident(got, np.concatenate([t_target, t_target]), n, decomp, kms, rns, kcc, mods, handle, modswitch, 2)
            assert (got[:result.size] == exp).all() and (got[result.size:] == exp).all(), (n, decomp, devices)
            with pytest.raises(hb.HexlB200Error):   # a sharded handle serves host buffers only
                hb.KeySwitchResident(dev(result), dev(t_target), n, decomp, kms, rns, kcc, mods, handle, modswitch)
            del handle


def test_key_switch_sharded_copy_engine_exchange():
    """By default the sharded key switch all-gathers its digits with P2P stores from the inverse transform's last kernel
    (NttMulti::mirror); HEXL_B200_KS_PEER_COPIES=1 selects the copy-engine exchange (cudaMemcpyPeerAsync behind the
    transform), which is also what runs between GPUs without peer access.  The switch is read once per process."""
    import os
    import subprocess
    import sys
    here = os.path.abspath(__file__)
    res = subprocess.run([sys.executable, "-m", "pytest", here, "-m", "gpu", "-x", "-q", "-k", "test_key_switch_sharded_by_modulus"],
                         env={**os.environ, "HEXL_B200_KS_PEER_COPIES": "1"}, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0 and "1 passed" in res.stdout, res.stdout[-2000:] + res.stderr[-2000:]
