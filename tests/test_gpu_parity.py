"""Parity of the sm_90a path against the oracle, through the C ABI.

Bar: bit-exact for every canonical output (NTT out_mf == 1, every eltwise op);
for the lazy outputs (forward out_mf == 4, inverse out_mf == 2, ReduceMod q->2)
congruent mod q and inside the advertised range -- the reference's own tests
compare lazy outputs only mod q (test/test-ntt.cpp:246-251,279-286) because its
tiers disagree bit-wise there.  The checker is the compiled reference when
oracle/_ref travelled with the repo, else the C restatement.
"""
import numpy as np
import pytest

from util import kat_modulus, kat_values, uniform_below

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64)).cuda()


def host(t):
    return t.cpu().numpy().view(np.uint64)


@pytest.fixture(scope="module", autouse=True)
def _need_cuda(hb):
    if not torch.cuda.is_available() or hb.device_count() == 0:
        pytest.fail("gpu-marked test collected on a machine without CUDA")


# ---------------------------------------------------------------- NTT: KATs
def test_ntt_reference_kats(hb, kats):
    """test/test-ntt.cpp:231-355 on the 14 tuples of :357-404, device and host buffers."""
    for c in kats["ntt_forward"]["cases"]:
        n, q = c["n"], c["q"]
        x = np.array(c["input"], dtype=np.uint64)
        exp = np.array(c["output"], dtype=np.uint64)
        t = hb.NTT(n, q)
        # in-place forward on the device
        d = dev(x)
        t.ComputeForward(d, d, 1, 1)
        assert (host(d) == exp).all(), c
        # lazy forward, compared mod q
        d = dev(x)
        t.ComputeForward(d, d, 2, 4)
        assert (host(d) % np.uint64(q) == exp).all() and (host(d) < np.uint64(4 * q)).all(), c
        # out of place + round trip
        o, d = dev(np.zeros_like(x)), dev(x)
        t.ComputeForward(o, d, 2, 1)
        assert (host(o) == exp).all() and (host(d) == x).all()
        t.ComputeInverse(d, o, 1, 1)
        assert (host(d) == x).all()
        t.ComputeInverse(d, o, 1, 2)
        assert (host(d) % np.uint64(q) == x).all() and (host(d) < np.uint64(2 * q)).all()
        # host-pointer path (what an unmodified caller of the reference API uses)
        y = np.zeros_like(x)
        t.ComputeForward(y, x, 1, 1)
        assert (y == exp).all()
        t.ComputeInverse(y, y, 1, 1)
        assert (y == x).all()


# ------------------------------------------- NTT: every size against the oracle
SIZES = [(1, 48), (2, 20), (3, 22), (4, 29), (5, 31), (6, 33), (7, 40), (8, 48), (9, 49), (10, 30),
         (10, 61), (11, 50), (12, 51), (12, 61), (13, 58), (13, 30), (14, 59), (14, 61), (15, 50), (16, 55),
         (16, 61), (17, 60), (17, 61), (18, 55), (19, 61), (20, 50),  # 2^20 = the reference's maximum degree
         # q < 2^30: the 32-bit-word kernels (GeneratePrimes(bits) returns primes just above 2^bits)
         (4, 12), (6, 20), (8, 29), (10, 29), (11, 22), (12, 28), (13, 29), (14, 25), (15, 29), (16, 29), (17, 29),
         (18, 29)]


@pytest.mark.parametrize("logn,bits", SIZES)
def test_ntt_matches_oracle(hb, checker, logn, bits):
    n = 1 << logn
    q = hb.GeneratePrimes(1, bits, True, n)[0]
    qq = np.uint64(q)
    t = hb.NTT(n, q)
    batch = max(1, min(37, (1 << 16) // n))  # ragged batch: not a multiple of the CTA packing
    for in_mf, out_mf in [(1, 1), (4, 1), (2, 4)]:
        x = uniform_below(logn * 10 + in_mf, n * batch, q * in_mf)
        exp = checker.ntt_forward(x, n, q, in_mf, 1)
        o = dev(np.zeros_like(x))
        t.ComputeForward(o, dev(x), in_mf, out_mf)
        got = host(o)
        if out_mf == 1:
            assert (got == exp).all(), (logn, in_mf, out_mf, int((got != exp).sum()))
        else:
            assert (got % qq == exp).all() and (got < np.uint64(4 * q)).all()
    for in_mf, out_mf in [(1, 1), (2, 1), (2, 2)]:
        x = uniform_below(logn * 20 + in_mf, n * batch, q * in_mf)
        exp = checker.ntt_inverse(x, n, q, in_mf, 1)
        o = dev(np.zeros_like(x))
        t.ComputeInverse(o, dev(x), in_mf, out_mf)
        got = host(o)
        if out_mf == 1:
            assert (got == exp).all(), (logn, in_mf, out_mf, int((got != exp).sum()))
        else:
            assert (got % qq == exp).all() and (got < np.uint64(2 * q)).all()
    # in place, device
    x = uniform_below(logn, n * batch, q)
    d = dev(x)
    t.ComputeForward(d, d, 1, 1)
    assert (host(d) == checker.ntt_forward(x, n, q)).all()
    t.ComputeInverse(d, d, 1, 1)
    assert (host(d) == x).all()


def test_device_calls_capture_into_a_cuda_graph(hb, checker):
    """Device-pointer calls only enqueue kernels on the caller's stream (no allocation,
    no synchronisation), so a FwdNTT -> MultMod -> InvNTT product can be captured once
    and replayed; the replayed graph is compared with the oracle on fresh inputs."""
    n, batch = 1 << 13, 6
    q = hb.GeneratePrimes(1, 50, True, n)[0]
    t = hb.NTT(n, q)
    a = torch.zeros(batch * n, dtype=torch.int64, device="cuda")
    b = torch.zeros_like(a)
    fa, fb, out = torch.empty_like(a), torch.empty_like(a), torch.empty_like(a)

    def product():
        t.ComputeForward(fa, a, 1, 4)
        t.ComputeForward(fb, b, 1, 4)
        hb.EltwiseMultMod(fa, fa, fb, batch * n, q, 4)
        t.ComputeInverse(out, fa, 1, 1)

    product()  # first use uploads the tables; not part of the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        product()
    for seed in (1, 2):
        x, y = uniform_below(seed, n * batch, q), uniform_below(seed + 10, n * batch, q)
        a.copy_(dev(x))
        b.copy_(dev(y))
        g.replay()
        torch.cuda.synchronize()
        exp = checker.ntt_inverse(
            checker.mult_mod(checker.ntt_forward(x, n, q), checker.ntt_forward(y, n, q), q), n, q)
        assert (host(out) == exp).all()


def test_ntt_extreme_inputs(hb, checker):
    """all-zero, all q-1, and lazy inputs at the top of their range (4q-1 / 2q-1), at the
    largest modulus of each arithmetic mode: q just below 2^62 (GENERIC butterflies) and
    q just below 2^56 (FAST butterflies, where the lazy ranges come closest to 2^64),
    including N = 2^17 whose column pass runs 5 unreduced stages."""
    # 60: q just below 2^61, 8q just below 2^64 (WIDE butterflies); 29: q just below 2^30 (32-bit-word kernels)
    for bits in (61, 60, 55, 29):
        for logn in (4, 10, 12, 15, 17):
            n = 1 << logn
            q = hb.GeneratePrimes(1, bits, False, n)[0]  # largest primes below 2^(bits+1)
            assert q < (1 << (bits + 1)) and q > (1 << (bits + 1)) - (1 << 40)
            t = hb.NTT(n, q)
            for fill, in_mf in [(0, 1), (q - 1, 1), (4 * q - 1, 4), (2 * q - 1, 2)]:
                x = np.full(n, fill, dtype=np.uint64)
                x[1::3] = 0  # mix extremes so sums and differences both hit their bounds
                o = dev(np.zeros_like(x))
                t.ComputeForward(o, dev(x), in_mf, 1)
                assert (host(o) == checker.ntt_forward(x, n, q, in_mf, 1)).all(), (bits, logn, fill)
                if in_mf <= 2:
                    t.ComputeInverse(o, dev(x), in_mf, 1)
                    assert (host(o) == checker.ntt_inverse(x, n, q, in_mf, 1)).all(), (bits, logn, fill)
                    t.ComputeInverse(o, dev(x), in_mf, 2)
                    got = host(o)
                    assert (got % np.uint64(q) == checker.ntt_inverse(x, n, q, in_mf, 1)).all()
                    assert (got < np.uint64(2 * q)).all()


def test_ntt_kernel_variants():
    """The pipelined kernels with a pipeline one polynomial deep, so that consumers actually wait on their producers'
    release/acquire handshake (at the default depth of 16 the producers finished long before).  The depth is read
    once per process, so tests/variant_check.py runs in its own process."""
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    res = subprocess.run([sys.executable, os.path.join(here, "variant_check.py")],
                         env={**os.environ, "HEXL_B200_PIPE_LOOKAHEAD": "1"}, capture_output=True, text=True,
                         timeout=600)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-2000:]
    assert "variant ok" in res.stdout


def test_unified_memory_buffers(hb, checker):
    """hexl_b200_managed_alloc: the host fills and reads the buffers directly, the kernels
    work on them in place, and a call without a stream returns with the result complete."""
    n, batch = 1 << 12, 3
    q = hb.GeneratePrimes(1, 55, True, n)[0]
    t = hb.NTT(n, q)
    a, b, r = hb.managed_empty(n * batch), hb.managed_empty(n * batch), hb.managed_empty(n * batch)
    try:
        x, y = uniform_below(5, n * batch, q), uniform_below(6, n * batch, q)
        a[:] = x
        b[:] = y
        t.ComputeForward(r, a, 1, 1)
        assert (r == checker.ntt_forward(x, n, q)).all()
        hb.EltwiseMultMod(r, a, b, n * batch, q, 1)
        assert (r == checker.mult_mod(x, y, q)).all()
        t.ComputeInverse(a, a, 1, 1)  # in place
        assert (a == checker.ntt_inverse(x, n, q)).all()
    finally:
        for arr in (a, b, r):
            hb.managed_free(arr)


@pytest.mark.parametrize("logn,group", [(2, 3), (3, 1), (6, 5), (10, 3), (12, 2), (13, 1), (14, 2), (16, 1)])
def test_multi_modulus_launch_matches_oracle(hb, checker, logn, group):
    """hexl_b200_ntt_forward/inverse_multi: polynomial u under ntts[u // group]; moduli of all
    three arithmetic classes mixed in one call (the launch then runs the GENERIC butterflies)
    and a FAST-only list; device and host pointers."""
    n = 1 << logn
    for bit_list in ([max(logn + 2, 20), 45, 61, 50, 29 if logn < 28 else 40], [40, 50, 55]):
        mods = [hb.GeneratePrimes(1, b, True, n)[0] for b in bit_list]
        ntts = [hb.NTT(n, q) for q in mods]
        x = np.concatenate([uniform_below(7 * i + logn, n * group, q) for i, q in enumerate(mods)])
        exp_f = np.concatenate([checker.ntt_forward(x[i * n * group:(i + 1) * n * group], n, q)
                                for i, q in enumerate(mods)])
        exp_i = np.concatenate([checker.ntt_inverse(x[i * n * group:(i + 1) * n * group], n, q)
                                for i, q in enumerate(mods)])
        o = dev(np.zeros_like(x))
        hb.ComputeForwardMulti(ntts, o, dev(x), 1, 1)
        assert (host(o) == exp_f).all(), (logn, bit_list)
        hb.ComputeInverseMulti(ntts, o, dev(x), 1, 1, batch_per_modulus=group)
        assert (host(o) == exp_i).all(), (logn, bit_list)
        d = dev(x)  # in place round trip, lazy forward output feeding the inverse is not allowed (< 4q): use 1
        hb.ComputeForwardMulti(ntts, d, d)
        hb.ComputeInverseMulti(ntts, d, d)
        assert (host(d) == x).all()
        y = np.zeros_like(x)  # host pointers: staged per modulus
        hb.ComputeForwardMulti(ntts, y, x)
        assert (y == exp_f).all()


@pytest.mark.parametrize("logn,group,nmods", [(3, 2, 3), (8, 3, 5), (12, 2, 4), (15, 1, 3), (7, 1, 70)])
def test_rns_product_pipeline_matches_oracle(hb, checker, logn, group, nmods):
    """hexl_b200_eltwise_mult_mod_multi and hexl_b200_poly_multiply_multi against the oracle's
    FwdNTT -> EltwiseMultMod -> InvNTT per modulus (BASELINE configs[3]); result separate,
    aliasing a, aliasing b; device and host pointers."""
    n = 1 << logn
    bits = [max(logn + 2, 20), 50, 60, 40, 29][:min(nmods, 5)]
    mods = [hb.GeneratePrimes(1, bb, True, n)[0] for bb in bits]
    if nmods > 5:
        mods += [q for q in hb.GeneratePrimes(nmods, 45, True, n) if q not in mods][:nmods - 5]
    ntts = [hb.NTT(n, q) for q in mods]
    sz = n * group
    a = np.concatenate([uniform_below(3 * i + 1, sz, q) for i, q in enumerate(mods)])
    b = np.concatenate([uniform_below(3 * i + 2, sz, q) for i, q in enumerate(mods)])
    prod = np.concatenate([checker.mult_mod(a[i * sz:(i + 1) * sz], b[i * sz:(i + 1) * sz], q) for i, q in enumerate(mods)])
    o = dev(np.zeros_like(a))
    hb.EltwiseMultModMulti(o, dev(a), dev(b), sz, mods)
    assert (host(o) == prod).all()
    h = np.zeros_like(a)
    hb.EltwiseMultModMulti(h, a, b, sz, mods)
    assert (h == prod).all()
    for fn, ref in ((hb.EltwiseAddModMulti, checker.add_mod), (hb.EltwiseSubModMulti, checker.sub_mod)):
        exp = np.concatenate([ref(a[i * sz:(i + 1) * sz], b[i * sz:(i + 1) * sz], q) for i, q in enumerate(mods)])
        fn(o, dev(a), dev(b), sz, mods)
        assert (host(o) == exp).all()
    conv = np.concatenate([
        checker.ntt_inverse(checker.mult_mod(checker.ntt_forward(a[i * sz:(i + 1) * sz], n, q),
                                             checker.ntt_forward(b[i * sz:(i + 1) * sz], n, q), q), n, q)
        for i, q in enumerate(mods)])
    da, db = dev(a), dev(b)
    hb.PolyMultiplyMulti(ntts, o, da, db, group)
    assert (host(o) == conv).all() and (host(da) == a).all() and (host(db) == b).all()
    hb.PolyMultiplyMulti(ntts, da, da, db)  # result aliases a
    assert (host(da) == conv).all()
    da = dev(a)
    hb.PolyMultiplyMulti(ntts, db, da, db)  # result aliases b
    assert (host(db) == conv).all() and (host(da) == a).all()
    hb.PolyMultiplyMulti(ntts, h, a, b, group)  # host pointers
    assert (h == conv).all()


@pytest.mark.parametrize("logn", [1, 3, 4, 9, 12, 13, 16])
@pytest.mark.parametrize("bits", [[50, 55], [60, 60], [33, 60], [20, 50]])
def test_product_multiplied_on_load_extremes(hb, checker, logn, bits):
    """The inverse transform that multiplies on load (NttMulti::mul; dyadic-multiply-internal.cpp:17-73 folded into the
    transform): all three 64-bit butterfly classes ([50,55] FAST, [60,60] and mixed WIDE), every kernel shape (one thread
    per polynomial, single row kernel, row + column kernels), operands at 0 / 1 / q-1 / random, against the checker."""
    n = 1 << logn
    mods = []
    for bb in bits:
        mods += [q for q in hb.GeneratePrimes(2, max(bb, logn + 6), True, n) if q not in mods][:1]
    ntts = [hb.NTT(n, q) for q in mods]
    group = 3
    sz = n * group
    parts_a, parts_b = [], []
    for i, q in enumerate(mods):
        a = uniform_below(40 + i, sz, q)
        b = uniform_below(50 + i, sz, q)
        a[:n] = q - 1                      # first polynomial: all q-1 times all q-1
        b[:n] = q - 1
        b[n:n + n // 2] = 0                # second: zeros, ones and q-1 mixed with random values
        b[n + n // 2:2 * n] = 1
        a[n:2 * n:2] = q - 1
        parts_a.append(a)
        parts_b.append(b)
    a, b = np.concatenate(parts_a), np.concatenate(parts_b)
    conv = np.concatenate([
        checker.ntt_inverse(checker.mult_mod(checker.ntt_forward(a[i * sz:(i + 1) * sz], n, q),
                                             checker.ntt_forward(b[i * sz:(i + 1) * sz], n, q), q), n, q)
        for i, q in enumerate(mods)])
    o = dev(np.zeros_like(a))
    hb.PolyMultiplyMulti(ntts, o, dev(a), dev(b), group)
    assert (host(o) == conv).all()
    h = np.zeros_like(a)
    hb.PolyMultiplyMulti(ntts, h, a, b, group)      # host pointers: per-modulus segments
    assert (h == conv).all()


def test_unfused_product_chain_still_matches():
    """HEXL_B200_NO_PRODUCT_FUSION=1 selects the chain of lazy transforms + MultMod kernel + inverse (read once per process)."""
    import os
    import subprocess
    import sys
    here = os.path.abspath(__file__)
    res = subprocess.run([sys.executable, "-m", "pytest", here, "-m", "gpu", "-x", "-q", "-k",
                          "test_rns_product_pipeline_matches_oracle or test_product_multiplied_on_load_extremes"],
                         env={**os.environ, "HEXL_B200_NO_PRODUCT_FUSION": "1"}, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0 and " passed" in res.stdout, res.stdout[-2000:] + res.stderr[-2000:]


def test_multi_modulus_more_than_one_parameter_block(hb, checker):
    n, group = 256, 2
    mods = hb.GeneratePrimes(70, 40, True, n)
    ntts = [hb.NTT(n, q) for q in mods]
    x = np.concatenate([uniform_below(i, n * group, q) for i, q in enumerate(mods)])
    o = dev(np.zeros_like(x))
    hb.ComputeForwardMulti(ntts, o, dev(x))
    exp = np.concatenate([checker.ntt_forward(x[i * n * group:(i + 1) * n * group], n, q) for i, q in enumerate(mods)])
    assert (host(o) == exp).all()


def test_concurrent_host_threads(hb, checker):
    """The reference is "single-threaded and thread-safe" (README.md:264-265): many host
    threads may call it at once.  Eight threads share one NTT object and the NTT cache and
    mix device-pointer calls (each on its own stream), host-pointer calls (which share the
    per-device staging buffers) and lookups in the NTT cache that race with its first
    creation of a handle; ctypes drops the GIL for the duration of every call, so the calls
    really overlap.  No composite runs here: the rotations from several threads, sharing
    the scratch pool and the staging slots, are in test_gpu_rotation_shapes.py."""
    import threading
    n = 1 << 12
    q = hb.GeneratePrimes(1, 55, True, n)[0]
    shared = hb.NTT(n, q)
    mods = hb.GeneratePrimes(3, 45, True, n)
    errors = []

    def worker(tid):
        try:
            stream = torch.cuda.Stream()
            for it in range(6):
                batch = 1 + (tid + it) % 4
                x = uniform_below(100 * tid + it, n * batch, q)
                exp = checker.ntt_forward(x, n, q)
                if (tid + it) % 2 == 0:
                    with torch.cuda.stream(stream):
                        d = dev(x)
                        o = torch.empty_like(d)
                        shared.ComputeForward(o, d, 1, 1, stream=stream)
                        hb.EltwiseAddMod(o, o, o, n * batch, q, stream=stream)
                        stream.synchronize()
                    got = host(o)
                    exp = (exp + exp) % np.uint64(q)
                else:
                    got = np.zeros_like(x)
                    shared.ComputeForward(got, x, 1, 1)
                assert (got == exp).all(), (tid, it)
                cached = hb.GetNTT(n, mods[(tid + it) % 3])  # cache hit or first creation, racing with the others
                y = uniform_below(tid + 1000 * it, n, cached.GetModulus())
                back = np.zeros_like(y)
                cached.ComputeForward(back, y, 1, 1)
                cached.ComputeInverse(back, back, 1, 1)
                assert (back == y).all(), (tid, it)
        except Exception as exc:  # noqa: BLE001 - reported by the main thread
            errors.append((tid, repr(exc)))

    threads = [threading.Thread(target=worker, args=(t,)) for t in range(8)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors


def test_ntt_user_root(hb, checker):
    n = 256
    q = hb.GeneratePrimes(1, 40, True, n)[0]
    root = hb.PowMod(hb.MinimalPrimitiveRoot(2 * n, q), 5, q)
    t = hb.NTT(n, q, root)
    x = uniform_below(5, n, q)
    o = dev(np.zeros_like(x))
    t.ComputeForward(o, dev(x), 1, 1)
    assert (host(o) == checker.ntt_forward(x, n, q, 1, 1, root=root)).all()


def test_ntt_linearity_and_roundtrip_full_size(hb):
    """Size-independent properties at BASELINE's N = 2^16 / 55-bit, on a batch
    large enough to span many waves: Inv(Fwd(x)) == x, and Fwd is linear."""
    n = 1 << 16
    q = hb.GeneratePrimes(1, 55, True, n)[0]
    t = hb.NTT(n, q)
    batch = 512
    g = torch.Generator(device="cuda").manual_seed(1)
    a = torch.randint(0, q, (batch, n), dtype=torch.int64, device="cuda", generator=g)
    b = torch.randint(0, q, (batch, n), dtype=torch.int64, device="cuda", generator=g)
    fa, fb, fs = torch.empty_like(a), torch.empty_like(a), torch.empty_like(a)
    s = torch.empty_like(a)
    hb.EltwiseAddMod(s, a, b, a.numel(), q)
    t.ComputeForward(fa, a, 1, 1)
    t.ComputeForward(fb, b, 1, 1)
    t.ComputeForward(fs, s, 1, 1)
    hb.EltwiseAddMod(fa, fa, fb, a.numel(), q)
    assert torch.equal(fa, fs)
    t.ComputeInverse(fs, fs, 1, 1)
    assert torch.equal(fs, s)
    assert int(fs.max()) < q and int(fs.min()) >= 0


def test_ntt_host_pointer_batches(hb, checker):
    """host buffers, batch spanning several staging chunks, pinned and pageable"""
    n = 1 << 12
    q = hb.GeneratePrimes(1, 50, True, n)[0]
    t = hb.NTT(n, q)
    batch = 3000  # 96 MB > 32 MiB chunks x 3 slots
    x = uniform_below(77, n * batch, q)
    exp = checker.ntt_forward(x, n, q)
    y = np.zeros_like(x)
    t.ComputeForward(y, x, 1, 1)
    assert (y == exp).all()
    px = hb.pinned_empty(n * batch)
    px[:] = x
    t.ComputeForward(px, px, 1, 1)
    assert (px == exp).all()
    t.ComputeInverse(px, px, 1, 1)
    assert (px == x).all()
    hb.pinned_free(px)


def test_mixed_pointers_rejected(hb):
    t = hb.NTT(16, hb.GeneratePrimes(1, 30, True, 16)[0])
    x = np.zeros(16, dtype=np.uint64)
    with pytest.raises(hb.HexlB200Error) as ei:
        t.ComputeForward(dev(x), x, 1, 1)
    assert ei.value.code == -5


def test_debug_bounds_checks(hb):
    """HEXL_DEBUG-style range checks (check.hpp:33-36; test-eltwise-mult-mod.cpp:66-76)"""
    hb.set_debug(True)
    try:
        q = 769
        t = hb.NTT(8, q)
        bad = dev(np.array([0, 1, 2, 3, 4, 5, 6, 770], dtype=np.uint64))
        good = dev(np.arange(8, dtype=np.uint64))
        with pytest.raises(hb.HexlB200Error):
            t.ComputeForward(good.clone(), bad, 1, 1)
        t.ComputeForward(good.clone(), bad, 2, 1)  # 770 < 2q is fine
        with pytest.raises(hb.HexlB200Error):
            hb.EltwiseMultMod(good.clone(), good, bad, 8, q, 1)
        with pytest.raises(hb.HexlB200Error):
            hb.EltwiseAddMod(good.clone(), bad, good, 8, q)
        with pytest.raises(hb.HexlB200Error):
            hb.EltwiseFMAMod(np.zeros(8, dtype=np.uint64), host(bad), 1, None, 8, q, 1)
    finally:
        hb.set_debug(False)


# ------------------------------------------------------------- eltwise: KATs
def test_eltwise_reference_kats(hb, kats):
    gp = hb.GeneratePrimes
    for c in kats["eltwise_mult_mod"]["cases"]:
        q = kat_modulus(c["q"], gp)
        a, b = kat_values(c["op1"], q), kat_values(c["op2"], q)
        d = dev(a)
        hb.EltwiseMultMod(d, d, dev(b), len(a), q, c["in_mf"])  # in place, as the reference tests
        assert (host(d) == kat_values(c["out"], q)).all(), c
        r = np.zeros_like(a)
        hb.EltwiseMultMod(r, a, b, len(a), q, c["in_mf"])  # host pointers
        assert (r == kat_values(c["out"], q)).all(), c
    for c in kats["eltwise_fma_mod"]["cases"]:
        q = c["q"]
        a1 = kat_values(c["arg1"], q)
        a3 = None if c["arg3"] is None else dev(kat_values(c["arg3"], q))
        d = dev(a1)
        hb.EltwiseFMAMod(d, d, c["arg2"], a3, len(a1), q, c["in_mf"])
        assert (host(d) == kat_values(c["out"], q)).all(), c
    s = kats["eltwise_fma_mod"]["in_mf_sweep"]
    for mf in s["in_mfs"]:
        q = s["q"]
        a1 = kat_values(s["arg1_base"], q) + np.uint64((mf - 1) * q)
        d = dev(a1)
        hb.EltwiseFMAMod(d, d, s["arg2"], dev(kat_values(s["arg3"], q)), len(a1), q, mf)
        assert (host(d) == kat_values(s["out"], q)).all(), mf
    for c in kats["eltwise_reduce_mod"]["cases"]:
        q = c["q"]
        in_mf = q if c["in_mf"] == "q" else c["in_mf"]
        op = kat_values(c["op"], q)
        r = dev(np.zeros_like(op))
        hb.EltwiseReduceMod(r, dev(op), len(op), q, in_mf, c["out_mf"])
        assert (host(r) == kat_values(c["out"], q)).all(), c
    for name, fn in (("eltwise_add_mod", hb.EltwiseAddMod), ("eltwise_sub_mod", hb.EltwiseSubMod)):
        for c in kats[name]["cases"]:
            q = kat_modulus(c["q"], gp)
            a, b = kat_values(c["op1"], q), kat_values(c["op2"], q)
            d = dev(a)
            fn(d, d, b if isinstance(b, int) else dev(b), len(a), q)
            assert (host(d) == kat_values(c["out"], q)).all(), c
    for c in kats["eltwise_cmp_add"]["cases"]:
        a = kat_values(c["op1"], 0)
        d = dev(a)
        hb.EltwiseCmpAdd(d, d, len(a), c["cmp"], c["bound"], c["diff"])
        assert (host(d) == kat_values(c["out"], 0)).all()
    for c in kats["eltwise_cmp_sub_mod"]["cases"]:
        a = kat_values(c["op1"], 0)
        d = dev(a)
        hb.EltwiseCmpSubMod(d, d, len(a), c["q"], c["cmp"], c["bound"], c["diff"])
        assert (host(d) == kat_values(c["out"], 0)).all()


# ------------------------------------------------ eltwise: random vs the oracle
@pytest.mark.parametrize("bits", [20, 30, 32, 40, 50, 55, 59, 60])
@pytest.mark.parametrize("n", [1, 7, 1024 + 7, 1 << 16])
def test_eltwise_matches_oracle(hb, checker, bits, n):
    q = hb.GeneratePrimes(1, bits, True, 1)[0]
    qq = np.uint64(q)
    a, b = uniform_below(1, n, q), uniform_below(2, n, q)
    da, db = dev(a), dev(b)
    r = torch.empty_like(da)
    assert (host(hb.EltwiseAddMod(r, da, db, n, q)) == checker.add_mod(a, b, q)).all()
    assert (host(hb.EltwiseAddMod(r, da, int(b[0]), n, q)) == checker.add_mod(a, int(b[0]), q)).all()
    assert (host(hb.EltwiseSubMod(r, da, db, n, q)) == checker.sub_mod(a, b, q)).all()
    assert (host(hb.EltwiseSubMod(r, da, int(b[0]), n, q)) == checker.sub_mod(a, int(b[0]), q)).all()
    for mf in (1, 2, 4):
        x, y = uniform_below(3, n, mf * q), uniform_below(4, n, mf * q)
        assert (host(hb.EltwiseMultMod(r, dev(x), dev(y), n, q, mf)) == checker.mult_mod(x, y, q, mf)).all()
    for mf in (1, 2, 4, 8):
        x, c = uniform_below(5, n, mf * q), uniform_below(6, n, mf * q)
        s = int(uniform_below(7, 1, mf * q)[0])
        assert (host(hb.EltwiseFMAMod(r, dev(x), s, dev(c), n, q, mf)) == checker.fma_mod(x, s, c, q, mf)).all()
        assert (host(hb.EltwiseFMAMod(r, dev(x), s, None, n, q, mf)) == checker.fma_mod(x, s, None, q, mf)).all()
    wide = uniform_below(8, n, 1 << 64)
    assert (host(hb.EltwiseReduceMod(r, dev(wide), n, q, q, 1)) == wide % qq).all()
    lazy = host(hb.EltwiseReduceMod(r, dev(wide), n, q, q, 2))
    assert (lazy % qq == wide % qq).all() and (lazy < np.uint64(2 * q)).all()
    x4 = uniform_below(9, n, 4 * q)
    assert (host(hb.EltwiseReduceMod(r, dev(x4), n, q, 4, 1)) == checker.reduce_mod(x4, q, 4, 1)).all()
    assert (host(hb.EltwiseReduceMod(r, dev(x4), n, q, 4, 2)) == checker.reduce_mod(x4, q, 4, 2)).all()
    x2 = uniform_below(10, n, 2 * q)
    assert (host(hb.EltwiseReduceMod(r, dev(x2), n, q, 2, 1)) == checker.reduce_mod(x2, q, 2, 1)).all()
    assert (host(hb.EltwiseReduceMod(r, dev(x2), n, q, 2, 2)) == x2).all()  # equal factors: copy
    w = uniform_below(11, n, 1 << 64)
    diff = int(b[n // 2]) or 1
    for cmp in range(8):
        bound = int(w[n // 3])
        assert (host(hb.EltwiseCmpAdd(r, dev(w), n, cmp, bound, diff)) == checker.cmp_add(w, cmp, bound, diff)).all()
        assert (host(hb.EltwiseCmpSubMod(r, dev(w), n, q, cmp, bound, diff))
                == checker.cmp_sub_mod(w, q, cmp, bound, diff)).all()


def test_eltwise_unaligned_and_inplace(hb, checker):
    """operands at odd 8-byte offsets take the scalar instantiation; in-place aliasing"""
    q = hb.GeneratePrimes(1, 55, True, 1)[0]
    n = 4099
    a, b = uniform_below(1, n + 1, q), uniform_below(2, n + 1, q)
    da, db = dev(a), dev(b)
    ra = da[1:]  # 8-byte aligned only
    hb.EltwiseMultMod(ra, ra, db[1:], n, q, 1)
    assert (host(da)[1:] == checker.mult_mod(a[1:], b[1:], q, 1)).all() and host(da)[0] == a[0]
    da = dev(a)
    hb.EltwiseFMAMod(da[:n], da[:n], 12345, db[1:], n, q, 1)
    assert (host(da)[:n] == checker.fma_mod(a[:n], 12345, b[1:], q, 1)).all()


def test_eltwise_host_pointers_large(hb, checker):
    q = hb.GeneratePrimes(1, 60, True, 1)[0]
    n = (40 << 20) // 8 * 3 + 5  # several staging chunks plus a ragged tail
    a, b = uniform_below(1, n, q), uniform_below(2, n, q)
    r = np.zeros_like(a)
    hb.EltwiseMultMod(r, a, b, n, q, 1)
    assert (r == checker.mult_mod(a, b, q, 1)).all()
    hb.EltwiseFMAMod(r, a, 987654321, b, n, q, 1)
    assert (r == checker.fma_mod(a, 987654321, b, q, 1)).all()
    hb.EltwiseReduceMod(r, a, n, q, q, 1)
    assert (r == a).all()


def test_polynomial_product_pipeline(hb):
    """FwdNTT -> EltwiseMultMod -> InvNTT equals the schoolbook negacyclic product
    (the shape of BASELINE config 4), lazy factors (4 on the forward outputs) included."""
    n = 64
    q = hb.GeneratePrimes(1, 50, True, n)[0]
    t = hb.NTT(n, q)
    a, b = uniform_below(1, n, q), uniform_below(2, n, q)
    exp = [0] * n
    for i in range(n):
        for j in range(n):
            k, v = (i + j) % n, int(a[i]) * int(b[j])
            exp[k] = (exp[k] + (v if i + j < n else -v)) % q
    da, db = dev(a), dev(b)
    t.ComputeForward(da, da, 1, 4)
    t.ComputeForward(db, db, 1, 4)
    hb.EltwiseMultMod(da, da, db, n, q, 4)
    t.ComputeInverse(da, da, 1, 1)
    assert [int(v) for v in host(da)] == exp


def test_kernels_really_launch(hb):
    before = hb.launch_count()
    q = hb.GeneratePrimes(1, 30, True, 1024)[0]
    d = dev(uniform_below(1, 1024, q))
    hb.NTT(1024, q).ComputeForward(d, d, 1, 1)
    torch.cuda.synchronize()
    assert hb.launch_count() > before


def test_cpp_drop_in_caller_runs(hb, tmp_path):
    """The reference-style C++ caller (tests/cpp/example_caller.cpp: the scenarios of
    example/example.cpp plus the N=32 known answer) through include/hexl/hexl.hpp,
    with plain host vectors exactly as an unmodified SEAL/OpenFHE-style caller passes."""
    import os
    import shutil
    import subprocess
    if not shutil.which("g++"):
        pytest.skip("g++ not present")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = tmp_path / "example_caller"
    libdir = os.path.dirname(hb.LIB_PATH)
    subprocess.run(["g++", "-std=c++17", "-O1", "-I", os.path.join(root, "include"),
                    os.path.join(root, "tests", "cpp", "example_caller.cpp"), "-o", str(exe),
                    "-L", libdir, "-lhexl_b200", f"-Wl,-rpath,{libdir}"], check=True)
    res = subprocess.run([str(exe), "run"], capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr


# ---------------------------------------------- SEAL-shaped composites (SURVEY 8(f)-1/-2)
def _seal_kats():
    import json
    import os
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    return json.load(open(os.path.join(root, "tests", "golden", "seal_kats.json")))


def test_dyadic_multiply_reference_kats(hb):
    """test/experimental/seal/test-dyadic-multiply.cpp:16-155, incl. result aliasing operand1/2"""
    for c in _seal_kats()["dyadic_multiply"]["cases"]:
        n, mods = c["coeff_count"], c["moduli"]
        bufs = {"op1": np.array(c["op1"], dtype=np.uint64)}
        bufs["op2"] = np.array(c["op2"], dtype=np.uint64) if c["op2"] is not None else None
        bufs["out"] = np.zeros(3 * n * len(mods), dtype=np.uint64)
        exp = np.array(c["exp_out"], dtype=np.uint64)
        # host pointers, same aliasing as the reference test
        h = {k: (None if v is None else v.copy()) for k, v in bufs.items()}
        hb.DyadicMultiply(h[c["call"]["result"]], h[c["call"]["operand1"]], h[c["call"]["operand2"]], n, mods)
        assert (h[c["call"]["result"]] == exp).all(), c["name"]
        # device pointers
        d = {k: (None if v is None else dev(v)) for k, v in bufs.items()}
        hb.DyadicMultiply(d[c["call"]["result"]], d[c["call"]["operand1"]], d[c["call"]["operand2"]], n, mods)
        assert (host(d[c["call"]["result"]]) == exp).all(), c["name"]


def test_dyadic_multiply_matches_oracle(hb, checker):
    n = 1 << 13
    mods = hb.GeneratePrimes(3, 50, True, n) + hb.GeneratePrimes(2, 60, True, n)
    a = np.concatenate([uniform_below(10 + i, n, q) for _ in range(2) for i, q in enumerate(mods)])
    b = np.concatenate([uniform_below(20 + i, n, q) for _ in range(2) for i, q in enumerate(mods)])
    exp = checker.dyadic_multiply(a, b, n, mods)
    out = torch.zeros(3 * n * len(mods), dtype=torch.int64, device="cuda")
    hb.DyadicMultiply(out, dev(a), dev(b), n, mods)
    assert (host(out) == exp).all()


def test_key_switch_reference_kat(hb):
    """test/experimental/seal/test-key-switch.cpp:16-186 through host and device pointers"""
    k = _seal_kats()["key_switch"]
    args = (k["coeff_count"], k["decomp_modulus_size"], k["key_modulus_size"], k["rns_modulus_size"],
            k["key_component_count"], k["moduli"])
    exp = np.array(k["expected_output"], dtype=np.uint64)
    keys = [np.array(x, dtype=np.uint64) for x in k["k_switch_keys"]]
    res = np.array(k["input"], dtype=np.uint64)
    hb.KeySwitch(res, np.array(k["t_target_iter_ptr"], dtype=np.uint64), *args, keys, k["modswitch_factors"])
    assert (res == exp).all()
    dres = dev(np.array(k["input"], dtype=np.uint64))
    hb.KeySwitch(dres, dev(np.array(k["t_target_iter_ptr"], dtype=np.uint64)), *args, [dev(x) for x in keys],
                 k["modswitch_factors"])
    assert (host(dres) == exp).all()


@pytest.mark.parametrize("logn,decomp,bits", [(12, 3, 50), (13, 4, 58), (15, 6, 50), (10, 67, 40)])  # 67 > one parameter block
def test_key_switch_matches_oracle(hb, checker, logn, decomp, bits):
    """CKKS key-switch shape of BASELINE config 5 (N = 2^15, many RNS moduli) against the
    compiled reference / oracle on random data."""
    n = 1 << logn
    kms = rns = decomp + 1
    kcc = 2
    mods = hb.GeneratePrimes(kms, bits, True, n)
    t_target = np.concatenate([uniform_below(30 + j, n, mods[j]) for j in range(decomp)])
    keys = [np.concatenate([uniform_below(100 * j + 7 * k + i, n, mods[i]) for k in range(kcc) for i in range(kms)])
            for j in range(decomp)]
    result = np.concatenate([uniform_below(500 + 10 * k + i, n, mods[i]) for k in range(kcc) for i in range(decomp)])
    modswitch = [hb.InverseMod(mods[-1] % mods[i], mods[i]) for i in range(decomp)]
    exp = checker.key_switch(result.copy(), t_target, n, decomp, kms, rns, kcc, mods, keys, modswitch)
    dres = dev(result)
    hb.KeySwitch(dres, dev(t_target), n, decomp, kms, rns, kcc, mods, [dev(x) for x in keys], modswitch)
    assert (host(dres) == exp).all()


def test_dyadic_multiply_odd_length_and_unaligned(hb, checker):
    """the scalar instantiation: odd coefficient count, and views that start 8 bytes off a 16-byte boundary"""
    for n, shift in ((13, 0), (64, 1)):
        mods = hb.GeneratePrimes(3, 40, True, 1)
        a = np.concatenate([uniform_below(3 + i, n, q) for _ in range(2) for i, q in enumerate(mods)])
        b = np.concatenate([uniform_below(9 + i, n, q) for _ in range(2) for i, q in enumerate(mods)])
        da = torch.zeros(a.size + 1, dtype=torch.int64, device="cuda")
        db = torch.zeros(b.size + 1, dtype=torch.int64, device="cuda")
        out = torch.zeros(3 * n * len(mods) + 1, dtype=torch.int64, device="cuda")
        da[shift:shift + a.size] = dev(a)
        db[shift:shift + b.size] = dev(b)
        hb.DyadicMultiply(out[shift:shift + 3 * n * len(mods)], da[shift:shift + a.size], db[shift:shift + b.size], n, mods)
        assert (host(out[shift:shift + 3 * n * len(mods)]) == checker.dyadic_multiply(a, b, n, mods)).all(), (n, shift)


def test_dyadic_multiply_many_moduli(hb, checker):
    """more moduli than one kernel-parameter block (64)"""
    n = 256
    mods = hb.GeneratePrimes(70, 45, True, n)
    a = np.concatenate([uniform_below(10 + i, n, q) for _ in range(2) for i, q in enumerate(mods)])
    b = np.concatenate([uniform_below(200 + i, n, q) for _ in range(2) for i, q in enumerate(mods)])
    out = torch.zeros(3 * n * len(mods), dtype=torch.int64, device="cuda")
    hb.DyadicMultiply(out, dev(a), dev(b), n, mods)
    assert (host(out) == checker.dyadic_multiply(a, b, n, mods)).all()


def test_key_switch_is_asynchronous_and_graph_capturable(hb, checker):
    """A device-pointer KeySwitch only enqueues work on the caller's stream (scratch comes
    from a stream-ordered pool, small tables ride in kernel parameters): it can be captured
    into a CUDA graph and replayed on new data."""
    n, decomp, kcc = 1 << 12, 4, 2
    kms = rns = decomp + 1
    mods = hb.GeneratePrimes(kms, 50, True, n)
    modswitch = [hb.InverseMod(mods[-1] % mods[i], mods[i]) for i in range(decomp)]
    keys = [np.concatenate([uniform_below(100 * j + 7 * k + i, n, mods[i]) for k in range(kcc) for i in range(kms)])
            for j in range(decomp)]
    dkeys = [dev(x) for x in keys]
    dt = torch.zeros(decomp * n, dtype=torch.int64, device="cuda")
    dres = torch.zeros(kcc * decomp * n, dtype=torch.int64, device="cuda")

    def call():
        hb.KeySwitch(dres, dt, n, decomp, kms, rns, kcc, mods, dkeys, modswitch)

    call()  # tables, pool and function attributes are set up outside the capture
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        call()
    for seed in (3, 4):
        t_target = np.concatenate([uniform_below(seed * 50 + j, n, mods[j]) for j in range(decomp)])
        result = np.concatenate([uniform_below(seed * 500 + 10 * k + i, n, mods[i])
                                 for k in range(kcc) for i in range(decomp)])
        dt.copy_(dev(t_target))
        dres.copy_(dev(result))
        g.replay()
        torch.cuda.synchronize()
        exp = checker.key_switch(result.copy(), t_target, n, decomp, kms, rns, kcc, mods, keys, modswitch)
        assert (host(dres) == exp).all()


def test_ntt_cache(hb):
    q = hb.GeneratePrimes(1, 40, True, 1024)[0]
    a, b = hb.GetNTT(1024, q), hb.GetNTT(1024, q)
    assert a._h.value == b._h.value and a.GetModulus() == q
