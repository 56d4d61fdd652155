"""The Galois automorphism model (tests/galois_exact.py) and the CPU-side checks of hexl_b200_apply_galois and
hexl_b200_apply_galois_key_switch.  CPU only.

The GPU tests compare ApplyGalois with the model bit for bit, so the model is pinned here: the NTT-form permutation
pi_g is the coefficient-form automorphism conjugated by the exact transform (ntt_exact.forward), with the minimal root
and with another one; pi_g has the aligned-block property the NTT-form kernel relies on; and the automorphisms compose
as a group.  Bad arguments are refused before any device is touched."""
import random

import numpy as np
import pytest

import galois_exact as gx
import ntt_exact
from util import uniform_below

U64 = np.uint64


def _prime(port, n):
    """a 40-bit prime that is 1 mod 2n"""
    return int(port.generate_primes(1, 39, True, n)[0])


def _roots(n, q):
    """the minimal primitive 2n-th root and a non-minimal one (its cube, also primitive since 3 is odd)"""
    r = ntt_exact.minimal_root(n, q)
    return [r, pow(r, 3, q)] if n > 1 else [r]


def _check_commutes(n, q, g, root, a, fa):
    got = ntt_exact.forward(gx.sigma_coef(a, n, g, [q]), n, q, root)
    assert (got == gx.sigma_ntt(fa, n, g)).all(), (n, g, root)


@pytest.mark.parametrize("logn", range(1, 9))
def test_ntt_form_is_the_transform_of_the_coefficient_form_for_every_g(port, logn):
    n = 1 << logn
    q = _prime(port, n)
    a = uniform_below(17 * n, n, q)
    for root in _roots(n, q):
        fa = ntt_exact.forward(a, n, q, root)
        for g in range(1, 2 * n, 2):
            _check_commutes(n, q, g, root, a, fa)


def _sampled_g(n, seed):
    rnd = random.Random(seed)
    return sorted({3, 5, pow(3, 7, 2 * n), 2 * n - 1, rnd.randrange(1, 2 * n, 2)})


@pytest.mark.parametrize("logn", range(10, 14))
def test_ntt_form_is_the_transform_of_the_coefficient_form_at_larger_degrees(port, logn):
    n = 1 << logn
    q = _prime(port, n)
    a = uniform_below(5 * n + 1, n, q)
    for root in _roots(n, q):
        fa = ntt_exact.forward(a, n, q, root)
        for g in _sampled_g(n, logn):
            _check_commutes(n, q, g, root, a, fa)


def _aligned_blocks(n, g):
    """every aligned block of 2^t output slots reads exactly one aligned block of 2^t input slots, for every t"""
    p = gx.pi(n, g)
    assert sorted(p) == list(range(n))
    t = 1
    while t <= n:
        rows = (p >> (t.bit_length() - 1)).reshape(-1, t)
        if not (rows == rows[:, :1]).all():
            return False
        t *= 2
    return True


@pytest.mark.parametrize("logn", range(1, 11))
def test_aligned_block_property_for_every_g(logn):
    n = 1 << logn
    for g in range(1, 2 * n, 2):
        assert _aligned_blocks(n, g), (n, g)
    # the pair form the kernel uses
    for g in range(1, 2 * n, 2):
        p = gx.pi(n, g)
        assert (p[1::2] == p[0::2] ^ 1).all()


@pytest.mark.parametrize("logn", range(11, 21))
def test_aligned_block_property_for_sampled_g(logn):
    n = 1 << logn
    for g in _sampled_g(n, 100 + logn):
        assert _aligned_blocks(n, g), (n, g)


def test_coefficient_form_equals_the_integer_definition(port):
    n = 64
    mods = [int(q) for q in port.generate_primes(3, 39, True, n)]
    coeffs = [int(v) - (1 << 30) for v in uniform_below(3, n, 1 << 31)]
    coeffs[0], coeffs[1] = 0, -1
    x = np.concatenate([np.array([c % q for c in coeffs], dtype=U64) for q in mods])
    for g in (1, 3, 5, 2 * n - 1, 77):
        exp = gx.sigma_int(coeffs, n, g)
        got = gx.sigma_coef(x, n, g, mods).reshape(len(mods), n)
        for i, q in enumerate(mods):
            assert [int(v) for v in got[i]] == [c % q for c in exp], (g, i)
            assert (got[i] < U64(q)).all()


@pytest.mark.parametrize("logn", [3, 6, 10])
def test_automorphisms_compose_and_one_is_the_identity(port, logn):
    n = 1 << logn
    mods = [int(q) for q in port.generate_primes(2, 39, True, n)]
    x = np.concatenate([uniform_below(i + 9, n, q) for i, q in enumerate(mods)])
    assert (gx.sigma_coef(x, n, 1, mods) == x).all()
    assert (gx.sigma_ntt(x, n, 1) == x).all()
    for g, h in [(3, 5), (2 * n - 1, 3), (5, 2 * n - 1), (7, 9)]:
        gh = g * h % (2 * n)
        assert (gx.sigma_coef(gx.sigma_coef(x, n, h, mods), n, g, mods) == gx.sigma_coef(x, n, gh, mods)).all()
        assert (gx.sigma_ntt(gx.sigma_ntt(x, n, h), n, g) == gx.sigma_ntt(x, n, gh)).all()


# ---------------------------------------------------------------- the C entry points without a GPU
def _galois(hb, n, mods, g, count=1, ntt_form=True, result=None, operand=None):
    op = np.zeros(max(count, 1) * len(mods) * max(n, 1), dtype=U64) if operand is None else operand
    return hb.ApplyGalois(op if result is None else result, op, n, mods, len(mods), count, g, ntt_form)


def _invalid(hb, fn, what, words=()):
    with pytest.raises(hb.HexlB200Error) as e:
        fn()
    assert e.value.code == -1, (what, str(e.value))
    for w in words:
        assert w in str(e.value), (what, str(e.value))


def test_apply_galois_refuses_bad_arguments(hb, port):
    n = 64
    mods = [int(q) for q in port.generate_primes(3, 39, True, n)]
    cases = {
        "even g": (n, mods, 4),
        "g = 0": (n, mods, 0),
        "g = 2n": (n, mods, 2 * n),
        "g = 2n + 1": (n, mods, 2 * n + 1),
        "n not a power of two": (48, mods, 3),
        "n above 2^20": (1 << 21, mods, 3),
        "n = 1": (1, mods, 1),
        "modulus 1": (n, [1] + mods[1:], 3),
        "modulus 2^62": (n, mods[:-1] + [1 << 62], 3),
    }
    for what, (nn, mm, g) in cases.items():
        for ntt_form in (True, False):
            _invalid(hb, lambda: _galois(hb, nn, mm, g, ntt_form=ntt_form,
                                         operand=np.zeros(len(mm) * max(nn, 1) if nn <= 1 << 20 else 1, dtype=U64)),
                     what)
    buf = np.zeros(3 * len(mods) * n, dtype=U64)
    _invalid(hb, lambda: hb.ApplyGalois(buf[n:], buf[:2 * len(mods) * n], n, mods, len(mods), 2, 3), "overlap",
             ["overlap"])
    # null pointers, through the C ABI directly
    lib, x = hb._lib, np.zeros(len(mods) * n, dtype=U64)
    m = np.array(mods, dtype=U64)
    for args in [(None, x.ctypes.data, m.ctypes.data), (x.ctypes.data, None, m.ctypes.data),
                 (x.ctypes.data, x.ctypes.data, None)]:
        assert lib.hexl_b200_apply_galois(args[0], args[1], n, args[2], len(mods), 1, 3, 1, None) == -1
    assert lib.hexl_b200_apply_galois(x.ctypes.data, x.ctypes.data, n, m.ctypes.data, 0, 1, 3, 1, None) == -1
    assert lib.hexl_b200_apply_galois(x.ctypes.data, x.ctypes.data, n, m.ctypes.data, len(mods), 1, 3, 2, None) == -1
    # nothing to do
    _galois(hb, n, mods, 3, count=0)


def test_apply_galois_key_switch_refuses_bad_arguments(hb, port):
    n, decomp = 64, 3
    mods = [int(q) for q in port.generate_primes(decomp + 1, 49, True, n)]
    ms = [1] * decomp
    ct = np.zeros(3 * decomp * n, dtype=U64)

    def call(kcc=2, g=3, nn=n, rns=decomp + 1, keys=None):
        return hb.ApplyGaloisKeySwitch(ct, nn, decomp, len(mods), rns, kcc, mods, keys, ms, g)

    _invalid(hb, lambda: call(kcc=3), "three components", ["key_component_count"])
    _invalid(hb, lambda: call(kcc=1), "one component", ["key_component_count"])
    _invalid(hb, lambda: call(g=4), "even g", ["galois_elt"])
    _invalid(hb, lambda: call(g=2 * n + 1), "g >= 2n", ["galois_elt"])
    _invalid(hb, lambda: call(nn=48), "n not a power of two")
    _invalid(hb, lambda: call(rns=decomp), "rns != decomp + 1")
    _invalid(hb, lambda: call(), "no key handle", ["galois_keys"])
    lib, m, msa = hb._lib, np.array(mods, dtype=U64), np.array(ms, dtype=U64)
    assert lib.hexl_b200_apply_galois_key_switch(None, n, decomp, len(mods), decomp + 1, 2, m.ctypes.data, None,
                                                 msa.ctypes.data, 3, 1, None) == -1


def test_without_a_gpu_the_call_fails_and_launches_nothing(hb, port):
    if hb.device_count() > 0:
        pytest.skip("a CUDA device is present")
    n = 64
    mods = [int(q) for q in port.generate_primes(3, 39, True, n)]
    for ntt_form in (False, True):
        before = hb.launch_count()
        with pytest.raises(hb.HexlB200Error) as e:
            _galois(hb, n, mods, 3, count=2, ntt_form=ntt_form)
        assert e.value.code == -2
        assert hb.launch_count() == before
