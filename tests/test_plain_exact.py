"""The model of the plaintext calls (tests/plain_exact.py) against big-integer statements and decryption, and the
compiler's resource report of their kernels.  CPU only.

(a) SEAL's split formula m [floor(Q/t)]_{q_i} + fix equals floor((Q m + floor((t+1)/2)) / t) mod q_i;
(b) the kernel's fix (a Shoup quotient corrected by one) is the true quotient at t = 2, 3, 2^61 - 1, m = 0 and t - 1,
    and Q mod t = 0 and t - 1;
(c) the lift is the centred value of [m c]_t mod each q_i, with t above, between and below the q_i;
(d) BFV add_plain / sub_plain decrypt to m1 +- m2 and multiply_plain to m1 m2 in R_t; BGV add_plain after a modulus
    switch decrypts correctly only with the correction factor, and BGV multiply_plain decrypts to m1 m2."""
import numpy as np
import pytest

import bgv_exact as gx
import plain_exact as px
from mul_relin_exact import negacyclic_product
from test_kernel_resources import kernel_resources
from util import uniform_below

U64 = np.uint64
T61 = (1 << 61) - 1


def _primes(port, n, count, bits):
    return [int(q) for q in port.generate_primes(count, bits, True, n)]


@pytest.mark.parametrize("t", [2, 3, 257, 65537, (1 << 40) + 15, T61])
def test_split_formula_is_the_rounded_quotient(port, t):
    n = 32
    Q = _primes(port, n, 3, 59)
    Qp = px._prod(Q)
    m = [int(v) for v in uniform_below(t, n, t)] + [0, t - 1]
    r, h = Qp % t, (t + 1) // 2
    for v in m:
        fix = px.fix_quotient(v, r, t)
        for q in Q:
            assert (v * (Qp // t % q) + fix) % q == ((Qp * v + h) // t) % q


@pytest.mark.parametrize("t", [2, 3, 65537, T61])
def test_fix_is_the_true_quotient_at_its_extremes(t):
    h = (t + 1) // 2
    for r in sorted({0, 1, t // 2, t - 1}):
        for m in sorted({0, 1, t // 2, t - 1}):
            assert px.fix_quotient(m, r, t) == (m * r + h) // t, (t, r, m)
    for m in (int(v) for v in uniform_below(7, 200, t)):
        for r in (int(v) for v in uniform_below(m + 1, 4, t)):
            assert px.fix_quotient(m, r, t) == (m * r + h) // t


@pytest.mark.parametrize("where", ["above", "between", "below"])
@pytest.mark.parametrize("cf", [1, 5])
def test_lift_is_the_centred_residue(port, where, cf):
    n = 64
    Q = _primes(port, n, 2, 30) + _primes(port, n, 1, 50)
    t = {"above": T61, "between": (1 << 40) + 15, "below": 65537}[where]
    pcc = n // 2 + 1
    plain = uniform_below(3, pcc, t)
    plain[0], plain[1], plain[2] = 0, t - 1, (t + 1) // 2
    got = px.lift(plain, pcc, n, Q, t, cf).reshape(len(Q), n)
    for j in range(n):
        m = int(plain[j]) * cf % t if j < pcc else 0
        centred = m - t if m >= (t + 1) // 2 else m
        for i, q in enumerate(Q):
            assert int(got[i, j]) == centred % q


def _secret(n, seed):
    return [int(v) - 1 for v in uniform_below(seed, n, 3)]


@pytest.mark.parametrize("n, l, t", [(16, 1, 2), (64, 2, 257), (256, 3, 65537), (128, 2, 1073741789)])
def test_bfv_calls_decrypt(port, n, l, t):
    Q = _primes(port, n, l, 60)
    s = _secret(n, n + l)
    m1 = [int(v) for v in uniform_below(11 + l, n, t)]
    pcc = n // 2 + 1
    m2 = uniform_below(12 + l, pcc, t)
    m2f = [int(v) for v in m2] + [0] * (n - pcc)
    ct = px.encrypt(port, m1, s, Q, n, t, 21)
    assert px.decrypt(port, ct, s, Q, n, t) == m1
    for sub in (False, True):
        got = px.decrypt(port, px.add_plain(ct, m2, pcc, n, Q, t, sub), s, Q, n, t)
        assert got == [(a - b if sub else a + b) % t for a, b in zip(m1, m2f)]
    prod = px.multiply_plain(port, ct, m2, pcc, n, Q, t)
    assert px.decrypt(port, prod, s, Q, n, t) == [v % t for v in negacyclic_product(m1, m2f, n)]
    fp = px.plain_lift(port, m2, pcc, n, Q, t, ntt_form=True)
    assert (px.multiply_plain(port, ct, fp, pcc, n, Q, t, plain_ntt_form=True) == prod).all()


@pytest.mark.parametrize("n, L, t", [(32, 3, 65537), (64, 2, 257), (16, 3, 1073741789)])
def test_bgv_chains_decrypt(port, n, L, t):
    """add_plain = PlainLift(correction factor, NTT form) + EltwiseAddModMulti on c0 after BgvModSwitch, and
    multiply_plain = PlainLift(NTT form) + EltwiseMultModMulti on both components"""
    mods = _primes(port, n, L + 1, 55)
    s = gx.secret(n, 5 + n)
    m1 = [int(v) for v in uniform_below(31, n, t)]
    m2 = uniform_below(32, n, t)
    ct = gx.encrypt(port, m1, s, n, mods, t, 41)
    sw = gx.mod_switch(port, ct, n, mods, 2, True, t).reshape(2, L + 1, n)[:, :L].reshape(-1)
    Q = mods[:L]
    c = pow(mods[L] % t, -1, t)  # the message picks up q_L^-1 in the switch
    assert gx.decrypt(port, sw, [None, s], n, Q, t) == [v * c % t for v in m1]
    for cf, ok in ((c, True), (1, False)):
        lifted = px.plain_lift(port, m2, n, n, Q, t, cf, ntt_form=True)
        out = sw.copy()
        for i, q in enumerate(Q):
            out[i * n:(i + 1) * n] = port.add_mod(sw[i * n:(i + 1) * n], lifted[i * n:(i + 1) * n], q)
        dec = [v * pow(c, -1, t) % t for v in gx.decrypt(port, out, [None, s], n, Q, t)]
        assert (dec == [(a + int(b)) % t for a, b in zip(m1, m2)]) == ok, f"correction factor {cf}"
    lifted = px.plain_lift(port, m2, n, n, mods, t, ntt_form=True)
    prod = ct.copy()
    for k in range(2):
        for i, q in enumerate(mods):
            o = (k * (L + 1) + i) * n
            prod[o:o + n] = port.mult_mod(ct[o:o + n], lifted[i * n:(i + 1) * n], q)
    expect = [v % t for v in negacyclic_product(m1, [int(v) for v in m2], n)]
    assert gx.decrypt(port, prod, [None, s], n, mods, t) == expect


@pytest.mark.parametrize("kernel", ["plain_lift_kernel", "bfv_add_plain_kernel"])
def test_plain_kernels_keep_no_local_memory(kernel):
    res = {name: r for name, r in kernel_resources("plain.cu").items() if kernel in name}
    assert res, f"no ptxas report for {kernel}"
    for name, (frame, stores, loads) in res.items():
        assert frame == 0 and stores == 0 and loads == 0, f"{name}: stack {frame}, spills {stores}/{loads}"
