"""The BGV model of tests/bgv_exact.py on the CPU: the t-corrected conversion's integer statement at its extremes, the
anchors that tie the model to SEAL's formula and to the existing calls, decryption of every operation, and the ptxas
report of the new kernel."""
import numpy as np
import pytest

import bgv_exact as bx
import hybrid_exact as hx
import mul_relin_exact as mr
from test_kernel_resources import kernel_resources
from util import uniform_below

U64 = np.uint64
TAUS = [2, 3, 65537, (1 << 61) - 1]


def _prod(values):
    out = 1
    for v in values:
        out *= int(v)
    return out


def _primes(port, count, bits, n=16):
    return [int(q) for q in port.generate_primes(count, bits, True, n)]


def _lift(limbs, moduli):
    """CRT lift in [0, prod) of one column per coefficient: limbs [len(moduli)][n] -> list of ints"""
    M = _prod(moduli)
    basis = [(M // q) * pow(M // q % q, -1, q) for q in moduli]
    return [sum(int(limbs[i][c]) * basis[i] for i in range(len(moduli))) % M for c in range(len(limbs[0]))]


@pytest.mark.parametrize("tau", TAUS)
@pytest.mark.parametrize("count", [1, 2, 63, 64])
def test_conversion_integer_statement(port, count, tau):
    """delta = X mod P_T, delta = 0 mod tau and 0 <= delta < P_T (|T| + tau - 1), read back from the limbs of delta
    over enough targets to lift it, at X = 0, X = P_T - 1, every source word q - 1 and random words"""
    src = _primes(port, count, 60)
    P = _prod(src)
    n = 8
    rows = [[0] * n, [P - 1] * n]
    inputs = [np.array([[X % q for X in row] for q in src], dtype=U64) for row in rows]
    inputs.append(np.array([[q - 1] * n for q in src], dtype=U64))
    inputs.append(np.array([uniform_below(7 * count + i, n, q) for i, q in enumerate(src)], dtype=U64))
    # targets whose product exceeds P_T (|T| + tau): the lift of delta over them is delta itself
    targets = [int(q) for q in port.generate_primes(count + 3, 60, False, n)]
    M = _prod(targets)
    assert M > P * (count + tau)
    for x in inputs:
        X = _lift(x, src)
        delta = bx.t_corrected_convert(port, x.reshape(-1), n, src, targets, tau).reshape(len(targets), n)
        for c, d in enumerate(_lift(delta, targets)):
            assert d % P == X[c], (count, tau, c)
            assert d % tau == 0, (count, tau, c)
            assert 0 <= d < P * (count + tau - 1), (count, tau, c)


@pytest.mark.parametrize("tau", TAUS)
def test_mod_switch_is_the_exact_division(port, tau):
    """(X - delta) / q_L mod every q_i, delta = x_L + q_L [-x_L q_L^-1]_tau, at the edge words and random words"""
    n, mods = 16, _primes(port, 4, 50)
    Q, q_last = _prod(mods), mods[-1]
    rows = [[0] * n, [Q - 1] * n, [q_last - 1] * n] + [[int(v) for v in uniform_below(3, n, 1 << 62)]]
    operand = np.array([[[X % q for X in row] for q in mods] for row in rows], dtype=U64).reshape(-1)
    got = bx.mod_switch(port, operand, n, mods, len(rows), False, tau).reshape(len(rows), 4, n)
    for p, row in enumerate(rows):
        for c, X in enumerate(row):
            X %= Q
            xl = X % q_last
            delta = xl + q_last * ((-xl * pow(q_last, -1, tau)) % tau)
            assert (X - delta) % q_last == 0
            for i, q in enumerate(mods[:-1]):
                assert int(got[p, i, c]) == (X - delta) // q_last % q


# ------------------------------------------------------------------------------------------------ anchors
@pytest.mark.parametrize("tau", TAUS)
@pytest.mark.parametrize("fill", [None, "q-1"])
def test_one_prime_conversion_is_seal(port, tau, fill):
    """T = {one prime}: the model's mod switch is SEAL's per-limb formula, in coefficient form"""
    n, mods = 32, _primes(port, 5, 60)
    operand = (np.concatenate([np.full(n, q - 1, dtype=U64) for _ in range(2) for q in mods]) if fill
               else np.concatenate([uniform_below(11 + i, n, q) for _ in range(2) for i, q in enumerate(mods)]))
    assert np.array_equal(bx.mod_switch(port, operand, n, mods, 2, False, tau),
                          bx.seal_mod_switch(operand, n, mods, 2, tau))


@pytest.mark.parametrize("tau", [2, 65537])
def test_ntt_mod_switch_is_inverse_coefficient_forward(port, tau):
    n, mods = 64, _primes(port, 4, 50, 64)
    operand = np.concatenate([uniform_below(21 + i, n, q) for i, q in enumerate(mods)])
    coef = np.concatenate([port.ntt_inverse(operand[i * n:(i + 1) * n], n, q) for i, q in enumerate(mods)])
    switched = bx.mod_switch(port, coef, n, mods, 1, False, tau)
    chain = np.concatenate([port.ntt_forward(switched[i * n:(i + 1) * n], n, q) for i, q in enumerate(mods[:-1])])
    got = bx.mod_switch(port, operand, n, mods, 1, True, tau)
    assert np.array_equal(got[:3 * n], chain)


@pytest.mark.parametrize("L, K, alpha, level", [(4, 1, 1, 4), (5, 2, 2, 3), (6, 3, 4, 6)])
def test_multiply_relinearize_is_dyadic_then_key_switch(port, L, K, alpha, level):
    n, tau = 32, 65537
    mods = _primes(port, L + K, 50, n)
    keys = hx.random_keys(mods, n, L, alpha, 2, 5)
    ct1 = np.concatenate([uniform_below(31 + i, n, mods[i % level]) for i in range(2 * level)])
    ct2 = np.concatenate([uniform_below(41 + i, n, mods[i % level]) for i in range(2 * level)])
    d = mr.tensor(port, ct1, ct2, n, level, mods)
    chain = bx.key_switch(port, np.concatenate([d[0], d[1]]), d[2], n, level, L, K, alpha, 2, mods, keys, tau)
    assert np.array_equal(bx.multiply_relinearize(port, ct1, ct2, n, level, L, K, alpha, mods, keys, tau, False),
                          chain)


def test_hoisted_identity_is_key_switch_of_c1(port):
    n, L, K, alpha, tau = 32, 5, 2, 2, 257
    mods = _primes(port, L + K, 50, n)
    keys = hx.random_keys(mods, n, L, alpha, 2, 6)
    ct = np.concatenate([uniform_below(51 + i, n, mods[i % L]) for i in range(2 * L)])
    comp = L * n
    chain = bx.key_switch(port, np.concatenate([ct[:comp], np.zeros(comp, dtype=U64)]), ct[comp:], n, L, L, K, alpha,
                          2, mods, keys, tau)
    assert np.array_equal(bx.hoisted(port, ct, n, L, L, K, alpha, mods, [1], [keys], tau), chain)


# ------------------------------------------------------------------------------------------------ decryption
def _setup(port, n, l, K, alpha, tau):
    mods = [q for q in port.generate_primes(l + K + 2, 50, True, n) if np.gcd(q, tau) == 1][:l + K]
    s = bx.secret(n, 3 + n)
    return [int(q) for q in mods], s


@pytest.mark.parametrize("alpha, K", [(1, 1), (2, 2)])
@pytest.mark.parametrize("tau", [2, 257, 65537, 1073479681])
@pytest.mark.parametrize("n, l", [(16, 2), (64, 3), (1024, 4)])
def test_operations_decrypt(port, n, l, tau, alpha, K):
    mods, s = _setup(port, n, l, K, alpha, tau)
    s2 = mr.negacyclic_product(s, s, n)
    m1 = [int(v) for v in uniform_below(5 + n, n, tau)]
    m2 = [int(v) for v in uniform_below(6 + n, n, tau)]
    prod = [v % tau for v in mr.negacyclic_product(m1, m2, n)]
    ct1, ct2 = bx.encrypt(port, m1, s, n, mods[:l], tau, 7), bx.encrypt(port, m2, s, n, mods[:l], tau, 8)
    assert bx.decrypt(port, ct1, [None, s], n, mods[:l], tau) == m1
    # fresh, mod-switched: m [q_L^-1]_tau
    switched = bx.mod_switch(port, ct1, n, mods[:l], 2, True, tau).reshape(2, l, n)[:, :l - 1].reshape(-1)
    inv = pow(mods[l - 1], -1, tau)
    assert bx.decrypt(port, switched, [None, s], n, mods[:l - 1], tau) == [v * inv % tau for v in m1]
    keys = bx.bgv_keys(port, s, s2, n, mods, l, alpha, tau, 40 + n, 8)
    for ms in (False, True):
        r = bx.multiply_relinearize(port, ct1, ct2, n, l, l, K, alpha, mods, keys, tau, ms)
        inv = pow(mods[l - 1], -1, tau) if ms else 1
        assert bx.decrypt(port, r, [None, s], n, mods[:l - ms], tau) == [v * inv % tau for v in prod], ms
    # hoisted rotation: sigma_g(m)
    g = 5
    gkeys = bx.bgv_keys(port, s, _sigma(s, n, g), n, mods, l, alpha, tau, 60 + n, 8)
    rot = bx.hoisted(port, ct1, n, l, l, K, alpha, mods, [g], [gkeys], tau)
    assert bx.decrypt(port, rot, [None, s], n, mods[:l], tau) == [v % tau for v in _sigma(m1, n, g)]
    # keys for another secret fail
    other = bx.secret(n, 99 + n)
    wrong = bx.bgv_keys(port, other, mr.negacyclic_product(other, other, n), n, mods, l, alpha, tau, 40 + n, 8)
    r = bx.multiply_relinearize(port, ct1, ct2, n, l, l, K, alpha, mods, wrong, tau, False)
    assert bx.decrypt(port, r, [None, s], n, mods[:l], tau) != prod
    # the rounded CKKS mod-down with the same keys loses the message
    if tau >= 257:
        d = mr.tensor(port, ct1, ct2, n, l, mods)
        ckks = hx.key_switch_hybrid(port, np.concatenate([d[0], d[1]]), d[2], n, l, l, K, alpha, 2, mods, keys)
        assert bx.decrypt(port, ckks, [None, s], n, mods[:l], tau) != prod


def _sigma(a, n, g):
    """a(X^g) in Z[X]/(X^n + 1), integer coefficients"""
    out = [0] * n
    for i, v in enumerate(a):
        k = i * g % (2 * n)
        if k < n:
            out[k] += v
        else:
            out[k - n] -= v
    return out


@pytest.mark.parametrize("kernel", ["base_conv_t_kernel"])
def test_t_corrected_kernel_keeps_no_local_memory(kernel):
    res = {name: r for name, r in kernel_resources("rns.cu").items() if kernel in name}
    assert len(res) == 2, f"ptxas reports for {kernel}: {sorted(res)}"
    for name, (frame, stores, loads) in res.items():
        assert frame == 0 and stores == 0 and loads == 0, f"{name}: stack {frame}, spills {stores}/{loads}"
