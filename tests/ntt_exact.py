"""The negacyclic NTT in Python integers for the tests, and the moduli and inputs the single- and multi-modulus tests
run.

forward() and inverse() are the transforms the library computes (hexl/ntt/ntt-internal.cpp): natural order in,
bit-reversed order out, X[k] = sum_j x_j psi^((2 brv(k) + 1) j) with psi the minimal primitive 2N-th root of unity (or
a given one).  Each stage is one vectorised step over numpy object arrays, and every operation is fully reduced, so
there is no lazy range, no quotient estimate and no word size to get wrong.  Inputs may be any value below 2^64; they
are reduced first, which is what a transform must do with its lazy inputs.  A polynomial of N = 2^20 takes a few
seconds.

tests/test_ntt_exact.py checks the model against the O(N^2) definition and pins the checkers to it at the moduli below;
the GPU tests then compare against the faster checkers.
"""
from __future__ import annotations

import functools

import numpy as np

from util import uniform_below

U64 = np.uint64
MAX_LOGN = 20

# Moduli lists of the multi-modulus tests: (name, [(bits, first)]) with GeneratePrimes(1, bits, first, 2^20), a prime
# just above 2^bits when `first`, else just below 2^(bits + 1).  Every prime is 1 mod 2^21, so each list serves every
# degree up to 2^20.
MODULUS_LISTS = [
    ("fast_edges", [(32, True), (55, False), (49, True)]),                # just above 2^32, just below 2^56, 50 bits
    ("wide_small", [(60, False), (59, True), (31, False), (29, False)]),  # below 2^61, 60 bits, [2^30, 2^32), < 2^30
    ("small_only", [(29, False), (29, True), (24, True)]),                # all below 2^30, one of 25 bits
    ("generic_mixed", [(61, False), (29, False), (49, True)]),            # just below 2^62, below 2^30, 50 bits
]
KINDS = ("top", "alternating", "uniform")

# Primes of the single-modulus tests, GeneratePrimes(1, bits, first, 2^20) as above: the prime on each side of every
# boundary of pick_mode (SMALL below 2^30, GENERIC in [2^30, 2^32), FAST in [2^32, 2^56), WIDE in [2^56, 2^61), GENERIC
# from 2^61), the largest GENERIC prime, and one mid-range prime per mode.  single_primes() adds, per degree, the
# smallest prime that is 1 mod 2N.
SINGLE_PRIMES = [
    ("below_2^30", (29, False)), ("above_2^30", (30, True)),
    ("below_2^32", (31, False)), ("above_2^32", (32, True)),
    ("below_2^56", (55, False)), ("above_2^56", (56, True)),
    ("below_2^61", (60, False)), ("above_2^61", (61, True)),
    ("below_2^62", (61, False)),
    ("small_25bit", (24, True)), ("fast_50bit", (49, True)), ("wide_60bit", (59, True)),
]
SINGLE_NAMES = [name for name, _ in SINGLE_PRIMES] + ["smallest"]


def smallest_prime(n):
    """the smallest prime q = 1 mod 2n"""
    q = 2 * n + 1
    while any(q % d == 0 for d in range(2, int(q ** 0.5) + 1)):
        q += 2 * n
    return q


@functools.lru_cache(maxsize=None)
def _fixed_primes(primes):
    return tuple((name, int(primes(1, bits, first, 1 << MAX_LOGN)[0])) for name, (bits, first) in SINGLE_PRIMES)


def single_primes(primes, logn):
    """[(name, q)] of SINGLE_NAMES for N = 2^logn; primes(num, bits, first, n) is GeneratePrimes"""
    return list(_fixed_primes(primes)) + [("smallest", smallest_prime(1 << logn))]


def single_polynomial(kind, seed, n, q, in_mf):
    """n values below in_mf * q whose residues mod q do not depend on in_mf, so one transform of the model serves
    every input factor: all at in_mf * q - 1, 0 alternating with that value, or uniform below q plus a uniform multiple
    of q below in_mf * q"""
    if kind != "uniform":
        return polynomial(kind, seed, n, in_mf * q)
    return uniform_below(seed, n, q) + U64(q) * uniform_below(seed + 1, n, in_mf)


def single_operand(seed, n, q, batch, in_mf):
    """`batch` polynomials under one modulus, polynomial u of kind KINDS[u % 3] and seed seed + 2u"""
    return np.concatenate([single_polynomial(KINDS[u % 3], seed + 2 * u, n, q, in_mf) for u in range(batch)])


def moduli(primes, spec):
    """the primes of one MODULUS_LISTS entry; primes(num, bits, first, n) is GeneratePrimes"""
    mods = [int(primes(1, bits, first, 1 << MAX_LOGN)[0]) for bits, first in spec]
    assert len(set(mods)) == len(mods)
    return mods


def polynomial(kind, seed, n, bound):
    """n values below `bound`: all at bound - 1, 0 alternating with bound - 1, or uniform"""
    if kind == "top":
        return np.full(n, bound - 1, dtype=U64)
    if kind == "alternating":
        x = np.zeros(n, dtype=U64)
        x[1::2] = bound - 1
        return x
    return uniform_below(seed, n, bound)


def operand(seed, n, mods, group, in_mf):
    """`group` polynomials per modulus, below in_mf * q; polynomial u of modulus i is of kind KINDS[(i + u) % 3], so a
    group of 3 holds every kind and a group of 1 cycles through them over the moduli"""
    return np.concatenate([polynomial(KINDS[(i + u) % 3], seed * 7919 + 100 * i + u, n, in_mf * q)
                           for i, q in enumerate(mods) for u in range(group)])


def _brv(n):
    """the bit-reversal permutation of [0, n)"""
    logn = n.bit_length() - 1
    r = np.zeros(n, dtype=np.int64)
    for b in range(logn):
        r |= ((np.arange(n) >> b) & 1) << (logn - 1 - b)
    return r


def _powers(base, n, q):
    """[base^0, ..., base^(n-1)] mod q as an object array"""
    p = np.array([1], dtype=object)
    while p.size < n:
        p = np.concatenate([p, p * pow(base, p.size, q) % q])
    return p[:n]


def minimal_root(n, q):
    """the smallest primitive 2n-th root of unity mod the prime q (the root NTT(n, q) uses)"""
    assert (q - 1) % (2 * n) == 0
    for g in range(2, q):
        r = pow(g, (q - 1) // (2 * n), q)
        if pow(r, n, q) == q - 1:
            break
    # the primitive 2n-th roots are the odd powers of r
    odd = _powers(r * r % q, n, q) * r % q
    return int(min(odd))


def _table(n, q, psi):
    """psi^brv(k) at slot k: the factor of the butterflies of group i at the stage with m groups is slot m + i"""
    return _powers(psi, n, q)[_brv(n)]


def forward(x, n, q, root=None):
    """the forward transform of every polynomial in x (back to back), in Python integers"""
    psi = root if root is not None else minimal_root(n, q)
    w = _table(n, q, psi)
    a = (np.asarray(x, dtype=U64).astype(object) % q).reshape(-1, n)
    m, t = 1, n // 2
    while m < n:
        v = a.reshape(-1, m, 2, t)
        X = v[:, :, 0, :]
        Y = v[:, :, 1, :] * w[m:2 * m, None] % q
        v[:, :, 0, :], v[:, :, 1, :] = (X + Y) % q, (X - Y) % q
        m, t = 2 * m, t // 2
    return a.reshape(-1).astype(U64)


def inverse(x, n, q, root=None):
    """the inverse of forward(): each stage undone in reverse order, then a multiplication by n^-1"""
    psi = root if root is not None else minimal_root(n, q)
    w_inv = _table(n, q, pow(psi, -1, q))
    a = (np.asarray(x, dtype=U64).astype(object) % q).reshape(-1, n)
    m, t = n // 2, 1
    while m >= 1:
        v = a.reshape(-1, m, 2, t)
        X, Y = v[:, :, 0, :], v[:, :, 1, :]
        v[:, :, 0, :], v[:, :, 1, :] = (X + Y) % q, (X - Y) * w_inv[m:2 * m, None] % q
        m, t = m // 2, 2 * t
    return (a * pow(n, -1, q) % q).reshape(-1).astype(U64)


def forward_definition(x, n, q, root):
    """X[k] = sum_j x_j psi^((2 brv(k) + 1) j), term by term (O(n^2))"""
    brv = _brv(n)
    xs = [int(v) % q for v in x]
    return np.array([sum(xs[j] * pow(root, (2 * int(brv[k]) + 1) * j, q) for j in range(n)) % q for k in range(n)],
                    dtype=U64)


def inverse_definition(X, n, q, root):
    """x_j = n^-1 sum_k X[k] psi^(-(2 brv(k) + 1) j), term by term (O(n^2))"""
    brv = _brv(n)
    Xs = [int(v) % q for v in X]
    inv_root, inv_n = pow(root, -1, q), pow(n, -1, q)
    return np.array([inv_n * sum(Xs[k] * pow(inv_root, (2 * int(brv[k]) + 1) * j, q) for k in range(n)) % q
                     for j in range(n)], dtype=U64)
