"""The negacyclic NTT in Python integers for the tests, and the moduli lists and inputs the multi-modulus tests run.

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
