"""Exact models of the element-wise operations and of DyadicMultiply, in plain Python integers (no GPU).

Every function states what the operation means mathematically, with none of the reference's algorithms: products and
sums are formed exactly and reduced with Python's `%`, so nothing here can wrap, estimate a quotient or stop one
subtraction short.  Arrays are numpy uint64 in and out; the arithmetic runs on object arrays of Python ints, so a
2^16-element case costs milliseconds.

Canonical outputs (every operation except ReduceMod with output_mod_factor 2) are compared word for word with
`equal_words`.  ReduceMod's lazy output is only defined up to congruence: `lazy_words_ok` checks it is congruent to the
input and below 2q.  CmpAdd is not modular: its sum wraps mod 2^64, as in the reference's definition.

The moduli the GPU tests sweep are here too, so the CPU tests can show which of them the unfixed arithmetic gets
wrong."""
import numpy as np

from util import uniform_below

M64 = (1 << 64) - 1


def big(a):
    """uint64 array (or int) -> object array of Python ints"""
    return np.asarray(a, dtype=np.uint64).astype(object)


def words(x):
    """object array of Python ints in [0, 2^64) -> uint64 array"""
    return np.asarray(x, dtype=object).astype(np.uint64)


# ------------------------------------------------------------------------------------------------ the operations
def mult_mod(a, b, q):
    """EltwiseMultMod for any input_mod_factor: a * b mod q"""
    return words(big(a) * big(b) % q)


def fma_mod(a, s, c, q):
    """EltwiseFMAMod: a * s + c mod q (c may be None: a * s mod q)"""
    r = big(a) * int(s)
    if c is not None:
        r = r + big(c)
    return words(r % q)


def add_mod(a, b, q):
    """EltwiseAddMod, b a vector or a scalar"""
    return words((big(a) + (int(b) if np.isscalar(b) else big(b))) % q)


def sub_mod(a, b, q):
    """EltwiseSubMod, b a vector or a scalar"""
    return words((big(a) - (int(b) if np.isscalar(b) else big(b))) % q)


def reduce_mod(x, q):
    """EltwiseReduceMod with output_mod_factor 1, whatever the input_mod_factor: x mod q"""
    return words(big(x) % q)


# CMPINT (hexl/include/hexl/util/util.hpp): EQ LT LE FALSE NE NLT NLE TRUE
_CMP = (lambda x, b: x == b, lambda x, b: x < b, lambda x, b: x <= b, lambda x, b: False,
        lambda x, b: x != b, lambda x, b: x >= b, lambda x, b: x > b, lambda x, b: True)


def cmp_holds(cmp, x, bound):
    """boolean array: CMPINT `cmp` of every x against bound (both unsigned 64-bit)"""
    x = np.asarray(x, dtype=np.uint64)
    return np.broadcast_to(_CMP[cmp](x, np.uint64(bound)), x.shape)


def cmp_add(x, cmp, bound, diff):
    """EltwiseCmpAdd: x + diff (mod 2^64) where cmp(x, bound) holds, else x"""
    hit = cmp_holds(cmp, x, bound)
    return words(np.where(hit, (big(x) + diff) & M64, big(x)))


def cmp_sub_mod(x, q, cmp, bound, diff):
    """EltwiseCmpSubMod: (x - diff) mod q where cmp(x, bound) holds, else x mod q (the test is on x before reduction)"""
    hit = cmp_holds(cmp, x, bound)
    return words(np.where(hit, (big(x) - diff) % q, big(x) % q))


def dyadic_multiply(op1, op2, n, moduli):
    """DyadicMultiply: operands hold 2 polynomials x len(moduli) x n words, the result 3:
    (x0 y0, x0 y1 + x1 y0, x1 y1), every coefficient mod its modulus"""
    m = len(moduli)
    x, y = big(op1).reshape(2, m, n), big(op2).reshape(2, m, n)
    q = np.array([int(v) for v in moduli], dtype=object).reshape(m, 1)
    out = np.stack([x[0] * y[0] % q, (x[0] * y[1] + x[1] * y[0]) % q, x[1] * y[1] % q])
    return words(out.reshape(-1))


def mont_mult(a, b, q, r):
    """EltwiseMontReduceMod: a * b * 2^-r mod q"""
    return words(big(a) * big(b) * pow(1 << r, -1, q) % q)


def mont_in(a, q, r):
    """EltwiseMontgomeryFormIn: a * 2^r mod q"""
    return words(big(a) * ((1 << r) % q) % q)


def mont_out(a, q, r):
    """EltwiseMontgomeryFormOut: a * 2^-r mod q"""
    return words(big(a) * pow(1 << r, -1, q) % q)


def neg_inv_mod(q, r):
    """-q^-1 mod 2^r, the Montgomery constant the entry points take"""
    return (-pow(q, -1, 1 << r)) % (1 << r)


# ---------------------------------------------------------------------------------------------------- checks
def wrong_words(got, exp):
    return int((np.asarray(got, dtype=np.uint64) != np.asarray(exp, dtype=np.uint64)).sum())


def wrong_lazy_words(got, exp, q):
    """ReduceMod with output_mod_factor 2 against the canonical result exp = x mod q: a word is right when it is
    congruent to x and below 2q, that is when it equals exp or exp + q"""
    got, exp, qq = np.asarray(got, dtype=np.uint64), np.asarray(exp, dtype=np.uint64), np.uint64(q)
    ok = (got == exp) | ((got >= qq) & (got - qq == exp))
    return int((~ok).sum())


# ---------------------------------------------------------------------------------------------------- operands
BAND = 1 << 20


def _span(lo, hi, seed, n):
    """n values in [lo, hi)"""
    return np.uint64(lo) + uniform_below(seed, n, hi - lo)


def operands(q, bound, seed, n, edges=()):
    """Two operand vectors of n words below `bound` (in_mf * q, or 2^64 for any word):
    every pair of edge values first, the largest first (0, 1, q - 1, q - 2, q, q + 1, bound - 1, bound - 2 and
    `edges`, where below bound); then a dense band of pairs with both operands within 2^20 of q (and, for lazy
    inputs, within 2^20 below bound); then uniform values."""
    e = sorted({v for v in (0, 1, q - 1, q - 2, q, q + 1, bound - 1, bound - 2, *edges) if 0 <= v < bound},
               reverse=True)
    a = np.array([x for x in e for _ in e], dtype=np.uint64)[:n]
    b = np.array([y for _ in e for y in e], dtype=np.uint64)[:n]
    rest = n - a.size
    near = rest // 2
    lo, hi = max(0, q - BAND), min(bound, q + BAND)
    parts_a, parts_b = [a], [b]
    if bound > q + BAND:   # half of the band at the top of the lazy range
        top = near // 2
        parts_a.append(_span(bound - BAND, bound, seed + 1, top))
        parts_b.append(_span(bound - BAND, bound, seed + 2, top))
        near -= top
    parts_a += [_span(lo, hi, seed + 3, near), _span(0, bound, seed + 5, rest - rest // 2)]
    parts_b += [_span(lo, hi, seed + 4, near), _span(0, bound, seed + 6, rest - rest // 2)]
    return np.concatenate(parts_a), np.concatenate(parts_b)


# ------------------------------------------------------------------------------------------------------ moduli
def is_prime(n):
    """deterministic Miller-Rabin for n < 2^64 (the first 12 prime bases suffice below 3.3 * 10^24)"""
    if n < 2:
        return False
    bases = (2, 3, 5, 7, 11, 13, 17, 19, 23, 29, 31, 37)
    for p in bases:
        if n % p == 0:
            return n == p
    d, s = n - 1, 0
    while d % 2 == 0:
        d, s = d // 2, s + 1
    for a in bases:
        x = pow(a, d, n)
        if x in (1, n - 1):
            continue
        for _ in range(s - 1):
            x = x * x % n
            if x == n - 1:
                break
        else:
            return False
    return True


def prime_below(x):
    p = x - 1
    while not is_prime(p):
        p -= 1
    return p


def prime_above(x):
    p = x + 1
    while not is_prime(p):
        p += 1
    return p


def band_moduli(powers):
    """the largest prime below and the smallest prime above 2^k for every k in `powers`, where the word arithmetic
    changes: 32-bit operands (2^30, 2^32), the transform's word classes (2^56, 2^60), the input_mod_factor limits and
    the generalised Barrett product's 62-bit case (2^61, 2^62), the sign bit (2^63)"""
    out = []
    for k in powers:
        out += [prime_below(1 << k), prime_above(1 << k)]
    return out


# Primes in [2^61.7, 2^62) at which the generalised Barrett product (alpha = 62, beta = -2) with one conditional
# subtraction leaves results in [q, 2q): with bits(q) = 62, alpha - bits(q) = 0 and its quotient estimate can be low by
# two.  Found by sampling primes in bands of 2^0.1 below 2^62 and running the product, as the reference's scalar tier
# computes it, on 4096 operand pairs within 2^20 of q: none were affected below 2^61.7, 2 of 60 in [2^61.7, 2^61.8),
# 6 of 60 in [2^61.8, 2^61.9) and 9 of 60 in [2^61.9, 2^62).  The largest primes below 2^62 (2^62 - 57, 2^62 - 87)
# are not affected.
BARRETT_62_BIT_WITNESSES = (4084223049772944437, 4513552570436316989, 4416645352417296419)

# the API does not require primes; the largest modulus each operation accepts (2^62 - 1, 2^63 - 1, 2^64 - 1) is
# composite as well
COMPOSITE_MODULI = (
    (1 << 30) + 1,                                                      # 5^2 * 13 * 41 * 61 * 1321
    3 * 5 * 7 * 11 * 13 * 17 * 19 * 23 * 29 * 31 * 37 * 41 * 43 * 47,   # the odd primes up to 47, about 2^58.1
)
