"""Exact CKKS KeySwitch (hexl/experimental/seal/key-switch-internal.cpp:25-201) for the tests, and the key-switch
cases the tests run.

The reference and the C restatement (oracle/hexl_oracle.c:orc_key_switch) add up each output modulus's digit x key
products in an unreduced 128-bit accumulator.  Each product is a lazy forward-transform output (< 4q) times a key word
(< q), so the sum can wrap 2^128 once q > 2^60 and there are more than 16 digits.  Where it wraps, both checkers are
wrong.  key_switch_exact() computes the same function with canonical modular operations only (every product and every
sum reduced), so nothing can wrap.  Its building blocks are the C restatement's canonical NTT, mult_mod, add_mod and
sub_mod, which the golden vectors pin; tests/test_ks_exact.py shows it equals both checkers wherever they do not wrap.
"""
from __future__ import annotations

from typing import NamedTuple

import numpy as np

from util import uniform_below

U64 = np.uint64


def key_switch_exact(port, result, t_target, n, decomp, key_modulus_size, rns, kcc, moduli, keys, modswitch):
    """KeySwitch with the argument layout of Port.key_switch; returns the updated result as a new array.
    Digits may be any representative below 2^64 (the reference takes them in [0, 2q))."""
    assert rns == decomp + 1
    moduli = [int(q) for q in moduli]
    t_target = np.asarray(t_target, dtype=U64)

    def slot(i):  # RNS modulus i lives in key / moduli slot `slot(i)`; the special prime is the last slot
        return key_modulus_size - 1 if i == decomp else i

    # every digit back to coefficient form under its own modulus
    coef = [port.ntt_inverse(t_target[j * n:(j + 1) * n] % U64(moduli[j]), n, moduli[j]) for j in range(decomp)]
    # prod[i, k] = sum over digits j of NTT_qi(coef_j mod qi) * key_j[component k, slot(i)]  (mod qi)
    prod = {}
    for i in range(rns):
        s = slot(i)
        q = moduli[s]
        ops = port.ntt_forward(np.concatenate([c % U64(q) for c in coef]), n, q)  # one transform call per modulus
        for k in range(kcc):
            off = (k * key_modulus_size + s) * n
            acc = np.zeros(n, dtype=U64)
            for j in range(decomp):
                key = np.asarray(keys[j][off:off + n], dtype=U64) % U64(q)
                acc = port.add_mod(acc, port.mult_mod(ops[j * n:(j + 1) * n], key, q), q)
            prod[i, k] = acc
    # mod-down by the special prime: result_i += (prod_i - NTT_qi(centred special part mod qi)) * modswitch_i
    q_last = moduli[key_modulus_size - 1]
    half = q_last >> 1
    out = np.array(result, dtype=U64, copy=True)
    for k in range(kcc):
        t_last = port.add_mod(port.ntt_inverse(prod[decomp, k], n, q_last), half, q_last)
        for i in range(decomp):
            qi = moduli[i]
            centred = port.sub_mod(t_last % U64(qi), half % qi, qi)
            d = port.sub_mod(prod[i, k], port.ntt_forward(centred, n, qi), qi)
            d = port.mult_mod(d, np.full(n, int(modswitch[i]) % qi, dtype=U64), qi)
            dst = slice(n * (decomp * k + i), n * (decomp * k + i + 1))
            out[dst] = port.add_mod(out[dst], d, qi)
    return out


class Case(NamedTuple):
    """One key-switch configuration: moduli, keys and modswitch factors; ciphertexts come from ciphertext()."""
    n: int
    decomp: int
    kms: int            # key_modulus_size
    kcc: int            # key_component_count
    mods: list
    keys: list
    modswitch: list
    digit_factor: int   # digits are drawn from [0, digit_factor * q_j)
    wraps: bool         # the checkers' 128-bit accumulator can wrap on this case (see can_wrap)

    @property
    def rns(self):
        return self.decomp + 1

    @property
    def shape(self):
        """(n, decomp, key_modulus_size, rns_modulus_size, key_component_count, moduli): the arguments every
        KeySwitch entry point takes between the buffers and the keys"""
        return self.n, self.decomp, self.kms, self.rns, self.kcc, self.mods


def can_wrap(mods, decomp):
    """Whether decomp lazy products (4q - 1)(q - 1) can exceed a 128-bit sum for the largest modulus the switch uses
    (the digits' and the special prime's; the unused key slots are never read)"""
    q = max(mods[:decomp] + [mods[-1]])
    return decomp * (4 * q - 1) * (q - 1) > (1 << 128) - 1


def make_case(port, name, n=None):
    """The named configuration at degree n (default: the degree the GPU tests use).

    uniform       4 digits of 50-bit primes: the shape every older test has
    kcc1, kcc3    3 digits of 50-bit primes with key_component_count 1 and 3
    one_digit     1 digit (SEAL's level above the bottom) of a 50-bit prime, so rns_modulus_size = 2
    slots         kcc3 with 3 unused key slots between the digits and the special prime
                  (key_modulus_size = rns_modulus_size + 3)
    slots2        slots with key_component_count 2, the only count the rotations take
    small_special 3 digits of 50-bit primes and a 29-bit special prime, smaller than every digit: its inverse transform
                  runs the 32-bit-word kernels, and the mod-down moves values into larger moduli
    kcc3_wrap     17 digits just below 2^61 with key_component_count 3: one multiply-accumulate launch holds 16 digits
                  there, so every modulus takes two launches
    wrap17        kcc3_wrap with key_component_count 2: the rotations' two launches (16 + 1 digits) per element
    seal_chain    a SEAL-style chain: first digit just below 2^61, larger than the special prime (just above 2^60),
                  then 40-bit digits, so the multi-modulus transforms run in WIDE mode; digits in [0, 2q); one unused
                  key slot between the digits and the special prime (key_modulus_size = rns_modulus_size + 1)
    word_classes  a 58-bit, a 29-bit and a 50-bit digit (the three word classes of the transforms) and a 45-bit
                  special prime, larger than one digit and smaller than the others
    wrap_keys     29 digits + the special prime, the largest NTT primes below 2^61, every key word q - 1: the
                  checkers' accumulator wraps (a sum of more than 16 products can reach 2^128)
    wrap_blocks   70 digits (more than one 64-entry parameter block) of primes just below 2^61, random keys
    """
    primes = port.generate_primes
    kcc, digit_factor, key_fill = 2, 1, None
    if name == "uniform":
        n = n or 1 << 12
        mods = primes(5, 50, True, n)
        decomp = 4
    elif name in ("kcc1", "kcc3", "slots", "slots2"):
        n = n or 1 << 12
        decomp, kcc = 3, {"kcc1": 1, "slots2": 2}.get(name, 3)
        mods = primes(7 if name in ("slots", "slots2") else 4, 50, True, n)
    elif name == "one_digit":
        n = n or 1 << 12
        decomp = 1
        mods = primes(2, 50, True, n)
    elif name == "small_special":
        n = n or 1 << 12
        decomp = 3
        mods = primes(3, 50, True, n) + primes(1, 29, True, n)
        assert mods[-1] < 1 << 30 and mods[-1] < min(mods[:decomp])
    elif name in ("kcc3_wrap", "wrap17"):
        n = n or 1 << 12
        decomp, kcc = 17, 3 if name == "kcc3_wrap" else 2
        mods = primes(18, 60, False, n)
    elif name == "seal_chain":
        n = n or 1 << 12
        decomp = 4
        mods = (primes(1, 60, False, n) + primes(3, 40, True, n) + primes(1, 45, True, n)
                + primes(1, 60, True, n))
        assert mods[0] > mods[-1] > 1 << 60
        digit_factor = 2
    elif name == "word_classes":
        n = n or 1 << 12
        decomp = 3
        mods = (primes(1, 58, True, n) + primes(1, 29, True, n) + primes(1, 50, True, n)
                + primes(1, 45, True, n))
    elif name == "wrap_keys":
        n = n or 1 << 12
        decomp = 29
        mods = primes(30, 60, False, n)
        key_fill = "q-1"
    elif name == "wrap_blocks":
        n = n or 1 << 11
        decomp = 70
        mods = primes(71, 60, False, n)
    else:
        raise ValueError(name)
    mods = [int(q) for q in mods]
    kms = len(mods)
    assert kms >= decomp + 1 and len(set(mods)) == kms
    seed = 1000 * sum(map(ord, name)) + n

    def key_word(j, k, i):
        if key_fill == "q-1":
            return np.full(n, mods[i] - 1, dtype=U64)
        return uniform_below(seed + 100000 * j + 1000 * k + i, n, mods[i])

    keys = [np.concatenate([key_word(j, k, i) for k in range(kcc) for i in range(kms)]) for j in range(decomp)]
    modswitch = [port.inverse_mod(mods[-1] % mods[i], mods[i]) for i in range(decomp)]
    return Case(n, decomp, kms, kcc, mods, keys, modswitch, digit_factor, can_wrap(mods, decomp))


def ciphertext(case, seed):
    """(result, t_target) of one ciphertext: result canonical, digits below digit_factor * q_j"""
    n, d = case.n, case.decomp
    result = np.concatenate([uniform_below(seed * 7919 + 50 * k + i, n, case.mods[i])
                             for k in range(case.kcc) for i in range(d)])
    t_target = np.concatenate([uniform_below(seed * 104729 + j, n, case.digit_factor * case.mods[j]) for j in range(d)])
    return result, t_target


def expected(port, case, result, t_target):
    return key_switch_exact(port, result, t_target, *case.shape, case.keys, case.modswitch)
