"""Parity of the pipelined NTT kernels under the HEXL_B200_PIPE_LOOKAHEAD of the calling environment (run by
tests/test_gpu_parity.py::test_ntt_kernel_variants in its own process, since the library reads the variable once).

Every shape here is one where a pipelined kernel is the default: the single-modulus forward transform at N = 2^15,
2^16 and 2^17 of 64 polynomials, and the multi-modulus forward transform at N = 2^17 of 64 or more units (alone and
inside PolyMultiplyMulti).  Each polynomial of the batch goes through a forward and an inverse transform and must come
back unchanged; a spread of polynomials is compared with the checker."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import hexl_b200 as hb  # noqa: E402
import oracle  # noqa: E402
from util import uniform_below  # noqa: E402

checker = oracle.best_checker()
BATCH = 64
SPREAD = [0, 1, 31, 62, 63]  # polynomials / units compared with the checker


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.uint64).view(np.int64)).cuda()


def host(t):
    return t.cpu().numpy().view(np.uint64)


def poly(v, i, n):
    return v[i * n:(i + 1) * n]


# single modulus: FAST (just above 2^50, just below 2^56), WIDE (just above 2^60), GENERIC (just below 2^62)
for logn in (15, 16, 17):
    n = 1 << logn
    for bits, first in ((50, True), (55, False), (60, True), (61, False)):
        q = hb.GeneratePrimes(1, bits, first, n)[0]
        qq = np.uint64(q)
        t = hb.NTT(n, q)
        x = uniform_below(logn + bits, n * BATCH, q)
        exp = {i: checker.ntt_forward(poly(x, i, n), n, q) for i in SPREAD}
        o = dev(np.zeros_like(x))
        t.ComputeForward(o, dev(x), 1, 1)
        g = host(o)
        assert all((poly(g, i, n) == exp[i]).all() for i in SPREAD), ("fwd", logn, bits)
        t.ComputeInverse(o, o, 1, 1)
        assert (host(o) == x).all(), ("round trip", logn, bits)
        t.ComputeForward(o, dev(x), 1, 4)
        g = host(o)
        assert all((poly(g, i, n) % qq == exp[i]).all() for i in SPREAD) and (g < np.uint64(4) * qq).all(), \
            ("fwd lazy", logn, bits)
        d = dev(x)
        t.ComputeForward(d, d, 1, 1)
        g = host(d)
        assert all((poly(g, i, n) == exp[i]).all() for i in SPREAD), ("fwd in place", logn, bits)
        t.ComputeInverse(d, d, 1, 1)
        assert (host(d) == x).all(), ("round trip in place", logn, bits)
        # extreme inputs: polynomial 0 has every coefficient at the top of its allowed range (the largest lazy growth
        # inside the kernels), the others are uniform in that range
        for in_mf in (1, 4):
            xe = uniform_below(logn + bits + in_mf, n * BATCH, q * in_mf)
            xe[:n] = q * in_mf - 1
            o = dev(np.zeros_like(xe))
            t.ComputeForward(o, dev(xe), in_mf, 1)
            g = host(o)
            for i in (0, 1, BATCH - 1):
                assert (poly(g, i, n) == checker.ntt_forward(poly(xe, i, n), n, q, in_mf, 1)).all(), \
                    ("fwd extreme", logn, bits, in_mf, i)

# multi-modulus batches of 64 or more units at N = 2^17 under WIDE, FAST and GENERIC moduli lists, and the product
# pipeline
n = 1 << 17
for bit_list in ((60, 60, 55), (50, 55), (61, 55)):
    mods = []
    for b in bit_list:
        first = b != 61  # 61: the largest primes below 2^62 (GENERIC)
        for cand in hb.GeneratePrimes(4, b, first, n):
            if cand not in mods:
                mods.append(cand)
                break
    ntts = [hb.NTT(n, q) for q in mods]
    group = -(-BATCH // len(mods))
    sz = n * group
    units = len(mods) * group
    a = np.concatenate([uniform_below(5 * i + 17, sz, q) for i, q in enumerate(mods)])
    b = np.concatenate([uniform_below(5 * i + 18, sz, q) for i, q in enumerate(mods)])
    spread = [0, 1, units // 2, units - 2, units - 1]
    exp_f = {u: checker.ntt_forward(poly(a, u, n), n, mods[u // group]) for u in spread}
    o = dev(np.zeros_like(a))
    hb.ComputeForwardMulti(ntts, o, dev(a), 1, 1, batch_per_modulus=group)
    g = host(o)
    assert all((poly(g, u, n) == exp_f[u]).all() for u in spread), ("multi fwd", bit_list)
    hb.ComputeInverseMulti(ntts, o, o, 1, 1, batch_per_modulus=group)
    assert (host(o) == a).all(), ("multi round trip", bit_list)
    d = dev(a)
    hb.ComputeForwardMulti(ntts, d, d, 1, 4, batch_per_modulus=group)
    g = host(d)
    qs = np.concatenate([np.full(sz, q, dtype=np.uint64) for q in mods])
    assert all((poly(g, u, n) % np.uint64(mods[u // group]) == exp_f[u]).all() for u in spread), \
        ("multi fwd lazy in place", bit_list)
    assert (g < qs * np.uint64(4)).all(), ("multi fwd lazy range", bit_list)
    if max(mods) < (1 << 61):
        hb.PolyMultiplyMulti(ntts, o, dev(a), dev(b), group)
        g = host(o)
        for u in spread:
            q = mods[u // group]
            conv = checker.ntt_inverse(checker.mult_mod(exp_f[u], checker.ntt_forward(poly(b, u, n), n, q), q), n, q)
            assert (poly(g, u, n) == conv).all(), ("poly multiply", bit_list, u)
print("variant ok", {k: v for k, v in os.environ.items() if k.startswith("HEXL_B200_")})
