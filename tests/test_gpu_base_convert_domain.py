"""FastBaseConvert across the domain its API accepts, against plain Python integers.

The call takes any pairwise-coprime sources and any targets in (1, 2^61): not only the NTT primes the key switch feeds
it.  The reference is hybrid_exact.fast_base_convert_int,
    result_t = (sum_i [x_i (Q/q_i)^-1]_{q_i} (Q/q_i)) mod t,
with no modular helper that assumes odd or NTT-friendly moduli (tests/test_hybrid_exact.py pins it to the modular
model on primes).  Covered: targets 2, 3, 4, 2^60, even 61-bit and 5-bit ones far below 60-bit sources (so every
y_i >= t), composite and even sources, one source, 64 sources of q - 1, a target equal to a source, n on both sides of
the 64-slot tile and the scalar path, on device buffers, 8-byte offset views and host buffers."""
import math

import numpy as np
import pytest

import hybrid_exact as hx
from test_gpu_hybrid_key_switch import SENTINEL, _check, dev, host
from util import uniform_below

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

U64 = np.uint64


@pytest.fixture(scope="module", autouse=True)
def _need_cuda(hb):
    if not torch.cuda.is_available() or hb.device_count() == 0:
        pytest.fail("gpu-marked test collected on a machine without CUDA")


def _case(port, name):
    """(sources, targets)"""
    p60 = [int(q) for q in port.generate_primes(67, 60, False, 2)]
    p50 = [int(q) for q in port.generate_primes(8, 50, True, 2)]
    if name == "small_targets":      # 60-bit sources into targets far below them, powers of two and an even 61-bit one
        return p60[:3], [2, 3, 4, 17, 31, 16, 1 << 60, (1 << 61) - 2, (1 << 61) - 1]
    if name == "composite_sources":  # pairwise coprime, none prime but 2^20 even
        return ([15, (1 << 40) + 1, 7 * 11 * 13 * 17 * 19 * 23, 1000003 * 1000033, 1 << 20],
                [p50[0], 9, 1 << 33, (1 << 61) - 3, 6])
    if name == "one_source":
        return [p60[0]], [p50[0], 2, (1 << 61) - 2, p60[1]]
    if name == "sixty_four":         # every word q - 1, into 3 targets that are neither prime NTT moduli nor odd
        return p60[:64], [(1 << 61) - 1, 1 << 60, 3]
    if name == "target_is_a_source":
        return p50[:3], [p50[1], p50[5], p50[0] * 2]
    if name == "ntt_primes":         # the key switch's own domain
        return p50[:3], p50[3:8]
    raise KeyError(name)


CASES = ["small_targets", "composite_sources", "one_source", "sixty_four", "target_is_a_source", "ntt_primes"]


def _inputs(src, n, count, name):
    if name == "sixty_four":
        return np.concatenate([np.full(n, q - 1, dtype=U64) for _ in range(count) for q in src])
    x = np.concatenate([uniform_below(977 * p + i, n, q) for p in range(count) for i, q in enumerate(src)])
    per = len(src) * n
    for p in range(count):  # the extremes of every limb
        for i, q in enumerate(src):
            x[p * per + i * n] = q - 1
            x[p * per + (i + 1) * n - 1] = 0 if n > 1 else q - 1
    return x


@pytest.mark.parametrize("n", [1, 63, 64, 65, (1 << 16) + 1])
@pytest.mark.parametrize("name", CASES)
def test_fast_base_convert_domain(hb, port, name, n):
    src, dst = _case(port, name)
    assert all(math.gcd(a, b) == 1 for i, a in enumerate(src) for b in src[:i])
    assert all(1 < m < 1 << 61 for m in src + dst)
    if name == "sixty_four" and n > 65:
        pytest.skip("64 sources are covered up to n = 65; the tile edges are what n adds")
    count = 2
    x = _inputs(src, n, count, name)
    per = len(src) * n
    exp = np.concatenate([hx.fast_base_convert_int(x[p * per:(p + 1) * per], n, src, dst) for p in range(count)])
    # device buffers (16-byte accesses when n is even)
    out = torch.full((exp.size,), -1, dtype=torch.int64, device="cuda")
    xin = dev(x)
    hb.FastBaseConvert(out, xin, n, src, dst, count)
    torch.cuda.synchronize()
    _check(host(out), exp, f"{name}, n = {n}, device")
    assert torch.equal(xin, dev(x)), "the operand changed"
    # 8-byte offset views between guard words: the word-at-a-time kernel
    buf = torch.full((exp.size + 2,), SENTINEL - (1 << 64), dtype=torch.int64, device="cuda")
    xo = torch.full((x.size + 2,), SENTINEL - (1 << 64), dtype=torch.int64, device="cuda")
    xo[1:-1] = dev(x)
    hb.FastBaseConvert(buf[1:-1], xo[1:-1], n, src, dst, count)
    torch.cuda.synchronize()
    got = host(buf)
    _check(got[1:-1], exp, f"{name}, n = {n}, offset view")
    assert got[0] == SENTINEL and got[-1] == SENTINEL, "a guard word next to the result was written"
    assert (host(xo)[1:-1] == x).all() and host(xo)[0] == SENTINEL and host(xo)[-1] == SENTINEL
    # host buffers, on one device and split over two
    for devices in ([], [0, 0]):
        try:
            hb.set_host_devices(devices)
            got = np.full(exp.size, SENTINEL, dtype=U64)
            hb.FastBaseConvert(got, x.copy(), n, src, dst, count)
        finally:
            hb.set_host_devices([])
        _check(got, exp, f"{name}, n = {n}, host {devices}")
