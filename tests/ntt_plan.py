"""The launch plan of the single-modulus transforms (hexl_b200/csrc/ntt.cu) restated in Python, and the parameter set of
tests/test_gpu_ntt_degrees.py.

kernels(q, log_n, batch, forward) lists the kernels one device call of NTT::ComputeForward / ComputeInverse launches, in
launch order, as the Itanium-mangled fragments of their names in the ptxas report (ntt_row_fwd<kFast, 12> is
"11ntt_row_fwdILi1ELi12EE", as in tests/test_kernel_resources.py).  It restates pick_mode, pick_row_log and
plan_col_passes (ntt_kernels.cuh) and plan_single_pass (ntt.cu).  The GPU test asserts that every call launches as many
kernels as the plan names; tests/test_ntt_plan.py asserts that the plan over the GPU test's parameter set names every
kernel ntt.cu compiles, and nothing else.
"""
from __future__ import annotations

import ntt_exact as nx

# ntt_kernels.cuh: enum { kGeneric = 0, kFast = 1, kSmall = 2, kWide = 3 }
GENERIC, FAST, SMALL, WIDE = 0, 1, 2, 3
DEEP = 64                           # plan_single_pass: the pipelined forward takes 64 <= batch < 2^31 polynomials
CHUNK_WORDS = (32 << 20) // 8       # capi.h: kChunkBytes of host-pointer staging, in 64-bit words

# ------------------------------------------------------------------------------------------------ the parameter set
LOGNS = list(range(1, nx.MAX_LOGN + 1))
# one degree per kernel shape: stage kernels, a row kernel alone, and N = 2^14 .. 2^17 (single-pass kernels, or the
# split of one radix-32 column pass at 2^17), and two column passes
SHAPE_LOGNS = (3, 11, 14, 15, 16, 17, 19)
HOST_LOGNS = SHAPE_LOGNS
ROOT_LOGNS = SHAPE_LOGNS
DEEP_LOGNS = (15, 16, 17)
DEEP_BATCHES = (DEEP - 1, DEEP)
# the primes of the batch-threshold test: each side of every boundary of the 64-bit modes (below 2^30 is SMALL's
# largest)
DEEP_PRIMES = ["below_2^30", "above_2^30", "below_2^32", "above_2^32", "below_2^56", "above_2^56", "below_2^61",
               "above_2^61", "below_2^62"]
# one prime per mode, for the calls with a non-minimal root and the host-pointer calls of many chunks
MODE_PRIMES = ["small_25bit", "fast_50bit", "wide_60bit", "below_2^62"]


def batches(log_n):
    """polynomials per device call: 1 and 3, and below N = 4096 one full row CTA (4096 / N rows) and one of one row"""
    n = 1 << log_n
    return [1, 3] + ([4096 // n + 1] if n < 4096 else [])


def chunk_polys(log_n):
    """polynomials per staging chunk of a host-pointer call (capi.h:run_host, staged by stage_items): whole
    polynomials up to kChunkBytes"""
    return max(1, CHUNK_WORDS >> log_n)


def host_chunks(log_n, batch):
    """the polynomials of each staging chunk of a host-pointer call of `batch` polynomials"""
    per = chunk_polys(log_n)
    return [min(per, batch - b) for b in range(0, batch, per)]


def host_batch(log_n, name):
    """polynomials of a host-pointer call: 3, except at 2^15 and 2^16 for MODE_PRIMES, where the pipelined forward
    starts, one full chunk (128 / 64 polynomials) and one of DEEP - 1, so the chunks fall on both sides of the
    threshold"""
    if log_n in (15, 16) and name in MODE_PRIMES:
        return chunk_polys(log_n) + DEEP - 1
    return 3


def cases(primes):
    """every (q, log_n, batch, forward) of one device call of the GPU test (host-pointer calls chunk into these);
    primes(num, bits, first, n) is GeneratePrimes"""
    fixed = nx.single_primes(primes, nx.MAX_LOGN)[:-1]   # all but the smallest prime do not depend on the degree
    table = dict(fixed)
    out = []
    for log_n in LOGNS:
        named = fixed + [("smallest", nx.smallest_prime(1 << log_n))]
        for _, q in named:
            for b in batches(log_n):
                out += [(q, log_n, b, True), (q, log_n, b, False)]
        if log_n in HOST_LOGNS:
            for name, q in named:
                for b in host_chunks(log_n, host_batch(log_n, name)):
                    out += [(q, log_n, b, True), (q, log_n, b, False)]
        if log_n in DEEP_LOGNS:
            out += [(table[name], log_n, b, True) for name in DEEP_PRIMES for b in DEEP_BATCHES]
        if log_n in ROOT_LOGNS:
            out += [(table[name], log_n, 1, fwd) for name in MODE_PRIMES for fwd in (True, False)]
    return out


# ------------------------------------------------------------------------------------------------ the plan
def mode(q):
    """pick_mode: SMALL below 2^30, FAST in [2^32, 2^56), WIDE in [2^56, 2^61), GENERIC otherwise"""
    if q < 1 << 30:
        return SMALL
    if 1 << 32 <= q < 1 << 56:
        return FAST
    return WIDE if 1 << 56 <= q < 1 << 61 else GENERIC


def row_log(log_n):
    """pick_row_log"""
    return log_n if log_n <= 13 else 12


def col_passes(top_stages):
    """plan_col_passes: the top stages in passes of at most 5, as even as possible, larger first"""
    if top_stages <= 0:
        return []
    passes = (top_stages + 4) // 5
    out, left = [], top_stages
    for p in range(passes):
        out.append((left + (passes - p) - 1) // (passes - p))
        left -= out[-1]
    return out


def single_pass(md, log_n, batch, forward):
    """plan_single_pass: ("split", 0) or (kernel, log2 R) with R = N / 4096"""
    lr = log_n - 12
    if lr < 2 or lr > 5:
        return "split", 0
    if md == SMALL:
        return "dsmem", lr
    if forward and lr >= 3 and DEEP <= batch < 1 << 31:
        return "pipe", lr
    if lr <= 3:
        return "dsmem", lr
    if lr == 4:
        return "fused", lr
    return "split", 0


def fragment(name, *args):
    """the mangled fragment of kernel template `name` with int (or bool) arguments: 7ntt_colILi1ELi4ELb1EE"""
    return f"{len(name)}{name}I" + "".join(f"Lb{int(a)}E" if isinstance(a, bool) else f"Li{a}E" for a in args) + "E"


def kernels(q, log_n, batch, forward):
    """the kernels one device call launches, in order (launch_ntt_forward / launch_ntt_inverse)"""
    if batch == 0:
        return []
    if log_n < 4:
        return [fragment("ntt_stage_simple", forward)] * log_n
    md = mode(q)
    kind, lr = single_pass(md, log_n, batch, forward)
    if kind != "split":
        return [fragment(f"ntt_{kind}_{'fwd' if forward else 'inv'}", md, lr)]
    lc = row_log(log_n)
    cols = [fragment("ntt_col", md, r, forward) for r in col_passes(log_n - lc)]
    row = fragment(f"ntt_row_{'fwd' if forward else 'inv'}", md, lc)
    # the inverse runs the row kernel first, then the column passes innermost first
    return cols + [row] if forward else [row] + cols[::-1]
