"""Multiplier-pipe budget of the flagship transform kernels, and the lazy ranges that budget relies on (CPU only).

H100 has no 64-bit integer multiplier: every IMAD and IMAD.WIDE of the 64-bit NTT kernels runs on the FMA-heavy
pipe, which bounds them (DESIGN.md 4.1).  The budget test counts, in the SASS of the built library, the heavy-pipe
cycles of the FAST-mode kernels of the N = 2^16 benchmark (ntt_pipe_fwd<kFast, 4>, ntt_fused_inv<kFast, 4>) with
the model's weights -- 4 per IMAD.WIDE, 2 per narrow IMAD (IMAD.X, IMAD.MOV, ... included) -- and holds them at or
below what the current code compiles to.  The kernels are straight-line per work item, so the static count is the
dynamic count of one column item plus one row item.

The range tests restate, on exact integers (tests/arith_model.py), the reductions that replaced multiplies there:
the two-product Barrett of the FAST forward output, the three-product quotient of the inverse root stage, and the
conditional subtractions of the FAST inverse pass fix-ups."""
import os
import random
import re
import shutil
import subprocess

import pytest

import arith_model as am
from test_kernel_resources import kernel_resources

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "hexl_b200", "lib", "libhexl_b200.so")

# heavy-pipe cycles per thread for one column item + one row item (128 butterflies, 5 wide + 4 narrow each = 3584)
HEAVY_BUDGET = {"12ntt_pipe_fwdILi1ELi4EE": 3886, "13ntt_fused_invILi1ELi4EE": 3998}
FRAME_BUDGET = {"12ntt_pipe_fwdILi1ELi4EE": 0, "13ntt_fused_invILi1ELi4EE": 24}
_INSN = re.compile(r"^\s+/\*[0-9a-f]{4}\*/\s+(?:@!?U?P[0-9T]\s+)?([A-Z0-9_.]+)")


def heavy_cycles(sass):
    wide = narrow = 0
    for line in sass.splitlines():
        m = _INSN.match(line)
        if not m:
            continue
        op = m.group(1)
        if op.startswith("IMAD.WIDE"):
            wide += 1
        elif op == "IMAD" or op.startswith("IMAD."):
            narrow += 1
    return 4 * wide + 2 * narrow, wide, narrow


def kernel_sass():
    if not os.path.exists(LIB):
        pytest.fail(f"{LIB} is missing: build the library first (python hexl_b200/build.py)")
    tool = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
    if not os.path.exists(tool):
        pytest.skip("cuobjdump not found")
    txt = subprocess.run([tool, "-sass", LIB], capture_output=True, text=True, check=True).stdout
    return {part.split("\n")[0].strip(): part for part in re.split(r"\n\s*Function : ", txt)[1:]}


@pytest.mark.parametrize("frag", sorted(HEAVY_BUDGET))
def test_heavy_pipe_budget(frag):
    hits = [(name, body) for name, body in kernel_sass().items() if frag in name]
    assert len(hits) == 1, f"{frag}: {len(hits)} kernels match"
    cycles, wide, narrow = heavy_cycles(hits[0][1])
    assert cycles <= HEAVY_BUDGET[frag], f"{frag}: {cycles} heavy-pipe cycles ({wide} wide, {narrow} narrow)"


@pytest.mark.parametrize("frag", sorted(FRAME_BUDGET))
def test_no_new_stack_frame(frag):
    hits = [r for name, r in kernel_resources("ntt.cu").items() if frag in name]
    assert len(hits) == 1, f"{frag}: {len(hits)} kernels match"
    assert hits[0][0] <= FRAME_BUDGET[frag], f"{frag}: {hits[0][0]} B stack frame"


def _moduli(lo_bits, hi_bits, rng, count=8):
    out = [(1 << lo_bits) + 1, (1 << hi_bits) - 1, (1 << hi_bits) - 59, (1 << (hi_bits - 1)) + 1]
    out += [rng.randrange(1 << lo_bits, 1 << hi_bits) | 1 for _ in range(count)]
    return out


def _below(bound, rng, count):
    """values below `bound`: its edges, then random ones"""
    vals = [0, 1, bound - 1, bound - 2, bound >> 1, (bound >> 1) - 1, (bound >> 1) + 1]
    vals += [rng.randrange(bound) for _ in range(count)]
    return [v for v in vals if 0 <= v < bound]


def _near_multiples(q, top, rng):
    """k*q - 1, k*q, k*q + 1 for every k up to `top`"""
    return [v for k in range(top + 1) for v in (k * q - 1, k * q, k * q + 1) if 0 <= v < (1 << 64)]


def test_fast_forward_output_two_product_barrett():
    """fwd_out<kFast>: barrett_lazy3_bigq lands below 3q for every value the FAST forward reaches (< 84q, and indeed
    any 64-bit word); two conditional subtractions (2q, q) then give the canonical value, and < 3q already meets
    output_mod_factor 4."""
    rng = random.Random(11)
    for q in _moduli(32, 56, rng):
        assert 84 * q < (1 << 63)
        for x in _near_multiples(q, 84, rng) + _below(84 * q, rng, 300) + _below(1 << 64, rng, 50):
            r = am.barrett_lazy3_bigq(x, q)
            assert r < 3 * q and (r - x) % q == 0, (q, x)
            assert am.csub_s(am.csub_s(r, 2 * q), q) == x % q


@pytest.mark.parametrize("lo_bits,hi_bits", [(32, 56), (56, 61)])   # FAST, WIDE
def test_root_stage_three_product_quotient(lo_bits, hi_bits):
    """inv_bfly_last<kFast / kWide>: x * N^-1 (or N^-1 w) with the three-product quotient is in [0,4q) for ANY
    64-bit x; inv_out then subtracts 2q -> [0,2q) (output_mod_factor 2) and q -> [0,q) (output_mod_factor 1)."""
    rng = random.Random(12)
    for q in _moduli(lo_bits, hi_bits, rng):
        assert 4 * q < (1 << 63)
        for w in [1, 2, q - 1, q - 2, q >> 1] + [rng.randrange(1, q) for _ in range(6)]:
            wp = am.shoup(w, q)
            for x in _below(1 << 64, rng, 120) + [(1 << 64) - 1 - k for k in range(4)] + _near_multiples(q, 8, rng):
                r = am.mul_tw(x, w, wp, q, approx=True)
                assert r < 4 * q and (r - x * w) % q == 0, (q, w, x)
                lazy = am.csub_s(r, 2 * q)
                assert lazy < 2 * q and am.csub_s(lazy, q) == (x * w) % q


def fixup(x, bound_q, q):
    """inv_pass_fixup<K, ...> on one slot bounded by bound_q * q: Barrett above 32q, else halving subtractions"""
    if bound_q > 32:
        return am.barrett_lazy3_bigq(x, q)
    if bound_q > 2 * am.K_FAST_BOUND:
        x = am.csub_s(x, 16 * q)
    if bound_q > am.K_FAST_BOUND:
        x = am.csub_s(x, 8 * q)
    return x


@pytest.mark.parametrize("K", [1, 2, 3, 4, 5])
def test_fast_inverse_fixup_by_subtraction(K):
    """Every slot of a K-stage FAST inverse pass is back below 8q after the fix-up, congruent, and only the slots
    whose bound exceeds 32q (the all-sum slot from K = 3 on; at K = 5 also the 64q slot) still take a multiply."""
    rng = random.Random(13)
    bounds = [am.inv_slot_bound(K, low) for low in range(1 << K)]
    sim, _, ok = am.simulate_inverse_pass_bounds(K, 1 << K)
    assert ok and sim == bounds
    assert all(b & (b - 1) == 0 for b in bounds)   # powers of two: each subtraction halves the bound
    barrett = [low for low, b in enumerate(bounds) if b > 32]
    assert barrett == {1: [], 2: [], 3: [0], 4: [0], 5: [0, 1]}[K]
    for q in _moduli(32, 56, rng, 4):
        for b in sorted(set(bounds)):
            assert b * q < (1 << 64)
            for x in _near_multiples(q, b, rng) + _below(b * q, rng, 200):
                if x >= b * q:
                    continue
                r = fixup(x, b, q)
                assert r < am.K_FAST_BOUND * q and (r - x) % q == 0, (K, b, q, x)
