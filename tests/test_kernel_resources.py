"""Compiler resource report of the NTT kernels (CPU only: reads the `ptxas -v` logs hexl_b200/build.py writes).

The transform kernels keep their coefficients in per-thread register arrays (`E v[16]`, `E v[R]`).  When an index
into such an array is not a compile-time constant, the array is placed in local memory and every butterfly stage
round-trips through L1/L2; ptxas then reports a stack frame with "0 bytes spill".  These tests fail on any kernel
whose stack frame is more than what ptxas spilled, and hold the kernels of the flagship workload (forward + inverse,
N = 2^16, 55-bit modulus) to at most a 16-byte genuine spill.
"""
import importlib.util
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_spec = importlib.util.spec_from_file_location("_hexl_b200_build", os.path.join(ROOT, "hexl_b200", "build.py"))
_build = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(_build)

TRANSFORM_SOURCES = ["ntt.cu", "ntt_multi.cu"]
# local memory not accounted for by spills: anything this large is at least a two-element 64-bit array
MAX_UNSPILLED_FRAME = 8
MAX_FLAGSHIP_FRAME = 16
# Itanium-mangled name fragments: ntt_row_fwd<kFast, 12>, ntt_row_inv<kFast, 12>, ntt_col<kFast, 4, true / false>
FLAGSHIP = ["11ntt_row_fwdILi1ELi12EE", "11ntt_row_invILi1ELi12EE", "7ntt_colILi1ELi4ELb1EE", "7ntt_colILi1ELi4ELb0EE"]

_PROPS = re.compile(r"Function properties for (\S+)\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                    r"(\d+) bytes spill loads")


def kernel_resources(src):
    """{mangled kernel name: (stack frame, spill stores, spill loads)} from the ptxas log of one source."""
    log = os.path.join(_build.OBJ, os.path.splitext(src)[0] + ".o.log")
    if not os.path.exists(log):
        pytest.fail(f"{log} is missing: build the library first (python -m hexl_b200.build)")
    with open(log) as f:
        txt = f.read()
    return {name: tuple(int(x) for x in rest) for name, *rest in _PROPS.findall(txt)}


@pytest.mark.parametrize("src", TRANSFORM_SOURCES)
def test_no_register_array_in_local_memory(src):
    res = kernel_resources(src)
    assert len(res) > 100, f"expected the ptxas report of every kernel of {src}, found {len(res)}"
    bad = [f"{name}: {frame} B frame, {st} B spill stores, {ld} B spill loads"
           for name, (frame, st, ld) in res.items() if frame > max(st, ld) + MAX_UNSPILLED_FRAME]
    assert not bad, f"{len(bad)} kernels of {src} hold local memory beyond their spills:\n" + "\n".join(bad)


def test_flagship_kernels_stay_in_registers():
    res = kernel_resources("ntt.cu")
    for frag in FLAGSHIP:
        hits = [(name, r) for name, r in res.items() if frag in name]
        assert len(hits) == 1, f"{frag}: {len(hits)} kernels match"
        name, (frame, st, ld) = hits[0]
        assert frame <= MAX_FLAGSHIP_FRAME, f"{name}: {frame} B stack frame ({st} B spill stores, {ld} B spill loads)"
