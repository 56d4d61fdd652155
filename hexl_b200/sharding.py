"""Host-side sharding of independent units (polynomials / RNS residues) over GPUs.

The hot path has no data dependence between units (SURVEY.md 8(e)), so scaling
is a contiguous block split with no data-path collective.  The same rule is
used by the C ABI for host-pointer calls over several devices
(hexl_b200_set_host_devices, csrc/capi.h stage_items) and by bench.py's ranks.
"""
from __future__ import annotations


def split_units(total: int, parts: int) -> list[tuple[int, int]]:
    """[lo, hi) of each of `parts` contiguous blocks covering range(total); block
    sizes differ by at most one unit (e.g. 30 moduli over 8 GPUs -> 4,4,4,4,4,4,3,3
    up to ordering)."""
    if parts <= 0:
        raise ValueError("parts must be positive")
    return [(total * p // parts, total * (p + 1) // parts) for p in range(parts)]


def rank_block(total: int, rank: int, world: int) -> tuple[int, int]:
    return split_units(total, world)[rank]
