"""Lane-major order of the deepest four twiddle levels in the device tables (CPU only).

Where the rows of a transform are 4096 points (N = 2^12 and N >= 2^14), the last register pass of every row
(ntt_kernels.cuh: reg_stages at LB = 0) reads, for thread-row U = (row in polynomial) * 256 + u and level
j = 0..3 of the deepest four (depth log_n - 4 + j), entry U * 2^j + g for g < 2^j.  In node order adjacent lanes
are 2^j entries apart.  The device copies (capi_ntt.cu: device_order) store that entry at lane_major(U, g, j)
(internal.h) instead, and the kernel reads it there from one per-thread base plus g << 5.  These tests restate the
mapping, the old and the new address of every fetch, and count the 128-byte lines each warp-wide load touches.
"""
import numpy as np
import pytest

ROW_THREADS = 256     # threads of a 4096-point row: 16 coefficients each


def lanes_major(log_n):
    """internal.h: twiddle_lanes_major, pick_row_log(log_n) == 12"""
    return (log_n if log_n <= 13 else 12) == 12


def lane_major(U, g, j):
    """internal.h: lane_major"""
    return ((U >> 5) << (j + 5)) + (g << 5) + (U & 31)


def device_order(log_n):
    """capi_ntt.cu: device_order -- node[k] is the tree node whose twiddle sits at position k of the device copy"""
    node = np.arange(1 << log_n, dtype=np.int64)
    if lanes_major(log_n):
        for j in range(4):
            level = 1 << (log_n - 4 + j)
            i = np.arange(level, dtype=np.int64)
            node[level + lane_major(i >> j, i & ((1 << j) - 1), j)] = level + i
    return node


LANE_LOGS = [log_n for log_n in range(1, 21) if lanes_major(log_n)]


def last_pass_fetches(log_n):
    """Every twiddle fetch of the last register pass of every row of one polynomial: yields (beta, g, old, new),
    old = the tree node in node order (the previous address), new = the position the kernel reads now; both are
    [rows, 256] arrays indexed by (row, u)."""
    rows = 1 << (log_n - 12)
    r = np.arange(rows, dtype=np.int64)[:, None]
    u = np.arange(ROW_THREADS, dtype=np.int64)[None, :]
    base = rows + r                                   # root node of the row
    for beta in (3, 2, 1, 0):                         # index bit of the stage; the level is j = 3 - beta
        j = 3 - beta
        for g in range(1 << j):
            old = (base << (11 - beta)) + (u << j) + g
            new = (base << (11 - beta)) + lane_major(u, 0, j) + (g << 5)
            yield beta, g, old, new


def lines_per_warp(pos, entry_bytes):
    """distinct 128-byte lines of each warp-wide load; pos is [rows, 256] (table positions), the table 128-byte aligned"""
    lines = (pos * entry_bytes) // 128
    warps = lines.reshape(lines.shape[0], ROW_THREADS // 32, 32)
    return np.array([[len(set(w)) for w in row] for row in warps])


def test_lane_major_transforms():
    assert LANE_LOGS == [12, 14, 15, 16, 17, 18, 19, 20]


@pytest.mark.parametrize("log_n", LANE_LOGS)
def test_mapping_is_a_bijection_on_each_level(log_n):
    for j in range(4):
        level = 1 << (log_n - 4 + j)
        i = np.arange(level, dtype=np.int64)
        pos = lane_major(i >> j, i & ((1 << j) - 1), j)
        assert np.array_equal(np.sort(pos), i), (log_n, j)
        # the additive split the kernel relies on: g enters as g << 5
        assert np.array_equal(pos, lane_major(i >> j, 0, j) + ((i & ((1 << j) - 1)) << 5))
    node = device_order(log_n)
    assert np.array_equal(node[: 1 << (log_n - 4)], np.arange(1 << (log_n - 4)))   # the levels above keep node order


@pytest.mark.parametrize("log_n", LANE_LOGS)
def test_new_address_reads_the_same_node(log_n):
    node = device_order(log_n)
    for beta, g, old, new in last_pass_fetches(log_n):
        # the pass reads the deepest four levels only
        depth = np.floor(np.log2(old)).astype(np.int64)
        assert (depth == log_n - 1 - beta).all()
        assert np.array_equal(node[new], old), (log_n, beta, g)


@pytest.mark.parametrize("entry_bytes", [16, 8])    # Twiddle (64-bit modes), Twiddle32 (SMALL)
@pytest.mark.parametrize("log_n", [12, 14, 16, 17, 20])
def test_each_warp_load_touches_the_fewest_lines(log_n, entry_bytes):
    fewest = 32 * entry_bytes // 128
    old_total = new_total = 0
    for beta, g, old, new in last_pass_fetches(log_n):
        per_warp = lines_per_warp(new, entry_bytes)
        assert (per_warp == fewest).all(), (log_n, entry_bytes, beta, g)
        old_total += lines_per_warp(old, entry_bytes)
        new_total += per_warp
    # per warp and row: 15 loads; node order needed 340 line requests of 16-byte entries (170 of 8-byte ones)
    assert (new_total == 15 * fewest).all()
    assert (old_total == {16: 340, 8: 170}[entry_bytes]).all()


@pytest.mark.parametrize("log_n", [2, 3, 8, 11, 13])
def test_other_row_lengths_keep_node_order(log_n):
    assert np.array_equal(device_order(log_n), np.arange(1 << log_n))
