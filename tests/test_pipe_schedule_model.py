"""Host-side model of the persistent pipelined forward transform's work queue (ntt_kernels.cuh:ntt_pipe_fwd,
ntt_multi.cu:ntt_pipe_multi): item -> (polynomial, role) mapping, coverage, and freedom from deadlock with any number of
resident CTAs.  The 16 column tiles of a polynomial produce, its R rows consume.  No GPU: the kernels' control flow is restated with a cooperative scheduler that lets CTAs claim items
in counter order and run or block exactly as the device code does."""
import random

import pytest


def item_of(i, slots, kprod, units, lookahead):
    """what work item i is: None (skipped), ('prod', poly, j) or ('cons', poly, j)"""
    blk, j = divmod(i, slots)
    producer = j < kprod
    if (blk >= units) if producer else (blk < lookahead):
        return None
    return ("prod", blk, j) if producer else ("cons", blk - lookahead, j - kprod)


@pytest.mark.parametrize("logr", [2, 3, 4, 5])
@pytest.mark.parametrize("units,lookahead", [(1, 1), (3, 1), (5, 2), (7, 48), (64, 48)])
def test_every_work_unit_exactly_once_and_producers_first(logr, units, lookahead):
    ct, r = 4096 // 256, 1 << logr
    slots = ct + r
    kprod = ct
    ncons = slots - kprod
    total = (units + lookahead) * slots
    seen = {}
    for i in range(total):
        it = item_of(i, slots, kprod, units, lookahead)
        if it:
            assert it not in seen
            seen[it] = i
    assert len(seen) == units * slots
    for p in range(units):
        last_prod = max(seen[("prod", p, j)] for j in range(kprod))
        first_cons = min(seen[("cons", p, j)] for j in range(ncons))
        assert last_prod < first_cons             # every producer item is claimed before any consumer of its polynomial
    assert item_of(total, slots, kprod, units, lookahead) is None or total // slots >= units + lookahead


@pytest.mark.parametrize("ctas", [1, 2, 3, 7, 148 * 3])
@pytest.mark.parametrize("units,lookahead", [(1, 1), (4, 1), (9, 3), (40, 48)])
def test_no_deadlock_under_any_interleaving(ctas, units, lookahead):
    """CTAs claim items from one atomic counter; a consumer blocks until its polynomial's producers have all
    FINISHED; producers never block.  Whatever the interleaving (here: random), all work completes."""
    slots, kprod = 16 + 4, 16
    total = (units + lookahead) * slots
    rng = random.Random(ctas * 1000 + units * 10 + lookahead)
    counter = 0
    done = [0] * units
    state = [None] * ctas                          # per CTA: None (idle), ('run', item) or ('wait', item)
    finished = 0
    exited = [False] * ctas
    for _ in range(20 * total + 100 * ctas):
        live = [c for c in range(ctas) if not exited[c]]
        if not live:
            break
        c = rng.choice(live)
        st = state[c]
        if st is None:
            if counter >= total:
                exited[c] = True
                continue
            it = item_of(counter, slots, kprod, units, lookahead)
            counter += 1
            if it is None:
                continue
            state[c] = ("wait", it) if it[0] == "cons" else ("run", it)
        elif st[0] == "wait":
            if done[st[1][1]] == kprod:
                state[c] = ("run", st[1])
        else:
            it = st[1]
            if it[0] == "prod":
                done[it[1]] += 1
            finished += 1
            state[c] = None
    assert all(exited) and finished == units * slots and all(d == kprod for d in done)
