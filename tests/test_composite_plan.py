"""The scratch rounds of the RNS composites, restated in tests/composite_plan.py, against the host sources that run them
and against the shapes of tests/test_gpu_composite_rounds.py (CPU only).

The GPU test is only worth its time if every one of its calls runs more than one round and the last round is shorter
than the others, so that a round that reads or writes the first round's polynomials (or moduli) again gives a wrong
answer somewhere.  This file asserts that of every shape, and that the formulas are still the ones the host sources run."""
import os

import pytest

import composite_plan as plan
import rescale_exact as rx

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _several_uneven(rounds):
    return len(rounds) >= 2 and rounds[-1] < rounds[0] and all(r == rounds[0] for r in rounds[:-1])


def test_formulas_are_the_ones_the_host_sources_run():
    csrc = os.path.join(ROOT, "hexl_b200", "csrc")
    with open(os.path.join(csrc, "internal.h")) as f:
        assert f"constexpr int kParamBlock = {plan.PARAM_BLOCK};" in f.read()
    for what, (name, lines) in plan.SOURCE.items():
        with open(os.path.join(csrc, name)) as f:
            src = f.read()
        for line in lines:
            assert line in src, f"{what}: {name} no longer has `{line}`; restate the change in composite_plan.py"


def test_spot_values():
    assert plan.rescale_rounds(1 << 16, 31, 35) == [16, 16, 3]
    assert plan.rescale_rounds(1 << 14, 70, 33) == [31, 2]
    assert plan.rescale_rounds(1 << 16, 31, 2) == [2]            # test_gpu_rescale.py's seal_n16: one round
    assert plan.rescale_rounds(1 << 20, 6, 1) == [1]
    assert plan.galois_inplace_rounds(1 << 16, 31, 35) == [16, 16, 3]
    assert plan.galois_inplace_rounds(1 << 20, 6, 3) == [3]       # test_gpu_galois.py's largest in-place call
    assert plan.key_switch_rounds(1 << 16, 30, 31) == [17, 14]
    assert plan.key_switch_rounds(1 << 17, 29, 30) == [8, 8, 8, 6]
    assert plan.key_switch_rounds(1 << 12, 29, 30) == [30]
    assert plan.ks_mac_digits_per_launch((1 << 61) - 1) == 16
    assert plan.ks_mac_digits_per_launch((1 << 60) - 1) == 64
    assert plan.ks_mac_launches(30, (1 << 61) - 1) == [16, 14]


@pytest.mark.parametrize("shape", sorted(plan.RESCALE_SHAPES))
def test_rescale_shapes_run_several_uneven_rounds(port, shape):
    n, name, limbs, count = plan.RESCALE_SHAPES[shape]
    mods = rx.chain(port.generate_primes, n, name, limbs)
    assert len(mods) == limbs
    rounds = plan.rescale_rounds(n, limbs, count)
    assert _several_uneven(rounds), rounds
    assert sum(rounds) == count


def test_rescale_blocks_shape_splits_every_round_into_parameter_blocks():
    n, _, limbs, _ = plan.RESCALE_SHAPES["blocks_n14"]
    assert limbs - 1 > plan.PARAM_BLOCK


def test_galois_shape_runs_several_uneven_rounds():
    n, _, limbs, count = plan.GALOIS_SHAPE
    assert _several_uneven(plan.galois_inplace_rounds(n, limbs, count))


@pytest.mark.parametrize("shape", sorted(plan.KS_SHAPES))
def test_key_switch_shapes_run_several_uneven_rounds(port, shape):
    logn, decomp = plan.KS_SHAPES[shape]
    n = 1 << logn
    mods = [int(q) for q in port.generate_primes(decomp + 1, 60, False, n)]
    assert all((1 << 60) < q < (1 << 61) for q in mods)
    rounds = plan.key_switch_rounds(n, decomp, decomp + 1)
    assert _several_uneven(rounds), rounds
    # within every round the multiply-accumulate takes more than one launch, the last one shorter
    assert _several_uneven(plan.ks_mac_launches(decomp, max(mods)))
    # with moduli below 2^60 it takes one: the GPU test counts the difference
    assert plan.ks_mac_launches(decomp, (1 << 60) - 1) == [decomp]
