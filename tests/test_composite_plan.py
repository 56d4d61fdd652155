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


# ------------------------------------------------------------------------------ the hybrid family
def _hybrid_mods(port, shape):
    logn, L, K, alpha, dbits, sbits, levels = plan.HYBRID_SHAPES[shape]
    n = 1 << logn
    data = [int(q) for q in port.generate_primes(L, dbits, dbits < 60, n)]
    special = [int(q) for q in port.generate_primes(K + 128, sbits, sbits < 60, n)][-K:]
    return n, L, K, alpha, data + special, levels


def test_hybrid_spot_values():
    assert plan.base_conv_targets(10) == 29 and plan.base_conv_targets(11) == 27
    assert plan.base_conv_targets(1) == 79 and plan.base_conv_targets(64) == 3
    assert plan.base_conv_blocks(11, 29) == [27, 2]
    assert plan.base_conv_blocks(10, 30) == [29, 1]
    assert plan.hybrid_digit_widths(29, 2) == [2] * 14 + [1]
    assert plan.hybrid_mod_up_rounds(1 << 16, 30, 10, 10) == [40]
    assert plan.hybrid_mod_up_rounds(1 << 10, 70, 2, 64) == [64, 8]     # the 64-modulus cap
    assert plan.hybrid_round_slots(28, 30, 25, 6) == [25, 26, 27, 30, 31, 32]
    assert plan.hybrid_mod_down_blocks(30, 10) == [[29, 1]]
    assert plan.hybrid_mod_down_blocks(30, 10, True) == [[27, 2]]
    assert plan.hybrid_mod_down_blocks(70, 2, True) == [[58, 6], [5]]  # 3 sources: 58 targets a launch
    assert plan.relin_tensor_data(28, 25, 6) == 3 and plan.relin_tensor_data(28, 28, 3) == 0
    assert plan.relin_mac_launches(20, (1 << 61) - 1) == [16, 4]
    # 20 digits below 2^61: chunks of 16 and 4 digits, 4 elements per launch, so 6 elements take 2 launches each
    assert plan.weighted_mac_launches(20, 6, (1 << 61) - 1) == [(16, 4), (16, 2), (4, 4), (4, 2)]
    assert plan.weighted_mac_launches(3, 66, (1 << 50) - 1) == [(3, 21), (3, 21), (3, 21), (3, 3)]


def test_hybrid_launches_agree_with_the_earlier_counts():
    """below 2^60 the plan gives the counts the per-call test files derive on their own (one multiply-accumulate per
    round, base_conv_targets from the digit widths), with one launch per transform"""
    import hybrid_exact as hx

    def ntt(forward, units):
        return 1

    def targets(s):
        return (480 - 4 * s) // (5 + s)

    for L, K, alpha, level in [(6, 2, 2, 6), (30, 10, 10, 30), (70, 2, 64, 70), (70, 2, 64, 5), (12, 1, 1, 12)]:
        n = 1 << 12
        basis = [(1 << 45) + 1] * (level + K)
        groups = hx.digits(level, alpha)
        nb = level + K
        ichunk = min(max(1, (256 << 20) // (len(groups) * n * 8)), nb, 64)
        exp = -(-level // 64)
        for b0 in range(0, nb, ichunk):
            cnt = min(ichunk, nb - b0)
            exp += sum(-(-cnt // targets(len(S))) for S in groups) + 2
        exp += 1 + sum(-(-min(64, level - i0) // targets(K)) + 2 for i0 in range(0, level, 64))
        assert plan.hybrid_launches("switch", n, level, K, alpha, basis, ntt) == exp


@pytest.mark.parametrize("shape", sorted(plan.HYBRID_SHAPES))
def test_hybrid_shapes_have_the_plan_their_names_claim(port, shape):
    n, L, K, alpha, mods, levels = _hybrid_mods(port, shape)
    assert len(set(mods)) == L + K
    rounds = {level: plan.hybrid_mod_up_rounds(n, level, K, alpha) for level in levels}
    if shape == "bench_rescale":
        assert rounds == {30: [40]}
        assert plan.hybrid_mod_down_blocks(30, K, True) == [[27, 2]]
        assert plan.hybrid_mod_down_blocks(30, K) == [[29, 1]]
    elif shape == "budget_a2":
        assert rounds == {30: [34, 6], 29: [34, 5]}
        assert plan.hybrid_digit_widths(29, alpha)[-1] == 1
        # the second round holds special primes only, at both levels
        assert plan.hybrid_round_slots(29, L, 34, 5) == [L + j for j in range(5, 10)]
    elif shape == "budget_a3":
        assert rounds == {30: [25, 8], 28: [25, 6]}
        # at level 28 the second round mixes three data limbs with the three special primes, whose key slots are not
        # their positions in B
        assert plan.hybrid_round_slots(28, L, 25, 6) == [25, 26, 27, 30, 31, 32]
        assert plan.relin_tensor_data(28, 25, 6) == 3 and plan.relin_tensor_data(30, 25, 8) == 5
    elif shape == "mixed_chunks":
        assert rounds == {24: [21, 5]}
        assert all(q < 1 << 51 for q in mods[:L]) and all((1 << 60) < q < (1 << 61) for q in mods[L:])
        first, second = max(mods[:21]), max(mods[21:26])
        assert plan.ks_mac_launches(24, first) == [24] and plan.ks_mac_launches(24, second) == [16, 8]
        assert plan.relin_mac_launches(24, first) == [24] and plan.relin_mac_launches(24, second) == [16, 8]
        assert plan.weighted_mac_launches(24, 3, first) == [(24, 2), (24, 1)]
        assert plan.weighted_mac_launches(24, 3, second) == [(16, 3), (8, 3)]
    # every named shape but bench_rescale runs several rounds at every level it is tested at, the last one shorter
    if shape != "bench_rescale":
        assert all(_several_uneven(r) for r in rounds.values()), rounds


def test_every_level_sweep_crosses_each_block_boundary():
    """(L, K, alpha) = (30, 10, 10): the levels of the sweep sit on both sides of the mod-up's 29-target block, the
    mod-down's 29 block and the merged rescale's 27 block"""
    widest = {level: max(len(plan.base_conv_blocks(w, level + 10)) for w in plan.hybrid_digit_widths(level, 10))
              for level in range(1, 31)}
    assert widest[19] == 1 and widest[20] == 2             # 10-modulus digits into 29 and 30 targets
    assert len(plan.hybrid_mod_down_blocks(29, 10)[0]) == 1 and len(plan.hybrid_mod_down_blocks(30, 10)[0]) == 2
    assert len(plan.hybrid_mod_down_blocks(28, 10, True)[0]) == 1
    assert len(plan.hybrid_mod_down_blocks(29, 10, True)[0]) == 2
