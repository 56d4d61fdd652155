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


# ------------------------------------------------------------------------------ the evaluator calls
def _recorder():
    calls = []

    def ntt(forward, units):
        calls.append((forward, units))
        return 1
    return calls, ntt


def test_evaluator_spot_values():
    assert [plan.base_conv_t_targets(f) for f in (1, 2, 3, 4, 10, 11, 64)] == [67, 58, 51, 45, 27, 25, 3]
    assert plan.base_conv_t_blocks(10, 30) == [27, 3] and plan.base_conv_t_blocks(11, 29) == [25, 4]
    assert plan.hybrid_mod_down_blocks(30, 10, tau=True) == [[27, 3]]
    assert plan.hybrid_mod_down_blocks(30, 10, True, tau=True) == [[25, 4]]
    assert plan.bgv_mod_switch_rounds(1 << 16, 31, 35) == [16, 16, 3]
    assert plan.bgv_mod_switch_rounds(1 << 14, 70, 33) == [31, 2]
    assert plan.bgv_mod_switch_rounds(1 << 12, 6, 8) == [8]            # test_gpu_bgv.py's in-place counts: one chunk
    # per chunk: the last limbs' inverse transform, then per block of moduli one conversion, a forward transform of
    # delta and the finish; coefficient form: the conversion and the finish
    calls, ntt = _recorder()
    assert plan.bgv_mod_switch_launches(1 << 16, 31, 35, True, ntt) == 3 * (1 + 3)
    assert calls == [(False, 16), (True, 30 * 16), (False, 16), (True, 30 * 16), (False, 3), (True, 30 * 3)]
    assert plan.bgv_mod_switch_launches(1 << 16, 31, 35, False, _one) == 3 * 2
    calls, ntt = _recorder()
    assert plan.bgv_mod_switch_launches(1 << 14, 70, 33, True, ntt) == 2 * (1 + 2 * 3)
    assert calls == [(False, 31), (True, 64 * 31), (True, 5 * 31), (False, 2), (True, 64 * 2), (True, 5 * 2)]
    assert plan.bgv_mod_switch_launches(1 << 14, 70, 33, False, _one) == 2 * 2 * 2
    assert [plan.relin_sum_launches(30, k) for k in (1, 2, 32, 33)] == [0, 1, 1, 2]
    assert plan.relin_sum_launches(70, 65) == 2 * 3
    # BEHZ: the transforms run one handle per polynomial, 64 handles a launch set
    calls, ntt = _recorder()
    assert plan.bfv_launches(62, False, ntt) == 2 + 4 + 1 + 3 + 1
    assert calls == [(True, 64)] * 3 + [(True, 56)] + [(False, 64)] * 2 + [(False, 58)]
    assert plan.bfv_launches(62, True, _one) == 1 + 2 + 1 + 3 + 1
    assert plan.bfv_launches(129, False, _one) == 2 + 9 + 3 + 7 + 1
    # the relinearized BFV call: no inverse transform of the target, the mod-down's per-block transform inverse
    basis = [(1 << 45) + 1] * 8
    calls, ntt = _recorder()
    plan.hybrid_launches("bfv_relin", 1 << 12, 6, 2, 2, basis, ntt, M=13, square=True)
    assert calls == [(True, 26), (False, 39),                  # BfvMultiply: 2M forward, 3M inverse
                     (True, 24),                               # the mod-up's one round: 8 moduli x 3 digits
                     (False, 4), (False, 12)]                  # the mod-down: K x 2, then 6 x 2 data limbs back
    calls, ntt = _recorder()
    plan.hybrid_launches("mul_relin_sum", 1 << 12, 6, 2, 2, basis, ntt, pairs=3)
    assert calls == [(False, 6), (True, 24), (False, 4), (True, 12)]


def test_t_blocks_of_every_hybrid_shape():
    """the t-corrected mod-down's blocks at each HYBRID_SHAPES level, without and with the merged modulus switch: one
    more source (6 + F words per target instead of 5 + F, 6 more for tau) than CKKS's rounded conversion"""
    want = {("bench_rescale", 30): ([[27, 3]], [[25, 4]]),
            ("budget_a2", 30): ([[27, 3]], [[25, 4]]), ("budget_a2", 29): ([[27, 2]], [[25, 3]]),
            ("budget_a3", 30): ([[30]], [[29]]), ("budget_a3", 28): ([[28]], [[27]]),
            ("mixed_chunks", 24): ([[24]], [[23]])}
    got = {(name, level): (plan.hybrid_mod_down_blocks(level, K, tau=True),
                           plan.hybrid_mod_down_blocks(level, K, True, tau=True))
           for name, (_, _, K, _, _, _, levels) in plan.HYBRID_SHAPES.items() for level in levels}
    assert got == want
    # at K = 10 both differ from CKKS's 29 + 1 and 27 + 2
    assert plan.hybrid_mod_down_blocks(30, 10) == [[29, 1]] and plan.hybrid_mod_down_blocks(30, 10, True) == [[27, 2]]


def _earlier_relin(n, level, K, alpha, rescale, fwd, inv, t_sources=False):
    """tests/test_gpu_mul_relin.py's relin_launches (and with t_sources tests/test_gpu_bgv.py's multiply count) below
    2^60: the mod-up with one multiply-accumulate per round, and the mod-down from K + rescale special limbs"""
    import hybrid_exact as hx

    def targets(s):
        return (474 - 4 * s) // (6 + s) if t_sources else (480 - 4 * s) // (5 + s)

    groups, nb = hx.digits(level, alpha), level + K
    ichunk = min(max(1, (256 << 20) // (len(groups) * n * 8)), nb, 64)
    up = inv * -(-level // 64) + sum(sum(-(-min(ichunk, nb - b0) // ((480 - 4 * len(S)) // (5 + len(S))))
                                         for S in groups) + fwd + 1 for b0 in range(0, nb, ichunk))
    lv, k = level - int(rescale), K + int(rescale)
    return up, inv + sum(-(-min(64, lv - i0) // targets(k)) + fwd + 1 for i0 in range(0, lv, 64))


def test_evaluator_launches_agree_with_the_earlier_counts():
    """below 2^60 the plan gives the counts the per-call GPU files derived on their own: test_gpu_mul_relin_sum.py's
    sum_launches, test_gpu_bfv.py's bfv_launches and relinearized count, and test_gpu_bgv.py's switch, rotation,
    multiply and modulus-switch counts, with transforms of different launch counts in each direction"""
    fwd, inv = 2, 3

    def ntt(forward, units):
        return fwd if forward else inv

    n = 1 << 12
    for L, K, alpha, level in [(6, 2, 2, 6), (6, 2, 2, 5), (30, 10, 10, 30), (70, 2, 64, 70), (70, 2, 64, 65),
                               (12, 1, 1, 12), (20, 2, 5, 12), (30, 1, 1, 30)]:
        basis = [(1 << 45) + 1] * (level + K)
        for rescale in (False, True):
            up, down = _earlier_relin(n, level, K, alpha, rescale, fwd, inv)
            for pairs in (1, 2, 33, 65):
                extra = 0 if pairs == 1 else -(-level // 64) * -(-pairs // 32)
                got = plan.hybrid_launches("mul_relin_sum", n, level, K, alpha, basis, ntt, rescale=rescale,
                                           pairs=pairs)
                assert got == up + down + extra, (L, K, alpha, level, rescale, pairs)
            up, down = _earlier_relin(n, level, K, alpha, rescale, fwd, inv, t_sources=True)
            assert plan.hybrid_launches("mul_relin", n, level, K, alpha, basis, ntt, rescale=rescale, tau=True) == \
                up + down
        up, down = _earlier_relin(n, level, K, alpha, False, fwd, inv, t_sources=True)
        assert plan.hybrid_launches("switch", n, level, K, alpha, basis, ntt, tau=True) == up + down
        up2 = up + sum(1 for _ in range(0, level + K, min(max(1, (256 << 20) // (-(-level // alpha) * n * 8)),
                                                          level + K, 64)))   # a second multiply-accumulate per round
        assert plan.hybrid_launches("hoisted", n, level, K, alpha, basis, ntt, elts=2, tau=True) == 2 + up2 + 2 * down
        blocks = -(-(level - 1) // 64)
        assert plan.bgv_mod_switch_launches(n, level, 2, True, ntt) == inv + blocks * (2 + fwd)
        assert plan.bgv_mod_switch_launches(n, level, 2, False, ntt) == 2 * blocks
        for k in (level, level + 1):
            M = level + k + 1
            for square in (False, True):
                inputs = 2 if square else 4
                bfv = (1 if square else 2) + fwd * -(-inputs * M // 64) + -(-M // 64) + inv * -(-3 * M // 64) + 1
                assert plan.bfv_launches(M, square, ntt) == bfv
                up, down = _earlier_relin(n, level, K, alpha, False, fwd, inv)
                lb = -(-level // 64)
                assert plan.hybrid_launches("bfv_relin", n, level, K, alpha, basis, ntt, M=M, square=square) == \
                    bfv + up + down - inv * lb - fwd * lb + inv * lb


def _divisible(units):
    """the GPU tests measure a transform of `units` polynomials as c copies, c a divisor in [2, 64]"""
    return any(max(units, 2) % d == 0 for d in range(2, 65))


def test_evaluator_shapes_have_the_plan_their_names_claim(port):
    import bfv_exact as bfx
    import inner_sum_exact as ix
    # BgvModSwitch: several chunks at both RESCALE_SHAPES, blocks_n14's each in two parameter blocks
    for shape, (n, _, limbs, count) in plan.RESCALE_SHAPES.items():
        assert _several_uneven(plan.bgv_mod_switch_rounds(n, limbs, count)), shape
    assert plan.RESCALE_SHAPES["blocks_n14"][2] - 1 > plan.PARAM_BLOCK
    # the sums: 33 pairs take two tensor-sum chunks, the second shorter; at g = 5 and k = 7, bit 1 has a keyed
    # doubling and a keyed shift (one mod-up for both), and k = 16 doubles four times
    assert _several_uneven(plan._split(33, plan.RELIN_SUM_PAIRS))
    for logn in {v[0] for v in plan.HYBRID_SHAPES.values()}:
        bits = ix.inner_sum_bits(5, 7, 1 << logn)
        assert all(e not in (None, 1) for e in bits[1]), bits
        assert [d is not None for d, _ in ix.inner_sum_bits(5, 16, 1 << logn)] == [True] * 4 + [False]
    # BEHZ_TILES: 129 moduli, tensor blocks 64 + 64 + 1
    logn, l, k = plan.BEHZ_TILES
    assert l == k == plan.PARAM_BLOCK and _several_uneven(plan._split(l + k + 1, plan.PARAM_BLOCK))
    # the host batch: one ciphertext per slot, the last slot of the wrap shorter
    name, level, batch = plan.EVALUATOR_HOST_BATCH
    assert level in plan.HYBRID_SHAPES[name][-1]
    assert _several_uneven(plan._split(batch, plan.STAGING_SLOTS))
    # every transform the plan asks of the new file has a unit count the GPU test can measure
    units = []

    def ntt(forward, u):
        units.append(u)
        return 1
    for name in plan.HYBRID_SHAPES:
        n, L, K, alpha, mods, levels = _hybrid_mods(port, name)
        for level in levels:
            basis = mods[:level] + mods[L:]
            M = level + bfx.seal_base_b_size(mods[:level], 65537) + 1
            for rs in (False, True):
                plan.hybrid_launches("mul_relin_sum", n, level, K, alpha, basis, ntt, rescale=rs, pairs=33)
                plan.hybrid_launches("mul_relin", n, level, K, alpha, basis, ntt, rescale=rs, tau=True)
                for k in (7, 16):
                    ix.inner_sum_launches(n, level, K, alpha, basis, ntt, 5, k, rs)
            plan.hybrid_launches("hoisted", n, level, K, alpha, basis, ntt, elts=2, tau=True)
            for square in (False, True):
                plan.hybrid_launches("bfv_relin", n, level, K, alpha, basis, ntt, M=M, square=square)
    for n, _, limbs, count in plan.RESCALE_SHAPES.values():
        for form in (True, False):
            plan.bgv_mod_switch_launches(n, limbs, count, form, ntt)
    plan.hybrid_launches("bfv_relin", 1 << logn, l, 2, 32, [(1 << 57) + 1] * (l + 2), ntt, M=l + k + 1)
    assert units and all(_divisible(u) for u in units), sorted(u for u in set(units) if not _divisible(u))


# ------------------------------------------------------------------------------ LinearTransformHybridBSGS
def _one(forward, units):
    return 1


def test_bsgs_spot_values():
    below60, above60 = [(1 << 45) + 1] * 8, [(1 << 61) - 1] * 40
    n = 1 << 12
    # (6, 2, 2): one mod-up round of 3 digits (1 + 3 + 1 + 1 launches) and one mod-down block (1 + 1 + 1 + 1)
    babies, giants = (False, True), (False, True)
    # row 0: the identity over the identity, 1 sum launch; row 1: keyed over keyed: baby mod-up 6, 1 sum launch over B,
    # the kcc = 1 mod-down 4, the giant's mod-up 6; the final mod-down 4
    assert plan.bsgs_launches(n, 6, 2, 2, below60, _one, babies, giants, {(0, 0), (1, 1)}) == 6 + 1 + 1 + 4 + 6 + 4
    assert plan.bsgs_launches(n, 6, 2, 2, below60, _one, babies, giants, {(0, 0), (1, 1)}, True) == 22
    # identity rows only: the sums alone, and with the rescale the mod-down by q_5 P of X folded into Y
    assert plan.bsgs_launches(n, 6, 2, 2, below60, _one, babies, giants, {(0, 0)}) == 1
    assert plan.bsgs_launches(n, 6, 2, 2, below60, _one, babies, giants, {(0, 0)}, True) == 1 + 4
    # a keyed giant over the identity baby: no baby mod-up, no kcc = 1 mod-down
    assert plan.bsgs_launches(n, 6, 2, 2, below60, _one, babies, giants, {(1, 0)}) == 1 + 6 + 4
    # no pair at all: nothing
    assert plan.bsgs_launches(n, 6, 2, 2, below60, _one, babies, giants, set()) == 0
    # 30 one-modulus digits below 2^61: 16 + 14 digits per multiply-accumulate, per stored baby and per giant; 65
    # babies in a row: two chunks of sums per block of moduli
    grid = ((True,) * 65, (True,), None)
    up = 1 + 30 * 1 + 1                                                      # one round of 40 moduli at n = 2^12
    down1, down2 = 1 + 2 + 1 + 1, 1 + 2 + 1 + 1                              # base_conv_blocks(10, 30) == [29, 1]
    assert plan.bsgs_launches(n, 30, 10, 1, above60, _one, *grid) == \
        (up + 65 * 2) + 2 * 1 + down1 + (up + 2) + down2
    # every launch of a transform counts: the plan asks for each transform's units
    seen = []
    plan.bsgs_launches(n, 6, 2, 2, below60, lambda f, u: seen.append((f, u)) or 1, babies, giants, {(1, 1)}, True)
    assert seen == [(False, 6), (True, 24),                                  # baby mod-up: 8 moduli x 3 digits
                    (False, 2), (True, 6),                                   # kcc = 1 mod-down: K x 1, 6 x 1
                    (False, 6), (True, 24),                                  # giant mod-up
                    (False, 6), (True, 10)]                                  # merged mod-down: (K + 1) x 2, 5 x 2


def _bsgs_launches_below_2_60(n, level, K, alpha, bspec, gspec, present, rescale, fwd, inv):
    """the count tests/test_gpu_bsgs.py derived on its own before the plan held BSGS: moduli below 2^60, so
    ceil(D / 64) digit chunks per multiply-accumulate, and fwd / inv launches per transform"""
    import hybrid_exact as hx

    def targets(s):
        return (480 - 4 * s) // (5 + s)

    def up(macs):
        groups, nb = hx.digits(level, alpha), level + K
        ichunk = min(max(1, (256 << 20) // (len(groups) * n * 8)), nb, 64)
        return inv * -(-level // 64) + sum(sum(-(-min(ichunk, nb - b0) // targets(len(S))) for S in groups)
                                           + fwd + macs for b0 in range(0, nb, ichunk))

    def down(lv, k):
        return inv + sum(-(-min(64, lv - i0) // targets(k)) + fwd + 1 for i0 in range(0, lv, 64))

    chunks, nb = -(-(-(-level // alpha)) // 64), level + K
    stored = [i for i, (_, k) in enumerate(bspec)
              if k is not None and any((j, i) in present for j in range(len(gspec)))]
    total = up(len(stored) * chunks) if stored else 0
    y_used = False
    for j, (_, gk) in enumerate(gspec):
        row = [i for i in range(len(bspec)) if (j, i) in present]
        if not row:
            continue
        keyed_baby = any(bspec[i][1] is not None for i in row)
        total += -(-(nb if keyed_baby else level) // 64) * -(-len(row) // 64)
        y_used = y_used or keyed_baby or gk is not None
        if gk is not None:
            total += (down(level, K) if keyed_baby else 0) + up(chunks)
    if rescale:
        return total + down(level - 1, K + 1)
    return total + (down(level, K) if y_used else 0)


def test_bsgs_launches_agree_with_the_earlier_counts():
    """below 2^60 the plan gives the counts tests/test_gpu_bsgs.py expected from its own formula, on the grids of its
    test_launch_counts, with transforms of different launch counts in each direction"""
    n = 1 << 12
    bspec = [(1, None), (3, 0), (2 * n - 1, 1), (5, 2), (3, 1)]
    gspec = [(1, None), (9, 0), (25, 1), (2 * n - 1, 2)]
    sparse = {(0, 0), (0, 1), (0, 2), (0, 4), (1, 0), (2, 0), (2, 1), (2, 3), (2, 4)}
    many = [(pow(5, i + 1, 2 * n), i % 3) for i in range(66)]
    grids = [("sparse", bspec, gspec, sparse),
             ("identity rows only", bspec, [(1, None), (1, None)], {(0, 0), (1, 0)}),
             ("keyed giants over the identity baby", bspec, gspec, {(1, 0), (2, 0), (3, 0)}),
             ("66 babies", many, gspec[:2], {(j, i) for j in range(2) for i in range(66)})]
    for L, K, alpha, level in [(6, 2, 2, 6), (30, 10, 10, 30), (70, 2, 64, 70), (12, 1, 1, 12)]:
        basis = [(1 << 45) + 1] * (level + K)
        for name, bspec, gspec, present in grids:
            for rescale in (False, True):
                exp = _bsgs_launches_below_2_60(n, level, K, alpha, bspec, gspec, present, rescale, 2, 3)
                got = plan.bsgs_launches(n, level, K, alpha, basis, lambda f, u: 2 if f else 3,
                                         [k is not None for _, k in bspec], [k is not None for _, k in gspec],
                                         present, rescale)
                assert got == exp, (L, K, alpha, name, rescale)


def test_bsgs_grids_have_the_plan_their_names_claim(port):
    babies, giants, present = plan.BSGS_SPARSE
    rows, stored = plan.bsgs_rows(babies, giants, present)
    assert stored == [1, 3, 4, 5] and babies[2]                 # a keyed baby without a diagonal stores nothing
    assert rows[0] == [0, 1, 5] and not giants[0]              # the identity giant over the identity and keyed babies
    assert rows[1] == [0] and giants[1]                        # a keyed giant, no kcc = 1 mod-down
    assert rows[2] == [0, 3, 4, 5] and giants[2]               # a keyed giant over keyed babies
    assert rows[3] == [] and giants[3]                         # an absent last row: the fold goes to row 2
    babies, giants, present = plan.BSGS_SWEEP
    rows, stored = plan.bsgs_rows(babies, giants, present)
    assert stored == [1, 2] and all(giants[j] and any(babies[i] for i in rows[j]) for j in (1, 2))
    babies, giants, present = plan.BSGS_BENCH
    rows, stored = plan.bsgs_rows(babies, giants, present)
    assert stored == list(range(1, 8)) and all(row == list(range(8)) for row in rows)
    # tools/bsgs_bench.py's shape: the seven kcc = 1 mod-downs and the final one convert into 29 + 1 targets, the
    # merged rescale's into 27 + 2
    logn, L, K, alpha, _, _, level = plan.BSGS_BENCH_SHAPE
    assert (L, K, alpha, level) == (30, 10, 10, 30)
    assert plan.hybrid_mod_down_blocks(level, K) == [[29, 1]]
    assert plan.hybrid_mod_down_blocks(level, K, True) == [[27, 2]]
    # the giants' mod-ups take the 16 + 8 digit chunks of mixed_chunks' second round as the stored babies' do: one
    # launch more per stored baby and per keyed giant with a pair than with the moduli below 2^60
    n, L, K, alpha, mods, levels = _hybrid_mods(port, "mixed_chunks")
    level = levels[0]
    basis = mods[:level] + mods[L:]
    low = [(1 << 50) + 1] * len(basis)
    for rescale in (False, True):
        diff = (plan.bsgs_launches(n, level, K, alpha, basis, _one, *plan.BSGS_SPARSE, rescale)
                - plan.bsgs_launches(n, level, K, alpha, low, _one, *plan.BSGS_SPARSE, rescale))
        assert diff == 4 + 2


def test_bsgs_every_level_sweep_crosses_the_one_component_mod_down_block():
    """(30, 10, 10): the kcc = 1 mod-down of BSGS_SWEEP's keyed giants converts into one block of 29 targets at level 29
    and two at level 30, like the final mod-down"""
    ntt_calls = []

    def ntt(forward, units):
        ntt_calls.append((forward, units))
        return 1

    n = 1 << 8
    for level in (29, 30):
        ntt_calls.clear()
        plan.bsgs_launches(n, level, 10, 10, [(1 << 50) + 1] * (level + 10), ntt, *plan.BSGS_SWEEP)
        assert ntt_calls.count((False, 10)) == 2               # the two keyed giants' kcc = 1 mod-downs
        assert len(plan.hybrid_mod_down_blocks(level, 10)[0]) == level - 28
