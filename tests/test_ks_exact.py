"""The exact KeySwitch model (tests/ks_exact.py) against the checkers, and the shapes where the checkers are wrong.
CPU only.

The GPU key-switch tests compare against the exact model, so the model itself is pinned here: it gives the reference's
known answer, and it equals the C restatement and the compiled reference bit for bit on every shape where their
128-bit accumulator cannot wrap.  On the wrapping shapes the GPU tests use, the C restatement is shown to differ from
it, so a lazy 128-bit checker could not say what the right answer is there."""
import json
import os

import numpy as np
import pytest

import ks_exact

NON_WRAPPING = ("uniform", "seal_chain", "word_classes", "kcc1", "kcc3", "one_digit", "slots", "slots2",
                "small_special")
# the older cases run at two row-kernel degrees; the shape variants also at the tiny-kernel degrees 2, 4 and 8
DEGREES = {name: (1 << 8, 1 << 11) for name in ("uniform", "seal_chain", "word_classes")}
WRAPPING = ("wrap_keys", "wrap_blocks", "kcc3_wrap", "wrap17")


def test_exact_model_gives_the_reference_kat(port):
    """test/experimental/seal/test-key-switch.cpp:16-186"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(root, "tests", "golden", "seal_kats.json")) as f:
        k = json.load(f)["key_switch"]
    got = ks_exact.key_switch_exact(port, np.array(k["input"], dtype=np.uint64), k["t_target_iter_ptr"],
                                    k["coeff_count"], k["decomp_modulus_size"], k["key_modulus_size"],
                                    k["rns_modulus_size"], k["key_component_count"], k["moduli"], k["k_switch_keys"],
                                    k["modswitch_factors"])
    assert (got == np.array(k["expected_output"], dtype=np.uint64)).all()


@pytest.mark.parametrize("name", NON_WRAPPING)
@pytest.mark.parametrize("checker_kind", ["port", "ref"])
def test_exact_model_equals_checkers_where_they_do_not_wrap(request, port, checker_kind, name):
    """uniform moduli; a SEAL-style chain with a digit prime larger than the special prime, digits in [0, 2q) and
    key_modulus_size > rns_modulus_size; moduli of all three word classes in one switch; key_component_count 1 and 3;
    one digit; three unused key slots, with three components and with two; a special prime smaller than every digit"""
    chk = port if checker_kind == "port" else request.getfixturevalue("ref")
    if checker_kind == "ref" and not chk.has_seal:
        pytest.skip("oracle/_ref was built without the experimental/seal sources")
    for n in DEGREES.get(name, (2, 4, 8, 64, 1 << 12)):
        case = ks_exact.make_case(port, name, n)
        assert not case.wraps
        for seed in (1, 2):
            result, t_target = ks_exact.ciphertext(case, seed)
            exp = ks_exact.expected(port, case, result, t_target)
            got = chk.key_switch(result.copy(), t_target, *case.shape, case.keys, case.modswitch)
            assert (got == exp).all(), (name, n, seed, int((got != exp).sum()))
            assert (exp != result).any()   # the switch changed something


@pytest.mark.parametrize("name", NON_WRAPPING + WRAPPING)
def test_cases_have_the_shapes_their_names_say(port, name):
    """wraps is set exactly on the cases whose 128-bit sum can wrap, so the GPU tests compare the checkers with the
    model on every other case; kcc3_wrap and wrap17 need two multiply-accumulate launches of 16 digits and 1 digit"""
    case = ks_exact.make_case(port, name)
    assert case.wraps == (name in WRAPPING)
    shape = {"kcc1": (3, 4, 1), "kcc3": (3, 4, 3), "one_digit": (1, 2, 2), "slots": (3, 7, 3), "slots2": (3, 7, 2),
             "small_special": (3, 4, 2), "kcc3_wrap": (17, 18, 3), "wrap17": (17, 18, 2)}
    if name in shape:
        assert (case.decomp, case.kms, case.kcc) == shape[name]
    if name == "small_special":
        assert case.mods[-1] < 1 << 30 < min(case.mods[:case.decomp])
    if name in ("kcc3_wrap", "wrap17"):
        q = max(case.mods)
        assert (1 << 60) < min(case.mods) and q < (1 << 61)
        per_launch = ((1 << 128) - 1) // ((4 * q - 1) * (q - 1))
        assert per_launch == 16 and -(-case.decomp // per_launch) == 2


@pytest.mark.parametrize("name", ["wrap_keys", "wrap_blocks"])
def test_lazy_128_bit_checker_is_wrong_at_the_wrapping_shapes(port, name):
    """At the degrees the GPU tests run, moduli just below 2^61 with 29 digits and keys at q - 1, or with 70 digits
    and random keys, make the C restatement's unreduced sum of digit x key products wrap 2^128."""
    case = ks_exact.make_case(port, name)
    assert case.wraps and all((1 << 60) < q < (1 << 61) for q in case.mods)
    result, t_target = ks_exact.ciphertext(case, 1)
    exp = ks_exact.expected(port, case, result, t_target)
    lazy = port.key_switch(result.copy(), t_target, *case.shape, case.keys, case.modswitch)
    wrong = int((lazy != exp).sum())
    # one wrapped sum under the special prime spreads over every coefficient of every modulus
    assert wrong > exp.size // 2, (name, wrong, exp.size)
    for i, q in enumerate(case.mods[:case.decomp]):
        part = exp.reshape(case.kcc, case.decomp, case.n)[:, i]
        assert (part < np.uint64(q)).all()
