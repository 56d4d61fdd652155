"""The hoisted-rotation model (tests/hoist_exact.py) against an independent model and against the rotation, and the
compiler report of the permuted multiply-accumulate kernel.  CPU only.

The GPU applies the automorphism after the digits' transforms, inside the multiply-accumulate; the model does the same.
Here it is shown to equal the key switch of the signed lift sigma_g(a_j) computed on Python integers, for every odd g
at the small degrees and sampled g at 2^10.  At g = 1 it is the rotation [sigma(c0), 0] + KS(sigma(c1)) of
ApplyGaloisKeySwitch bit for bit; at other elements it is not, so the two calls really differ."""
import numpy as np
import pytest

import galois_exact as gx
import hoist_exact as hx
import ks_exact
from test_kernel_resources import kernel_resources

U64 = np.uint64
CASES = ("uniform", "seal_chain", "word_classes")


def _elements(n):
    if n <= 1 << 6:
        return list(range(1, 2 * n, 2))
    return [1, 3, 5, 2 * n - 1, n + 1, 2 * int(hx.uniform_below(n, 1, n)[0]) + 1]


def _rotation(port, case, ct, g):
    """[sigma(c0), 0] + KS(sigma(c1)), the function of ApplyGaloisKeySwitch"""
    comp = case.decomp * case.n
    r = np.concatenate([gx.sigma_ntt(ct[:comp], case.n, g), np.zeros(comp, dtype=U64)])
    return ks_exact.key_switch_exact(port, r, gx.sigma_ntt(ct[comp:], case.n, g), *case.shape, case.keys,
                                     case.modswitch)


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("logn", [1, 2, 3, 6, 10])
def test_permuting_after_the_transforms_is_the_signed_lift(port, name, logn):
    case = ks_exact.make_case(port, name, 1 << logn)
    ct = hx.ciphertexts(case, 1, logn)
    elts = _elements(case.n)
    got = hx.hoisted_exact(port, ct, case.n, case.decomp, case.kms, case.mods, elts, [case.keys] * len(elts),
                           case.modswitch).reshape(len(elts), -1)
    for r, g in enumerate(elts):
        exp = hx.signed_lift_exact(port, ct, case.n, case.decomp, case.kms, case.mods, g, case.keys, case.modswitch)
        assert (got[r] == exp).all(), (name, case.n, g, int((got[r] != exp).sum()))


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("logn", [1, 3, 10])
def test_identity_element_is_the_rotation(port, name, logn):
    case = ks_exact.make_case(port, name, 1 << logn)
    ct = hx.ciphertexts(case, 1, 5)
    got = hx.hoisted_exact(port, ct, case.n, case.decomp, case.kms, case.mods, [1], [case.keys], case.modswitch)
    assert (got == _rotation(port, case, ct, 1)).all()


@pytest.mark.parametrize("name", CASES)
def test_other_elements_differ_from_the_rotation(port, name):
    """sigma_g of the unsigned digit lift is the signed lift plus q_j where sigma_g negates a nonzero coefficient, so
    every extended limb of a random ciphertext's rotation differs somewhere"""
    case = ks_exact.make_case(port, name, 1 << 6)
    ct = hx.ciphertexts(case, 1, 9)
    for g in (3, 2 * case.n - 1):
        got = hx.hoisted_exact(port, ct, case.n, case.decomp, case.kms, case.mods, [g], [case.keys], case.modswitch)
        rot = _rotation(port, case, ct, g)
        differ = (got != rot).reshape(2, case.decomp, case.n).any(axis=2)
        assert differ.all(), (name, g, differ)


def test_permuted_multiply_accumulate_has_no_stack_frame():
    res = kernel_resources("seal.cu")
    macs = {name: r for name, r in res.items() if "13ks_mac_kernel" in name}
    # ks_mac_kernel<false> (the key switch) and ks_mac_kernel<true> (the hoisted rotations)
    assert sorted(("ILb0E" in name, "ILb1E" in name) for name in macs) == [(False, True), (True, False)], list(macs)
    for name, (frame, st, ld) in macs.items():
        assert frame == 0 and st == 0 and ld == 0, f"{name}: {frame} B stack frame, {st} B spill stores, {ld} B loads"
