"""The rescale model (tests/rescale_exact.py) against the integer definition, and the CPU-side checks of
hexl_b200_divide_and_round_q_last: argument validation, no device, and the compiler's resource report of its kernels.
CPU only.

The GPU tests compare DivideAndRoundQLast with rescale_exact() bit for bit, so the model is pinned here: in
coefficient form it equals floor((X + h) / q_L) mod q_i computed with Python integers, its NTT form is the coefficient
form conjugated by the transforms, and it gives the same words built on the C restatement and on the compiled
reference."""
import os
import re

import numpy as np
import pytest

import rescale_exact as rx

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CHAINS = ("seal", "classes", "wide", "small")
U64 = np.uint64


def _mods(port, name, n):
    return rx.chain(port.generate_primes, n, name)


@pytest.mark.parametrize("name", CHAINS)
@pytest.mark.parametrize("n", [8, 64])
def test_coefficient_form_equals_integer_definition(port, name, n):
    mods = _mods(port, name, n)
    count = 3
    x = rx.random_operand(n + 17, n, mods, count)
    exp = rx.rescale_integer(x, n, mods, count)
    got = rx.rescale_exact(port, x, n, mods, count, ntt_form=False)
    assert (got == exp).all(), (name, n, int((got != exp).sum()))
    L = len(mods) - 1
    lim = got.reshape(count, L + 1, n)
    assert all((lim[:, i] < U64(q)).all() for i, q in enumerate(mods[:L]))
    assert (lim[:, L] == x.reshape(count, L + 1, n)[:, L]).all()   # limb L carried through untouched


@pytest.mark.parametrize("name", CHAINS)
def test_edge_inputs_equal_integer_definition(port, name):
    n = 16
    mods = _mods(port, name, n)
    rows = rx.edge_values(mods, n, 5)
    x = rx.limbs_of(rows, mods)
    exp = rx.rescale_integer(x, n, mods, len(rows))
    assert (rx.rescale_exact(port, x, n, mods, len(rows), ntt_form=False) == exp).all()
    assert (rx.rescale_per_limb(x, n, mods, len(rows)) == exp).all()
    # the edges themselves: X = 0 -> 0; X = Q - 1 -> floor((Q - 1 + h) / q_L) = Q / q_L, which is 0 mod every q_i
    e = exp.reshape(len(rows), len(mods), n)
    assert (e[0, :-1] == 0).all() and (e[1, :-1] == 0).all()
    # q_L is odd: X mod q_L = h - 1 and h round down, h + 1 up; adding ceil(q_L / 2) instead of h would round h up
    assert mods[-1] % 2 == 1
    for row, up in zip(rows[2:], (0, 0, 1)):
        assert all((v + (mods[-1] >> 1)) // mods[-1] == v // mods[-1] + up for v in row)


PER_LIMB_LISTS = {
    "tiny q_i": [2, 3, (1 << 61) - 1],
    "tiny q_L": [(1 << 61) - 1, 2, 3],
    "even q_L": [(1 << 61) - 1, 1000003, 1 << 40],
    "composite": [3 * 5 * 7 * 11 * 13 * 17 * 19 * 23, 29 * 31 * 37 * 41 * 43 * 47, 53 * 59 * 61 * 67 * 71],
}


@pytest.mark.parametrize("name", sorted(PER_LIMB_LISTS))
def test_per_limb_formula_equals_integer_definition(name):
    """the GPU domain test's reference where the moduli share factors; here on pairwise coprime moduli"""
    mods, n = PER_LIMB_LISTS[name], 16
    x = np.concatenate([rx.limbs_of(rx.edge_values(mods, n, 3), mods), rx.random_operand(4, n, mods, 2)])
    count = x.size // (len(mods) * n)
    assert (rx.rescale_per_limb(x, n, mods, count) == rx.rescale_integer(x, n, mods, count)).all()


def test_q_last_between_the_other_moduli(port):
    mods = _mods(port, "classes", 32)
    assert min(mods[:-1]) < mods[-1] < max(mods[:-1])


@pytest.mark.parametrize("name", CHAINS)
@pytest.mark.parametrize("n", [8, 64])
def test_ntt_form_is_the_coefficient_form_between_transforms(port, name, n):
    mods = _mods(port, name, n)
    count = 2
    rns = len(mods)
    x = rx.random_operand(3 * n + 1, n, mods, count).reshape(count, rns, n)
    got = rx.rescale_exact(port, x.reshape(-1), n, mods, count, ntt_form=True).reshape(count, rns, n)
    coef = np.stack([np.stack([port.ntt_inverse(x[p, i], n, q) for i, q in enumerate(mods)]) for p in range(count)])
    exp_coef = rx.rescale_integer(coef.reshape(-1), n, mods, count).reshape(count, rns, n)
    for i, q in enumerate(mods[:-1]):
        exp = port.ntt_forward(np.ascontiguousarray(exp_coef[:, i]).reshape(-1), n, q).reshape(count, n)
        assert (got[:, i] == exp).all(), (name, n, i)
    assert (got[:, -1] == x[:, -1]).all()


@pytest.mark.parametrize("ntt_form", [False, True])
@pytest.mark.parametrize("name", CHAINS)
def test_model_on_port_equals_model_on_reference(port, ref, name, ntt_form):
    n = 64
    mods = _mods(port, name, n)
    x = rx.random_operand(99, n, mods, 2)
    a = rx.rescale_exact(port, x, n, mods, 2, ntt_form)
    b = rx.rescale_exact(ref, x, n, mods, 2, ntt_form)
    assert (a == b).all()


# ---------------------------------------------------------------- the C entry point without a GPU
def _call(hb, n, mods, count=1, ntt_form=True, result=None, operand=None):
    size = count * len(mods) * n
    op = np.zeros(size, dtype=U64) if operand is None else operand
    res = op if result is None else result
    return hb.DivideAndRoundQLast(res, op, n, mods, len(mods), count, ntt_form)


def test_bad_arguments_raise_invalid_arg(hb, port):
    n = 64
    good = _mods(port, "seal", n)
    bad = {
        "one limb": (n, good[:1], True),
        "modulus 1": (n, [1] + good[1:], False),
        "modulus 2^61": (n, [(1 << 61) + 1] + good[1:], False),
        "not coprime to q_L": (n, [6, 9, 15], False),
        "q_i == q_L": (n, [good[-1]] + good[1:], True),
        "n not a power of two": (48, good, True),
        "n above 2^20": (1 << 21, [97, 193], True),
        "n = 1 in NTT form": (1, [97, 193], True),
        "not NTT-friendly": (n, good[:-1] + [good[-1] + 2 * n + 2], True),
        "n = 0 in coefficient form": (0, good, False),
    }
    for what, (nn, mods, ntt) in bad.items():
        with pytest.raises(hb.HexlB200Error) as e:
            _call(hb, nn, mods, 1, ntt, operand=np.zeros(max(nn, 1) * len(mods), dtype=U64))
        assert e.value.code == -1, (what, str(e.value))
    # overlapping buffers that are not the same buffer
    buf = np.zeros(3 * len(good) * n, dtype=U64)
    with pytest.raises(hb.HexlB200Error) as e:
        hb.DivideAndRoundQLast(buf[n:], buf[:2 * len(good) * n], n, good, len(good), 2, True)
    assert e.value.code == -1
    # nothing to do
    _call(hb, n, good, count=0)


def test_without_a_gpu_the_call_fails_and_launches_nothing(hb, port):
    if hb.device_count() > 0:
        pytest.skip("a CUDA device is present")
    n = 64
    for ntt_form in (False, True):
        mods = _mods(port, "classes", n)
        before = hb.launch_count()
        with pytest.raises(hb.HexlB200Error) as e:
            _call(hb, n, mods, 2, ntt_form)
        assert e.value.code == -2
        assert hb.launch_count() == before


# ---------------------------------------------------------------- compiler resources
_PROPS = re.compile(r"Function properties for (\S+)\n\s+(\d+) bytes stack frame, (\d+) bytes spill stores, "
                    r"(\d+) bytes spill loads")
RESCALE_KERNELS = ("ks_round_kernel", "ks_finish_kernel", "rescale_coef_kernel")


def test_rescale_kernels_hold_no_stack_frame_beyond_spills(hb):
    """seal.o.log is the `ptxas -v` report the library build writes for seal.cu"""
    log = os.path.join(ROOT, "hexl_b200", "_obj", "seal.o.log")
    if not os.path.exists(log):
        pytest.fail(f"{log} is missing: build the library first (python -m hexl_b200.build)")
    with open(log) as f:
        props = {name: tuple(int(v) for v in rest) for name, *rest in _PROPS.findall(f.read())}
    for kernel in RESCALE_KERNELS:
        hits = [(name, r) for name, r in props.items() if kernel in name]
        assert len(hits) == 1, f"{kernel}: {len(hits)} entries in the ptxas report"
        name, (frame, st, ld) = hits[0]
        assert frame <= max(st, ld), f"{name}: {frame} B stack frame, {st} B spill stores, {ld} B spill loads"
