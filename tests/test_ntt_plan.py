"""Every kernel of ntt.cu is launched by tests/test_gpu_ntt_degrees.py (CPU only: the plan restated in tests/ntt_plan.py
against the ptxas report hexl_b200/build.py writes).

The GPU test checks each call's launch count against ntt_plan.kernels; here the union of the plan over that test's
parameter set must be exactly the set of kernels the compiler reports for ntt.cu.  A kernel added without a case that
launches it, or a plan that names a kernel which does not exist, fails."""
import ntt_exact as nx
import ntt_plan as plan
from test_kernel_resources import kernel_resources


def test_plan_restates_the_launch_table():
    """spot checks of ntt.cu's table: the split above 2^17, the deep threshold, SMALL's distributed shared memory"""
    fast, small = 1 << 55, (1 << 29) + 1
    assert plan.col_passes(8) == [4, 4] and plan.col_passes(7) == [4, 3] and plan.col_passes(5) == [5]
    assert plan.kernels(fast, 17, 63, True) == ["7ntt_colILi1ELi5ELb1EE", "11ntt_row_fwdILi1ELi12EE"]
    assert plan.kernels(fast, 17, 64, True) == ["12ntt_pipe_fwdILi1ELi5EE"]
    assert plan.kernels(fast, 18, 64, False) == ["11ntt_row_invILi1ELi12EE", "7ntt_colILi1ELi3ELb0EE",
                                                 "7ntt_colILi1ELi3ELb0EE"]
    assert plan.kernels(small, 17, 64, True) == ["13ntt_dsmem_fwdILi2ELi5EE"]
    assert plan.kernels(fast, 3, 5, False) == ["16ntt_stage_simpleILb0EE"] * 3
    assert plan.host_chunks(15, plan.host_batch(15, "fast_50bit")) == [128, 63]
    assert plan.host_chunks(16, plan.host_batch(16, "fast_50bit")) == [64, 63]


def test_every_kernel_of_ntt_cu_is_launched(hb):
    launched = {k for case in plan.cases(hb.GeneratePrimes) for k in plan.kernels(*case)}
    compiled = list(kernel_resources("ntt.cu"))
    matches = {frag: [name for name in compiled if frag in name] for frag in launched}
    missing = sorted(frag for frag, names in matches.items() if len(names) != 1)
    assert not missing, f"the plan names kernels ntt.cu does not compile exactly once: {missing}"
    untested = sorted(name for name in compiled if not any(frag in name for frag in launched))
    assert not untested, f"{len(untested)} kernels of ntt.cu are launched by no case of the GPU test: {untested}"
    assert len(launched) == len(compiled)


def test_every_mode_and_prime_side(hb):
    """each boundary prime sits on the side of pick_mode's boundary its name says"""
    primes = dict(nx.single_primes(hb.GeneratePrimes, nx.MAX_LOGN))
    want = {"below_2^30": plan.SMALL, "above_2^30": plan.GENERIC, "below_2^32": plan.GENERIC,
            "above_2^32": plan.FAST, "below_2^56": plan.FAST, "above_2^56": plan.WIDE, "below_2^61": plan.WIDE,
            "above_2^61": plan.GENERIC, "below_2^62": plan.GENERIC, "small_25bit": plan.SMALL,
            "fast_50bit": plan.FAST, "wide_60bit": plan.WIDE, "smallest": plan.SMALL}
    assert {name: plan.mode(q) for name, q in primes.items()} == want
    for name, q in primes.items():
        if name.startswith(("below_", "above_")):
            edge = 1 << int(name.split("^")[1])
            assert q < edge if name.startswith("below_") else q > edge, (name, q)
