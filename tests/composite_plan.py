"""The scratch rounds of the RNS composites (hexl_b200/csrc/capi_keyswitch.cu, capi_galois.cu) restated in Python, and the shapes of
tests/test_gpu_composite_rounds.py.

Each composite splits one device call into rounds that fit about 256 MiB of pool scratch:

    rescale_rounds          divide_and_round_on_device, NTT form: polynomials per round
    galois_inplace_rounds   apply_galois_on_device, in place: polynomials copied into scratch per round
    key_switch_rounds       key_switch_on_device, step 2: RNS moduli per round
    ks_mac_launches         the digits of each ks_mac_kernel launch within one round (ks_mac_digits_per_launch)

Every function returns the list of round (or launch) sizes.  SOURCE holds the source file under hexl_b200/csrc and the
lines of it each formula restates;
tests/test_composite_plan.py asserts they are still there, so a change of the budget or of a formula fails on the CPU
before the GPU test silently runs a single round.
"""
from __future__ import annotations

PARAM_BLOCK = 64          # internal.h: kParamBlock, moduli per kernel parameter block
SCRATCH_BYTES = 256 << 20

SOURCE = {
    "rescale": ("capi_keyswitch.cu",
                ["const uint64_t block = std::min<uint64_t>(L, kParamBlock);",
                 "uint64_t chunk = std::max<uint64_t>(1, (256ull << 20) / ((block + 1) * n * 8));",
                 "chunk = std::min(chunk, count);"]),
    "galois": ("capi_galois.cu",
               ["const uint64_t chunk = std::min<uint64_t>(count, std::max<uint64_t>(1, (256ull << 20) / (unit * 8)));"]),
    "key_switch": ("capi_keyswitch.cu",
                   ["uint64_t ichunk = std::max<uint64_t>(1, (256ull << 20) / (per_mod * 8));",
                    "ichunk = std::min<uint64_t>({ichunk, rns, (uint64_t)kParamBlock});"]),
    "ks_mac": ("capi_keyswitch.cu",
               ["const unsigned __int128 largest_product = (unsigned __int128)(4 * q - 1) * (q - 1);",
                "return (uint64_t)std::min<unsigned __int128>(kParamBlock, ~(unsigned __int128)0 / largest_product);"]),
}


def _split(total, per):
    return [min(per, total - i) for i in range(0, total, per)]


def rescale_rounds(n, rns, count):
    """NTT form: the gathered last limbs plus one block of rounded limbs of `chunk` polynomials fit the budget"""
    block = min(rns - 1, PARAM_BLOCK)
    chunk = min(max(1, SCRATCH_BYTES // ((block + 1) * n * 8)), count)
    return _split(count, chunk)


def galois_inplace_rounds(n, rns, count):
    """in place: whole polynomials are copied into scratch, as many as fit the budget"""
    return _split(count, min(count, max(1, SCRATCH_BYTES // (rns * n * 8))))


def key_switch_rounds(n, decomp, rns):
    """step 2: every digit under `ichunk` moduli at a time (decomp x n words per modulus), at most one parameter block"""
    ichunk = min(max(1, SCRATCH_BYTES // (decomp * n * 8)), rns, PARAM_BLOCK)
    return _split(rns, ichunk)


def ks_mac_digits_per_launch(largest_q):
    """digits one ks_mac_kernel launch sums unreduced in 128 bits: lazy products (4q - 1)(q - 1) of the round's largest
    modulus, at most one parameter block of key pointers"""
    return min(PARAM_BLOCK, ((1 << 128) - 1) // ((4 * largest_q - 1) * (largest_q - 1)))


def ks_mac_launches(decomp, largest_q):
    """the digits of each multiply-accumulate launch of one step-2 round"""
    return _split(decomp, ks_mac_digits_per_launch(largest_q))


# ------------------------------------------------------------------------------ the GPU test's shapes
# name -> (n, chain, limbs, count): the rescale in NTT and coefficient form
RESCALE_SHAPES = {
    "seal_n16": (1 << 16, "seal", 31, 35),      # rounds 16, 16, 3
    "blocks_n14": (1 << 14, "blocks", 70, 33),  # rounds 31, 2, each with two parameter blocks
}
# ApplyGalois in place
GALOIS_SHAPE = (1 << 16, "seal", 31, 35)        # rounds 16, 16, 3
# name -> (log2 n, digits): KeySwitch / KeySwitchResident / ApplyGaloisKeySwitch, primes just below 2^61
KS_SHAPES = {
    "ckks_n16": (16, 30),   # moduli rounds 17, 14; digits per launch 16, 14
    "ckks_n17": (17, 29),   # moduli rounds 8, 8, 8, 6
}
