"""The scratch rounds of the RNS composites (hexl_b200/csrc/capi_keyswitch.cu, capi_galois.cu, capi_hybrid.cu,
capi_bfv.cu) restated in Python, and the shapes of tests/test_gpu_composite_rounds.py, tests/test_gpu_hybrid_rounds.py,
tests/test_gpu_bsgs_rounds.py and tests/test_gpu_evaluator_rounds.py.

Each composite splits one device call into rounds that fit about 256 MiB of pool scratch:

    rescale_rounds          divide_and_round_on_device, NTT form: polynomials per round
    galois_inplace_rounds   apply_galois_on_device, in place: polynomials copied into scratch per round
    key_switch_rounds       key_switch_on_device, step 2: RNS moduli per round
    ks_mac_launches         the digits of each ks_mac_kernel launch within one round (ks_mac_digits_per_launch)

and the hybrid family (KeySwitchHybrid, the hoisted hybrid rotations, LinearTransformHybrid and
MultiplyRelinearizeHybrid) around one mod-up and one mod-down:

    hybrid_mod_up_rounds    hybrid_mod_up: moduli of the extended basis B per round, and hybrid_round_slots their keys
    base_conv_blocks        base_convert_on_device: targets per launch (base_conv_targets of the source count)
    hybrid_mod_down_blocks  hybrid_mod_down: blocks of 64 data moduli, each in base-conversion launches from K (or
                            K + 1 with the merged rescale) special limbs
    relin_mac_launches, weighted_mac_launches, ks_mac_launches
                            the multiply-accumulate launches of one round of each call
    hybrid_launches         the kernel launches of one ciphertext of each call, from all of the above
    bsgs_launches           the same for LinearTransformHybridBSGS: a baby mod-up, per row the sums, per keyed giant
                            a one-component mod-down and a mod-up, and the final mod-down (bsgs_rows: what it runs)

and the evaluator calls built on them (tests/test_gpu_evaluator_rounds.py):

    base_conv_t_blocks      BGV's t-corrected conversion: base_conv_t_targets of the source count per launch; the tau
                            option of hybrid_mod_down_blocks / _launches and hybrid_launches uses it
    bgv_mod_switch_rounds   BgvModSwitch: polynomials per chunk, in both forms (bgv_mod_switch_launches)
    relin_sum_launches      MultiplyRelinearizeSumHybrid's tensor sums (hybrid_launches "mul_relin_sum")
    bfv_launches            the BEHZ product of BfvMultiply; hybrid_launches "bfv_relin" adds the switch of d2 in
                            coefficient form (the coef option of hybrid_mod_up_launches / hybrid_mod_down_launches)
    inner_sum_exact.inner_sum_launches restates InnerSumHybrid from these primitives; its host lines are pinned here.

Every function returns the list of round (or launch) sizes.  SOURCE holds the source file under hexl_b200/csrc and the
lines of it each formula restates;
tests/test_composite_plan.py asserts they are still there, so a change of the budget or of a formula fails on the CPU
before the GPU test silently runs a single round.
"""
from __future__ import annotations

PARAM_BLOCK = 64          # internal.h: kParamBlock, moduli per kernel parameter block
SCRATCH_BYTES = 256 << 20
RELIN_SUM_PAIRS = 32      # hybrid_rotation.h: kRelinSumPairs, pairs per tensor-sum launch
STAGING_SLOTS = 3         # capi.h: kSlots, the rotating staging slots of a device

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
    # ks_mac_products, which the hybrid switch and the hoisted hybrid rotations run once per mod-up round
    "ks_mac_products": ("capi_keyswitch.cu",
                        ["const uint64_t per_mod = decomp * n, jmax = ks_mac_digits_per_launch(mods, cnt);",
                         "for (uint64_t r = 0; r < elts; ++r)",
                         "for (uint64_t j0 = 0; j0 < decomp; j0 += jmax) {"]),
    "base_conv_targets": ("internal.h",
                          ["constexpr int kBaseConvWords = 480;",
                           "inline u64 base_conv_targets(u64 from) { return (kBaseConvWords - 4 * from) / (5 + from); }"]),
    "base_conv_blocks": ("capi_hybrid.cu",
                         ["const uint64_t F = from_count, block = base_conv_targets(F);",
                          "for (uint64_t e0 = 0; e0 < to_count; e0 += block) {",
                          "const uint64_t cnt = std::min(block, to_count - e0);"]),
    "hybrid_mod_up": ("capi_hybrid.cu",
                      ["const uint64_t D = (level + alpha - 1) / alpha, nb = level + p_size;",
                       "const uint64_t per_mod = D * n;",
                       "uint64_t ichunk = std::max<uint64_t>(1, (256ull << 20) / (per_mod * 8));",
                       "ichunk = std::min<uint64_t>({ichunk, nb, (uint64_t)kParamBlock});",
                       "const uint64_t lo = d * alpha, width = std::min(alpha, level - lo);",
                       "for (uint64_t e = 0; e < cnt; ++e) slots[e] = b0 + e < level ? b0 + e : q_size + (b0 + e - level);"]),
    "hybrid_mod_down": ("capi_hybrid.cu",
                        ["for (uint64_t i0 = 0; i0 < level; i0 += kParamBlock) {",
                         "const uint64_t cnt = std::min<uint64_t>(kParamBlock, level - i0);",
                         "if (rescale) return hybrid_mod_down(dev, result, prod, tmp, n, level - 1, p_size + 1, 2, h, bmods, false, s);"]),
    "relin_mac": ("capi_hybrid.cu",
                  ["tensor.data = b0 < level ? std::min(cnt, level - b0) : 0;",
                   "const uint64_t jc = std::min(ks_mac_digits_per_launch(mods, cnt), D);",
                   "for (uint64_t j0 = 0; j0 < D; j0 += jc) {  // key pointers ride in the kernel parameters"]),
    "weighted_mac": ("capi_hybrid.cu",
                     ["for (uint64_t r0 = 0; r0 < elts; r0 += kParamBlock) {",
                      "const uint64_t per = std::max<uint64_t>(1, kParamBlock / jc);",
                      "for (uint64_t j0 = 0; j0 < D; j0 += jc) {",
                      "for (uint64_t k0 = 0; k0 < keyed.size(); k0 += per) {"]),
    # BGV: the t-corrected conversion's table holds 4 words per source, 6 for tau and 6 + F per target
    "base_conv_t_targets": ("internal.h",
                            ["inline u64 base_conv_t_targets(u64 from) "
                             "{ return (kBaseConvWords - 4 * from - 6) / (6 + from); }"]),
    "base_conv_t_blocks": ("capi_hybrid.cu",
                           ["const uint64_t tau = plain_modulus, tblock = base_conv_t_targets(F);",
                            "for (uint64_t e0 = 0; e0 < to_count; e0 += tblock) {\n"
                            "      const uint64_t cnt = std::min(tblock, to_count - e0);"]),
    "bgv_mod_down": ("capi_hybrid.cu",
                     ["hybrid_mod_down(dev, results[r], prod + r * nb * kcc * n, tmp, n, level, p_size, kcc, h, bmods, "
                      "true, s,\n                            false, plain_modulus))",
                      "if (plain_modulus)  // BGV: the t-corrected mod-down by P, or by q_{level-1} P (the merged "
                      "modulus switch)\n    return hybrid_mod_down(dev, result, prod, tmp, n, level - rescale, "
                      "p_size + rescale, 2, h, bmods, false, s, false,\n                           plain_modulus);"]),
    # BgvModSwitch: one multi-line pin per step, each unique in the file (DivideAndRoundQLast shares single lines)
    "bgv_mod_switch": ("capi_keyswitch.cu",
                       ["const uint64_t L = rns - 1, q_last = moduli[L];\n"
                        "  const uint64_t block = std::min<uint64_t>(L, kParamBlock);\n"
                        "  uint64_t chunk = std::max<uint64_t>(1, (256ull << 20) / ((block + 1) * n * 8));\n"
                        "  chunk = std::min(chunk, count);",
                        "if (ntt_form) {\n"
                        "      CU(cudaMemcpy2DAsync(t_last, n * 8, last, rns * n * 8, n * 8, cnt, cudaMemcpyDeviceToDevice,"
                        " s));\n"
                        "      if (int rc = ntt_multi_on_device(false, dev, h + L, 1, t_last, t_last, 1, cnt, s)) return rc;",
                        "for (uint64_t i0 = 0; i0 < L; i0 += kParamBlock) {\n"
                        "      const uint64_t cm = std::min<uint64_t>(kParamBlock, L - i0);\n"
                        "      if (int rc = base_convert_on_device(tmp, cnt * n, n, last, n, last_poly, n, cnt, &q_last, 1,"
                        " moduli + i0, cm,\n"
                        "                                          false, s, plain_modulus))\n"
                        "        return rc;\n"
                        "      if (ntt_form)\n"
                        "        if (int rc = ntt_multi_on_device(true, dev, h + i0, cm, tmp, tmp, 4, cnt, s)) return rc;",
                        "launch_ks_finish(result + p0 * rns * n, op, tmp, n, cnt, rns, i0, cm, fin, true, false, s);"]),
    "mul_relin_sum": ("capi_hybrid.cu",
                      ["if (pairs == 1)\n    return multiply_relinearize_hybrid_on_device(",
                       "for (uint64_t i0 = 0; i0 < level; i0 += kParamBlock) {\n"
                       "    const uint64_t cnt = std::min<uint64_t>(kParamBlock, level - i0);\n"
                       "    const KsModuli mods = ks_mac_moduli(bmods + i0, nullptr, cnt);\n"
                       "    for (uint64_t r0 = 0; r0 < pairs; r0 += kRelinSumPairs) {\n"
                       "      const uint64_t rcnt = std::min<uint64_t>(kRelinSumPairs, pairs - r0);"]),
    "relin_sum_pairs": ("hybrid_rotation.h", [f"constexpr int kRelinSumPairs = {RELIN_SUM_PAIRS};"]),
    # the host-buffer switches stage one ciphertext per slot, the slots rotating
    "staging_slots": ("capi.h", [f"constexpr int kSlots = {STAGING_SLOTS};",
                                 "for (u64 first = lo; first < hi; first += per_chunk, slot = (slot + 1) % kSlots)"]),
    "host_switch_chunk": ("capi_keyswitch.cu", ["return stage_items(use, batch, 1, [&](int dev, u64, u64, auto&& stage) {"]),
    "bfv": ("capi_bfv.cu",
            ["const uint64_t inputs = square ? 2 : 4;",
             "cudaError_t e = launch_bfv_extend(ext, poly, ct1, comp, n, 2, l, k, ext_tab, s);\n"
             "  if (e == cudaSuccess && !square) e = launch_bfv_extend(",
             "for (uint64_t p = 0; p < inputs; ++p) hs.insert(hs.end(), pl.h.data(), pl.h.data() + M);\n"
             "  if (int rc = ntt_multi_on_device(true, dev, hs.data(), inputs * M, ext, ext, 1, 1, s)) return rc;\n"
             "  for (uint64_t first = 0; first < M; first += kParamBlock) {",
             "for (uint64_t p = 0; p < 3; ++p) hs.insert(hs.end(), pl.h.data(), pl.h.data() + M);\n"
             "  if (int rc = ntt_multi_on_device(false, dev, hs.data(), 3 * M, tensor, tensor, 1, 1, s)) return rc;\n"
             "  e = launch_bfv_scale(out, tensor, poly, n, 3, l, k, scale_tab, s);"]),
    # one launch_ntt_multi per block of 64 handles: the BFV transforms' handles run one polynomial each
    "ntt_multi_blocks": ("capi_ntt.cu",
                         ["for (uint64_t first = 0; first < count; first += kParamBlock) {\n"
                          "    const uint64_t cnt = std::min<uint64_t>(kParamBlock, count - first);\n"
                          "    NttMulti multi{};"]),
    "bfv_relin": ("capi_hybrid.cu",
                  ["if (!coef)\n    if (int rc = ws.get(&t_coef, level * n)) return rc;",
                   "if (!coef)\n    if (int rc = ntt_multi_on_device(false, dev, h.data(), level, t_coef, target, 1, 1, s, "
                   "nullptr, false, mul))",
                   "if (coef) {\n      uint64_t* data = prod + i0 * kcc * n;\n"
                   "      if (int rc = ntt_multi_on_device(false, dev, h.data() + i0, cnt, data, data, 1, kcc, s)) "
                   "return rc;\n"
                   "    } else if (int rc = ntt_multi_on_device(true, dev, h.data() + i0, cnt, tmp, tmp, 4, kcc, s)) {",
                   "if (int rc = bfv_product_on_device(dev, plan, BfvOutputs{{result, result + comp, d2}}, ct1, ct2, s)) "
                   "return rc;\n  if (int rc = hybrid_mod_up(dev, d2, n, level, q_size, p_size, alpha, h, bmods, ws,",
                   "prod + b0 * 2 * n, nb * 2 * n, &keys, nullptr, 1, s);\n"
                   "                             },\n"
                   "                             s, nullptr, true))\n"
                   "    return rc;\n"
                   "  return hybrid_mod_down(dev, result, prod, tmp, n, level, p_size, 2, h, bmods, true, s, true);"]),
    # restated by inner_sum_exact.inner_sum_launches
    "inner_sum": ("capi_hybrid.cu",
                  ["const uint64_t span = (mode & (kSumNextY | kSumRYWrite | kSumCopy1)) ? nb : level;\n"
                   "    for (uint64_t b0 = 0; b0 < span; b0 += kParamBlock) {",
                   "if (d_keyed || s_keyed) {\n      const uint64_t* c1 = xa + comp;\n      if (y_a) {\n"
                   "        if (int rc = hybrid_mod_down(dev, xa_own + comp, y1, tmp, n, level, p_size, 1, h, bmods, "
                   "true, s)) return rc;",
                   "uint64_t* prod = d_keyed ? yn : yr;",
                   "const uint64_t pstride = (uint64_t)(yr - yn);",
                   "prod + b0 * 2 * n, pstride, keys, elts, count, s, true);",
                   "if (rescale) return hybrid_mod_down(dev, result, yr, tmp, n, level - 1, p_size + 1, 2, h, bmods, "
                   "false, s);\n  if (!y_r) return 0;\n"
                   "  return hybrid_mod_down(dev, result, yr, tmp, n, level, p_size, 2, h, bmods, true, s);"]),
    "bsgs": ("capi_hybrid.cu",
             ["if (!baby_keys[i]) continue;",                                         # stored: a keyed baby ...
              "if (diag[j * n1 + i]) {\n        stored[i] = used_keys.size();",       # ... with a diagonal
              "used_elts.data(), used_keys.size(), s);",                             # their products per round
              "if (present.empty()) continue;  // an absent row costs nothing",
              "const uint64_t span = keyed_baby ? nb : level;",
              "for (uint64_t b0 = 0; b0 < span; b0 += kParamBlock) {",
              "for (uint64_t r0 = 0; r0 < present.size(); r0 += kParamBlock) {",
              "if (!keyed_giant) continue;",
              "if (keyed_baby)\n"
              "      if (int rc = hybrid_mod_down(dev, x1, y1, tmp, n, level, p_size, 1, h, bmods, true, s))",
              "stride, &giant_keys[j], &h_elt, 1, s, true);",                         # one set per giant round
              "if (rescale) return hybrid_mod_down(dev, result, y, tmp, n, level - 1, p_size + 1, 2, h, bmods, false, s);",
              "if (!y_used) return 0;"]),
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


# ------------------------------------------------------------------------------ the hybrid family (capi_hybrid.cu)
BASE_CONV_WORDS = 480     # internal.h: kBaseConvWords, the parameter table of one base-conversion launch


def base_conv_targets(from_count):
    """targets one base-conversion launch takes: 4 words per source, 5 + from_count per target"""
    return (BASE_CONV_WORDS - 4 * from_count) // (5 + from_count)


def base_conv_blocks(from_count, to_count):
    """the targets of each launch of base_convert_on_device"""
    return _split(to_count, base_conv_targets(from_count))


def base_conv_t_targets(from_count):
    """targets one t-corrected conversion launch takes (BGV): 4 words per source, 6 for tau, 6 + from_count per
    target"""
    return (BASE_CONV_WORDS - 4 * from_count - 6) // (6 + from_count)


def base_conv_t_blocks(from_count, to_count):
    """the targets of each t-corrected launch of base_convert_on_device"""
    return _split(to_count, base_conv_t_targets(from_count))


def hybrid_digit_widths(level, alpha):
    """the moduli of each digit at `level`: alpha each, the last one partial"""
    return [min(alpha, level - lo) for lo in range(0, level, alpha)]


def hybrid_mod_up_rounds(n, level, K, alpha):
    """hybrid_mod_up: the moduli of B = {q_0..q_{level-1}, p_0..p_{K-1}} per round, every digit (D x n words per
    modulus) under `ichunk` moduli at a time, at most one parameter block"""
    D, nb = -(-level // alpha), level + K
    ichunk = min(max(1, SCRATCH_BYTES // (D * n * 8)), nb, PARAM_BLOCK)
    return _split(nb, ichunk)


def hybrid_round_slots(level, q_size, b0, cnt):
    """the key slot of each modulus of the round starting at b0: data modulus b < level in slot b, special prime j in
    slot q_size + j"""
    return [b if b < level else q_size + (b - level) for b in range(b0, b0 + cnt)]


def hybrid_mod_down_blocks(level, K, rescale=False, tau=False):
    """hybrid_mod_down: per block of 64 data moduli, the targets of each base-conversion launch, from K special limbs,
    or K + 1 with the merged rescale (q_{level-1} joins P and leaves the targets); tau: BGV's t-corrected conversion"""
    targets, sources = level - int(rescale), K + int(rescale)
    blocks = base_conv_t_blocks if tau else base_conv_blocks
    return [blocks(sources, cnt) for cnt in _split(targets, PARAM_BLOCK)]


def relin_tensor_data(level, b0, cnt):
    """the data limbs of a mod-up round that the relinearization's storing launch adds the tensor terms into"""
    return min(cnt, level - b0) if b0 < level else 0


def relin_mac_launches(D, largest_q):
    """MultiplyRelinearizeHybrid: the digits of each ks_relin_mac launch of one round"""
    return _split(D, min(ks_mac_digits_per_launch(largest_q), D))


def weighted_mac_launches(D, keyed, largest_q):
    """LinearTransformHybrid: (digits, elements) of each ks_weighted_mac launch of one round: a digit chunk within the
    128-bit bound, times chunks of 64 // jc keyed elements"""
    jc = min(ks_mac_digits_per_launch(largest_q), D)
    per = max(1, PARAM_BLOCK // jc)
    return [(j, e) for j in _split(D, jc) for e in _split(keyed, per)]


def hybrid_mod_up_launches(n, level, K, alpha, basis, ntt, macs, coef=False):
    """hybrid_mod_up: the target's inverse transform (none with coef: the target is already in coefficient form), then
    per round one base conversion per digit and block of targets, the forward transform of the round's digits and
    macs(D, largest) multiply-accumulate launches, largest the round's largest modulus"""
    D = -(-level // alpha)
    total = 0 if coef else sum(ntt(False, cnt) for cnt in _split(level, PARAM_BLOCK))  # the target to coefficients
    b0 = 0
    for cnt in hybrid_mod_up_rounds(n, level, K, alpha):
        total += sum(len(base_conv_blocks(w, cnt)) for w in hybrid_digit_widths(level, alpha))
        total += ntt(True, cnt * D) + macs(D, max(basis[b0:b0 + cnt]))
        b0 += cnt
    return total


def hybrid_mod_down_launches(level, K, kcc, ntt, rescale=False, tau=False, coef=False):
    """hybrid_mod_down of kcc components: the special limbs' inverse transform, then per block of 64 data moduli the
    rounding (tau: t-corrected) base conversions, a forward transform of the correction (coef: an inverse transform of
    the products' data limbs instead) and the finish; with the merged rescale q_{level-1} joins P"""
    total = ntt(False, (K + int(rescale)) * kcc)
    for cnt, blocks in zip(_split(level - int(rescale), PARAM_BLOCK), hybrid_mod_down_blocks(level, K, rescale, tau)):
        total += len(blocks) + ntt(not coef, cnt * kcc) + 1
    return total


def relin_sum_launches(level, pairs):
    """MultiplyRelinearizeSumHybrid's tensor sums: none for one pair (it is MultiplyRelinearizeHybrid), else one launch
    per block of 64 data limbs and chunk of RELIN_SUM_PAIRS pairs"""
    return 0 if pairs == 1 else -(-level // PARAM_BLOCK) * -(-pairs // RELIN_SUM_PAIRS)


def ntt_handles(ntt, forward, handles):
    """one transform of `handles` polynomials under a handle each (group 1): one multi-modulus launch set per block of
    64 handles, each block its own unit count"""
    return sum(ntt(forward, cnt) for cnt in _split(handles, PARAM_BLOCK))


def bfv_launches(M, square, ntt):
    """bfv_product_on_device of one pair over M = l + k + 1 moduli (Q, B and m_sk): one extension launch per distinct
    input ciphertext, the forward transforms of the lifted polynomials (2M, or 4M, one handle each), one tensor launch
    per block of 64 moduli, the inverse transforms of the tensor's 3M polynomials and one scaling launch"""
    inputs = 2 if square else 4
    return ((1 if square else 2) + ntt_handles(ntt, True, inputs * M) + -(-M // PARAM_BLOCK)
            + ntt_handles(ntt, False, 3 * M) + 1)


def hybrid_launches(call, n, level, K, alpha, basis, ntt, elts=1, keyed=None, rescale=False, kcc=2, tau=False,
                    pairs=1, M=None, square=False):
    """kernel launches of one ciphertext of `call` ("switch", "hoisted", "linear", "mul_relin", "mul_relin_sum",
    "bfv_relin"): basis holds the moduli of B (level data, then K special); ntt(forward, units) is the launch count of
    one multi-modulus transform of `units` polynomials.  "switch" and "hoisted" run `elts` switches over one mod-up;
    "linear" takes `elts` elements, `keyed` of them with keys; "mul_relin_sum" sums `pairs` products; "bfv_relin" is
    the BEHZ product over M moduli (square: ct1 = ct2), then the switch of d2 in coefficient form.  tau: BGV's
    t-corrected mod-downs (rescale is then the merged modulus switch)."""
    total = 0
    if call == "mul_relin_sum":
        total += relin_sum_launches(level, pairs)
        call = "mul_relin"
    if call == "bfv_relin":
        total += bfv_launches(M, square, ntt)
    if call == "hoisted":
        total += elts                                                      # one automorphism launch per element
    if call == "linear":
        total += -(-level // PARAM_BLOCK) * -(-elts // PARAM_BLOCK)        # the permuted sums
        if not keyed:
            return total

    def macs(D, largest):
        if call == "mul_relin":
            return len(relin_mac_launches(D, largest))
        if call == "linear":
            return len(weighted_mac_launches(D, keyed, largest))
        return elts * len(ks_mac_launches(D, largest))

    coef = call == "bfv_relin"
    total += hybrid_mod_up_launches(n, level, K, alpha, basis, ntt, macs, coef)
    downs = 1 if call in ("linear", "mul_relin", "bfv_relin") else elts
    return total + downs * hybrid_mod_down_launches(level, K, kcc if call == "switch" else 2, ntt, rescale, tau, coef)


def bgv_mod_switch_rounds(n, rns, count):
    """BgvModSwitch: polynomials per chunk, in both forms: the gathered last limbs plus one block of deltas of `chunk`
    polynomials fit the budget"""
    block = min(rns - 1, PARAM_BLOCK)
    chunk = min(max(1, SCRATCH_BYTES // ((block + 1) * n * 8)), count)
    return _split(count, chunk)


def bgv_mod_switch_launches(n, rns, count, ntt_form, ntt):
    """BgvModSwitch: per chunk, in NTT form the last limbs' inverse transform (cnt units); per block of 64 moduli the
    t-corrected conversion from the one last limb, in NTT form the forward transform of delta (cm x cnt units), and the
    finish"""
    total = 0
    for cnt in bgv_mod_switch_rounds(n, rns, count):
        total += ntt(False, cnt) if ntt_form else 0
        for cm in _split(rns - 1, PARAM_BLOCK):
            total += len(base_conv_t_blocks(1, cm)) + (ntt(True, cm * cnt) if ntt_form else 0) + 1
    return total


def bsgs_rows(babies, giants, present):
    """the present babies of each giant's row, and the keyed babies with a diagonal (whose products the baby mod-up
    stores), in baby order"""
    rows = [[i for i in range(len(babies)) if present is None or (j, i) in present] for j in range(len(giants))]
    return rows, [i for i, keyed in enumerate(babies) if keyed and any(i in row for row in rows)]


def bsgs_launches(n, level, K, alpha, basis, ntt, babies, giants, present, rescale=False):
    """LinearTransformHybridBSGS: kernel launches of one ciphertext.  babies[i] (giants[j]) is true for a keyed term,
    false for an identity one; present is the set of (giant j, baby i) pairs with a diagonal, or None for all of them.
      - the baby mod-up only when some keyed baby has a pair, storing the products of each such baby per round;
      - per row with a pair, one sum launch per block of 64 moduli of the span (B with a keyed baby in the row, the
        data moduli without) and chunk of 64 present babies;
      - per keyed giant with a pair, the one-component (kcc = 1) mod-down of y_1 when the row has a keyed baby, then a
        mod-up with one multiply-accumulate set per round;
      - the final mod-down: none while Y is empty, or over (level - 1, K + 1) with the merged rescale."""
    rows, stored = bsgs_rows(babies, giants, present)
    stored = len(stored)
    total = 0
    if stored:
        total += hybrid_mod_up_launches(n, level, K, alpha, basis, ntt,
                                        lambda D, q: stored * len(ks_mac_launches(D, q)))
    y_used = False
    for row, keyed_giant in zip(rows, giants):
        if not row:
            continue
        keyed_baby = any(babies[i] for i in row)
        span = level + K if keyed_baby else level
        total += -(-span // PARAM_BLOCK) * -(-len(row) // PARAM_BLOCK)
        y_used = y_used or keyed_baby or bool(keyed_giant)
        if keyed_giant:
            if keyed_baby:
                total += hybrid_mod_down_launches(level, K, 1, ntt)
            total += hybrid_mod_up_launches(n, level, K, alpha, basis, ntt, lambda D, q: len(ks_mac_launches(D, q)))
    if rescale:
        return total + hybrid_mod_down_launches(level, K, 2, ntt, True)
    return total + (hybrid_mod_down_launches(level, K, 2, ntt) if y_used else 0)


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
# name -> (log2 n, L, K, alpha, data prime bits, special prime bits, levels): the hybrid calls of
# tests/test_gpu_hybrid_rounds.py; tests/test_composite_plan.py pins the plan each name stands for
HYBRID_SHAPES = {
    "bench_rescale": (16, 30, 10, 10, 50, 50, (30,)),   # one round; merged rescale's mod-down targets 27 + 2
    "budget_a2": (16, 30, 10, 2, 50, 50, (30, 29)),     # rounds 34 + 6, and 34 + 5 with a one-modulus last digit
    "budget_a3": (17, 30, 3, 3, 50, 50, (30, 28)),      # rounds 25 + 8, and 25 + 6 mixing data and special moduli
    "mixed_chunks": (16, 24, 2, 1, 50, 60, (24,)),      # rounds 21 + 5; multiply-accumulate 1, then 16 + 8 launches
}
# the grids of LinearTransformHybridBSGS in tests/test_gpu_bsgs_rounds.py: (keyed babies, keyed giants, present pairs
# (giant j, baby i), None for all).  BSGS_SPARSE runs at every HYBRID_SHAPES level: the identity baby under the identity
# giant, keyed babies under it, a keyed giant over the identity baby alone (no kcc = 1 mod-down), a keyed giant over
# keyed babies (baby 5 repeats baby 1's element), a keyed baby without a diagonal (stored index != baby index) and an
# absent last row (the rescale folds into row 2, not the last).  BSGS_SWEEP runs at every level of the sweep, its keyed
# giants over keyed babies; BSGS_BENCH is tools/bsgs_bench.py's full 8 x 8 grid, the first baby and giant identities.
BSGS_SPARSE = ((False, True, True, True, True, True), (False, True, True, True),
               {(0, 0), (0, 1), (0, 5), (1, 0), (2, 0), (2, 3), (2, 4), (2, 5)})
BSGS_SWEEP = ((False, True, True), (False, True, True), {(0, 0), (0, 1), (1, 0), (1, 2), (2, 1)})
BSGS_BENCH = ((False,) + (True,) * 7, (False,) + (True,) * 7, None)
BSGS_BENCH_SHAPE = (16, 30, 10, 10, 50, 50, 30)   # (log2 n, L, K, alpha, data bits, special bits, level)
# tests/test_gpu_evaluator_rounds.py: BEHZ with full tiles, (log2 n, l, k): M = l + k + 1 = 129 moduli, tensor blocks
# 64 + 64 + 1; and one host-buffer batch at production size, (HYBRID_SHAPES name, level, batch): one ciphertext per
# staging slot, so the slots wrap (3 + 1)
BEHZ_TILES = (12, 64, 64)
EVALUATOR_HOST_BATCH = ("budget_a2", 30, 4)
