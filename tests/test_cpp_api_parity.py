"""The intel::hexl drop-in headers against the reference library, through the C++ API a SEAL- or OpenFHE-style caller
compiles.

tests/cpp/api_parity.cpp is written against the public intel::hexl API only.  oracle/Makefile compiles it against the
reference's headers and library (oracle/_ref/api_parity_ref, and api_parity_ref_scalar for the reference's scalar
tier); this test compiles it against include/hexl/** and libhexl_b200.so.  Both programs write every result as a
record of 64-bit words, and the records are compared:

* exact records word for word;
* lazy records (the representative is the implementation's choice): each side below out_mf * q, the sides congruent;
* property records (GeneratePrimitiveRoot, random in the reference): every root is primitive on each side.

The documented deviations (README) are checked against exact arithmetic rather than against the reference:
EltwiseMultMod at 62-bit moduli above about 2^61.7 (ours is canonical), EltwiseReduceMod with input_mod_factor 4 at
q >= 2^63, MSB and Log2 of words just below 2^k for k >= 60 and IsPrime(1) (the reference's are off), and
NTT::CheckArguments on invalid arguments (the reference's release build returns true whatever the arguments; ours
returns the precondition).  The reference's scalar tier leaves the AVX-512 tables empty; there the
tables are checked against their definition below.

The host-only run (inline arithmetic, number theory, NTT tables and constants) needs no GPU; the full run adds every
GPU entry point."""
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

import eltwise_exact as ee

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "api_parity.cpp")
REF_DIR = os.path.join(ROOT, "oracle", "_ref")
REF_AVX = os.path.join(REF_DIR, "api_parity_ref")
REF_SCALAR = os.path.join(REF_DIR, "api_parity_ref_scalar")

# the tables the reference fills only when its CPU has the AVX-512 extension that uses them
AVX_ONLY_TABLES = ("_AVX512Precon32RootOfUnityPowers", "_AVX512Precon52RootOfUnityPowers",
                   "_AVX512Precon64RootOfUnityPowers", "_Precon52InvRootOfUnityPowers")

# every function and constant the drop-in headers declare that the reference also declares, and the pattern of the
# records that exercise it; a run must write at least one record matching each pattern
HOST_NAMES = {
    "MultiplyUInt64Hi<32>": "MultiplyUInt64Hi_32", "MultiplyUInt64Hi<52>": "MultiplyUInt64Hi_52",
    "MultiplyUInt64Hi<64>": "MultiplyUInt64Hi_64", "MultiplyUInt64": "MultiplyUInt64", "AddUInt64": "AddUInt64",
    "MaximumValue": "MaximumValue", "MSB": "MSB_Log2", "Log2": "MSB_Log2", "IsPowerOfTwo": "IsPowerOfTwo_",
    "IsPowerOfFour": "IsPowerOfTwo_IsPowerOfFour", "Not": "CMPINT_Not",
    "DivideUInt128UInt64Lo": "DivideUInt128UInt64Lo", "BarrettReduce128": "DivideUInt128UInt64Lo_BarrettReduce128",
    "MultiplyMod(x, y, y_precon, q)": "MultiplyMod_precon_", "MultiplyModLazy<BitShift>(x, y, factor, q)":
    "MultiplyModLazy_factor_", "MultiplyModLazy<BitShift>(x, y, q)": "MultiplyModLazy_", "BarrettReduce64<1>":
    "BarrettReduce64_1_", "BarrettReduce64<2>": "BarrettReduce64_2_", "ReduceMod<1>": "ReduceMod_1_",
    "ReduceMod<2>": "ReduceMod_2_", "ReduceMod<4>": "ReduceMod_4_", "ReduceMod<8>": "ReduceMod_8_",
    "MultiplyFactor": "MultiplyFactor_", "ReverseBits": "ReverseBits", "InverseMod": "InverseMod_",
    "MultiplyMod": "MultiplyMod_q", "AddUIntMod": "AddUIntMod_", "SubUIntMod": "SubUIntMod_", "PowMod": "PowMod_",
    "HenselLemma2adicRoot": "HenselLemma2adicRoot_", "MontgomeryReduce<64>": "MontgomeryReduce_64_",
    "HashPair": "HashPair", "RWLock": "HashPair", "IsPrime": "IsPrime", "GeneratePrimes": "GeneratePrimes", "MinimalPrimitiveRoot": "MinimalPrimitiveRoot",
    "IsPrimitiveRoot": "IsPrimitiveRoot", "GeneratePrimitiveRoot": "GeneratePrimitiveRoot",
    "NTT(degree, q)": "NTT_n", "NTT(degree, q, root)": "NTT_root3_", "NTT copy/move/assignment": "NTT_copy",
    "NTT::CheckArguments": "NTT_CheckArguments", "NTT constants and caps": "NTT_constants",
    **{f"NTT::Get{t}": rf"NTT_n\d+_q\d+_{t}$" for t in (
        "RootOfUnityPowers", "Precon32RootOfUnityPowers", "Precon64RootOfUnityPowers", "AVX512RootOfUnityPowers",
        "AVX512Precon32RootOfUnityPowers", "AVX512Precon52RootOfUnityPowers", "AVX512Precon64RootOfUnityPowers",
        "InvRootOfUnityPowers", "Precon32InvRootOfUnityPowers", "Precon52InvRootOfUnityPowers",
        "Precon64InvRootOfUnityPowers")},
    "NTT::GetMinimalRootOfUnity/GetDegree/GetModulus/GetRootOfUnityPower/GetInvRootOfUnityPower": r"NTT_n\d+_q\d+_scalars$",
}
GPU_NAMES = {
    "NTT::ComputeForward": "Forward_in", "NTT::ComputeInverse": "Inverse_in", "GetNTT": "Forward_inplace_cached",
    "EltwiseAddMod": "EltwiseAddMod_n", "EltwiseAddMod(scalar)": "EltwiseAddMod_scalar",
    "EltwiseSubMod": "EltwiseSubMod_n", "EltwiseSubMod(scalar)": "EltwiseSubMod_scalar",
    "EltwiseMultMod": "EltwiseMultMod_in", "EltwiseFMAMod": "EltwiseFMAMod_in",
    "EltwiseFMAMod(arg3 = nullptr)": "EltwiseFMAMod_noarg3", "EltwiseReduceMod": "EltwiseReduceMod_in",
    "EltwiseCmpAdd": "EltwiseCmpAdd_cmp", "EltwiseCmpSubMod": "EltwiseCmpSubMod_cmp",
    "EltwiseMontReduceMod": "EltwiseMontReduceMod", "EltwiseMontgomeryFormIn": "EltwiseMontgomeryFormIn",
    "EltwiseMontgomeryFormOut": "EltwiseMontgomeryFormOut", "DyadicMultiply": "DyadicMultiply",
    "KeySwitch": "KeySwitch", "internal::DyadicMultiply": "internal_DyadicMultiply",
    "internal::KeySwitch": "internal_KeySwitch",
}
ALL_CMPINT = [f"_cmp{c}_" for c in range(8)]


# ---------------------------------------------------------------------------------------------------- fixtures
@pytest.fixture(scope="module")
def ours(hb, tmp_path_factory):
    """tests/cpp/api_parity.cpp compiled against include/hexl/** and libhexl_b200.so"""
    if not shutil.which("g++"):
        pytest.skip("g++ not present")
    exe = tmp_path_factory.mktemp("api_parity") / "api_parity"
    libdir = os.path.dirname(hb.LIB_PATH)
    subprocess.run(["g++", "-std=c++17", "-O1", "-I", os.path.join(ROOT, "include"), SRC, "-o", str(exe),
                    "-L", libdir, "-lhexl_b200", f"-Wl,-rpath,{libdir}"], check=True)
    return str(exe)


def _reference_binary(tier):
    """the reference build of the caller: the AVX-512 one where the host has the extensions (as oracle.Ref picks
    its library), or the scalar tier"""
    import oracle
    path = REF_AVX if tier == "dispatch" and oracle._host_has_avx512() else REF_SCALAR
    if not os.path.exists(path):
        pytest.skip(f"{os.path.relpath(path, ROOT)} not built: oracle.build() compiles it where the reference source "
                    "tree is present, and it must be copied with the repository")
    return path, path == REF_SCALAR


def _run(exe, outdir, host_only):
    os.makedirs(outdir)
    args = [exe, str(outdir)] + (["--host-only"] if host_only else [])
    subprocess.run(args, check=True, stdout=subprocess.DEVNULL, timeout=1800)


# ---------------------------------------------------------------------------------------------------- records
def _index(d):
    out = {}
    with open(os.path.join(d, "index.txt")) as f:
        for line in f:
            tag, kind, q, out_mf = line.split()
            out[tag] = (kind, int(q), int(out_mf))
    return out


def _words(d, tag):
    return np.fromfile(os.path.join(d, tag + ".bin"), dtype="<u8")


def _first_difference(a, b):
    if a.size != b.size:
        return f"{a.size} words against {b.size}"
    i = int(np.flatnonzero(a != b)[0])
    return f"first difference at word {i}: {int(a[i])} against {int(b[i])}"


def _barrett_factors(values, shift, q):
    """floor(v * 2^shift / q) for every v (the precomputed factors of the NTT tables)"""
    return ee.words((ee.big(values) << shift) // q)


def _avx512_layout(w):
    """the reference's AVX-512 forward table: the powers w[i] for i in [N/8, N/4) appear four times in a row, those in
    [N/4, N/2) twice, and every other power once"""
    n = w.size
    reps = np.ones(n, dtype=np.int64)
    reps[n // 8:n // 4] = 4
    reps[n // 4:n // 2] = 2
    return np.repeat(w, reps)


def _check_tables(d, prefix, q):
    """the derived tables of one NTT against their definitions from its forward and inverse powers"""
    w, iw = _words(d, prefix + "_RootOfUnityPowers"), _words(d, prefix + "_InvRootOfUnityPowers")
    avx = _avx512_layout(w)
    want = {"_AVX512RootOfUnityPowers": avx, "_AVX512Precon32RootOfUnityPowers": _barrett_factors(avx, 32, q),
            "_AVX512Precon52RootOfUnityPowers": _barrett_factors(avx, 52, q),
            "_AVX512Precon64RootOfUnityPowers": _barrett_factors(avx, 64, q),
            "_Precon52InvRootOfUnityPowers": _barrett_factors(iw, 52, q)}
    bad = []
    for suffix, exp in want.items():
        got = _words(d, prefix + suffix)
        if got.size != exp.size or (got != exp).any():
            bad.append(f"{prefix}{suffix}: {_first_difference(got, exp)} (its definition)")
    return bad


def _is_primitive_root(root, degree, q):
    return degree >= 2 and pow(int(root), int(degree) // 2, int(q)) == int(q) - 1


def _check_arguments_holds(degree, q):
    """NTT's preconditions; ours needs a degree of at least 2"""
    return (degree > 1 and degree & (degree - 1) == 0 and degree <= 1 << 20 and q <= 1 << 62 and
            q % (2 * degree) == 1 and ee.is_prime(q))


def _deviation(tag, q, ours_dir, ref_dir, o, r):
    """None where the tag is compared with the reference; else the list of what is wrong with our side, checked
    against exact arithmetic (the reference side is only required to be congruent where it returns a residue)"""
    if tag == "NTT_CheckArguments":
        rows_o, rows_r = o.reshape(-1, 3), r.reshape(-1, 3)
        bad = []
        for (degree, qq, got), (_, _, ref_got) in zip(rows_o.tolist(), rows_r.tolist()):
            exp = _check_arguments_holds(degree, qq)
            if got != exp or (exp and ref_got != 1):
                bad.append(f"{tag}: CheckArguments({degree}, {qq}) = {got}, reference {ref_got}, expected {int(exp)}")
        return bad
    if tag == "MSB_Log2":
        # the reference rounds log2 in long double, so words just below 2^k for k >= 60 come out as k
        rows_o, rows_r = o.reshape(-1, 3).tolist(), r.reshape(-1, 3).tolist()
        bad = [f"{tag}: MSB/Log2({x}) = {m}, {l}" for x, m, l in rows_o if m != x.bit_length() - 1 or l != m]
        bad += [f"{tag}: reference MSB/Log2({x}) = {m}, {l}" for (x, m, l), (_, mo, _) in zip(rows_r, rows_o)
                if (m, l) != (mo, mo) and not (x >= (1 << 59) and m == l == mo + 1)]
        return bad
    if tag == "IsPrime":
        # the reference calls 1 a prime
        rows_o, rows_r = o.reshape(-1, 2).tolist(), r.reshape(-1, 2).tolist()
        bad = [f"{tag}: IsPrime({n}) = {p}" for n, p in rows_o if p != ee.is_prime(n)]
        bad += [f"{tag}: reference IsPrime({n}) = {p}" for (n, p), (_, po) in zip(rows_r, rows_o) if p != po and n != 1]
        return bad
    if tag.startswith("EltwiseMultMod_in") and q > 2 ** 61.7:
        suffix = tag[len("EltwiseMultMod"):]
        exp = ee.mult_mod(_words(ours_dir, "EltwiseMultMod_a" + suffix), _words(ours_dir, "EltwiseMultMod_b" + suffix),
                          q)
        bad = [f"{tag}: {ee.wrong_words(o, exp)} words differ from a * b mod q"] if ee.wrong_words(o, exp) else []
        if ee.wrong_lazy_words(r, exp, q):
            bad.append(f"{tag}: the reference's words are not congruent below 2q")
        return bad
    if tag.startswith("EltwiseReduceMod_in4_") and q >= 1 << 63:
        suffix = tag[len("EltwiseReduceMod"):]
        exp = ee.reduce_mod(_words(ours_dir, "EltwiseReduceMod_a" + suffix), q)
        wrong = ee.wrong_words(o, exp) if "_out1_" in tag else ee.wrong_lazy_words(o, exp, q)
        return [f"{tag}: {wrong} words differ from x mod q"] if wrong else []
    return None


def compare(ours_dir, ref_dir, ref_is_scalar):
    """every difference between the two runs, as readable lines"""
    io, ir = _index(ours_dir), _index(ref_dir)
    bad = [f"{t}: written only by our side" for t in io if t not in ir]
    bad += [f"{t}: written only by the reference" for t in ir if t not in io]
    for tag, (kind, q, out_mf) in io.items():
        if tag not in ir:
            continue
        if ir[tag] != (kind, q, out_mf):
            bad.append(f"{tag}: index line {ir[tag]} in the reference, {(kind, q, out_mf)} in ours")
            continue
        o, r = _words(ours_dir, tag), _words(ref_dir, tag)
        dev = _deviation(tag, q, ours_dir, ref_dir, o, r)
        if dev is not None:
            bad += dev
        elif kind == "exact":
            if ref_is_scalar and tag.endswith(AVX_ONLY_TABLES) and r.size == 0:
                continue  # checked against the definition below
            if o.size != r.size or (o != r).any():
                bad.append(f"{tag}: {_first_difference(o, r)}")
        elif kind == "lazy":
            top = np.uint64(out_mf * q) if out_mf * q < 1 << 64 else None
            for side, w in (("ours", o), ("reference", r)):
                if top is not None and (w >= top).any():
                    i = int(np.flatnonzero(w >= top)[0])
                    bad.append(f"{tag}: {side} word {i} = {int(w[i])} is not below {out_mf} * q")
            if o.size != r.size or (o % np.uint64(q) != r % np.uint64(q)).any():
                bad.append(f"{tag}: not congruent mod q, {_first_difference(o % np.uint64(q), r % np.uint64(q))}")
        elif kind == "property":
            for side, w in (("ours", o), ("reference", r)):
                for degree, qq, root in w.reshape(-1, 3).tolist():
                    if not _is_primitive_root(root, degree, qq):
                        bad.append(f"{tag}: {side} root {root} is not a primitive {degree}-th root mod {qq}")
        else:
            bad.append(f"{tag}: unknown kind {kind}")
    # the derived NTT tables against their definitions, on our side (and the reference's where it fills them)
    for tag, (kind, q, _) in io.items():
        if tag.startswith("NTT_") and tag.endswith("_RootOfUnityPowers") and "AVX" not in tag and "Precon" not in tag:
            prefix = tag[:-len("_RootOfUnityPowers")]
            bad += _check_tables(ours_dir, prefix, q)
            if not ref_is_scalar and prefix + "_RootOfUnityPowers" in ir:
                bad += [f"reference {b}" for b in _check_tables(ref_dir, prefix, q)]
    return io, bad


def _assert_covers(index, names):
    missing = [name for name, pattern in names.items() if not any(re.match(pattern, t) for t in index)]
    assert not missing, f"no record exercises {missing}"


def _report(bad):
    assert not bad, f"{len(bad)} records differ from the reference:\n" + "\n".join(bad[:40])


# ---------------------------------------------------------------------------------------------------- tests
@pytest.mark.parametrize("tier", ["dispatch", "scalar"])
def test_host_api_matches_reference(ours, tmp_path, tier):
    """inline arithmetic, number theory, NTT tables and constants: no GPU needed"""
    ref_exe, ref_is_scalar = _reference_binary(tier)
    _run(ours, tmp_path / "ours", True)
    _run(ref_exe, tmp_path / "ref", True)
    index, bad = compare(str(tmp_path / "ours"), str(tmp_path / "ref"), ref_is_scalar)
    _assert_covers(index, HOST_NAMES)
    _report(bad)


@pytest.mark.gpu
def test_full_api_matches_reference(ours, tmp_path, hb):
    """everything above plus every GPU entry point, called the way SEAL calls them"""
    if hb.device_count() == 0:
        pytest.fail("gpu-marked test collected on a machine without CUDA")
    ref_exe, ref_is_scalar = _reference_binary("dispatch")
    _run(ours, tmp_path / "ours", False)
    _run(ref_exe, tmp_path / "ref", False)
    index, bad = compare(str(tmp_path / "ours"), str(tmp_path / "ref"), ref_is_scalar)
    _assert_covers(index, {**HOST_NAMES, **GPU_NAMES})
    cmp_tags = [t for t in index if t.startswith("EltwiseCmpSubMod_cmp")]
    assert all(any(c in t for t in cmp_tags) for c in ALL_CMPINT)
    _report(bad)
