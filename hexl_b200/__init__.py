"""hexl_b200 -- Python (ctypes) view of libhexl_b200.so.

The product is the C-ABI shared library (include/hexl_b200.h) and the C++
drop-in headers (include/hexl/).  This module only binds that ABI for the test
suite and bench.py, keeping the reference's names and argument order
(``NTT.ComputeForward``, ``EltwiseMultMod`` ...; hexl/include/hexl/ntt/ntt.hpp,
hexl/include/hexl/eltwise/*.hpp).  Buffers may be

* torch CUDA tensors (int64 or uint64 storage) -> device-pointer path, enqueued
  on the current torch stream, no synchronisation;
* numpy uint64 arrays / torch CPU tensors      -> host-pointer path, staged
  through the GPU by the library, synchronous.

There is no CPU compute path: if the library is missing this import fails, and
if there is no CUDA device every compute call raises ``HexlB200Error``.
"""
from __future__ import annotations

import ctypes as C
import os
from enum import IntEnum

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("HEXL_B200_LIB") or os.path.join(_HERE, "lib", "libhexl_b200.so")

if not os.path.exists(LIB_PATH):
    raise ImportError(
        f"{LIB_PATH} is missing: build it with `python -m hexl_b200.build` "
        "(hexl_b200 has no fallback implementation)")

_lib = C.CDLL(LIB_PATH)
_u64, _vp, _int = C.c_uint64, C.c_void_p, C.c_int


class HexlB200Error(RuntimeError):
    """A call into libhexl_b200 failed (the C++ shim throws std::runtime_error
    in the same situations, mirroring HEXL_CHECK in debug builds)."""

    def __init__(self, code: int, msg: str):
        super().__init__(f"[{code}] {msg}")
        self.code = code


class CMPINT(IntEnum):
    """hexl/include/hexl/util/util.hpp:16-25"""
    EQ = 0
    LT = 1
    LE = 2
    FALSE = 3
    NE = 4
    NLT = 5
    NLE = 6
    TRUE = 7


def _sig(name, restype, argtypes):
    f = getattr(_lib, name)
    f.restype, f.argtypes = restype, argtypes
    return f


_sig("hexl_b200_version", C.c_char_p, [])
_sig("hexl_b200_last_error", C.c_char_p, [])
_sig("hexl_b200_device_count", _int, [])
_sig("hexl_b200_set_host_devices", _int, [C.POINTER(_int), _int])
_sig("hexl_b200_set_debug", None, [_int])
_sig("hexl_b200_sync", _int, [_vp])
_sig("hexl_b200_host_alloc", _vp, [C.c_size_t])
_sig("hexl_b200_host_free", None, [_vp])
_sig("hexl_b200_managed_alloc", _vp, [C.c_size_t])
_sig("hexl_b200_managed_free", None, [_vp])
_sig("hexl_b200_launch_count", _u64, [])
for _n in ("multiply_mod", "add_uint_mod", "sub_uint_mod", "pow_mod", "multiply_factor"):
    _sig("hexl_b200_" + _n, _u64, [_u64, _u64, _u64])
_sig("hexl_b200_inverse_mod", _u64, [_u64, _u64])
_sig("hexl_b200_reverse_bits", _u64, [_u64, _u64])
_sig("hexl_b200_is_prime", _int, [_u64])
_sig("hexl_b200_is_primitive_root", _int, [_u64, _u64, _u64])
_sig("hexl_b200_generate_primitive_root", _u64, [_u64, _u64])
_sig("hexl_b200_minimal_primitive_root", _u64, [_u64, _u64])
_sig("hexl_b200_generate_primes", _int, [_vp, C.c_size_t, C.c_size_t, _int, C.c_size_t])
_sig("hexl_b200_ntt_create", _int, [C.POINTER(_vp), _u64, _u64])
_sig("hexl_b200_ntt_create_with_root", _int, [C.POINTER(_vp), _u64, _u64, _u64])
_sig("hexl_b200_ntt_retain", None, [_vp])
_sig("hexl_b200_ntt_release", None, [_vp])
_sig("hexl_b200_ntt_check_arguments", _int, [_u64, _u64])
_sig("hexl_b200_ntt_degree", _u64, [_vp])
_sig("hexl_b200_ntt_modulus", _u64, [_vp])
_sig("hexl_b200_ntt_minimal_root", _u64, [_vp])
_sig("hexl_b200_ntt_table", C.POINTER(_u64), [_vp, _int])
_sig("hexl_b200_ntt_prepare", _int, [_vp, _int])
_sig("hexl_b200_ntt_forward", _int, [_vp, _vp, _vp, _u64, _u64, _u64, _vp])
_sig("hexl_b200_ntt_inverse", _int, [_vp, _vp, _vp, _u64, _u64, _u64, _vp])
_sig("hexl_b200_ntt_forward_multi", _int, [C.POINTER(_vp), _u64, _vp, _vp, _u64, _u64, _u64, _vp])
_sig("hexl_b200_ntt_inverse_multi", _int, [C.POINTER(_vp), _u64, _vp, _vp, _u64, _u64, _u64, _vp])
_sig("hexl_b200_eltwise_mult_mod_multi", _int, [_vp, _vp, _vp, _u64, _vp, _u64, _u64, _vp])
_sig("hexl_b200_eltwise_add_mod_multi", _int, [_vp, _vp, _vp, _u64, _vp, _u64, _vp])
_sig("hexl_b200_eltwise_sub_mod_multi", _int, [_vp, _vp, _vp, _u64, _vp, _u64, _vp])
_sig("hexl_b200_poly_multiply_multi", _int, [C.POINTER(_vp), _u64, _vp, _vp, _vp, _u64, _vp])
_sig("hexl_b200_eltwise_add_mod", _int, [_vp, _vp, _vp, _u64, _u64, _vp])
_sig("hexl_b200_eltwise_add_mod_scalar", _int, [_vp, _vp, _u64, _u64, _u64, _vp])
_sig("hexl_b200_eltwise_sub_mod", _int, [_vp, _vp, _vp, _u64, _u64, _vp])
_sig("hexl_b200_eltwise_sub_mod_scalar", _int, [_vp, _vp, _u64, _u64, _u64, _vp])
_sig("hexl_b200_eltwise_mult_mod", _int, [_vp, _vp, _vp, _u64, _u64, _u64, _vp])
_sig("hexl_b200_eltwise_fma_mod", _int, [_vp, _vp, _u64, _vp, _u64, _u64, _u64, _vp])
_sig("hexl_b200_eltwise_reduce_mod", _int, [_vp, _vp, _u64, _u64, _u64, _u64, _vp])
_sig("hexl_b200_eltwise_cmp_add", _int, [_vp, _vp, _u64, _int, _u64, _u64, _vp])
_sig("hexl_b200_eltwise_cmp_sub_mod", _int, [_vp, _vp, _u64, _u64, _int, _u64, _u64, _vp])

_sig("hexl_b200_ntt_get_cached", _int, [C.POINTER(_vp), _u64, _u64])
_sig("hexl_b200_dyadic_multiply", _int, [_vp, _vp, _vp, _u64, _vp, _u64, _vp])
_sig("hexl_b200_key_switch", _int, [_vp, _vp, _u64, _u64, _u64, _u64, _u64, _vp, _vp, _vp, _vp])
_sig("hexl_b200_divide_and_round_q_last", _int, [_vp, _vp, _u64, _vp, _u64, _u64, _int, _vp])
_sig("hexl_b200_apply_galois", _int, [_vp, _vp, _u64, _vp, _u64, _u64, _u64, _int, _vp])

_sig("hexl_b200_hensel_lemma_2adic_root", _u64, [C.c_uint32, _u64])
_sig("hexl_b200_montgomery_reduce", _u64, [_u64, _u64, _u64, _int, _u64])
_sig("hexl_b200_eltwise_mont_reduce_mod", _int, [_vp, _vp, _vp, _u64, _u64, _int, _u64, _vp])
_sig("hexl_b200_eltwise_montgomery_form_in", _int, [_vp, _vp, _u64, _u64, _u64, _int, _u64, _vp])
_sig("hexl_b200_eltwise_montgomery_form_out", _int, [_vp, _vp, _u64, _u64, _int, _u64, _vp])
_sig("hexl_b200_keys_upload", _int, [C.POINTER(_vp), _vp, _u64, _u64, _u64, _u64])
_sig("hexl_b200_keys_upload_sharded", _int, [C.POINTER(_vp), _vp, _u64, _u64, _u64, _u64])
_sig("hexl_b200_keys_release", None, [_vp])
_sig("hexl_b200_key_switch_resident", _int, [_vp, _vp, _u64, _u64, _u64, _u64, _u64, _vp, _vp, _vp, _u64, _vp])
_sig("hexl_b200_apply_galois_key_switch", _int, [_vp, _u64, _u64, _u64, _u64, _u64, _vp, _vp, _vp, _u64, _u64, _vp])
_sig("hexl_b200_apply_galois_key_switch_hoisted", _int,
     [_vp, _vp, _u64, _u64, _u64, _u64, _u64, _vp, _vp, _vp, _u64, _vp, _u64, _vp])
_sig("hexl_b200_fast_base_convert", _int, [_vp, _vp, _u64, _vp, _u64, _vp, _u64, _u64, _vp])
_sig("hexl_b200_key_switch_hybrid", _int, [_vp, _vp, _u64, _u64, _u64, _u64, _u64, _u64, _vp, _vp, _u64, _vp])
_sig("hexl_b200_apply_galois_key_switch_hybrid_hoisted", _int,
     [_vp, _vp, _u64, _u64, _u64, _u64, _u64, _vp, _vp, _vp, _u64, _u64, _vp])
_sig("hexl_b200_linear_transform_hybrid", _int,
     [_vp, _vp, _u64, _u64, _u64, _u64, _u64, _vp, _vp, _vp, _u64, _vp, _u64, _vp])
_sig("hexl_b200_linear_transform_hybrid_bsgs", _int,
     [_vp, _vp, _u64, _u64, _u64, _u64, _u64, _vp, _vp, _vp, _u64, _vp, _vp, _u64, _vp, _int, _u64, _vp])
_sig("hexl_b200_multiply_relinearize_hybrid", _int,
     [_vp, _vp, _vp, _u64, _u64, _u64, _u64, _u64, _vp, _vp, _int, _u64, _vp])
_sig("hexl_b200_multiply_relinearize_sum_hybrid", _int,
     [_vp, _vp, _vp, _u64, _u64, _u64, _u64, _u64, _u64, _vp, _vp, _int, _u64, _vp])
_sig("hexl_b200_inner_sum_hybrid", _int,
     [_vp, _vp, _u64, _u64, _u64, _u64, _u64, _vp, _u64, _u64, _vp, _vp, _u64, _int, _u64, _vp])
_sig("hexl_b200_bfv_multiply", _int, [_vp, _vp, _vp, _u64, _vp, _u64, _vp, _u64, _u64, _u64, _u64, _vp])
_sig("hexl_b200_bfv_multiply_relinearize_hybrid", _int,
     [_vp, _vp, _vp, _u64, _u64, _u64, _u64, _u64, _vp, _vp, _u64, _u64, _u64, _vp, _u64, _vp])
_sig("hexl_b200_bgv_mod_switch", _int, [_vp, _vp, _u64, _vp, _u64, _u64, _u64, _int, _vp])
_sig("hexl_b200_bgv_key_switch_hybrid", _int,
     [_vp, _vp, _u64, _u64, _u64, _u64, _u64, _u64, _vp, _u64, _vp, _u64, _vp])
_sig("hexl_b200_bgv_apply_galois_key_switch_hybrid_hoisted", _int,
     [_vp, _vp, _u64, _u64, _u64, _u64, _u64, _vp, _u64, _vp, _vp, _u64, _u64, _vp])
_sig("hexl_b200_bgv_multiply_relinearize_hybrid", _int,
     [_vp, _vp, _vp, _u64, _u64, _u64, _u64, _u64, _vp, _u64, _vp, _int, _u64, _vp])
_sig("hexl_b200_plain_lift", _int, [_vp, _vp, _u64, _u64, _vp, _u64, _u64, _u64, _int, _u64, _vp])
_sig("hexl_b200_bfv_add_plain", _int, [_vp, _vp, _vp, _u64, _u64, _u64, _vp, _u64, _u64, _int, _u64, _vp])
_sig("hexl_b200_bfv_multiply_plain", _int, [_vp, _vp, _vp, _u64, _u64, _int, _u64, _vp, _u64, _u64, _u64, _vp])

#: every symbol include/hexl_b200.h declares (checked against the header by the tests)
EXPORTED = sorted(n for n in dir(_lib) if n.startswith("hexl_b200_"))


def _check(rc: int) -> None:
    if rc != 0:
        raise HexlB200Error(rc, _lib.hexl_b200_last_error().decode())


# ------------------------------------------------------------------ buffers
def _is_torch(x) -> bool:
    return type(x).__module__.startswith("torch")


def _buf(x):
    """-> (address, number of 64-bit elements, is_cuda).  None -> (None, 0, None)."""
    if x is None:
        return None, 0, None
    if _is_torch(x):
        assert x.is_contiguous(), "tensor must be contiguous"
        assert x.element_size() == 8, "tensor must hold 64-bit integers"
        return x.data_ptr(), x.numel(), x.is_cuda
    assert isinstance(x, np.ndarray) and x.dtype == np.uint64 and x.flags["C_CONTIGUOUS"], \
        "host buffers must be C-contiguous numpy uint64 arrays"
    return x.ctypes.data, x.size, False


def _need(what: str, have: int, want: int) -> None:
    if have < want:
        raise HexlB200Error(-1, f"{what}: buffer holds {have} elements, the call needs {want}")


def _stream(stream, any_cuda: bool):
    if stream is not None:
        return int(getattr(stream, "cuda_stream", stream))
    if any_cuda:
        import torch
        return int(torch.cuda.current_stream().cuda_stream)
    return None


# ---------------------------------------------------------------- library info
def version() -> str:
    return _lib.hexl_b200_version().decode()


def device_count() -> int:
    return _lib.hexl_b200_device_count()


def set_host_devices(devices) -> None:
    arr = (_int * len(devices))(*devices)
    _check(_lib.hexl_b200_set_host_devices(arr, len(devices)))


def set_debug(on: bool) -> None:
    _lib.hexl_b200_set_debug(int(on))


def launch_count() -> int:
    return int(_lib.hexl_b200_launch_count())


def pinned_empty(n: int) -> np.ndarray:
    """uint64 numpy array of n elements in page-locked host memory."""
    ptr = _lib.hexl_b200_host_alloc(n * 8)
    if not ptr:
        raise HexlB200Error(-4, "hexl_b200_host_alloc failed")
    arr = np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint64)), shape=(n,))
    return arr  # freed at process exit; call pinned_free(arr) to release earlier


def pinned_free(arr: np.ndarray) -> None:
    _lib.hexl_b200_host_free(arr.ctypes.data)


def managed_empty(n: int) -> np.ndarray:
    """uint64 numpy array of n elements in unified memory: host code reads and writes it
    like any array, the kernels work on it in place (no staging copy)."""
    ptr = _lib.hexl_b200_managed_alloc(n * 8)
    if not ptr:
        raise HexlB200Error(-4, "hexl_b200_managed_alloc failed")
    return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_uint64)), shape=(n,))


def managed_free(arr: np.ndarray) -> None:
    _lib.hexl_b200_managed_free(arr.ctypes.data)


# --------------------------------------------------------------- number theory
def MultiplyMod(x, y, q): return int(_lib.hexl_b200_multiply_mod(x, y, q))
def AddUIntMod(x, y, q): return int(_lib.hexl_b200_add_uint_mod(x, y, q))
def SubUIntMod(x, y, q): return int(_lib.hexl_b200_sub_uint_mod(x, y, q))
def PowMod(b, e, q): return int(_lib.hexl_b200_pow_mod(b, e, q))
def InverseMod(x, q): return int(_lib.hexl_b200_inverse_mod(x, q))
def ReverseBits(x, w): return int(_lib.hexl_b200_reverse_bits(x, w))
def IsPrime(n): return bool(_lib.hexl_b200_is_prime(n))
def IsPrimitiveRoot(r, d, q): return bool(_lib.hexl_b200_is_primitive_root(r, d, q))
def GeneratePrimitiveRoot(d, q): return int(_lib.hexl_b200_generate_primitive_root(d, q))
def MinimalPrimitiveRoot(d, q): return int(_lib.hexl_b200_minimal_primitive_root(d, q))
def MultiplyFactor(operand, bit_shift, q): return int(_lib.hexl_b200_multiply_factor(operand, bit_shift, q))


def GeneratePrimes(num_primes, bit_size, prefer_small_primes, ntt_size=1):
    out = np.zeros(num_primes, dtype=np.uint64)
    got = _lib.hexl_b200_generate_primes(out.ctypes.data, num_primes, bit_size,
                                         int(bool(prefer_small_primes)), ntt_size)
    if got != num_primes:
        raise HexlB200Error(-1, "Failed to find enough primes")
    return [int(v) for v in out]


# -------------------------------------------------------------------- NTT
class NTT:
    """intel::hexl::NTT (hexl/include/hexl/ntt/ntt.hpp:22-293)."""

    def __init__(self, degree: int, q: int, root_of_unity: int | None = None):
        h = _vp()
        if root_of_unity is None:
            _check(_lib.hexl_b200_ntt_create(C.byref(h), degree, q))
        else:
            _check(_lib.hexl_b200_ntt_create_with_root(C.byref(h), degree, q, root_of_unity))
        self._h = h

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h and _lib is not None:  # module globals are already gone at interpreter shutdown
            _lib.hexl_b200_ntt_release(h)

    @staticmethod
    def CheckArguments(degree, modulus) -> bool:
        return bool(_lib.hexl_b200_ntt_check_arguments(degree, modulus))

    def Prepare(self, device: int = -1):
        """upload the tables to `device` now (needed before capturing a cold handle into a CUDA graph)"""
        _check(_lib.hexl_b200_ntt_prepare(self._h, device))
        return self

    def GetDegree(self): return int(_lib.hexl_b200_ntt_degree(self._h))
    def GetModulus(self): return int(_lib.hexl_b200_ntt_modulus(self._h))
    def GetMinimalRootOfUnity(self): return int(_lib.hexl_b200_ntt_minimal_root(self._h))

    def _table(self, which):
        p = _lib.hexl_b200_ntt_table(self._h, which)
        return np.ctypeslib.as_array(p, shape=(self.GetDegree(),)).copy()

    def GetRootOfUnityPowers(self): return self._table(0)
    def GetPrecon64RootOfUnityPowers(self): return self._table(1)
    def GetInvRootOfUnityPowers(self): return self._table(2)
    def GetPrecon64InvRootOfUnityPowers(self): return self._table(3)

    def _compute(self, fn, result, operand, in_mf, out_mf, stream):
        rp, rn, rc = _buf(result)
        op, on, oc = _buf(operand)
        n = self.GetDegree()
        assert rn == on and on % n == 0, "buffers must hold a whole number of polynomials"
        _check(fn(self._h, rp, op, in_mf, out_mf, on // n, _stream(stream, bool(rc or oc))))
        return result

    def ComputeForward(self, result, operand, input_mod_factor=1, output_mod_factor=1, stream=None):
        return self._compute(_lib.hexl_b200_ntt_forward, result, operand, input_mod_factor,
                             output_mod_factor, stream)

    def ComputeInverse(self, result, operand, input_mod_factor=1, output_mod_factor=1, stream=None):
        return self._compute(_lib.hexl_b200_ntt_inverse, result, operand, input_mod_factor,
                             output_mod_factor, stream)


def _multi(fn, ntts, result, operand, in_mf, out_mf, batch_per_modulus, stream):
    rp, rn, rc = _buf(result)
    op, on, oc = _buf(operand)
    n = ntts[0].GetDegree()
    if batch_per_modulus is None:
        assert on % (n * len(ntts)) == 0, "operand length must be a multiple of len(ntts) * degree"
        batch_per_modulus = on // (n * len(ntts))
    assert rn >= batch_per_modulus * n * len(ntts) and on >= batch_per_modulus * n * len(ntts)
    hs = (_vp * len(ntts))(*[t._h for t in ntts])
    _check(fn(hs, len(ntts), rp, op, in_mf, out_mf, batch_per_modulus, _stream(stream, rc or oc)))
    return result


def ComputeForwardMulti(ntts, result, operand, input_mod_factor=1, output_mod_factor=1, batch_per_modulus=None,
                        stream=None):
    """One launch for an RNS batch: polynomial u is transformed under ntts[u // batch_per_modulus]
    (hexl_b200_ntt_forward_multi; the reference needs one NTT::ComputeForward call per unit)."""
    return _multi(_lib.hexl_b200_ntt_forward_multi, ntts, result, operand, input_mod_factor, output_mod_factor,
                  batch_per_modulus, stream)


def ComputeInverseMulti(ntts, result, operand, input_mod_factor=1, output_mod_factor=1, batch_per_modulus=None,
                        stream=None):
    return _multi(_lib.hexl_b200_ntt_inverse_multi, ntts, result, operand, input_mod_factor, output_mod_factor,
                  batch_per_modulus, stream)


def EltwiseMultModMulti(result, operand1, operand2, n_per_modulus, moduli, input_mod_factor=1, stream=None):
    """EltwiseMultMod over an RNS batch in one launch: block e (n_per_modulus elements) under moduli[e]"""
    mods = np.ascontiguousarray(moduli, dtype=np.uint64)
    rp, rn, rc = _buf(result); ap, an, ac = _buf(operand1); bp, bn, _ = _buf(operand2)
    for what, have in (("result", rn), ("operand1", an), ("operand2", bn)):
        _need(what, have, n_per_modulus * mods.size)
    _check(_lib.hexl_b200_eltwise_mult_mod_multi(rp, ap, bp, n_per_modulus, mods.ctypes.data, mods.size,
                                                 input_mod_factor, _stream(stream, rc or ac)))
    return result


def _addsub_multi(fn, result, operand1, operand2, n_per_modulus, moduli, stream):
    mods = np.ascontiguousarray(moduli, dtype=np.uint64)
    rp, rn, rc = _buf(result); ap, an, ac = _buf(operand1); bp, bn, _ = _buf(operand2)
    for what, have in (("result", rn), ("operand1", an), ("operand2", bn)):
        _need(what, have, n_per_modulus * mods.size)
    _check(fn(rp, ap, bp, n_per_modulus, mods.ctypes.data, mods.size, _stream(stream, rc or ac)))
    return result


def EltwiseAddModMulti(result, operand1, operand2, n_per_modulus, moduli, stream=None):
    return _addsub_multi(_lib.hexl_b200_eltwise_add_mod_multi, result, operand1, operand2, n_per_modulus, moduli, stream)


def EltwiseSubModMulti(result, operand1, operand2, n_per_modulus, moduli, stream=None):
    return _addsub_multi(_lib.hexl_b200_eltwise_sub_mod_multi, result, operand1, operand2, n_per_modulus, moduli, stream)


def PolyMultiplyMulti(ntts, result, a, b, batch_per_modulus=None, stream=None):
    """Negacyclic products InvNTT(FwdNTT(a) .* FwdNTT(b)), polynomial u under ntts[u // batch_per_modulus]; result
    may be a, b or a separate buffer, and a may be b (a square), with or without result."""
    rp, rn, rc = _buf(result); ap, an, ac = _buf(a); bp, bn, _ = _buf(b)
    n = ntts[0].GetDegree()
    if batch_per_modulus is None:
        batch_per_modulus = an // (n * len(ntts))
    for what, have in (("result", rn), ("a", an), ("b", bn)):
        _need(what, have, batch_per_modulus * n * len(ntts))
    hs = (_vp * len(ntts))(*[t._h for t in ntts])
    _check(_lib.hexl_b200_poly_multiply_multi(hs, len(ntts), rp, ap, bp, batch_per_modulus, _stream(stream, rc or ac)))
    return result


# ---------------------------------------------------------------- element-wise
def _scalar(x) -> bool:
    return isinstance(x, (int, np.integer))


def EltwiseAddMod(result, operand1, operand2, n, modulus, stream=None):
    rp, rn, rc = _buf(result); ap, an, ac = _buf(operand1)
    _need("result", rn, n); _need("operand1", an, n)
    if not _scalar(operand2):
        _need("operand2", _buf(operand2)[1], n)
    if _scalar(operand2):
        _check(_lib.hexl_b200_eltwise_add_mod_scalar(rp, ap, int(operand2), n, modulus, _stream(stream, rc or ac)))
    else:
        bp, _, _ = _buf(operand2)
        _check(_lib.hexl_b200_eltwise_add_mod(rp, ap, bp, n, modulus, _stream(stream, rc or ac)))
    return result


def EltwiseSubMod(result, operand1, operand2, n, modulus, stream=None):
    rp, rn, rc = _buf(result); ap, an, ac = _buf(operand1)
    _need("result", rn, n); _need("operand1", an, n)
    if not _scalar(operand2):
        _need("operand2", _buf(operand2)[1], n)
    if _scalar(operand2):
        _check(_lib.hexl_b200_eltwise_sub_mod_scalar(rp, ap, int(operand2), n, modulus, _stream(stream, rc or ac)))
    else:
        bp, _, _ = _buf(operand2)
        _check(_lib.hexl_b200_eltwise_sub_mod(rp, ap, bp, n, modulus, _stream(stream, rc or ac)))
    return result


def EltwiseMultMod(result, operand1, operand2, n, modulus, input_mod_factor=1, stream=None):
    rp, rn, rc = _buf(result); ap, an, ac = _buf(operand1); bp, bn, _ = _buf(operand2)
    _need("result", rn, n); _need("operand1", an, n); _need("operand2", bn, n)
    _check(_lib.hexl_b200_eltwise_mult_mod(rp, ap, bp, n, modulus, input_mod_factor, _stream(stream, rc or ac)))
    return result


def EltwiseFMAMod(result, arg1, arg2, arg3, n, modulus, input_mod_factor=1, stream=None):
    rp, rn, rc = _buf(result); ap, an, ac = _buf(arg1); cp, cn, _ = _buf(arg3)
    _need("result", rn, n); _need("arg1", an, n)
    if arg3 is not None:
        _need("arg3", cn, n)
    _check(_lib.hexl_b200_eltwise_fma_mod(rp, ap, int(arg2), cp, n, modulus, input_mod_factor,
                                          _stream(stream, rc or ac)))
    return result


def EltwiseReduceMod(result, operand, n, modulus, input_mod_factor, output_mod_factor, stream=None):
    rp, rn, rc = _buf(result); ap, an, ac = _buf(operand)
    _need("result", rn, n); _need("operand", an, n)
    _check(_lib.hexl_b200_eltwise_reduce_mod(rp, ap, n, modulus, input_mod_factor, output_mod_factor,
                                             _stream(stream, rc or ac)))
    return result


def EltwiseCmpAdd(result, operand1, n, cmp, bound, diff, stream=None):
    rp, rn, rc = _buf(result); ap, an, ac = _buf(operand1)
    _need("result", rn, n); _need("operand1", an, n)
    _check(_lib.hexl_b200_eltwise_cmp_add(rp, ap, n, int(cmp), bound, diff, _stream(stream, rc or ac)))
    return result


def EltwiseCmpSubMod(result, operand1, n, modulus, cmp, bound, diff, stream=None):
    rp, rn, rc = _buf(result); ap, an, ac = _buf(operand1)
    _need("result", rn, n); _need("operand1", an, n)
    _check(_lib.hexl_b200_eltwise_cmp_sub_mod(rp, ap, n, modulus, int(cmp), bound, diff,
                                              _stream(stream, rc or ac)))
    return result


# ------------------------------------------------------- Montgomery-form helpers
def HenselLemma2adicRoot(r, q): return int(_lib.hexl_b200_hensel_lemma_2adic_root(r, q))
def MontgomeryReduce(T_hi, T_lo, q, r, inv_mod): return int(_lib.hexl_b200_montgomery_reduce(T_hi, T_lo, q, r, inv_mod))


def EltwiseMontReduceMod(result, a, b, n, modulus, r, neg_inv_mod, stream=None):
    """a*b*R^-1 mod q, R = 2^r (EltwiseMontReduceModAVX512<64, r>, eltwise-reduce-mod-avx512.hpp:156)"""
    rp, rn, rc = _buf(result); ap, an, ac = _buf(a); bp, bn, _ = _buf(b)
    _need("result", rn, n); _need("a", an, n); _need("b", bn, n)
    _check(_lib.hexl_b200_eltwise_mont_reduce_mod(rp, ap, bp, n, modulus, r, neg_inv_mod, _stream(stream, rc or ac)))
    return result


def EltwiseMontgomeryFormIn(result, a, R2_mod_q, n, modulus, r, neg_inv_mod, stream=None):
    rp, rn, rc = _buf(result); ap, an, ac = _buf(a)
    _need("result", rn, n); _need("a", an, n)
    _check(_lib.hexl_b200_eltwise_montgomery_form_in(rp, ap, R2_mod_q, n, modulus, r, neg_inv_mod, _stream(stream, rc or ac)))
    return result


def EltwiseMontgomeryFormOut(result, a, n, modulus, r, neg_inv_mod, stream=None):
    rp, rn, rc = _buf(result); ap, an, ac = _buf(a)
    _need("result", rn, n); _need("a", an, n)
    _check(_lib.hexl_b200_eltwise_montgomery_form_out(rp, ap, n, modulus, r, neg_inv_mod, _stream(stream, rc or ac)))
    return result


# ------------------------------------------------------- SEAL-shaped composites
def GetNTT(N: int, modulus: int) -> NTT:
    """hexl/include/hexl/experimental/seal/ntt-cache.hpp:27-53: process-wide cache"""
    h = _vp()
    _check(_lib.hexl_b200_ntt_get_cached(C.byref(h), N, modulus))
    obj = NTT.__new__(NTT)
    obj._h = h
    return obj


def DyadicMultiply(result, operand1, operand2, n, moduli, num_moduli=None, stream=None):
    """hexl/include/hexl/experimental/seal/dyadic-multiply.hpp:26"""
    mods = np.ascontiguousarray(moduli, dtype=np.uint64)
    rp, rn, rc = _buf(result); ap, an, ac = _buf(operand1); bp, bn, _ = _buf(operand2)
    nm = num_moduli or mods.size
    _need("moduli", mods.size, nm); _need("result", rn, 3 * n * nm)
    _need("operand1", an, 2 * n * nm); _need("operand2", bn, 2 * n * nm)
    _check(_lib.hexl_b200_dyadic_multiply(rp, ap, bp, n, mods.ctypes.data, nm,
                                          _stream(stream, rc or ac)))
    return result


def KeySwitch(result, t_target_iter_ptr, n, decomp_modulus_size, key_modulus_size, rns_modulus_size,
              key_component_count, moduli, k_switch_keys, modswitch_factors, stream=None):
    """hexl/include/hexl/experimental/seal/key-switch.hpp:34; k_switch_keys is a list of buffers"""
    mods = np.ascontiguousarray(moduli, dtype=np.uint64)
    ms = np.ascontiguousarray(modswitch_factors, dtype=np.uint64)
    rp, rn, rc = _buf(result); tp, tn, tc = _buf(t_target_iter_ptr)
    _need("moduli", mods.size, key_modulus_size); _need("modswitch_factors", ms.size, decomp_modulus_size)
    _need("k_switch_keys", len(k_switch_keys), decomp_modulus_size)
    _need("result", rn, key_component_count * decomp_modulus_size * n)
    _need("t_target_iter_ptr", tn, decomp_modulus_size * n)
    for k in k_switch_keys[:decomp_modulus_size]:
        _need("k_switch_keys[j]", _buf(k)[1], key_component_count * key_modulus_size * n)
    key_ptrs = (_vp * len(k_switch_keys))(*[_buf(k)[0] for k in k_switch_keys])
    _check(_lib.hexl_b200_key_switch(rp, tp, n, decomp_modulus_size, key_modulus_size, rns_modulus_size,
                                     key_component_count, mods.ctypes.data, key_ptrs, ms.ctypes.data,
                                     _stream(stream, rc or tc)))
    return result


def DivideAndRoundQLast(result, operand, n, moduli, rns_modulus_size, count=1, ntt_form=True, stream=None):
    """Rescale `count` polynomials of rns_modulus_size limbs (n words each) by their last modulus
    (hexl_b200_divide_and_round_q_last; SEAL's divide_and_round_q_last(_ntt)_inplace).  Limbs 0..L-1 of every
    polynomial of result are written, limb L is not; result may be operand."""
    mods = np.ascontiguousarray(moduli, dtype=np.uint64)
    rp, rn, rc = _buf(result); op, on, oc = _buf(operand)
    _need("moduli", mods.size, rns_modulus_size)
    _need("result", rn, count * rns_modulus_size * n); _need("operand", on, count * rns_modulus_size * n)
    _check(_lib.hexl_b200_divide_and_round_q_last(rp, op, n, mods.ctypes.data, rns_modulus_size, count,
                                                  int(bool(ntt_form)), _stream(stream, rc or oc)))
    return result


class KeySwitchKeys:
    """Key-switch keys uploaded once (hexl_b200_keys_upload): to the current device, or to every device
    named with set_host_devices.  k_switch_keys: list of host or device buffers, each
    key_component_count x key_modulus_size x n words."""

    def __init__(self, k_switch_keys, n, decomp_modulus_size, key_modulus_size, key_component_count,
                 sharded_by_modulus=False):
        """sharded_by_modulus: split the RNS moduli of ONE key switch over the devices of set_host_devices
        (hexl_b200_keys_upload_sharded); such a handle serves host buffers only."""
        for k in k_switch_keys[:decomp_modulus_size]:
            _need("k_switch_keys[j]", _buf(k)[1], key_component_count * key_modulus_size * n)
        _need("k_switch_keys", len(k_switch_keys), decomp_modulus_size)
        ptrs = (_vp * len(k_switch_keys))(*[_buf(k)[0] for k in k_switch_keys])
        h = _vp()
        fn = _lib.hexl_b200_keys_upload_sharded if sharded_by_modulus else _lib.hexl_b200_keys_upload
        _check(fn(C.byref(h), ptrs, n, decomp_modulus_size, key_modulus_size, key_component_count))
        self._h = h
        self.shape = (n, decomp_modulus_size, key_modulus_size, key_component_count)

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h and _lib is not None:
            _lib.hexl_b200_keys_release(h)


def KeySwitchResident(result, t_target_iter_ptr, n, decomp_modulus_size, key_modulus_size, rns_modulus_size,
                      key_component_count, moduli, keys: KeySwitchKeys, modswitch_factors, batch=1, stream=None):
    """`batch` key switches against resident keys (hexl_b200_key_switch_resident): ciphertext c uses
    result[c * kcc*decomp*n:] and t_target[c * decomp*n:]; host buffers are pipelined and split over the devices."""
    mods = np.ascontiguousarray(moduli, dtype=np.uint64)
    ms = np.ascontiguousarray(modswitch_factors, dtype=np.uint64)
    rp, rn, rc = _buf(result); tp, tn, tc = _buf(t_target_iter_ptr)
    _need("moduli", mods.size, key_modulus_size); _need("modswitch_factors", ms.size, decomp_modulus_size)
    _need("result", rn, batch * key_component_count * decomp_modulus_size * n)
    _need("t_target_iter_ptr", tn, batch * decomp_modulus_size * n)
    _check(_lib.hexl_b200_key_switch_resident(rp, tp, n, decomp_modulus_size, key_modulus_size, rns_modulus_size,
                                              key_component_count, mods.ctypes.data, keys._h, ms.ctypes.data, batch,
                                              _stream(stream, rc or tc)))
    return result


def ApplyGalois(result, operand, n, moduli, rns_modulus_size, count, galois_elt, ntt_form=True, stream=None):
    """The Galois automorphism a(X) -> a(X^galois_elt) of `count` polynomials of rns_modulus_size limbs (n words each),
    in NTT or coefficient form (hexl_b200_apply_galois); result may be operand."""
    mods = np.ascontiguousarray(moduli, dtype=np.uint64)
    rp, rn, rc = _buf(result); op, on, oc = _buf(operand)
    _need("moduli", mods.size, rns_modulus_size)
    _need("result", rn, count * rns_modulus_size * n); _need("operand", on, count * rns_modulus_size * n)
    _check(_lib.hexl_b200_apply_galois(rp, op, n, mods.ctypes.data, rns_modulus_size, count, galois_elt,
                                       int(bool(ntt_form)), _stream(stream, rc or oc)))
    return result


def ApplyGaloisKeySwitch(ciphertexts, n, decomp_modulus_size, key_modulus_size, rns_modulus_size, key_component_count,
                         moduli, galois_keys: KeySwitchKeys, modswitch_factors, galois_elt, batch=1, stream=None):
    """Rotation or conjugation of `batch` ciphertexts in place (hexl_b200_apply_galois_key_switch): ciphertext c is
    ciphertexts[c * 2*decomp*n:], c0 <- sigma(c0) + KS_0(sigma(c1)), c1 <- KS_1(sigma(c1))."""
    mods = np.ascontiguousarray(moduli, dtype=np.uint64)
    ms = np.ascontiguousarray(modswitch_factors, dtype=np.uint64)
    cp, cn, cc = _buf(ciphertexts)
    _need("moduli", mods.size, key_modulus_size); _need("modswitch_factors", ms.size, decomp_modulus_size)
    _need("ciphertexts", cn, batch * key_component_count * decomp_modulus_size * n)
    _check(_lib.hexl_b200_apply_galois_key_switch(cp, n, decomp_modulus_size, key_modulus_size, rns_modulus_size,
                                                  key_component_count, mods.ctypes.data,
                                                  galois_keys._h if galois_keys is not None else None, ms.ctypes.data,
                                                  galois_elt, batch, _stream(stream, cc)))
    return ciphertexts


def ApplyGaloisKeySwitchHoisted(results, ciphertexts, n, decomp_modulus_size, key_modulus_size, rns_modulus_size,
                                key_component_count, moduli, galois_keys, modswitch_factors, galois_elts, batch=1,
                                stream=None):
    """Hoisted rotations (hexl_b200_apply_galois_key_switch_hoisted): ciphertext c of `ciphertexts` (2*decomp*n words
    each) rotated by every galois_elts[r] with galois_keys[r] (a list of KeySwitchKeys), into
    results[(c * len(galois_elts) + r) * 2*decomp*n:], its digits decomposed once for all elements.  Not bit-identical
    to ApplyGaloisKeySwitch: digits are lifted to signed integers under sigma_g (equal for g = 1)."""
    mods = np.ascontiguousarray(moduli, dtype=np.uint64)
    ms = np.ascontiguousarray(modswitch_factors, dtype=np.uint64)
    elts = np.ascontiguousarray(galois_elts, dtype=np.uint64)
    rp, rn, rc = _buf(results); cp, cn, cc = _buf(ciphertexts)
    per = key_component_count * decomp_modulus_size * n
    _need("moduli", mods.size, key_modulus_size); _need("modswitch_factors", ms.size, decomp_modulus_size)
    _need("galois_keys", len(galois_keys), elts.size)
    _need("results", rn, batch * elts.size * per); _need("ciphertexts", cn, batch * per)
    keys = (_vp * max(1, len(galois_keys)))(*[k._h if k is not None else None for k in galois_keys])
    _check(_lib.hexl_b200_apply_galois_key_switch_hoisted(rp, cp, n, decomp_modulus_size, key_modulus_size,
                                                          rns_modulus_size, key_component_count, mods.ctypes.data,
                                                          keys, elts.ctypes.data, elts.size, ms.ctypes.data, batch,
                                                          _stream(stream, rc or cc)))
    return results


def FastBaseConvert(result, operand, n, from_moduli, to_moduli, count=1, stream=None):
    """Fast base conversion (hexl_b200_fast_base_convert) of `count` polynomials, coefficient form: polynomial p of
    operand holds len(from_moduli) limbs of n words, its result len(to_moduli) limbs,
    result_e = [sum_i [x_i (Q/q_i)^-1]_{q_i} [Q/q_i]_{t_e}]_{t_e}."""
    src = np.ascontiguousarray(from_moduli, dtype=np.uint64)
    dst = np.ascontiguousarray(to_moduli, dtype=np.uint64)
    rp, rn, rc = _buf(result); op, on, oc = _buf(operand)
    _need("result", rn, count * dst.size * n); _need("operand", on, count * src.size * n)
    _check(_lib.hexl_b200_fast_base_convert(rp, op, n, src.ctypes.data, src.size, dst.ctypes.data, dst.size, count,
                                            _stream(stream, rc or oc)))
    return result


def KeySwitchHybrid(result, target, n, level_size, q_size, p_size, digit_size, key_component_count, moduli,
                    keys: KeySwitchKeys, batch=1, stream=None):
    """Hybrid key switch (hexl_b200_key_switch_hybrid) of `batch` ciphertexts at level level_size: moduli holds the
    q_size data moduli, then the p_size special primes; keys were uploaded with decomp = ceil(q_size / digit_size) and
    key_modulus_size = q_size + p_size.  Ciphertext c reads target[c * level_size*n:] and accumulates into
    result[c * key_component_count*level_size*n:]."""
    mods = np.ascontiguousarray(moduli, dtype=np.uint64)
    rp, rn, rc = _buf(result); tp, tn, tc = _buf(target)
    _need("moduli", mods.size, q_size + p_size)
    _need("result", rn, batch * key_component_count * level_size * n); _need("target", tn, batch * level_size * n)
    _check(_lib.hexl_b200_key_switch_hybrid(rp, tp, n, level_size, q_size, p_size, digit_size, key_component_count,
                                            mods.ctypes.data, keys._h if keys is not None else None, batch,
                                            _stream(stream, rc or tc)))
    return result


def ApplyGaloisKeySwitchHybridHoisted(results, ciphertexts, n, level_size, q_size, p_size, digit_size, moduli,
                                      galois_keys, galois_elts, batch=1, stream=None):
    """Hoisted rotations with hybrid keys (hexl_b200_apply_galois_key_switch_hybrid_hoisted): ciphertext c of
    `ciphertexts` (2*level_size*n words each) rotated by every galois_elts[r] with galois_keys[r] (a list of hybrid
    KeySwitchKeys, key_component_count 2), into results[(c * len(galois_elts) + r) * 2*level_size*n:], its mod-up done
    once for all elements.  Not bit-identical to ApplyGalois + KeySwitchHybrid for g != 1 (signed digit lift)."""
    mods = np.ascontiguousarray(moduli, dtype=np.uint64)
    elts = np.ascontiguousarray(galois_elts, dtype=np.uint64)
    rp, rn, rc = _buf(results); cp, cn, cc = _buf(ciphertexts)
    per = 2 * level_size * n
    _need("moduli", mods.size, q_size + p_size); _need("galois_keys", len(galois_keys), elts.size)
    _need("results", rn, batch * elts.size * per); _need("ciphertexts", cn, batch * per)
    keys = (_vp * max(1, len(galois_keys)))(*[k._h if k is not None else None for k in galois_keys])
    _check(_lib.hexl_b200_apply_galois_key_switch_hybrid_hoisted(rp, cp, n, level_size, q_size, p_size, digit_size,
                                                                 mods.ctypes.data, keys, elts.ctypes.data, elts.size,
                                                                 batch, _stream(stream, rc or cc)))
    return results


def LinearTransformHybrid(result, ciphertexts, n, level_size, q_size, p_size, digit_size, moduli, galois_keys,
                          galois_elts, diagonals, batch=1, stream=None):
    """sum_r w_r (.) Rot_{g_r}(ct) with hybrid keys and one mod-down (hexl_b200_linear_transform_hybrid): ciphertext c
    of `ciphertexts` (2*level_size*n words each) goes to result[c * 2*level_size*n:].  diagonals holds
    len(galois_elts) x (level_size + p_size) x n words in NTT form (limb i < level_size under q_i, then the special
    primes).  galois_keys[r] is None for an identity term (galois_elts[r] = 1, adds w_r (.) ct without a key switch)."""
    mods = np.ascontiguousarray(moduli, dtype=np.uint64)
    elts = np.ascontiguousarray(galois_elts, dtype=np.uint64)
    rp, rn, rc = _buf(result); cp, cn, cc = _buf(ciphertexts); dp, dn, dc = _buf(diagonals)
    per = 2 * level_size * n
    _need("moduli", mods.size, q_size + p_size); _need("galois_keys", len(galois_keys), elts.size)
    _need("result", rn, batch * per); _need("ciphertexts", cn, batch * per)
    _need("diagonals", dn, elts.size * (level_size + p_size) * n)
    keys = (_vp * max(1, len(galois_keys)))(*[k._h if k is not None else None for k in galois_keys])
    _check(_lib.hexl_b200_linear_transform_hybrid(rp, cp, n, level_size, q_size, p_size, digit_size, mods.ctypes.data,
                                                  keys, elts.ctypes.data, elts.size, dp, batch,
                                                  _stream(stream, rc or cc or dc)))
    return result


def LinearTransformHybridBSGS(result, ciphertexts, n, level_size, q_size, p_size, digit_size, moduli, baby_keys,
                              baby_elts, giant_keys, giant_elts, diagonals, rescale=False, batch=1, stream=None):
    """sum_j sigma_{h_j}(sum_i w_{j,i} (.) sigma_{b_i}(ct)) with hybrid keys, baby-step giant-step and double-hoisted
    (hexl_b200_linear_transform_hybrid_bsgs): ciphertext c of `ciphertexts` (2*level_size*n words each) is stored at
    result[c * 2*l'*n:], l' = level_size - rescale.  diagonals lists len(giant_elts) x len(baby_elts) buffers (flat,
    row j = giant j, or one list per giant), each None (absent) or (level_size + p_size) x n words in NTT form.  A key
    of None is an identity term (element 1) on either side.  rescale=True divides by the last limb in the final
    mod-down."""
    mods = np.ascontiguousarray(moduli, dtype=np.uint64)
    be = np.ascontiguousarray(baby_elts, dtype=np.uint64)
    ge = np.ascontiguousarray(giant_elts, dtype=np.uint64)
    rp, rn, rc = _buf(result); cp, cn, cc = _buf(ciphertexts)
    flat = [d for row in diagonals for d in row] if diagonals and isinstance(diagonals[0], (list, tuple)) \
        else list(diagonals)
    per, dwords = 2 * level_size * n, (level_size + p_size) * n
    _need("moduli", mods.size, q_size + p_size)
    _need("baby_keys", len(baby_keys), be.size); _need("giant_keys", len(giant_keys), ge.size)
    _need("diagonals", len(flat), be.size * ge.size)
    _need("result", rn, batch * 2 * (level_size - int(bool(rescale))) * n); _need("ciphertexts", cn, batch * per)
    ptrs, any_cuda = [], False
    for r, d in enumerate(flat[:be.size * ge.size]):
        dp, dn, dc = _buf(d)
        if dp is not None:
            _need(f"diagonals[{r}]", dn, dwords)
        ptrs.append(dp)
        any_cuda = any_cuda or bool(dc)
    table = (_vp * max(1, len(ptrs)))(*ptrs)
    babies = (_vp * max(1, len(baby_keys)))(*[k._h if k is not None else None for k in baby_keys])
    giants = (_vp * max(1, len(giant_keys)))(*[k._h if k is not None else None for k in giant_keys])
    _check(_lib.hexl_b200_linear_transform_hybrid_bsgs(rp, cp, n, level_size, q_size, p_size, digit_size,
                                                       mods.ctypes.data, babies, be.ctypes.data, be.size, giants,
                                                       ge.ctypes.data, ge.size, table, int(bool(rescale)), batch,
                                                       _stream(stream, rc or cc or any_cuda)))
    return result


def MultiplyRelinearizeHybrid(result, ct1, ct2, n, level_size, q_size, p_size, digit_size, moduli,
                              relin_keys: KeySwitchKeys, rescale=False, batch=1, stream=None):
    """ct1 x ct2 relinearized with hybrid keys (hexl_b200_multiply_relinearize_hybrid): pair c reads
    ct1[c * 2*level_size*n:] and ct2[c * 2*level_size*n:] and its product is stored at result[c * 2*l'*n:],
    l' = level_size - rescale.  relin_keys switches s^2 to s (key_component_count 2).  rescale=True divides by the last
    limb in the same mod-down (one rounding, not bit-identical to a separate DivideAndRoundQLast).  ct1 may be ct2."""
    mods = np.ascontiguousarray(moduli, dtype=np.uint64)
    rp, rn, rc = _buf(result); ap, an, ac = _buf(ct1); bp, bn, bc = _buf(ct2)
    per = 2 * level_size * n
    _need("moduli", mods.size, q_size + p_size)
    _need("result", rn, batch * 2 * (level_size - int(bool(rescale))) * n)
    _need("ct1", an, batch * per); _need("ct2", bn, batch * per)
    _check(_lib.hexl_b200_multiply_relinearize_hybrid(rp, ap, bp, n, level_size, q_size, p_size, digit_size,
                                                      mods.ctypes.data,
                                                      relin_keys._h if relin_keys is not None else None,
                                                      int(bool(rescale)), batch, _stream(stream, rc or ac or bc)))
    return result


def MultiplyRelinearizeSumHybrid(result, ct1, ct2, n, level_size, q_size, p_size, digit_size, moduli,
                                 relin_keys: KeySwitchKeys, rescale=False, batch=1, stream=None):
    """sum_r ct1_r x ct2_r relinearized once with hybrid keys (hexl_b200_multiply_relinearize_sum_hybrid): ct1 and ct2
    list batch x num_pairs ciphertexts (flat, entry c * num_pairs + r = pair r of output c, or one list per output),
    each 2*level_size*n words; output c is stored at result[c * 2*l'*n:], l' = level_size - rescale.  relin_keys
    switches s^2 to s.  num_pairs = 1 is MultiplyRelinearizeHybrid bit for bit; rescale=False is DyadicMultiply of every
    pair, the sums and KeySwitchHybrid bit for bit.  Entries may repeat, and ct1[x] may be ct2[x]."""
    mods = np.ascontiguousarray(moduli, dtype=np.uint64)
    rp, rn, rc = _buf(result)

    def flat(cts):
        return [x for row in cts for x in row] if cts and isinstance(cts[0], (list, tuple)) else list(cts)

    a, b = flat(ct1), flat(ct2)
    if len(a) != len(b):
        raise HexlB200Error(-1, f"ct1 lists {len(a)} ciphertexts and ct2 {len(b)}")
    if batch and len(a) % batch:
        raise HexlB200Error(-1, f"{len(a)} pairs do not split into {batch} outputs")
    pairs = len(a) // batch if batch else 0
    per = 2 * level_size * n
    _need("moduli", mods.size, q_size + p_size)
    _need("result", rn, batch * 2 * (level_size - int(bool(rescale))) * n)
    ptrs, any_cuda = [[], []], bool(rc)
    for side, cts in enumerate((a, b)):
        for x, ct in enumerate(cts):
            p, cn, cc = _buf(ct)
            if p is not None:
                _need(f"ct{side + 1}[{x}]", cn, per)
            ptrs[side].append(p)
            any_cuda = any_cuda or bool(cc)
    t1 = (_vp * max(1, len(a)))(*ptrs[0])
    t2 = (_vp * max(1, len(b)))(*ptrs[1])
    _check(_lib.hexl_b200_multiply_relinearize_sum_hybrid(rp, t1, t2, pairs, n, level_size, q_size, p_size,
                                                          digit_size, mods.ctypes.data,
                                                          relin_keys._h if relin_keys is not None else None,
                                                          int(bool(rescale)), batch, _stream(stream, any_cuda)))
    return result


def InnerSumHybrid(result, ciphertexts, n, level_size, q_size, p_size, digit_size, moduli, galois_elt, sum_count,
                   galois_keys, key_elts, rescale=False, batch=1, stream=None):
    """sum_{j < sum_count} sigma_{g^j}(ct) with hybrid keys, g = galois_elt (hexl_b200_inner_sum_hybrid): ciphertext c
    of `ciphertexts` (2*level_size*n words each) is stored at result[c * 2*l'*n:], l' = level_size - rescale.
    (key_elts[r], galois_keys[r]) is a table of available keys; the call looks up the powers of g it needs there.  The
    log-step rotate-and-sum stays in the extended basis and is rounded once; rescale=True divides by the last limb in
    that mod-down."""
    mods = np.ascontiguousarray(moduli, dtype=np.uint64)
    ke = np.ascontiguousarray(key_elts, dtype=np.uint64)
    rp, rn, rc = _buf(result); cp, cn, cc = _buf(ciphertexts)
    _need("moduli", mods.size, q_size + p_size)
    _need("galois_keys", len(galois_keys), ke.size)
    _need("result", rn, batch * 2 * (level_size - int(bool(rescale))) * n)
    _need("ciphertexts", cn, batch * 2 * level_size * n)
    keys = (_vp * max(1, ke.size))(*[k._h if k is not None else None for k in list(galois_keys)[:ke.size]])
    _check(_lib.hexl_b200_inner_sum_hybrid(rp, cp, n, level_size, q_size, p_size, digit_size, mods.ctypes.data,
                                           galois_elt, sum_count, keys, ke.ctypes.data, ke.size,
                                           int(bool(rescale)), batch, _stream(stream, rc or cc)))
    return result


def BfvMultiply(result, ct1, ct2, n, moduli, level_size, base_b, m_sk, plain_modulus, batch=1, stream=None):
    """BFV ct1 x ct2 by BEHZ (hexl_b200_bfv_multiply): pair c reads ct1[c * 2*level_size*n:] and ct2[c * 2*level_size*n:]
    (coefficient form) and its tensor scaled by t/Q, (d0, d1, d2), is stored at result[c * 3*level_size*n:].  Q is the
    first level_size entries of moduli; base_b (B) and m_sk are the BEHZ bases, plain_modulus is t.  ct1 may be ct2."""
    mods = np.ascontiguousarray(moduli, dtype=np.uint64)
    bb = np.ascontiguousarray(base_b, dtype=np.uint64)
    rp, rn, rc = _buf(result); ap, an, ac = _buf(ct1); bp, bn, bc = _buf(ct2)
    per = 2 * level_size * n
    _need("moduli", mods.size, level_size)
    _need("result", rn, batch * 3 * level_size * n)
    _need("ct1", an, batch * per); _need("ct2", bn, batch * per)
    _check(_lib.hexl_b200_bfv_multiply(rp, ap, bp, n, mods.ctypes.data, level_size, bb.ctypes.data, bb.size, m_sk,
                                       plain_modulus, batch, _stream(stream, rc or ac or bc)))
    return result


def BfvMultiplyRelinearizeHybrid(result, ct1, ct2, n, level_size, q_size, p_size, digit_size, moduli, base_b, m_sk,
                                 plain_modulus, relin_keys: KeySwitchKeys, batch=1, stream=None):
    """BFV ct1 x ct2 by BEHZ relinearized with hybrid keys (hexl_b200_bfv_multiply_relinearize_hybrid): pair c's
    (d0, d1) + KS(d2) is stored at result[c * 2*level_size*n:], coefficient form.  moduli holds q_size data moduli then
    p_size special primes, as for MultiplyRelinearizeHybrid; base_b, m_sk and plain_modulus as for BfvMultiply.  Bit for
    bit BfvMultiply, the forward transform of d2, KeySwitchHybrid, the inverse transform and the addition of (d0, d1)."""
    mods = np.ascontiguousarray(moduli, dtype=np.uint64)
    bb = np.ascontiguousarray(base_b, dtype=np.uint64)
    rp, rn, rc = _buf(result); ap, an, ac = _buf(ct1); bp, bn, bc = _buf(ct2)
    per = 2 * level_size * n
    _need("moduli", mods.size, q_size + p_size)
    _need("result", rn, batch * per)
    _need("ct1", an, batch * per); _need("ct2", bn, batch * per)
    _check(_lib.hexl_b200_bfv_multiply_relinearize_hybrid(rp, ap, bp, n, level_size, q_size, p_size, digit_size,
                                                          mods.ctypes.data, bb.ctypes.data, bb.size, m_sk,
                                                          plain_modulus,
                                                          relin_keys._h if relin_keys is not None else None, batch,
                                                          _stream(stream, rc or ac or bc)))
    return result


# ------------------------------------------------------------------ plaintexts of BFV and BGV
def PlainLift(result, plain, plain_coeff_count, n, moduli, level_size, plain_modulus, correction_factor=1,
              ntt_form=False, count=1, stream=None):
    """Lift `count` plaintexts (plain_coeff_count words each, mod plain_modulus) into level_size limbs of n words each
    (hexl_b200_plain_lift): m' = [m correction_factor]_t, limb i = [m' - t]_{q_i} if m' >= floor((t + 1) / 2) else
    [m']_{q_i}; ntt_form=True then applies the forward transform.  Plaintext p is stored at result[p * level_size*n:]."""
    mods = np.ascontiguousarray(moduli, dtype=np.uint64)
    rp, rn, rc = _buf(result); pp, pn, pc = _buf(plain)
    _need("moduli", mods.size, level_size)
    _need("result", rn, count * level_size * n); _need("plain", pn, count * plain_coeff_count)
    _check(_lib.hexl_b200_plain_lift(rp, pp, plain_coeff_count, n, mods.ctypes.data, level_size, plain_modulus,
                                     correction_factor, int(bool(ntt_form)), count, _stream(stream, rc or pc)))
    return result


def BfvAddPlain(result, ct, plain, plain_coeff_count, n, moduli, level_size, plain_modulus, subtract=False,
                plain_count=1, batch=1, stream=None):
    """BFV add_plain / sub_plain (hexl_b200_bfv_add_plain): c0 of ciphertext c (ct[c * 2*level_size*n:], coefficient
    form) +- round(Q m / t) over the first plain_coeff_count coefficients, stored at result[c * 2*level_size*n:].  One
    plaintext for all ciphertexts (plain_count=1) or one each (plain_count=batch, at plain[c * plain_coeff_count:]).
    result may be ct."""
    mods = np.ascontiguousarray(moduli, dtype=np.uint64)
    rp, rn, rc = _buf(result); cp, cn, cc = _buf(ct); pp, pn, pc = _buf(plain)
    per = 2 * level_size * n
    _need("moduli", mods.size, level_size)
    _need("result", rn, batch * per); _need("ct", cn, batch * per); _need("plain", pn, plain_count * plain_coeff_count)
    _check(_lib.hexl_b200_bfv_add_plain(rp, cp, pp, plain_coeff_count, plain_count, n, mods.ctypes.data, level_size,
                                        plain_modulus, int(bool(subtract)), batch, _stream(stream, rc or cc or pc)))
    return result


def BfvMultiplyPlain(result, ct, plain, plain_coeff_count, n, moduli, level_size, plain_modulus, plain_ntt_form=False,
                     plain_count=1, batch=1, stream=None):
    """BFV multiply_plain (hexl_b200_bfv_multiply_plain): ciphertext c (coefficient form) times the lifted plaintext,
    negacyclic per limb, stored at result[c * 2*level_size*n:] in coefficient form.  plain_ntt_form=True takes
    PlainLift(ntt_form=True) outputs (level_size*n words each) and ignores plain_coeff_count.  result may be ct."""
    mods = np.ascontiguousarray(moduli, dtype=np.uint64)
    rp, rn, rc = _buf(result); cp, cn, cc = _buf(ct); pp, pn, pc = _buf(plain)
    per = 2 * level_size * n
    _need("moduli", mods.size, level_size)
    _need("result", rn, batch * per); _need("ct", cn, batch * per)
    _need("plain", pn, plain_count * (level_size * n if plain_ntt_form else plain_coeff_count))
    _check(_lib.hexl_b200_bfv_multiply_plain(rp, cp, pp, plain_coeff_count, plain_count, int(bool(plain_ntt_form)), n,
                                             mods.ctypes.data, level_size, plain_modulus, batch,
                                             _stream(stream, rc or cc or pc)))
    return result


# ------------------------------------------------------------------ BGV
def BgvModSwitch(result, operand, n, moduli, rns_modulus_size, plain_modulus, count=1, ntt_form=True, stream=None):
    """BGV modulus switch of `count` polynomials of rns_modulus_size limbs (n words each) by their last modulus
    (hexl_b200_bgv_mod_switch; SEAL's mod_t_and_divide_q_last(_ntt)_inplace): DivideAndRoundQLast's layout with the
    rounding replaced by a correction that is 0 mod plain_modulus.  Limb L of result is not written; result may be
    operand.  The message picks up [q_L^-1]_t."""
    mods = np.ascontiguousarray(moduli, dtype=np.uint64)
    rp, rn, rc = _buf(result); op, on, oc = _buf(operand)
    _need("moduli", mods.size, rns_modulus_size)
    _need("result", rn, count * rns_modulus_size * n); _need("operand", on, count * rns_modulus_size * n)
    _check(_lib.hexl_b200_bgv_mod_switch(rp, op, n, mods.ctypes.data, rns_modulus_size, plain_modulus, count,
                                         int(bool(ntt_form)), _stream(stream, rc or oc)))
    return result


def BgvKeySwitchHybrid(result, target, n, level_size, q_size, p_size, digit_size, key_component_count, moduli,
                       plain_modulus, keys: KeySwitchKeys, batch=1, stream=None):
    """KeySwitchHybrid for BGV (hexl_b200_bgv_key_switch_hybrid): the same layouts, with the mod-down by P subtracting
    a correction that is 0 mod plain_modulus.  Accumulates into result."""
    mods = np.ascontiguousarray(moduli, dtype=np.uint64)
    rp, rn, rc = _buf(result); tp, tn, tc = _buf(target)
    _need("moduli", mods.size, q_size + p_size)
    _need("result", rn, batch * key_component_count * level_size * n); _need("target", tn, batch * level_size * n)
    _check(_lib.hexl_b200_bgv_key_switch_hybrid(rp, tp, n, level_size, q_size, p_size, digit_size,
                                                key_component_count, mods.ctypes.data, plain_modulus,
                                                keys._h if keys is not None else None, batch,
                                                _stream(stream, rc or tc)))
    return result


def BgvApplyGaloisKeySwitchHybridHoisted(results, ciphertexts, n, level_size, q_size, p_size, digit_size, moduli,
                                         plain_modulus, galois_keys, galois_elts, batch=1, stream=None):
    """ApplyGaloisKeySwitchHybridHoisted for BGV (hexl_b200_bgv_apply_galois_key_switch_hybrid_hoisted): SEAL's
    rotate_rows / rotate_columns for every element of galois_elts with one mod-up, the same layouts."""
    mods = np.ascontiguousarray(moduli, dtype=np.uint64)
    elts = np.ascontiguousarray(galois_elts, dtype=np.uint64)
    rp, rn, rc = _buf(results); cp, cn, cc = _buf(ciphertexts)
    per = 2 * level_size * n
    _need("moduli", mods.size, q_size + p_size); _need("galois_keys", len(galois_keys), elts.size)
    _need("results", rn, batch * elts.size * per); _need("ciphertexts", cn, batch * per)
    keys = (_vp * max(1, len(galois_keys)))(*[k._h if k is not None else None for k in galois_keys])
    _check(_lib.hexl_b200_bgv_apply_galois_key_switch_hybrid_hoisted(rp, cp, n, level_size, q_size, p_size,
                                                                     digit_size, mods.ctypes.data, plain_modulus,
                                                                     keys, elts.ctypes.data, elts.size, batch,
                                                                     _stream(stream, rc or cc)))
    return results


def BgvMultiplyRelinearizeHybrid(result, ct1, ct2, n, level_size, q_size, p_size, digit_size, moduli, plain_modulus,
                                 relin_keys: KeySwitchKeys, mod_switch=False, batch=1, stream=None):
    """MultiplyRelinearizeHybrid for BGV (hexl_b200_bgv_multiply_relinearize_hybrid): the same layouts, the mod-down
    t-corrected; mod_switch=True drops the last limb in the same mod-down (the message picks up [q_{l-1}^-1]_t).
    mod_switch=False equals DyadicMultiply followed by BgvKeySwitchHybrid bit for bit.  ct1 may be ct2."""
    mods = np.ascontiguousarray(moduli, dtype=np.uint64)
    rp, rn, rc = _buf(result); ap, an, ac = _buf(ct1); bp, bn, bc = _buf(ct2)
    per = 2 * level_size * n
    _need("moduli", mods.size, q_size + p_size)
    _need("result", rn, batch * 2 * (level_size - int(bool(mod_switch))) * n)
    _need("ct1", an, batch * per); _need("ct2", bn, batch * per)
    _check(_lib.hexl_b200_bgv_multiply_relinearize_hybrid(rp, ap, bp, n, level_size, q_size, p_size, digit_size,
                                                          mods.ctypes.data, plain_modulus,
                                                          relin_keys._h if relin_keys is not None else None,
                                                          int(bool(mod_switch)), batch,
                                                          _stream(stream, rc or ac or bc)))
    return result
