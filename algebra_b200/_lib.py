"""ctypes binding of libalgebra_b200.so (the C ABI in include/algebra_b200.h).

There is no CPU fallback: if the shared library is missing this module raises at import of the first
symbol, and every compute entry point fails with a CUDA error when no device is present."""
from __future__ import annotations

import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("B200_LIB_PATH") or os.path.join(_HERE, "libalgebra_b200.so")   # (override: build-variant debugging)

EINVAL, ETOOLARGE, ENOMEM = -1, -2, -3
SCALARS_FR_MONT, SCALARS_BIGINT, SCALARS_U8, SCALARS_U16, SCALARS_U32, SCALARS_U64 = range(6)

# every symbol include/algebra_b200.h declares: name -> (restype, argtypes)
_c = ctypes
_u64p = _c.POINTER(_c.c_uint64)
_vp = _c.c_void_p
SIGNATURES = {
    "b200_version": (_c.c_char_p, []),
    "b200_last_error": (_c.c_char_p, []),
    "b200_msm_sw_g1": (_c.c_int, [_c.c_int, _vp, _vp, _c.c_size_t, _vp]),
    "b200_msm_sw_g1_dev": (_c.c_int, [_c.c_int, _vp, _vp, _c.c_size_t, _vp, _vp]),
    "b200_msm_sw_g1_scalars": (_c.c_int, [_c.c_int, _c.c_int, _vp, _vp, _c.c_size_t, _vp]),
    "b200_msm_sw_g1_scalars_dev": (_c.c_int, [_c.c_int, _c.c_int, _vp, _vp, _c.c_size_t, _vp, _vp]),
    "b200_msm_sw_g2": (_c.c_int, [_vp, _vp, _c.c_size_t, _vp]),
    "b200_msm_sw_g2_dev": (_c.c_int, [_vp, _vp, _c.c_size_t, _vp, _vp]),
    "b200_device_count": (_c.c_int, []),
    "b200_msm_sw_g1_multi": (_c.c_int, [_c.c_int, _c.c_int, _vp, _vp, _c.c_size_t, _vp]),
    "b200_bases_upload": (_c.c_int, [_c.c_int, _c.c_int, _vp, _c.c_size_t, _c.POINTER(_vp)]),
    "b200_msm_bases": (_c.c_int, [_vp, _c.c_int, _vp, _c.c_size_t, _vp]),
    "b200_bases_free": (_c.c_int, [_vp]),
    "b200_msm_stream_begin": (_c.c_int, [_c.c_int, _c.c_int, _c.c_size_t, _c.c_size_t, _c.POINTER(_vp)]),
    "b200_msm_stream_push": (_c.c_int, [_vp, _vp, _vp, _c.c_size_t]),
    "b200_msm_stream_finish": (_c.c_int, [_vp, _vp]),
    "b200_msm_stream_abort": (_c.c_int, [_vp]),
    "b200_set_msm_window": (_c.c_int, [_c.c_int]),
    "b200_set_msm_affine_levels": (_c.c_int, [_c.c_int]),
    "b200_set_msm_bucket_slice": (_c.c_int, [_c.c_int, _c.c_int]),
    "b200_msm_window_for": (_c.c_int, [_c.c_int, _c.c_size_t]),
    "b200_g1_sum": (_c.c_int, [_c.c_int, _vp, _c.c_size_t, _vp]),
    "b200_g1_into_affine": (_c.c_int, [_c.c_int, _vp, _vp]),
    "b200_ntt_fr": (_c.c_int, [_c.c_int, _vp, _c.c_uint32, _c.c_int, _vp]),
    "b200_ntt_fr_padded": (_c.c_int, [_c.c_int, _vp, _c.c_size_t, _vp, _c.c_uint32, _c.c_int, _vp]),
    "b200_ntt_fr_dev": (_c.c_int, [_c.c_int, _vp, _c.c_uint32, _c.c_int, _vp, _vp]),
    "b200_ntt_g1": (_c.c_int, [_c.c_int, _vp, _c.c_uint32, _c.c_int, _vp]),
    "b200_ntt_g1_dev": (_c.c_int, [_c.c_int, _vp, _c.c_uint32, _c.c_int, _vp, _vp]),
    "b200_clear_cache": (_c.c_int, []),
    "b200_poly_mul_size": (_c.c_size_t, [_c.c_int, _c.c_size_t, _c.c_size_t]),
    "b200_poly_mul_fr": (_c.c_int, [_c.c_int, _vp, _c.c_size_t, _vp, _c.c_size_t, _vp]),
    "b200_poly_mul_fr_dev": (_c.c_int, [_c.c_int, _vp, _c.c_size_t, _vp, _c.c_size_t, _vp, _vp]),
    "b200_gen_bases_dev": (_c.c_int, [_c.c_int, _c.c_uint64, _c.c_size_t, _vp, _vp, _vp]),
    "b200_gen_scalars_dev": (_c.c_int, [_c.c_int, _c.c_uint64, _c.c_size_t, _vp, _vp]),
    "b200_g1_batch_mul_dev": (_c.c_int, [_c.c_int, _vp, _vp, _c.c_size_t, _vp, _vp]),
    "b200_g1_normalize_batch_dev": (_c.c_int, [_c.c_int, _vp, _c.c_size_t, _vp, _vp]),
    "b200_fp_op_dev": (_c.c_int, [_c.c_int, _c.c_int, _vp, _vp, _vp, _c.c_size_t, _c.c_int, _vp]),
    "b200_ec_op_dev": (_c.c_int, [_c.c_int, _c.c_int, _vp, _vp, _vp, _c.c_size_t, _vp]),
    "b200_msm_last_timings": (_c.c_int, [_c.POINTER(_c.c_float), _c.POINTER(_c.c_int), _c.POINTER(_c.c_int),
                                         _c.POINTER(_c.c_ulonglong)]),
    "b200_launch_count": (_c.c_ulonglong, []),
}

_lib = None


class B200Error(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"algebra_b200 error {code}: {msg}")
        self.code = code


def lib() -> ctypes.CDLL:
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(or `make -C algebra_b200/csrc`). algebra_b200 has no CPU fallback.")
        l = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def check(rc: int) -> None:
    if rc != 0:
        raise B200Error(rc, lib().b200_last_error().decode(errors="replace"))
