"""ctypes binding of libanovos_b200.so (include/anovos_b200.h).

There is NO CPU fallback: importing works anywhere (so argument handling can be
tested on a CPU box), but every compute entry point raises if the CUDA library or a
CUDA device is missing.
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("ANOVOS_B200_LIB") or os.path.join(HERE, "libanovos_b200.so")

ANV_F32, ANV_F64, ANV_I32, ANV_I64 = 0, 1, 2, 3
MAX_LAUNCH_COLS = 65535   # ANV_MAX_LAUNCH_COLS of the header: columns per call of an entry point taking descriptors
MAX_BINS = 16384          # ANV_MAX_BINS of the header: bins per column of anv_hist / anv_moments_hist / anv_bin_assign


class AnvColumn(C.Structure):
    _fields_ = [("data", C.c_void_p), ("validity", C.c_void_p), ("dtype", C.c_int32), ("reserved", C.c_int32)]


class AnvMoments(C.Structure):
    _fields_ = [("n_valid", C.c_int64), ("n_nonzero", C.c_int64), ("min", C.c_double), ("max", C.c_double),
                ("mean", C.c_double), ("m2", C.c_double), ("m3", C.c_double), ("m4", C.c_double)]


class AnvBinspec(C.Structure):
    _fields_ = [("n_bins", C.c_int32), ("mode", C.c_int32), ("lo", C.c_double), ("inv_w", C.c_double),
                ("cut_offset", C.c_int64)]


class AnvDrift(C.Structure):
    _fields_ = [("psi", C.c_double), ("hd", C.c_double), ("jsd", C.c_double), ("ks", C.c_double),
                ("n_rows", C.c_int32), ("reserved", C.c_int32)]


class AnvImputeSpec(C.Structure):
    _fields_ = [("out_dtype", C.c_int32), ("flags", C.c_int32), ("fill", C.c_uint64)]


IMPUTE_NAN_MISSING, IMPUTE_ROUND_DOUBLE = 1, 2   # ANV_IMPUTE_* flags of the header


class AnvScaleSpec(C.Structure):
    _fields_ = [("mode", C.c_int32), ("out_dtype", C.c_int32), ("flags", C.c_int32), ("reserved", C.c_int32),
                ("a", C.c_double), ("b", C.c_double), ("c", C.c_double)]


SCALE_DIV, SCALE_AFFINE, SCALE_CONST = 0, 1, 2   # ANV_SCALE_* modes of the header
SCALE_NAN_TO_NULL = 1                            # ANV_SCALE_NAN_TO_NULL


# ANV_TF_* ops of the header
(TF_LN, TF_LOG10, TF_LOG2, TF_EXP, TF_POW_BASE, TF_POW, TF_SQRT, TF_CBRT, TF_SIN, TF_COS, TF_TAN, TF_ASIN, TF_ACOS, TF_ATAN,
 TF_RADIANS, TF_MUL_INV, TF_FLOOR, TF_CEIL, TF_FACTORIAL, TF_REMAINDER, TF_ROUND) = range(21)
TF_MAKES_NULLS = (TF_LN, TF_LOG10, TF_LOG2, TF_MUL_INV, TF_FACTORIAL)


class AnvError(RuntimeError):
    pass


_lib = None

_P, _I, _L, _SZ = C.c_void_p, C.c_int, C.c_int64, C.c_size_t
_SIGNATURES = {
    "anv_version": (C.c_int, []),
    "anv_source_hash": (C.c_char_p, []),
    "anv_last_error": (C.c_char_p, []),
    "anv_device_info": (C.c_int, [_P, _P, _P, _P]),
    "anv_moments_workspace_bytes": (_SZ, [_I, _L]),
    "anv_moments": (C.c_int, [_P, _I, _L, _P, _P, _SZ, _P]),
    "anv_hist": (C.c_int, [_P, _P, _P, _I, _L, _P, _I, _P]),
    "anv_moments_hist": (C.c_int, [_P, _P, _P, _I, _L, _P, _P, _I, _P, _SZ, _P]),
    "anv_bin_assign": (C.c_int, [_P, _P, _P, _I, _L, _I, _P, _L, _P]),
    "anv_hist_codes": (C.c_int, [_P, _P, _I, _L, _P, _I, _P]),
    "anv_drift_reduce": (C.c_int, [_P, _P, _P, _I, _P, _P, _I, _I, _L, _L, _P, _P]),
    "anv_select_workspace_bytes": (_SZ, [_I, _I]),
    "anv_select_ranks": (C.c_int, [_P, _I, _L, _P, _I, _I, _P, _P, _SZ, _P]),
    "anv_select_passes": (C.c_int, [_I]),
    "anv_select_begin": (C.c_int, [_I, _I, _P, _SZ, _P]),
    "anv_select_hist_region": (C.c_int, [_I, _I, _I, _P, _P]),
    "anv_select_accumulate": (C.c_int, [_P, _I, _L, _I, _I, _I, _P, _SZ, _P]),
    "anv_select_advance": (C.c_int, [_P, _I, _P, _I, _I, _I, _P, _P, _SZ, _P]),
    "anv_hll_registers": (C.c_int, [_P, _I, _L, _I, _P, _P]),
    "anv_xxh64_utf8": (C.c_int, [_P, _P, _L, _P]),
    "anv_gk_partition_sketch": (C.c_longlong, [_P, C.c_longlong, C.c_longlong, C.c_double, C.c_longlong, _P, _P, _P, C.c_longlong]),
    "anv_mode_distinct_workspace_bytes": (_SZ, [_I, _L, _I]),
    "anv_mode_distinct": (C.c_int, [_P, _I, _L, _I, _P, _P, _P, _P, _I, _P, _P, _SZ, _P]),
    "anv_mode_distinct_hll": (C.c_int, [_P, _I, _L, _I, _P, _P, _P, _P, _I, _P, _I, _P, _P, _SZ, _P]),
    "anv_mode_distinct_partition_workspace_bytes": (_SZ, [_I, _L]),
    "anv_mode_distinct_partition": (C.c_int, [_P, _I, _L, _P, _P, _P, _P, _I, _P, _P, _SZ, _P]),
    "anv_mode_distinct_partition_hll": (C.c_int, [_P, _I, _L, _P, _P, _P, _P, _I, _P, _I, _P, _P, _SZ, _P]),
    "anv_row_null_counts": (C.c_int, [_P, _I, _I, _L, _I, _P, _P, _P]),
    "anv_row_distinct_workspace_bytes": (_SZ, [_L]),
    "anv_row_distinct": (C.c_int, [_P, _I, _L, _I, _P, _P, _P, _SZ, _P]),
    "anv_impute_fill": (C.c_int, [_P, _P, _P, _I, _L, _P]),
    "anv_valid_not_nan": (C.c_int, [_P, _I, _L, _P, _P, _P]),
    "anv_scale_columns": (C.c_int, [_P, _P, _P, _P, _P, _I, _L, _P]),
    "anv_transform_columns": (C.c_int, [_P, _P, _P, _P, _P, _I, _L, _P]),
    "anv_ks_candidates_workspace_bytes": (_SZ, [_L]),
    "anv_ks_candidates": (C.c_int, [_P, _I, _L, _L, _P, _I, _P, _P, _P, _SZ, _P]),
    "anv_code_map": (C.c_int, [_P, _P, _P, _I, _L, _P]),
    "anv_one_hot": (C.c_int, [_P, _P, _I, _L, _P]),
    "anv_flag_members": (C.c_int, [_P, _P, _I, _L, _P]),
    "anv_flag_members_smem_keys": (C.c_int, []),
    "anv_class_hist": (C.c_int, [_P, _P, _P, _P, _I, _L, _P]),
    "anv_class_hist_max_thresholds": (C.c_int, []),
    "anv_spark_hash_seed": (C.c_uint64, [_L]),
    "anv_spark_sample_mask": (C.c_int, [_L, _L, _P, _P, _I, _P, _P]),
    "anv_synth_f32": (C.c_int, [_P, _P, _L, C.c_uint64, C.c_uint32, _I, C.c_float, C.c_float, C.c_float, _P]),
    "anv_synth_codes": (C.c_int, [_P, _P, _L, C.c_uint64, C.c_uint32, _I, C.c_float, C.c_float, _P]),
    "anv_synth_f32_rows": (C.c_int, [_P, _P, _L, _L, C.c_uint64, C.c_uint32, _I, C.c_float, C.c_float, C.c_float, _P]),
    "anv_synth_codes_rows": (C.c_int, [_P, _P, _L, _L, C.c_uint64, C.c_uint32, _I, C.c_float, C.c_float, _P]),
}


def lib():
    """Load (once) and return the ctypes handle; raise loudly when it is not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            try:  # build in-tree when a CUDA toolkit is around; never fall back to a CPU path
                from . import build as _build
                _build.build()
            except Exception as e:
                raise AnvError("libanovos_b200.so is not built (%s) and building it failed (%s). Run "
                               "`python -m anovos_b200.build` (needs nvcc). There is no CPU fallback." % (LIB_PATH, e))
        h = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            f = getattr(h, name)
            f.restype, f.argtypes = res, args
        if not os.environ.get("ANOVOS_B200_LIB"):
            # a stale binary (built from older .cu sources) would load silently and its struct layouts / workspace
            # sizing could have drifted from this binding: compare the source hash baked into the .so
            from . import build as _build
            want, have = _build.source_hash(), h.anv_source_hash().decode()
            if have != want:
                raise AnvError("libanovos_b200.so is stale: built from sources %s, the tree holds %s. Run "
                               "`python -m anovos_b200.build`." % (have[:12], want[:12]))
        _lib = h
    return _lib


def exported_symbols():
    return sorted(_SIGNATURES)


def check(rc: int, what: str = ""):
    if rc != 0:
        msg = lib().anv_last_error().decode("utf-8", "replace")
        raise AnvError("%s failed (%d): %s" % (what or "libanovos_b200", rc, msg))


def require_cuda():
    """The product path needs a CUDA device: fail loudly, never fall back."""
    import torch
    lib()
    if not torch.cuda.is_available():
        raise AnvError("anovos_b200 needs a CUDA device (sm_90a); torch.cuda.is_available() is False. "
                       "There is no CPU fallback.")
    return torch
