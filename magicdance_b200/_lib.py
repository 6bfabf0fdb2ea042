"""ctypes binding of the C ABI declared in include/magicdance_b200.h.

There is deliberately no fallback: if the shared library is missing or the device is not
sm_90, every compute entry point raises.
"""
from __future__ import annotations

import ctypes as C
import os

from . import build as _build

c_void_p, c_int32, c_int64, c_float = C.c_void_p, C.c_int32, C.c_int64, C.c_float


class GemmDesc(C.Structure):
    _fields_ = [
        ("a", c_void_p), ("lda", c_int64), ("a2", c_void_p), ("lda2", c_int64),
        ("k1", c_int32), ("conv", c_int32), ("nb", c_int32), ("h", c_int32), ("w", c_int32), ("c", c_int32),
        ("b", c_void_p), ("ldb", c_int64), ("d", c_void_p), ("ldd", c_int64),
        ("bias", c_void_p), ("bias_batch_stride", c_int64), ("rows_per_batch", c_int32), ("epilogue", c_int32),
        ("residual", c_void_p), ("ldr", c_int64),
        ("m", c_int32), ("n", c_int32), ("k", c_int32), ("splits", c_int32), ("splitk_ws", c_void_p),
        ("ln_u", c_void_p), ("ln_eps", c_float),
    ]


class AttnDesc(C.Structure):
    _fields_ = [
        ("q", c_void_p), ("ldq", c_int64),
        ("k0", c_void_p), ("ldk0", c_int64), ("vt0", c_void_p), ("ldvt0", c_int64),
        ("n0", c_int32), ("kv0_batches", c_int32), ("ldv0_batch", c_int32),
        ("k1", c_void_p), ("ldk1", c_int64), ("vt1", c_void_p), ("ldvt1", c_int64),
        ("n1", c_int32), ("kv1_batches", c_int32), ("ldv1_batch", c_int32),
        ("out", c_void_p), ("ldo", c_int64),
        ("batch", c_int32), ("heads", c_int32), ("d", c_int32), ("nq", c_int32), ("bank_batches", c_int32),
        ("scale", c_float),
    ]


class AttnBwdDesc(C.Structure):
    _fields_ = [
        ("fwd", AttnDesc),
        ("dout", c_void_p), ("lddout", c_int64),
        ("lse", c_void_p),
        ("dq", c_void_p), ("lddq", c_int64),
        ("dk0", c_void_p), ("lddk0", c_int64), ("dvt0", c_void_p), ("lddvt0", c_int64),
        ("dk1", c_void_p), ("lddk1", c_int64), ("dvt1", c_void_p), ("lddvt1", c_int64),
        ("ws", c_void_p),
    ]


class GemmBwdDesc(C.Structure):
    _fields_ = [
        ("fwd", GemmDesc),
        ("dd", c_void_p), ("lddd", c_int64),
        ("da", c_void_p), ("ldda", c_int64), ("da_dtype", c_int32), ("da_accumulate", c_int32),
        ("da2", c_void_p), ("ldda2", c_int64), ("da2_dtype", c_int32), ("da2_accumulate", c_int32),
        ("db", c_void_p), ("lddb", c_int64), ("db_dtype", c_int32), ("db_accumulate", c_int32),
        ("dbias", c_void_p), ("dbias_accumulate", c_int32),
        ("splits", c_int32),
        ("ws", c_void_p),
    ]


class GroupNormBwdDesc(C.Structure):
    _fields_ = [
        ("x1", c_void_p), ("x2", c_void_p), ("c1", c_int32), ("c2", c_int32),
        ("gamma", c_void_p), ("beta", c_void_p),
        ("dy", c_void_p),
        ("batch", c_int32), ("hw", c_int32), ("eps", c_float), ("silu", c_int32),
        ("dx1", c_void_p), ("dx1_dtype", c_int32), ("dx1_accumulate", c_int32),
        ("dx2", c_void_p), ("dx2_dtype", c_int32), ("dx2_accumulate", c_int32),
        ("dgamma", c_void_p), ("dbeta", c_void_p), ("dgamma_accumulate", c_int32), ("dbeta_accumulate", c_int32),
        ("ws", c_void_p),
    ]


class LayerNormBwdDesc(C.Structure):
    _fields_ = [
        ("x", c_void_p), ("gamma", c_void_p), ("dy", c_void_p),
        ("rows", c_int64), ("c", c_int32), ("eps", c_float),
        ("dx", c_void_p), ("dx_dtype", c_int32), ("dx_accumulate", c_int32),
        ("dgamma", c_void_p), ("dbeta", c_void_p), ("dgamma_accumulate", c_int32), ("dbeta_accumulate", c_int32),
        ("ws", c_void_p),
    ]


class Conv3x3BwdDesc(C.Structure):
    _fields_ = [
        ("x", c_void_p), ("wt", c_void_p), ("wt_t", c_void_p), ("bias", c_void_p), ("dy", c_void_p),
        ("batch", c_int32), ("h", c_int32), ("w", c_int32), ("cin", c_int32), ("cout", c_int32), ("stride", c_int32),
        ("silu", c_int32),
        ("dx", c_void_p),
        ("dw", c_void_p), ("dw_accumulate", c_int32),
        ("dbias", c_void_p), ("dbias_accumulate", c_int32),
        ("ws", c_void_p),
    ]


class SkinnyBwdDesc(C.Structure):
    _fields_ = [
        ("x", c_void_p), ("w", c_void_p), ("dy", c_void_p),
        ("rows", c_int32), ("n", c_int32), ("k", c_int32), ("silu_in", c_int32),
        ("dx", c_void_p), ("dx_accumulate", c_int32),
        ("dw", c_void_p), ("dw_accumulate", c_int32),
        ("dbias", c_void_p), ("dbias_accumulate", c_int32),
        ("ws", c_void_p),
    ]


# name -> (restype, argtypes); every symbol include/magicdance_b200.h declares
SIGNATURES = {
    "mdb_abi_version": (c_int32, []),
    "mdb_last_error": (C.c_char_p, []),
    "mdb_device_check": (c_int32, []),
    "mdb_launch_count": (c_int64, []),
    "mdb_abi_struct_bytes": (c_int64, [c_int32]),
    "mdb_set_tuning": (c_int32, [c_int32, c_int32]),
    "mdb_get_tuning": (c_int32, [c_int32]),
    "mdb_gemm_f16": (c_int32, [C.POINTER(GemmDesc), c_void_p]),
    "mdb_gemm_bwd_f16": (c_int32, [C.POINTER(GemmBwdDesc), c_void_p]),
    "mdb_gemm_bwd_ws_floats": (c_int64, [C.POINTER(GemmBwdDesc)]),
    "mdb_conv3x3_igemm_f16": (c_int32, [C.POINTER(GemmDesc), c_void_p]),
    "mdb_conv3x3_igemm_bwd_f16": (c_int32, [C.POINTER(GemmBwdDesc), c_void_p]),
    "mdb_conv3x3_igemm_bwd_ws_floats": (c_int64, [C.POINTER(GemmBwdDesc)]),
    "mdb_attention_f16": (c_int32, [C.POINTER(AttnDesc), c_void_p]),
    "mdb_attention_lse_f16": (c_int32, [C.POINTER(AttnDesc), c_void_p, c_void_p]),
    "mdb_attention_bwd_f16": (c_int32, [C.POINTER(AttnBwdDesc), c_void_p]),
    "mdb_attention_bwd_ws_floats": (c_int64, [c_int32, c_int32, c_int32]),
    "mdb_groupnorm_f16": (c_int32, [c_void_p, c_int32, c_void_p, c_int32, c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_int32, c_int32, c_float, c_int32, c_int32, c_void_p]),
    "mdb_groupnorm_ws_floats": (c_int64, [c_int32, c_int32, c_int32]),
    "mdb_layernorm_f16": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int32, c_float, c_void_p]),
    "mdb_groupnorm_bwd_f16": (c_int32, [C.POINTER(GroupNormBwdDesc), c_void_p]),
    "mdb_groupnorm_bwd_ws_floats": (c_int64, [C.POINTER(GroupNormBwdDesc)]),
    "mdb_layernorm_bwd_f16": (c_int32, [C.POINTER(LayerNormBwdDesc), c_void_p]),
    "mdb_layernorm_bwd_ws_floats": (c_int64, [C.POINTER(LayerNormBwdDesc)]),
    "mdb_geglu_f16": (c_int32, [c_void_p, c_int64, c_void_p, c_int64, c_int64, c_int32, c_void_p]),
    "mdb_geglu_bwd_f16": (c_int32, [c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64, c_int64, c_int32,
                                    c_void_p]),
    "mdb_conv3x3_direct_f16": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32,
                                         c_int32, c_int32, c_int32, c_int32, c_void_p]),
    "mdb_conv3x3_direct_bwd_f16": (c_int32, [C.POINTER(Conv3x3BwdDesc), c_void_p]),
    "mdb_conv3x3_direct_bwd_ws_floats": (c_int64, [C.POINTER(Conv3x3BwdDesc)]),
    "mdb_im2col3x3_f16": (c_int32, [c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32, c_int32, c_void_p]),
    "mdb_im2col3x3_br_f16": (c_int32, [c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32, c_int32, c_void_p]),
    "mdb_upsample2x_f16": (c_int32, [c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32, c_void_p]),
    "mdb_upsample2x_bwd_f16": (c_int32, [c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32, c_int32, c_int32,
                                         c_void_p]),
    "mdb_add_f16": (c_int32, [c_void_p, c_void_p, c_void_p, c_int64, c_int32, c_int32, c_void_p]),
    "mdb_timestep_embedding_f32": (c_int32, [c_void_p, c_int32, c_void_p, c_int32, c_int32, c_void_p]),
    "mdb_skinny_linear_f32": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32,
                                        c_int32, c_void_p]),
    "mdb_skinny_linear_bwd_f32": (c_int32, [C.POINTER(SkinnyBwdDesc), c_void_p]),
    "mdb_skinny_linear_bwd_ws_floats": (c_int64, [C.POINTER(SkinnyBwdDesc)]),
    "mdb_nchw_f32_to_nhwc_f16": (c_int32, [c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32, c_int32, c_void_p]),
    "mdb_nhwc_f16_to_nchw_f32": (c_int32, [c_void_p, c_void_p, c_int32, c_int32, c_int32, c_int32, c_void_p]),
    "mdb_softmax_rows_f16": (c_int32, [c_void_p, c_int64, c_int32, c_int32, c_float, c_void_p]),
    "mdb_cfg_ddim_update_f32": (c_int32, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64,
                                          c_void_p, c_int32, c_void_p]),
}

_lib = None
ABI_VERSION = 2
TUNE_GEMM_PAIR_MIN_TILES, TUNE_ATTN40_2Q_MIN_CTAS, TUNE_GEMM_BN80_BELOW = 1, 3, 4
TUNE_GEMM_SKINNY_CTAS, TUNE_GEMM_SPLIT_MIN_CHUNKS = 5, 6


def library_path() -> str:
    return os.environ.get("MAGICDANCE_B200_LIB", _build.LIB_PATH)


def load():
    """dlopen the kernel library and bind every declared symbol (no CUDA calls happen here)."""
    global _lib
    if _lib is not None:
        return _lib
    path = library_path()
    if not os.path.isfile(path):
        raise RuntimeError(
            f"magicdance_b200: kernel library {path} is missing — run `python -m magicdance_b200.build` "
            "(there is no CPU/PyTorch fallback for the hot path)")
    if path == _build.LIB_PATH and os.path.isdir(_build.CSRC) and not _build.is_fresh():
        # the descriptor structs below mirror the sources next to the library: a library built from other sources
        # would be called with mismatched layouts (memory corruption, not an error) — refuse it
        raise RuntimeError(f"magicdance_b200: {path} was not built from the sources in {_build.CSRC} "
                           "(stamp mismatch) — run `python -m magicdance_b200.build`")
    lib = C.CDLL(path)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the .so does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    if lib.mdb_abi_version() != ABI_VERSION:
        raise RuntimeError(f"magicdance_b200: ABI version mismatch ({lib.mdb_abi_version()} != {ABI_VERSION}); "
                           "rebuild the library")
    for which, mirror in ((0, GemmDesc), (1, AttnDesc), (2, AttnBwdDesc), (3, GemmBwdDesc), (4, GroupNormBwdDesc),
                          (5, LayerNormBwdDesc), (6, Conv3x3BwdDesc), (7, SkinnyBwdDesc)):
        if lib.mdb_abi_struct_bytes(which) != C.sizeof(mirror):
            raise RuntimeError(f"magicdance_b200: {mirror.__name__} mirrors {C.sizeof(mirror)} bytes, the library's "
                               f"struct has {lib.mdb_abi_struct_bytes(which)}: the binding and the library disagree")
    _lib = lib
    return lib


def check(rc: int, what: str):
    if rc != 0:
        msg = load().mdb_last_error().decode(errors="replace")
        raise RuntimeError(f"magicdance_b200.{what} failed (code {rc}): {msg}")
