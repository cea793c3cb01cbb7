"""
ctypes binding of libct_b200.so (include/ct_b200.h) -- the only route from the Python host
layer to the sm_90a kernels.

There is NO CPU implementation behind these functions: if the shared library is missing,
or no H100 is visible, every compute call raises.  Nothing here imports `oracle/`.
"""
from __future__ import annotations

import ctypes
import os
from typing import Optional

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
# CT_B200_LIB loads another build of the library, for example the parent commit's, for A/B timing
LIB_PATH = os.environ.get("CT_B200_LIB") or os.path.join(_HERE, "libct_b200.so")

INF = (1 << 63) - 1  # CT_DIV_INF

# ct_status_t
CT_OK = 0
CT_E_DTYPE, CT_E_BITS, CT_E_SHAPE, CT_E_ALIGN, CT_E_CUDA, CT_E_ARG, CT_E_NODEV, CT_E_UNSUPPORTED = -1, -2, -3, -4, -5, -6, -7, -8

# ct_dtype_t
DT_NONE = -1
DT = {
    torch.float32: 0,
    torch.float16: 1,
    torch.bfloat16: 2,
    torch.int8: 3,
    torch.float8_e4m3fn: 4,
    torch.int32: 5,
    torch.uint8: 6,
    torch.bool: 6,
    torch.int64: 7,
}

# ct_batch_op_t
(OP_QUANTIZE_PACK, OP_UNPACK_DEQUANTIZE, OP_QUANTIZE, OP_DEQUANTIZE, OP_FAKE_QUANTIZE, OP_PACK_INT32, OP_UNPACK_INT32,
 OP_OBSERVE_QUANTIZE_PACK, OP_QUANTIZE_PACK_FP4, OP_UNPACK_DEQUANTIZE_FP4, OP_OBSERVE_QUANTIZE_PACK_FP4,
 OP_SPARSE24_QUANTIZE_PACK, OP_SPARSE24_UNPACK_DEQUANTIZE, OP_OBSERVE_QUANTIZE_BLOCK, OP_OBSERVE_QUANTIZE_MX) = range(15)

Q_INT, Q_FLOAT, Q_FP4 = 0, 1, 2
DT_E8M0 = 8  # uint8 MX scale exponent as stored (CT_E8M0)
DT_F64 = 9   # compute precision of ct_hadamard_transform (CT_F64)
# bytes per element of each ct_dtype_t a tensor can hold
DT_SIZE = {code: torch.empty((), dtype=dt).element_size() for dt, code in DT.items()} | {DT_E8M0: 1}


class QuantDesc(ctypes.Structure):
    """mirror of `struct ct_quant_desc` (include/ct_b200.h)"""

    _fields_ = [
        ("rows", ctypes.c_int64),
        ("cols", ctypes.c_int64),
        ("rdiv", ctypes.c_int64),
        ("cdiv", ctypes.c_int64),
        ("s_row_stride", ctypes.c_int64),
        ("x_dtype", ctypes.c_int32),
        ("scale_dtype", ctypes.c_int32),
        ("zp_dtype", ctypes.c_int32),
        ("compute_dtype", ctypes.c_int32),
        ("q_dtype", ctypes.c_int32),
        ("out_dtype", ctypes.c_int32),
        ("qtype", ctypes.c_int32),
        ("num_bits", ctypes.c_int32),
        ("global_scale", ctypes.c_void_p),
        ("seff_dtype", ctypes.c_int32),
        ("_reserved", ctypes.c_int32),
        ("aux", ctypes.c_void_p),
    ]


MSE_MAX_STEPS = 64


class MseBlock(ctypes.Structure):
    """mirror of `struct ct_mse_block` (include/ct_b200.h): the MSE observer's search, pointed to by ct_quant_desc.aux"""

    _fields_ = [
        ("shrink", ctypes.c_float * MSE_MAX_STEPS),
        ("steps", ctypes.c_int32),
        ("patience", ctypes.c_int32),
        ("norm", ctypes.c_float),
        ("_reserved", ctypes.c_int32),
        ("any", ctypes.c_uint64),
        ("masks", ctypes.c_void_p),
        ("errors", ctypes.c_void_p),
    ]


class HeadJob(ctypes.Structure):
    """mirror of `struct ct_head_job` (include/ct_b200.h)"""

    _fields_ = [
        ("x", ctypes.c_void_p),
        ("out", ctypes.c_void_p),
        ("scale", ctypes.c_void_p),
        ("zp", ctypes.c_void_p),
        ("shape", ctypes.c_int64 * 4),
        ("stride", ctypes.c_int64 * 4),
        ("per_head", ctypes.c_int32),
        ("x_dtype", ctypes.c_int32),
        ("scale_dtype", ctypes.c_int32),
        ("zp_dtype", ctypes.c_int32),
        ("qtype", ctypes.c_int32),
        ("num_bits", ctypes.c_int32),
    ]


class HadamardJob(ctypes.Structure):
    """mirror of `struct ct_hadamard_job` (include/ct_b200.h)"""

    _fields_ = [
        ("x", ctypes.c_void_p),
        ("out", ctypes.c_void_p),
        ("shape", ctypes.c_int64 * 4),
        ("stride", ctypes.c_int64 * 4),
        ("sign", ctypes.c_void_p),
        ("perm", ctypes.c_void_p),
        ("dtype", ctypes.c_int32),
        ("precision", ctypes.c_int32),
        ("log2_n", ctypes.c_int32),
        ("inverse", ctypes.c_int32),
        ("core", ctypes.c_void_p),
        ("core_order", ctypes.c_int32),
    ]


class NativeLibraryError(RuntimeError):
    pass


_lib: Optional[ctypes.CDLL] = None

_vp, _i64, _int = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int
_descp = ctypes.POINTER(QuantDesc)

_PROTOS = {
    "ct_version": (ctypes.c_char_p, []),
    "ct_last_error": (ctypes.c_char_p, []),
    "ct_device_count": (_int, []),
    "ct_device_ok": (_int, [_int]),
    "ct_launch_count": (_i64, []),
    "ct_pack_int32": (_int, [_vp, _vp, _i64, _i64, _int, _int, _int, _vp]),
    "ct_unpack_int32": (_int, [_vp, _vp, _i64, _i64, _int, _int, _int, _vp]),
    "ct_quantize": (_int, [_descp, _vp, _vp, _vp, _vp, _vp, _int, _vp]),
    "ct_dequantize": (_int, [_descp, _vp, _vp, _vp, _vp, _vp, _int, _vp]),
    "ct_fake_quantize": (_int, [_descp, _vp, _vp, _vp, _vp, _vp, _int, _vp]),
    "ct_fake_quantize_heads": (_int, [_int, ctypes.POINTER(HeadJob), _int, _vp]),
    "ct_hadamard_transform": (_int, [ctypes.POINTER(HadamardJob), _int, _vp]),
    "ct_quantize_pack_int32": (_int, [_descp, _vp, _vp, _vp, _vp, _vp, _int, _vp]),
    "ct_unpack_dequantize_int32": (_int, [_descp, _vp, _vp, _vp, _vp, _vp, _int, _vp]),
    "ct_observe_quantize_pack_int32": (_int, [_descp, _vp, _vp, _vp, _vp, _int, _vp]),
    "ct_cast_to_fp4": (_int, [_vp, _int, _vp, _i64, _int, _vp]),
    "ct_pack_fp4": (_int, [_vp, _int, _vp, _i64, _i64, _int, _vp]),
    "ct_unpack_fp4": (_int, [_vp, _vp, _int, _i64, _i64, _int, _vp]),
    "ct_quantize_pack_fp4": (_int, [_descp, _vp, _vp, _vp, _vp, _vp, _int, _vp]),
    "ct_unpack_dequantize_fp4": (_int, [_descp, _vp, _vp, _vp, _vp, _vp, _int, _vp]),
    "ct_observe_quantize_pack_nvfp4": (_int, [_descp, _vp, _vp, _vp, _int, _vp]),
    "ct_mx_scale_compress": (_int, [_vp, _int, _vp, _i64, _int, _vp]),
    "ct_mx_scale_decompress": (_int, [_vp, _vp, _i64, _int, _vp]),
    "ct_awq_repack_int4": (_int, [_vp, _vp, _i64, _i64, _int, _vp]),
    "ct_awq_repack_zeros_int4": (_int, [_vp, _vp, _i64, _i64, _int, _vp]),
    "ct_observe_quantize_channel": (_int, [_descp, _vp, _vp, _vp, _vp, _int, _vp]),
    "ct_observe_quantize_block": (_int, [_descp, _vp, _vp, _vp, _int, _vp]),
    "ct_observe_quantize_mx": (_int, [_descp, _vp, _vp, _vp, _int, _vp]),
    "ct_observe_tensor": (_int, [_descp, _vp, _int, _vp, _vp, _int, _vp]),
    "ct_observe_quantize_tensor": (_int, [_descp, _vp, _vp, _vp, _vp, _int, _vp]),
    "ct_dynamic_fake_quantize": (_int, [_descp, _int, _int, _vp, _vp, _vp, _vp, _int, _vp]),
    "ct_batched": (_int, [_int, _int, _descp, _vp, _vp, _vp, _vp, _int, _vp]),
    "ct_pack_bitmasks": (_int, [_vp, _vp, _i64, _i64, _int, _vp]),
    "ct_unpack_bitmasks": (_int, [_vp, _vp, _i64, _i64, _int, _vp]),
    "ct_sparse24_compress": (_int, [_vp, _int, _vp, _vp, _i64, _i64, _int, _vp]),
    "ct_sparse24_decompress": (_int, [_vp, _int, _vp, _vp, _i64, _i64, _int, _vp]),
    "ct_sparse24_quantize_pack_int4": (_int, [_descp, _vp, _vp, _vp, _vp, _vp, _int, _vp]),
    "ct_sparse24_unpack_dequantize_int4": (_int, [_descp, _vp, _vp, _vp, _vp, _vp, _int, _vp]),
    "ct_bitmask_workspace_bytes": (_i64, [_i64, _i64]),
    "ct_bitmask_count": (_int, [_vp, _int, _vp, _vp, _vp, _vp, _i64, _i64, _int, _vp]),
    "ct_bitmask_compress": (_int, [_vp, _int, _vp, _vp, _vp, _i64, _i64, _int, _vp]),
    "ct_bitmask_decompress": (_int, [_vp, _int, _vp, _vp, _vp, _i64, _i64, _int, _vp]),
    "ct_bitmask_compress_onepass": (_int, [_vp, _int, _vp, _vp, _vp, _vp, _i64, _i64, _int, _vp]),
    "ct_semi_structured_from_dense": (_int, [_vp, _int, _vp, _vp, _i64, _i64, _int, _vp]),
    "ct_semi_structured_to_dense": (_int, [_vp, _int, _vp, _vp, _i64, _i64, _int, _vp]),
    "ct_host_run_many": (_int, [_int, _int, _descp, _vp, _vp, _vp, _vp, _int]),
    "ct_selftest_division": (_int, [_int, ctypes.POINTER(ctypes.c_uint64), _int]),
    "ct_selftest_fp4_division": (_int, [_int, _int, _int, ctypes.POINTER(ctypes.c_uint64), _int]),
}

EXPORTED_SYMBOLS = tuple(_PROTOS)


def lib() -> ctypes.CDLL:
    """Load libct_b200.so (built in-tree by compressed_tensors_b200._build). Fails loudly."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise NativeLibraryError(
                f"{LIB_PATH} is missing: build it with `python -m compressed_tensors_b200._build` "
                "(or __graft_entry__.build()). compressed_tensors_b200 has no CPU / eager fallback."
            )
        cdll = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _PROTOS.items():
            fn = getattr(cdll, name)  # AttributeError if the ABI is incomplete
            fn.restype = res
            fn.argtypes = args
        _lib = cdll
    return _lib


def last_error() -> str:
    return lib().ct_last_error().decode()


def check(rc: int, what: str = "") -> None:
    """translate ct_status_t into the exceptions the reference raises for the same condition"""
    if rc == CT_OK:
        return
    msg = last_error()
    if rc in (CT_E_BITS, CT_E_SHAPE, CT_E_DTYPE, CT_E_ARG):
        raise ValueError(f"{what}: {msg}" if what else msg)
    if rc == CT_E_NODEV:
        raise NativeLibraryError(msg)
    if rc == CT_E_UNSUPPORTED:
        raise NotImplementedError(msg)
    raise RuntimeError(f"{what}: {msg} (status {rc})")


def require_device(device: Optional[torch.device] = None) -> int:
    """index of the CUDA device the work will run on; raises when there is none"""
    if not torch.cuda.is_available():
        raise NativeLibraryError(
            "compressed_tensors_b200 needs a CUDA device (sm_90a / H100); it has no CPU code path"
        )
    if device is None or device.type != "cuda":
        return torch.cuda.current_device()
    return device.index if device.index is not None else torch.cuda.current_device()


def stream_ptr(device_index: int) -> ctypes.c_void_p:
    return ctypes.c_void_p(torch.cuda.current_stream(device_index).cuda_stream)


def ptr(t: Optional[torch.Tensor]) -> ctypes.c_void_p:
    if t is None:
        return ctypes.c_void_p(0)
    return ctypes.c_void_p(t.data_ptr())


def launch_count() -> int:
    return int(lib().ct_launch_count())

