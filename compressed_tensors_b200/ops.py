"""
Tensor-level front end of the C ABI: torch tensors in, torch tensors out, same argument meaning
and error behaviour as the reference's per-tensor functions

    compressors/pack_quantized/helpers.py : pack_to_int32 (:20-101), unpack_from_int32 (:104-180)
    quantization/lifecycle/forward.py     : quantize (:36-73), dequantize (:76-145),
                                            fake_quantize (:148-181), _process_quantization (:184-241)
    utils/helpers.py                      : pack_bitmasks (:306-317), unpack_bitmasks (:320-343)

(paths under src/compressed_tensors of the reference).  Host logic only: shape / dtype / strategy
resolution and output allocation.  All arithmetic happens in libct_b200.so on a H100.

Device policy: CUDA tensors run on their device and the current stream.  CPU tensors are staged
through the current CUDA device (large 2-D tensors via the pipelined ct_host_run_many) and the result
is returned on the CPU, as the reference would.  With no CUDA device the call raises; there is
no eager / CPU fallback.  Meta tensors only get their output shape and dtype computed.
"""
from __future__ import annotations

import ctypes
import functools
import math
import threading
from typing import NamedTuple, Optional, Sequence, Tuple

import torch

from . import _native as N

__all__ = [
    "pack_to_int32",
    "unpack_from_int32",
    "quantize",
    "dequantize",
    "fake_quantize",
    "fake_quantize_heads",
    "dynamic_fake_quantize",
    "hadamard_transform",
    "quantize_pack",
    "unpack_dequantize",
    "pack_bitmasks",
    "unpack_bitmasks",
    "sparse24_compress",
    "sparse24_decompress",
    "bitmask_compress",
    "bitmask_decompress",
    "sparse24_quantize_pack",
    "sparse24_unpack_dequantize",
    "batched",
    "BatchedPlan",
    "cast_to_fp4",
    "pack_fp4_to_uint8",
    "unpack_fp4_from_uint8",
    "quantize_pack_fp4",
    "unpack_dequantize_fp4",
    "compress_mx_scale",
    "decompress_mx_scale",
    "observe_quantize",
    "observe_quantize_pack",
    "observe_quantize_pack_nvfp4",
    "observe_quantize_mx",
    "observe_tensor_qparams",
    "observe_tensor_gparam",
    "dequantize_block_fp8",
    "awq_repack",
    "awq_repack_zeros",
]

_FLOAT_DTYPES = (torch.float32, torch.float16, torch.bfloat16)
# tensors at least this large take the pipelined host path when they live on the CPU
_HOST_PIPELINE_MIN_BYTES = 8 << 20


# --------------------------------------------------------------------------------------------
# device staging
# --------------------------------------------------------------------------------------------
_CPU = -1              # CT_DEVICE_CPU: the explicit host twins of the seven per-tensor hot-path entry points and of ct_hadamard_transform (csrc/cpu_twin.cu)
_mode = threading.local()


def _dev_index(*tensors: Optional[torch.Tensor]) -> int:
    """where the call runs: a CUDA device index, or _CPU when the eager body was selected (ImplBackend: no usable CUDA device, or
    CT_ENFORCE_EAGER).  Never a silent fallback: the CUDA backend on a GPU-less host raises."""
    if getattr(_mode, "cpu", False):
        return _CPU
    for t in tensors:
        if t is not None and t.is_cuda:
            return N.require_device(t.device)
    return N.require_device(None)


def _to_dev(t: Optional[torch.Tensor], idx: int) -> Optional[torch.Tensor]:
    if t is None:
        return None
    if idx == _CPU:
        return t.detach().cpu().contiguous()
    if t.is_cuda:
        if t.device.index != idx:
            raise ValueError(f"tensors live on different CUDA devices ({t.device} vs cuda:{idx})")
        return t if t.is_contiguous() else t.contiguous()
    return t.contiguous().to(f"cuda:{idx}", non_blocking=True)


def _back(out: torch.Tensor, like: torch.Tensor) -> torch.Tensor:
    return out if like.device == out.device else out.to(like.device)


def _stream(idx: int):
    return None if idx == _CPU else N.stream_ptr(idx)


# --------------------------------------------------------------------------------------------
# pack / unpack
# --------------------------------------------------------------------------------------------
def pack_to_int32(value: torch.Tensor, num_bits: int, packed_dim: int = 1) -> torch.Tensor:
    """reference: compressors/pack_quantized/helpers.py:20-101 (same checks, same messages)"""
    if value.dtype is not torch.int8:
        raise ValueError("Tensor must be quantized to torch.int8 before packing")
    if not 1 <= num_bits <= 8:
        raise ValueError(f"Packing is only supported for num_bits in [1, 8], got {num_bits}")
    if value.ndim > 2:
        return torch.stack([pack_to_int32(value[i], num_bits, packed_dim) for i in range(value.shape[0])])
    if value.ndim != 2:
        raise ValueError(f"expected a 2-D (or stacked 3-D) tensor, got shape {tuple(value.shape)}")
    rows, cols = value.shape
    if packed_dim == 1:
        out_shape = (rows, math.ceil(cols * num_bits / 32))
    elif packed_dim == 0:
        out_shape = (math.ceil(rows * num_bits / 32), cols)
    else:
        raise ValueError(f"packed_dim must be 0 or 1, got {packed_dim}")
    if value.device.type == "meta":
        out = torch.empty(out_shape, dtype=torch.int32, device="meta")
        return out
    idx = _dev_index(value)
    v = _to_dev(value, idx)
    out = torch.empty(out_shape, dtype=torch.int32, device=v.device)
    rc = N.lib().ct_pack_int32(N.ptr(v), N.ptr(out), rows, cols, int(num_bits), int(packed_dim), idx, _stream(idx))
    N.check(rc, "pack_to_int32")
    out = _back(out, value)
    if packed_dim == 0:
        # the reference returns the transpose of a [cols, words] buffer (helpers.py:98-99); keep
        # that (non-contiguous) memory format so `.contiguous()` callers behave identically
        out = out.t().contiguous().t()
    return out


def unpack_from_int32(value: torch.Tensor, num_bits: int, shape: Sequence[int], packed_dim: int = 1) -> torch.Tensor:
    """reference: compressors/pack_quantized/helpers.py:104-180"""
    if value.dtype is not torch.int32:
        raise ValueError(f"Expected {torch.int32} but got {value.dtype}, Aborting unpack.")
    if not 1 <= num_bits <= 8:
        raise ValueError(f"Unpacking is only supported for num_bits in [1, 8], got {num_bits}")
    shape = tuple(int(s) for s in shape)
    if value.ndim > 2:
        return torch.stack([unpack_from_int32(value[i], num_bits, shape[1:], packed_dim) for i in range(value.shape[0])])
    if packed_dim not in (0, 1):
        raise ValueError(f"packed_dim must be 0 or 1, got {packed_dim}")
    if packed_dim == 1:
        rows, cols = value.shape[0], shape[1]
        need = math.ceil(cols * num_bits / 32)
        if value.shape[1] < need:
            raise ValueError(f"packed tensor has {value.shape[1]} words per row, {need} needed for {cols} columns")
        if value.shape[1] != need:
            value = value[:, :need]
    else:
        rows, cols = shape[0], value.shape[1]
        need = math.ceil(rows * num_bits / 32)
        if value.shape[0] < need:
            raise ValueError(f"packed tensor has {value.shape[0]} word rows, {need} needed for {rows} rows")
        if value.shape[0] != need:
            value = value[:need]
    if value.device.type == "meta":
        return torch.empty((rows, cols), dtype=torch.int8, device="meta")
    idx = _dev_index(value)
    v = _to_dev(value, idx)
    out = torch.empty((rows, cols), dtype=torch.int8, device=v.device)
    rc = N.lib().ct_unpack_int32(N.ptr(v), N.ptr(out), rows, cols, int(num_bits), int(packed_dim), idx, _stream(idx))
    N.check(rc, "unpack_from_int32")
    return _back(out, value)


# --------------------------------------------------------------------------------------------
# strategy resolution (host logic of forward.py:184-241 and forward_helpers.py:62-177)
# --------------------------------------------------------------------------------------------
def _strategy_name(args) -> str:
    s = getattr(args, "strategy", None)
    return getattr(s, "value", s)


def _type_name(args) -> str:
    t = getattr(args, "type", "int")
    return getattr(t, "value", t)


class _Problem:
    """resolved 2-D view of one quantization call"""

    __slots__ = ("rows", "cols", "rdiv", "cdiv", "srs", "scale", "zp", "g_idx", "strategy", "gs")


def _resolve(x: torch.Tensor, scale: torch.Tensor, zero_point: Optional[torch.Tensor], args, g_idx) -> _Problem:
    strategy = _strategy_name(args)
    p = _Problem()
    p.strategy = strategy
    p.g_idx = None
    p.gs = None
    cols = x.shape[-1] if x.ndim >= 1 else 1
    rows = x.numel() // max(cols, 1) if x.numel() else 0
    p.rows, p.cols = rows, cols

    if zero_point is not None and zero_point.shape != scale.shape:
        scale, zero_point = torch.broadcast_tensors(scale, zero_point)

    if strategy == "block":
        bs = getattr(args, "block_structure", None)
        if bs is None or x.ndim != 2:
            raise ValueError("block quantization needs a 2-D tensor and a block_structure")
        bh, bw = int(bs[0]), int(bs[1])
        nrb, ncb = math.ceil(rows / bh), math.ceil(cols / bw)
        if scale.numel() != nrb * ncb:
            raise ValueError(f"block scale has {scale.numel()} elements, expected {nrb}x{ncb}")
        p.rdiv, p.cdiv, p.srs = bh, bw, ncb
        p.scale, p.zp = scale.reshape(nrb, ncb), (zero_point.reshape(nrb, ncb) if zero_point is not None else None)
        return p

    if strategy in ("group", "tensor_group"):
        group_size = int(getattr(args, "group_size"))
        while scale.ndim < 2:  # forward_helpers.py:137-139
            scale = scale.unsqueeze(1)
            zero_point = zero_point.unsqueeze(1) if zero_point is not None else None
        if cols >= group_size and cols % group_size != 0:
            raise ValueError(
                "tensor column shape must be divisble " f"by the given group_size {group_size} but got {cols}"
            )
        ngroups = math.ceil(cols / group_size)
        if g_idx is not None and g_idx.device.type != "meta" and not bool((g_idx == -1).any()):
            p.g_idx = g_idx
        last = scale.shape[-1]
        if last not in (1, ngroups):
            raise ValueError(f"group scale has {last} columns, expected {ngroups}")
        cdiv = group_size if last == ngroups else N.INF
        p.g_idx = p.g_idx if last == ngroups else None
    else:
        # tensor / channel / token / attn_head: plain broadcasting of x / scale
        last = scale.shape[-1] if scale.ndim >= 1 else 1
        if last == 1:
            cdiv = N.INF
        elif last == cols:
            cdiv = 1
        else:
            raise ValueError(f"scale of shape {tuple(scale.shape)} does not broadcast against {tuple(x.shape)}")

    lead = scale.shape[:-1] if scale.ndim >= 1 else ()
    if all(int(d) == 1 for d in lead):
        # one row of scales shared by every row of x
        p.rdiv, p.cdiv, p.srs = (1 if cdiv != N.INF or last != 1 else N.INF), cdiv, 0
        if last == 1:
            p.rdiv, p.cdiv, p.srs = N.INF, N.INF, 0
        p.scale = scale.reshape(-1)
        p.zp = zero_point.reshape(-1) if zero_point is not None else None
    else:
        target = tuple(x.shape[:-1]) + (last,)
        try:
            sc = scale.expand(target)
            zp = zero_point.expand(target) if zero_point is not None else None
        except RuntimeError as e:
            raise ValueError(f"scale of shape {tuple(scale.shape)} does not broadcast against {tuple(x.shape)}") from e
        p.rdiv, p.cdiv, p.srs = 1, cdiv, last
        p.scale = sc.reshape(rows, last)
        p.zp = zp.reshape(rows, last) if zp is not None else None
    return p


def _qparams(args) -> Tuple[int, int]:
    qtype = N.Q_FLOAT if _type_name(args) == "float" else N.Q_INT
    bits = int(getattr(args, "num_bits", 8))
    if qtype == N.Q_FLOAT and bits == 4:
        return N.Q_FP4, 4   # FP4 E2M1 (quant_args.py:484-485)
    if qtype == N.Q_FLOAT and bits != 8:
        raise NotImplementedError("Only num_bits in (4, 8) are supported")
    if qtype == N.Q_INT and not 1 <= bits <= 8:
        raise NotImplementedError(f"integer quantization on this path supports 1..8 bits, got {bits}")
    return qtype, bits


def _check_float(t: torch.Tensor, what: str):
    if t.dtype not in _FLOAT_DTYPES:
        raise NotImplementedError(f"{what} dtype {t.dtype} is not supported by compressed_tensors_b200 (fp32/fp16/bf16 only)")


_DT_FIELDS = ("x_dtype", "scale_dtype", "zp_dtype", "compute_dtype", "q_dtype", "out_dtype", "seff_dtype")


def _qdesc(rows: int, cols: int, rdiv: int, cdiv: int, srs: int, qtype: int = N.Q_INT, num_bits: int = 0, global_scale=None,
           **dtypes) -> N.QuantDesc:
    """a descriptor in which every field the caller does not name is absent: CT_NONE dtypes, no global scale, no aux.
    dtypes: the `*_dtype` fields, each a torch dtype or a ct_dtype_t code"""
    d = N.QuantDesc(rows=rows, cols=cols, rdiv=rdiv, cdiv=cdiv, s_row_stride=srs, qtype=qtype, num_bits=num_bits,
                    global_scale=global_scale)
    for f in _DT_FIELDS:
        v = dtypes.pop(f, None)
        setattr(d, f, N.DT_NONE if v is None else v if isinstance(v, int) else N.DT[v])
    if dtypes:
        raise TypeError(f"unknown descriptor fields {sorted(dtypes)}")
    return d


def _desc(p: _Problem, x_dt, s_dt, zp_dt, cd, q_dt, out_dt, qtype, bits, se_dt=None) -> N.QuantDesc:
    """se_dt: dtype of scale / global_scale (or, for stored fp8 / E8M0 scales, the float dtype they decode to)"""
    def code(t):
        return N.DT.get(t, N.DT_NONE)

    return _qdesc(p.rows, p.cols, p.rdiv, p.cdiv, p.srs, qtype, bits, x_dtype=code(x_dt), scale_dtype=N.DT[s_dt], zp_dtype=zp_dt,
                  compute_dtype=code(cd), q_dtype=code(q_dt), out_dtype=code(out_dt), seff_dtype=code(se_dt))


class _Call(NamedTuple):
    """one descriptor-driven kernel call as a public function resolved it: the entry point and its batched op, the descriptor, the
    streamed input as 2-D, the resolved qparams (p: scale, zero point, g_idx and the global-scale tensor, kept alive here), and the
    output's shape and dtype.  The per-tensor functions run it (`_run`); the whole-model launches batch it."""
    fn: str
    op: int
    desc: N.QuantDesc
    src: torch.Tensor
    p: _Problem
    out_shape: tuple
    out_dtype: torch.dtype


def _call(fn: str, op: int, p: _Problem, gs, src, out_shape, out_dtype, x_dt, cd, q_dt, out_dt, qtype, bits, se=None) -> _Call:
    p.gs = gs
    d = _desc(p, x_dt, p.scale.dtype, p.zp.dtype if p.zp is not None else None, cd, q_dt, out_dt, qtype, bits, se)
    return _Call(fn, op, d, src, p, tuple(out_shape), out_dtype)


def _run(c: _Call) -> torch.Tensor:
    lib = N.lib()
    p, src, d = c.p, c.src, c.desc
    on_cpu = not src.is_cuda
    idx = _dev_index(src, p.scale)
    if (
        idx != _CPU
        and on_cpu
        and p.g_idx is None
        and p.gs is None
        and c.op not in (N.OP_QUANTIZE_PACK_FP4, N.OP_UNPACK_DEQUANTIZE_FP4)
        and src.numel() * src.element_size() >= _HOST_PIPELINE_MIN_BYTES
        and not p.scale.is_cuda
    ):
        # pipelined H2D / kernel / D2H on host buffers
        srcc = src.contiguous()
        zp = p.zp.contiguous() if p.zp is not None else None
        out = torch.empty(c.out_shape, dtype=c.out_dtype, pin_memory=srcc.is_pinned())
        host_batched(c.op, [(d, srcc, p.scale.contiguous(), zp, out)], idx)
        return out
    s_dev = _to_dev(src, idx)
    sc = _to_dev(p.scale, idx)
    zp = _to_dev(p.zp, idx)
    gi = _to_dev(p.g_idx.to(torch.int32) if p.g_idx is not None else None, idx)
    gs_dev = _to_dev(p.gs, idx)   # one float32 on the device, read by the kernel (kept alive until the call returns)
    d.global_scale = gs_dev.data_ptr() if gs_dev is not None else None
    out = torch.empty(c.out_shape, dtype=c.out_dtype, device=s_dev.device)
    rc = getattr(lib, c.fn)(ctypes.byref(d), N.ptr(s_dev), N.ptr(sc), N.ptr(zp), N.ptr(gi), N.ptr(out), idx, _stream(idx))
    N.check(rc, c.fn)
    return _back(out, src)


def _global_scale(scale, global_scale):
    """
    `scale = scale / global_scale` (forward_helpers.py:535-536, 559-560, 196-197).  A float32 global scale of one
    element held in a >= 1-D tensor (what generate_gparam returns) is handed to the kernels, which form the quotient
    per group in registers; any other form is divided here with torch, exactly like the reference.
    Returns (scale, gs tensor or None, dtype of the effective scale).
    """
    if global_scale is None:
        return scale, None, scale.dtype
    if global_scale.dtype == torch.float32 and global_scale.numel() == 1 and global_scale.ndim >= 1 and scale.dtype in _FLOAT_DTYPES:
        return scale, global_scale.reshape(1).contiguous(), torch.result_type(scale, global_scale)
    scale = scale / global_scale
    return scale, None, scale.dtype


def _like(scale, dtype):
    """a stand-in with the scale's dimensionality for torch.result_type (0-dim tensors promote differently)"""
    return torch.empty(scale.shape, dtype=dtype, device="meta")


# --------------------------------------------------------------------------------------------
# quantize / dequantize / fake_quantize
# --------------------------------------------------------------------------------------------
def _quant_prologue(x, scale, global_scale, args):
    """the checks every quantizing op runs first, in order; returns (scale, gs, effective scale dtype, qtype, bits, compute dtype)"""
    scale, gs, se = _global_scale(scale, global_scale)
    _check_float(x, "input")
    _check_float(scale, "scale")
    qtype, bits = _qparams(args)
    cd = torch.result_type(x, scale if gs is None else _like(scale, se))
    return scale, gs, se, qtype, bits, cd


def _out_dtype(args, group_dtype, other_dtype):
    """the dtype a (fake) quantized or dequantized tensor comes back in: `group_dtype` on the group paths, `other_dtype` on the
    others (the effective scale's dtype, or for quantize the compute dtype)"""
    return group_dtype if _strategy_name(args) in ("group", "tensor_group") else other_dtype


def _quantize_call(x, scale, zero_point, args, dtype=None, g_idx=None, global_scale=None) -> _Call:
    scale, gs, se, qtype, bits, cd = _quant_prologue(x, scale, global_scale, args)
    out_dtype = dtype if dtype is not None else _out_dtype(args, x.dtype, cd)  # forward_helpers.py:134,171
    p = _resolve(x, scale, zero_point, args, g_idx)
    if x.device.type != "meta" and x.numel() and out_dtype not in N.DT:   # meta and empty inputs run no kernel
        raise NotImplementedError(f"quantize(dtype={out_dtype}) is not supported")
    return _call("ct_quantize", N.OP_QUANTIZE, p, gs, x.reshape(p.rows, p.cols), (p.rows, p.cols), out_dtype,
                 x.dtype, cd, out_dtype, out_dtype, qtype, bits, se)


@torch.no_grad()
def quantize(x, scale, zero_point, args, dtype: Optional[torch.dtype] = None, g_idx=None, global_scale=None) -> torch.Tensor:
    """reference: quantization/lifecycle/forward.py:36-73"""
    c = _quantize_call(x, scale, zero_point, args, dtype, g_idx, global_scale)
    if x.device.type == "meta" or x.numel() == 0:
        return torch.empty(x.shape, dtype=c.out_dtype, device=x.device)
    return _run(c).reshape(x.shape)


def _infer_dequant_args(x_q: torch.Tensor, scale: torch.Tensor):
    """strategy inference of forward.py:99-130 when args is None"""
    from types import SimpleNamespace

    if scale.ndim in (0, 1):
        return SimpleNamespace(strategy="tensor", group_size=None, block_structure=None)
    if scale.ndim == 2:
        if scale.shape[1] == 1:
            return SimpleNamespace(strategy="channel", group_size=None, block_structure=None)
        if scale.shape[0] == 1 or scale.shape[0] == x_q.shape[0]:
            return SimpleNamespace(strategy="group", group_size=int(x_q.shape[1] / scale.shape[1]), block_structure=None)
        rows, cols = x_q.shape[-2], x_q.shape[-1]
        return SimpleNamespace(strategy="block", group_size=None,
                               block_structure=[rows // scale.shape[0], cols // scale.shape[1]])
    raise ValueError(
        f"Could not infer a quantization strategy from scale with {scale.ndim} "
        "dimmensions. Expected 0 or 2 dimmensions."
    )


def _dequantize_call(x_q, scale, zero_point=None, args=None, dtype=None, g_idx=None, global_scale=None) -> _Call:
    if args is None:
        args = _infer_dequant_args(x_q, scale)
    if dtype is None:
        dtype = scale.dtype
    scale, gs, se = _global_scale(scale, global_scale)
    _check_float(scale, "scale")
    # the dtype argument is honoured only on the group path (SURVEY Appendix B4); inferred block sizes may not cover the tensor
    # (forward.py:118-126): the reference pads x to the block multiple, so the scale grid must be exactly ceil-div sized (_resolve)
    out_dtype = _out_dtype(args, dtype, se)
    p = _resolve(x_q, scale, zero_point, args, g_idx)
    if x_q.device.type != "meta" and x_q.numel() and (x_q.dtype not in N.DT or out_dtype not in _FLOAT_DTYPES):
        raise NotImplementedError(f"dequantize from {x_q.dtype} to {out_dtype} is not supported")
    return _call("ct_dequantize", N.OP_DEQUANTIZE, p, gs, x_q.reshape(p.rows, p.cols), (p.rows, p.cols), out_dtype,
                 None, None, x_q.dtype, out_dtype, N.Q_INT, 8, se)


@torch.no_grad()
def dequantize(x_q, scale, zero_point=None, args=None, dtype: Optional[torch.dtype] = None, g_idx=None, global_scale=None) -> torch.Tensor:
    """reference: quantization/lifecycle/forward.py:76-145"""
    c = _dequantize_call(x_q, scale, zero_point, args, dtype, g_idx, global_scale)
    if x_q.device.type == "meta" or x_q.numel() == 0:
        return torch.empty(x_q.shape, dtype=c.out_dtype, device=x_q.device)
    return _run(c).reshape(x_q.shape)


def _fake_quantize_call(x, scale, zero_point, args, g_idx=None, global_scale=None) -> _Call:
    scale, gs, se, qtype, bits, cd = _quant_prologue(x, scale, global_scale, args)
    out_dtype = _out_dtype(args, x.dtype, se)
    p = _resolve(x, scale, zero_point, args, g_idx)
    return _call("ct_fake_quantize", N.OP_FAKE_QUANTIZE, p, gs, x.reshape(p.rows, p.cols), (p.rows, p.cols), out_dtype,
                 x.dtype, cd, None, out_dtype, qtype, bits, se)


@torch.no_grad()
def fake_quantize(x, scale, zero_point, args, g_idx=None, global_scale=None) -> torch.Tensor:
    """reference: quantization/lifecycle/forward.py:148-181"""
    c = _fake_quantize_call(x, scale, zero_point, args, g_idx, global_scale)
    if x.device.type == "meta" or x.numel() == 0:
        return torch.empty(x.shape, dtype=c.out_dtype, device=x.device)
    return _run(c).reshape(x.shape)


def _head_job(x: torch.Tensor, scale: torch.Tensor, zp: Optional[torch.Tensor], args, out: torch.Tensor):
    """(the ct_head_job of one [B, H, S, D] tensor, the flattened scale / zero point it points into), or None when the strided kernel
    cannot take the tensor (the library checks the layout).  Scale shapes: one element (TENSOR), or [H, 1, 1] / [1, H, 1, 1] with the
    ATTN_HEAD strategy -- the shapes `fake_quantize` broadcasts one scale per head; any other shape takes `fake_quantize`."""
    if x.ndim != 4 or not x.is_cuda or x.dtype not in _FLOAT_DTYPES or scale.dtype != x.dtype or out.stride() != x.stride():
        return None
    if scale.device != x.device or (zp is not None and (zp.device != x.device or zp.dtype not in (torch.int8, torch.float8_e4m3fn))):
        return None
    if zp is not None and zp.shape != scale.shape:
        return None
    heads = x.shape[1]
    if scale.numel() == 1:
        per_head = 0
    elif _strategy_name(args) == "attn_head" and tuple(scale.shape) in ((heads, 1, 1), (1, heads, 1, 1)):
        per_head = 1
    else:
        return None
    qtype, bits = _qparams(args)
    if qtype == N.Q_FP4:
        return None
    flat_scale = scale.reshape(-1).contiguous()
    flat_zp = zp.reshape(-1).contiguous() if zp is not None else None
    j = N.HeadJob()
    j.x, j.out, j.scale = x.data_ptr(), out.data_ptr(), flat_scale.data_ptr()
    j.zp = flat_zp.data_ptr() if flat_zp is not None else None
    j.shape[:] = list(x.shape)
    j.stride[:] = list(x.stride())
    j.per_head = per_head
    j.x_dtype = j.scale_dtype = N.DT[x.dtype]
    j.zp_dtype = N.DT[zp.dtype] if zp is not None else N.DT_NONE
    j.qtype, j.num_bits = qtype, bits
    return j, (flat_scale, flat_zp)


@torch.no_grad()
def fake_quantize_heads(tensors: Sequence[torch.Tensor], scales: Sequence[torch.Tensor], zero_points: Sequence[Optional[torch.Tensor]],
                        args) -> list:
    """
    fake_quantize of one or two attention states (key and value, or query) of shape [B, H, S, D] in one launch, where they lie:
    transformers hands them over as transposed, non-contiguous views, and this reads and writes them with their own strides
    (ct_fake_quantize_heads) instead of copying each one to a contiguous buffer first.  Scales are per tensor ([1], TENSOR) or
    per head ([H, 1, 1], ATTN_HEAD); the outputs are `torch.empty_like` their inputs and equal `fake_quantize` bit for bit.
    Inputs the strided kernel does not take (CPU tensors, other strategies, scale shapes or dtypes, D % 8 != 0, unaligned or
    non-dense rows) run through `fake_quantize` one by one, with the scales and zero points exactly as given.
    """
    tensors, scales, zero_points = list(tensors), list(scales), list(zero_points)
    if not 1 <= len(tensors) <= 2 or len(scales) != len(tensors) or len(zero_points) != len(tensors):
        raise ValueError("fake_quantize_heads takes one or two tensors, each with its scale and zero point (or None)")
    if any(x.device.type == "meta" for x in tensors) or all(x.numel() == 0 for x in tensors):
        return [fake_quantize(x, s, z, args) for x, s, z in zip(tensors, scales, zero_points)]
    strategy = _strategy_name(args)
    if strategy in ("tensor", "attn_head") and len({x.device for x in tensors}) == 1 and not getattr(_mode, "cpu", False):
        outs = [torch.empty_like(x) for x in tensors]
        jobs = [_head_job(x, s, z, args, o) for x, s, z, o in zip(tensors, scales, zero_points, outs)]
        if all(j is not None for j in jobs):
            idx = tensors[0].device.index
            table = (N.HeadJob * len(jobs))(*(j for j, _ in jobs))   # `jobs` keeps the flattened qparams alive until the launch
            rc = N.lib().ct_fake_quantize_heads(len(jobs), table, idx, N.stream_ptr(idx))
            if rc != N.CT_E_UNSUPPORTED:
                N.check(rc, "ct_fake_quantize_heads")
                return outs
    return [fake_quantize(x, s, z, args) for x, s, z in zip(tensors, scales, zero_points)]


# args.scale_dtype -> how the library rounds a fresh scale (CT_NONE: it stays in x's dtype)
_SCALE_ROUNDING = {None: N.DT_NONE, torch.float8_e4m3fn: N.DT[torch.float8_e4m3fn], torch.uint8: N.DT_E8M0}
_DYNAMIC_ZP_DTYPES = (torch.int8, torch.float8_e4m3fn, torch.uint8)


def _dynamic_layout(x: torch.Tensor, args):
    """(rows, cols, rdiv, cdiv, s_row_stride, scale shape) of compute_dynamic_scales_and_zp's reduction (utils/helpers.py:140-195),
    or None for a strategy or shape the fused kernel does not take.  TOKEN reduces over every dim after the first two, so a 1-D or
    2-D value reduces over the whole tensor, as the reference's aminmax does, and gets one scale."""
    strategy, cols = _strategy_name(args), x.shape[-1]
    if strategy == "token" and x.ndim > 2:
        rows = x.shape[0] * x.shape[1]
        return rows, x.numel() // rows, 1, N.INF, 1, tuple(x.shape[:2]) + (1,) * (x.ndim - 2)
    if strategy in ("token", "tensor"):
        return x.numel() // cols, cols, N.INF, N.INF, 0, (1,)
    if strategy in ("group", "tensor_group"):
        g = int(getattr(args, "group_size", 0) or 0)
        if g <= 0 or cols % g != 0:
            return None   # the reference's unflatten raises for a ragged last group: the two-step path raises it
        return x.numel() // cols, cols, 1, g, cols // g, tuple(x.shape[:-1]) + (cols // g,)
    return None


@torch.no_grad()
def dynamic_fake_quantize(x: torch.Tensor, args, global_scale: Optional[torch.Tensor] = None):
    """
    compute_dynamic_scales_and_zp (utils/helpers.py:140-195) followed by fake_quantize (forward.py:148-181) in one pass over x on
    its GPU (`ct_dynamic_fake_quantize`): returns (out, scale, zero_point), the scale and zero point with the shapes and dtypes the
    reference's compute_dynamic_scales_and_zp returns and `out` equal bit for bit to fake_quantize with them.
    Returns None when the kernel does not take the input -- a CPU, non-contiguous or fp32 tensor, a last dimension not divisible by
    8, a strategy, scheme or group size it does not cover -- and the caller then runs the two steps, which also raise whatever the
    reference raises for the input.
    """
    if not x.is_cuda or not x.is_contiguous() or x.dtype not in (torch.bfloat16, torch.float16) or x.ndim == 0 or x.numel() == 0:
        return None
    if x.shape[-1] % 8 != 0 or getattr(_mode, "cpu", False):
        return None
    try:
        qtype, bits = _qparams(args)
    except (NotImplementedError, ValueError):
        return None
    layout = _dynamic_layout(x, args)
    scale_dtype_arg = getattr(args, "scale_dtype", None)
    zp_dtype = getattr(args, "zp_dtype", None)
    if layout is None or scale_dtype_arg not in _SCALE_ROUNDING or zp_dtype not in _DYNAMIC_ZP_DTYPES:
        return None
    rows, cols, rdiv, cdiv, srs, scale_shape = layout
    gs = None
    scale_dtype = x.dtype
    if global_scale is not None:
        # `global_scale * scales` (helpers.py:93-94): a float32 [1] global scale promotes the scale to float32
        if global_scale.dtype != torch.float32 or global_scale.numel() != 1 or global_scale.ndim == 0 or global_scale.device != x.device:
            return None
        gs = global_scale.reshape(1).contiguous()
        scale_dtype = torch.float32
    se = scale_dtype   # the effective scale dtype and compute dtype fake_quantize derives from that scale (ops.fake_quantize)
    cd = torch.promote_types(x.dtype, se)
    out = torch.empty_like(x)
    scale = torch.empty(scale_shape, dtype=scale_dtype, device=x.device)
    zero_point = torch.empty(scale_shape, dtype=zp_dtype, device=x.device)
    d = _qdesc(rows, cols, rdiv, cdiv, srs, qtype, bits, gs.data_ptr() if gs is not None else None, x_dtype=x.dtype, out_dtype=x.dtype,
               scale_dtype=scale_dtype, zp_dtype=zp_dtype, compute_dtype=cd, seff_dtype=se)
    idx = x.get_device()
    rc = N.lib().ct_dynamic_fake_quantize(ctypes.byref(d), int(not args.symmetric), _SCALE_ROUNDING[scale_dtype_arg], N.ptr(x), N.ptr(out),
                                          N.ptr(scale), N.ptr(zero_point), idx, N.stream_ptr(idx))
    if rc == N.CT_E_UNSUPPORTED:
        return None
    N.check(rc, "ct_dynamic_fake_quantize")
    return out, scale, zero_point


# --------------------------------------------------------------------------------------------
# Walsh-Hadamard transforms (transform/factory/hadamard.py, HadamardTransform.forward)
# --------------------------------------------------------------------------------------------
HADAMARD_MAX_ORDER = 1 << 15
HADAMARD_MAX_CORE = 256


def _hadamard_job(x: torch.Tensor, out: torch.Tensor, log2_n: int, sign, perm, inverse: bool, precision, core=None) -> N.HadamardJob:
    j = N.HadamardJob()
    j.x, j.out = x.data_ptr(), out.data_ptr()
    j.shape[:] = list(x.shape)
    j.stride[:] = list(x.stride())
    j.sign = sign.data_ptr() if sign is not None else None
    j.perm = perm.data_ptr() if perm is not None else None
    j.dtype = N.DT[x.dtype]
    j.precision = N.DT_F64 if precision == torch.float64 else N.DT[torch.float32]
    j.log2_n, j.inverse = log2_n, int(bool(inverse))
    if core is not None:
        j.core, j.core_order = core.data_ptr(), core.size(0)
    return j


def _verified_permutation(perm: torch.Tensor, n: int) -> torch.Tensor:
    """perm must be a permutation of 0 .. n-1: the kernel scatters and gathers shared memory through it.  Returns an int64 copy made
    when the values were checked, and the kernel reads only that copy.  The check runs once per version and storage of the tensor:
    callers that pass the same tensor every call (HadamardTransform) pay for one check.  A write through `perm.data` changes neither,
    as torch does not track it, so it is not seen; the copy keeps such a write from reaching the kernel unchecked."""
    if perm.dtype not in (torch.int64, torch.int32) or perm.ndim != 1 or perm.numel() != n:
        raise ValueError(f"perm must be a 1-D integer permutation of {n} indices, got shape {tuple(perm.shape)} and dtype {perm.dtype}")
    if perm.device.type == "meta":
        return perm
    key = (perm._version, perm.data_ptr())
    cached = getattr(perm, "_ct_checked_permutation", None)
    if cached is not None and cached[0] == key:
        return cached[1]
    if not torch.equal(torch.sort(perm).values, torch.arange(n, device=perm.device, dtype=perm.dtype)):
        raise ValueError(f"perm is not a permutation of 0 .. {n - 1}")
    checked = perm.detach().to(torch.int64, copy=True).contiguous()
    perm._ct_checked_permutation = (key, checked)
    return checked


def _verified_core(core: torch.Tensor, n: int) -> torch.Tensor:
    """core must be a K x K matrix of +-1 values with n = K * 2^m.  Returns an int8 copy made when it was checked, once per version
    and storage of the tensor, as _verified_permutation does for perm."""
    if core.ndim != 2 or core.size(0) != core.size(1) or core.size(0) < 1 or core.size(0) > HADAMARD_MAX_CORE:
        raise ValueError(f"core must be a square matrix of order 1 .. {HADAMARD_MAX_CORE}, got shape {tuple(core.shape)}")
    k = core.size(0)
    if n % k or (n // k) & (n // k - 1):
        raise ValueError(f"the order {n} is not {k} * 2^m for the core of order {k}")
    if core.device.type == "meta":
        return core
    key = (core._version, core.data_ptr())
    cached = getattr(core, "_ct_checked_core", None)
    if cached is not None and cached[0] == key:
        return cached[1]
    if core.is_complex() or core.dtype == torch.bool or not bool(((core == 1) | (core == -1)).all()):
        raise ValueError("core must hold +-1 values only")
    checked = core.detach().to(torch.int8, copy=True).contiguous()
    core._ct_checked_core = (key, checked)
    return checked


@torch.no_grad()
def hadamard_transform(x: torch.Tensor, n: int, sign: Optional[torch.Tensor] = None, perm: Optional[torch.Tensor] = None,
                       inverse: bool = False, precision: torch.dtype = torch.float32, core: Optional[torch.Tensor] = None) -> torch.Tensor:
    """
    `(x.to(precision) @ M / sqrt(n)).to(x.dtype)` along the last dimension, block-diagonal over its n-element blocks, for the structured
    matrices of the `hadamard` / `random-hadamard` factories: M = H (Sylvester), with rows and columns permuted by `perm` (a permutation
    of 0 .. n-1) and / or rows signed by `sign` (n values, negative -> -1, else +1: diag(sign) . H); `inverse` applies M^T.  A `sign`
    or `perm` of another length, or a `perm` that is not a permutation, raises ValueError.  `perm` is checked once per version of the
    tensor and the kernel uses the copy made at that check, so a write through `perm.data` (untracked by torch) is not seen until the
    tensor's next tracked write.  An O(n log n) butterfly
    (ct_hadamard_transform) instead of the dense product; precision fp32 or fp64.  The output has x's strides when x is dense (the
    transposed [B, H, S, D] attention states included), so no contiguous copy is made in or out.

    `core` (a K x K tensor of +-1 values, int8 or float) replaces H by (C ⊗ H_{2^m})^T for n = K * 2^m, the matrices the reference's
    random_hadamard_matrix builds for orders that are not powers of two: the butterflies run on each 2^m slice and the K slices are
    mixed with C (K additions per element).  A core that is not square, not +-1 or whose order K does not give n = K * 2^m raises
    ValueError; it is checked once per version of the tensor, like `perm`.
    """
    n = int(n)
    if core is not None:
        if n > HADAMARD_MAX_ORDER:
            raise NotImplementedError(f"hadamard_transform covers orders up to {HADAMARD_MAX_ORDER}, got {n}")
        core = _verified_core(core, n)
    else:
        if n <= 0 or n & (n - 1):
            raise ValueError("Cannot construct deterministic hadamard of size != 2^n")
        if n > HADAMARD_MAX_ORDER or n < 2:
            raise NotImplementedError(f"hadamard_transform covers orders 2 .. {HADAMARD_MAX_ORDER}, got {n}")
    _check_float(x, "input")
    if precision not in (torch.float32, torch.float64):
        raise NotImplementedError(f"hadamard_transform computes in float32 or float64, got {precision}")
    if x.ndim == 0 or x.shape[-1] % n:
        raise ValueError(f"{n} must divide the last dimension of a tensor of shape {tuple(x.shape)}")
    if sign is not None and (sign.numel() != n or sign.dtype not in (torch.int8, torch.float32, torch.float64, torch.float16, torch.bfloat16)):
        raise ValueError(f"sign must hold {n} signs, got {sign.numel()} of dtype {sign.dtype}")
    if perm is not None:
        perm = _verified_permutation(perm, n)
    if x.device.type == "meta" or x.numel() == 0:
        return torch.empty_like(x)
    idx = _dev_index(x)
    src = x
    if idx == _CPU or not x.is_cuda:
        src = _to_dev(x, idx)
    if src.ndim > 4:
        src = src.reshape(-1, *src.shape[-3:])
    v = src.view((1,) * (4 - src.ndim) + tuple(src.shape)) if src.ndim < 4 else src
    out = torch.empty_like(v)
    if out.stride() != v.stride():          # not dense (a slice): the output cannot keep the input's strides
        v = v.contiguous()
        out = torch.empty_like(v)
    sg = _to_dev(torch.where(sign < 0, -1, 1).to(torch.int8) if sign is not None and sign.dtype != torch.int8 else sign, idx)
    pm = _to_dev(perm, idx)
    cr = _to_dev(core, idx)
    log2_n = (n // core.size(0) if core is not None else n).bit_length() - 1
    rc = N.lib().ct_hadamard_transform(ctypes.byref(_hadamard_job(v, out, log2_n, sg, pm, inverse, precision, cr)), idx, _stream(idx))
    if rc == N.CT_E_UNSUPPORTED and not v.is_contiguous():
        v = v.contiguous()
        out = torch.empty_like(v)
        rc = N.lib().ct_hadamard_transform(ctypes.byref(_hadamard_job(v, out, log2_n, sg, pm, inverse, precision, cr)), idx, _stream(idx))
    N.check(rc, "hadamard_transform")
    return _back(out.view(x.shape), x)


# --------------------------------------------------------------------------------------------
# fused compressor bodies
# --------------------------------------------------------------------------------------------
@torch.no_grad()
def quantize_pack(x, scale, zero_point, args, g_idx=None, global_scale=None) -> torch.Tensor:
    """quantize(dtype=int8) -> pack_to_int32 in one pass (pack_quantized/base.py:96-104).
    x: [..., R, C] float; returns int32 [..., R, ceil(C*bits/32)]"""
    if x.ndim > 2:
        # N-D weights (MoE experts) pack slice by slice (helpers.py:44-51); scales follow the leading dim
        outs = []
        for i in range(x.shape[0]):
            sc = scale[i] if scale.ndim == x.ndim else scale
            zp = zero_point[i] if (zero_point is not None and zero_point.ndim == x.ndim) else zero_point
            outs.append(quantize_pack(x[i], sc, zp, args, g_idx, global_scale))
        return torch.stack(outs)
    c = _quantize_pack_call(x, scale, zero_point, args, g_idx, global_scale)
    if x.device.type == "meta":
        return torch.empty(c.out_shape, dtype=torch.int32, device="meta")
    return _run(c)


def _quantize_pack_call(x, scale, zero_point, args, g_idx=None, global_scale=None) -> _Call:
    scale, gs, se, qtype, bits, cd = _quant_prologue(x, scale, global_scale, args)
    if qtype != N.Q_INT:
        raise ValueError("pack-quantized compression needs integer quantization")
    p = _resolve(x, scale, zero_point, args, g_idx)
    return _call("ct_quantize_pack_int32", N.OP_QUANTIZE_PACK, p, gs, x.reshape(p.rows, p.cols), (p.rows, math.ceil(p.cols * bits / 32)),
                 torch.int32, x.dtype, cd, torch.int8, None, qtype, bits, se)


@torch.no_grad()
def unpack_dequantize(packed, scale, zero_point, num_bits: int, shape: Sequence[int], g_idx=None,
                      dtype: Optional[torch.dtype] = None) -> torch.Tensor:
    """unpack_from_int32 -> dequantize(args=None) in one pass (pack_quantized/base.py:159-166);
    the strategy is inferred from the scale shape exactly like forward.py:99-130."""
    shape = tuple(int(s) for s in shape)
    if packed.ndim > 2:
        _check_words(packed, num_bits)
        outs = []
        for i in range(packed.shape[0]):
            sc = scale[i] if scale.ndim == packed.ndim else scale
            zp = zero_point[i] if (zero_point is not None and zero_point.ndim == packed.ndim) else zero_point
            outs.append(unpack_dequantize(packed[i], sc, zp, num_bits, shape[1:], g_idx, dtype))
        return torch.stack(outs)
    c = _unpack_dequantize_call(packed, scale, zero_point, num_bits, shape, g_idx, dtype)
    if packed.device.type == "meta":
        return torch.empty(shape, dtype=c.out_dtype, device="meta")
    return _run(c)


def _check_words(packed, num_bits: int):
    if packed.dtype is not torch.int32:
        raise ValueError(f"Expected {torch.int32} but got {packed.dtype}, Aborting unpack.")
    if not 1 <= num_bits <= 8:
        raise ValueError(f"Unpacking is only supported for num_bits in [1, 8], got {num_bits}")


def _unpack_dequantize_call(packed, scale, zero_point, num_bits: int, shape, g_idx=None, dtype=None) -> _Call:
    """packed: 2-D; words past the last one `shape` needs are not read"""
    _check_words(packed, num_bits)
    _check_float(scale, "scale")
    like = torch.empty(shape, dtype=torch.int8, device="meta")
    args = _infer_dequant_args(like, scale)
    out_dtype = _out_dtype(args, dtype if dtype is not None else scale.dtype, scale.dtype)
    p = _resolve(like, scale, zero_point, args, g_idx)
    need = math.ceil(p.cols * num_bits / 32)
    if packed.shape[-1] < need:
        raise ValueError(f"packed tensor has {packed.shape[-1]} words per row, {need} needed")
    if packed.shape[-1] != need:
        packed = packed[:, :need]
    return _call("ct_unpack_dequantize_int32", N.OP_UNPACK_DEQUANTIZE, p, None, packed, shape, out_dtype,
                 None, None, torch.int8, out_dtype, N.Q_INT, int(num_bits))


# --------------------------------------------------------------------------------------------
# FP4 (E2M1) and MX formats
# --------------------------------------------------------------------------------------------
def _simple(fn_name: str, src: torch.Tensor, out_shape, out_dtype, call) -> torch.Tensor:
    """one elementwise FP4 / MX kernel on `src` (CPU tensors are staged through the GPU)"""
    if src.device.type == "meta":
        return torch.empty(out_shape, dtype=out_dtype, device="meta")
    idx = _dev_index(src)
    s_dev = _to_dev(src.contiguous(), idx)
    out = torch.empty(out_shape, dtype=out_dtype, device=s_dev.device)
    N.check(call(N.lib(), s_dev, out, idx), fn_name)
    return out.cpu() if not src.is_cuda else out


@torch.no_grad()
def cast_to_fp4(x: torch.Tensor) -> torch.Tensor:
    """reference: quantization/utils/fp4_utils.py:77-98 (returns a new tensor; the reference writes in place on a temporary)"""
    _check_float(x, "input")
    return _simple("ct_cast_to_fp4", x, x.shape, x.dtype,
                   lambda lib, a, o, i: lib.ct_cast_to_fp4(N.ptr(a), N.DT[a.dtype], N.ptr(o), a.numel(), i, N.stream_ptr(i)))


@torch.no_grad()
def pack_fp4_to_uint8(x: torch.Tensor) -> torch.Tensor:
    """reference: compressors/nvfp4/helpers.py:108-158"""
    m, n = x.shape
    if n % 2 != 0:
        raise ValueError("tensor must have an even number of columns for nvfp4 compression")
    _check_float(x, "input")
    return _simple("ct_pack_fp4", x, (m, n // 2), torch.uint8,
                   lambda lib, a, o, i: lib.ct_pack_fp4(N.ptr(a), N.DT[a.dtype], N.ptr(o), m, n, i, N.stream_ptr(i)))


@torch.no_grad()
def unpack_fp4_from_uint8(a: torch.Tensor, m: int, n: int, dtype: Optional[torch.dtype] = torch.bfloat16) -> torch.Tensor:
    """reference: compressors/nvfp4/helpers.py:162-193"""
    assert a.dtype == torch.uint8
    if dtype not in _FLOAT_DTYPES:
        raise NotImplementedError(f"unpack_fp4_from_uint8 to {dtype} is not supported")
    if a.numel() * 2 != m * n or n % 2 != 0:
        raise ValueError(f"{a.numel()} packed bytes do not hold a [{m}, {n}] fp4 tensor")
    return _simple("ct_unpack_fp4", a, (m, n), dtype,
                   lambda lib, t, o, i: lib.ct_unpack_fp4(N.ptr(t), N.ptr(o), N.DT[dtype], m, n, i, N.stream_ptr(i)))


@torch.no_grad()
def compress_mx_scale(scale: torch.Tensor, scale_dtype: torch.dtype = torch.uint8) -> torch.Tensor:
    """reference: compressors/mx_utils.py:18-31 (E8M0: 127 + floor(log2(scale)))"""
    _check_float(scale, "scale")
    out = _simple("ct_mx_scale_compress", scale, scale.shape, torch.uint8,
                  lambda lib, a, o, i: lib.ct_mx_scale_compress(N.ptr(a), N.DT[a.dtype], N.ptr(o), a.numel(), i, N.stream_ptr(i)))
    return out.to(scale_dtype)


@torch.no_grad()
def decompress_mx_scale(scale: torch.Tensor) -> torch.Tensor:
    """reference: compressors/mx_utils.py:34-44 (uint8 exponent -> bfloat16 power of two)"""
    if scale.dtype != torch.uint8:
        scale = scale.to(torch.uint8)
    return _simple("ct_mx_scale_decompress", scale, scale.shape, torch.bfloat16,
                   lambda lib, a, o, i: lib.ct_mx_scale_decompress(N.ptr(a), N.ptr(o), a.numel(), i, N.stream_ptr(i)))


@torch.no_grad()
def quantize_pack_fp4(x, scale, zero_point, args, g_idx=None, global_scale=None) -> torch.Tensor:
    """quantize(FP4 args) -> pack_fp4_to_uint8 in one pass (compressors/nvfp4/base.py:82-90): x [R, C] float ->
    uint8 [R, C/2].  NVFP4: group 16 + global_scale; MXFP4: group 32, power-of-two scales."""
    c = _quantize_pack_fp4_call(x, scale, zero_point, args, g_idx, global_scale)
    if x.device.type == "meta":
        return torch.empty(c.out_shape, dtype=torch.uint8, device="meta")
    return _run(c)


def _quantize_pack_fp4_call(x, scale, zero_point, args, g_idx=None, global_scale=None) -> _Call:
    if x.ndim != 2:
        raise ValueError("fp4 packing needs a 2-D weight")
    if x.shape[1] % 2 != 0:
        raise ValueError("tensor must have an even number of columns for nvfp4 compression")
    scale, gs, se, qtype, bits, cd = _quant_prologue(x, scale, global_scale, args)
    if qtype != N.Q_FP4:
        raise ValueError("fp4 packing needs FLOAT quantization with num_bits == 4")
    p = _resolve(x, scale, zero_point, args, g_idx)
    return _call("ct_quantize_pack_fp4", N.OP_QUANTIZE_PACK_FP4, p, gs, x.reshape(p.rows, p.cols), (p.rows, p.cols // 2), torch.uint8,
                 x.dtype, cd, x.dtype, None, qtype, bits, se)


@torch.no_grad()
def unpack_dequantize_fp4(packed, scale, global_scale=None, dtype: torch.dtype = torch.bfloat16, stored_scale: Optional[str] = None) -> torch.Tensor:
    """
    unpack_fp4_from_uint8 -> dequantize in one pass (compressors/nvfp4/base.py:111-128): uint8 [R, C/2] -> `dtype` [R, C].
    `scale` is either the float scale the reference hands to dequantize (scale.to(dtype)), or the STORED scale:
    stored_scale="fp8" (float8_e4m3fn, NVFP4) / "e8m0" (uint8 exponents, MX), decoded in registers to `dtype`
    exactly like _decompress_scale does.
    """
    c = _unpack_dequantize_fp4_call(packed, scale, global_scale, dtype, stored_scale)
    if packed.device.type == "meta":
        return torch.empty(c.out_shape, dtype=c.out_dtype, device="meta")
    return _run(c)


def _unpack_dequantize_fp4_call(packed, scale, global_scale=None, dtype: torch.dtype = torch.bfloat16, stored_scale=None) -> _Call:
    if packed.dtype != torch.uint8 or packed.ndim != 2:
        raise ValueError("packed fp4 weights are 2-D uint8")
    if dtype not in _FLOAT_DTYPES:
        raise NotImplementedError(f"unpack_dequantize_fp4 to {dtype} is not supported")
    m, n = packed.shape[0], packed.shape[1] * 2
    if stored_scale is None:
        _check_float(scale, "scale")
        s_code, base_dt = None, scale.dtype
    elif stored_scale == "fp8":
        if scale.dtype != torch.float8_e4m3fn:
            raise ValueError("stored NVFP4 scales are float8_e4m3fn")
        s_code, base_dt = N.DT[torch.float8_e4m3fn], dtype
    elif stored_scale == "e8m0":
        if scale.dtype != torch.uint8:
            raise ValueError("stored MX scales are uint8 exponents")
        s_code, base_dt = N.DT_E8M0, dtype
    else:
        raise ValueError(f"unknown stored_scale {stored_scale!r}")
    if global_scale is not None:
        if not (global_scale.dtype == torch.float32 and global_scale.numel() == 1 and global_scale.ndim >= 1):
            raise NotImplementedError("global_scale must be a float32 tensor of shape [1]")
        gs, se = global_scale.reshape(1).contiguous(), torch.result_type(_like(scale, base_dt), global_scale)
    else:
        gs, se = None, base_dt
    like = torch.empty((m, n), dtype=torch.int8, device="meta")
    args = _infer_dequant_args(like, scale)
    out_dtype = _out_dtype(args, dtype, se)
    p = _resolve(like, scale, None, args, None)
    c = _call("ct_unpack_dequantize_fp4", N.OP_UNPACK_DEQUANTIZE_FP4, p, gs, packed, (m, n), out_dtype, None, None, None, out_dtype,
              N.Q_FP4, 4, se)
    c.desc.scale_dtype = s_code if s_code is not None else N.DT[scale.dtype]
    return c


# --------------------------------------------------------------------------------------------
# checkpoint-format conversions (entrypoints/convert)
# --------------------------------------------------------------------------------------------
@torch.no_grad()
def dequantize_block_fp8(weight: torch.Tensor, scale_inv: torch.Tensor, block_size: Sequence[int], dtype: torch.dtype = torch.bfloat16) -> torch.Tensor:
    """(weight.to(float32) * scale_inv.to(float32) per block).to(dtype): entrypoints/convert/converters/fp8block_dequantizer.py:111-158.
    weight float8_e4m3fn [R, C], scale_inv [ceil(R/bh), ceil(C/bw)]; one kernel, no padded copy."""
    c = _dequantize_block_fp8_call(weight, scale_inv, block_size, dtype)
    if weight.device.type == "meta" or weight.numel() == 0:
        return torch.empty(weight.shape, dtype=dtype, device=weight.device)
    return _run(c)


def _dequantize_block_fp8_call(weight, scale_inv, block_size, dtype=torch.bfloat16) -> _Call:
    from types import SimpleNamespace

    if weight.ndim != 2 or weight.dtype != torch.float8_e4m3fn:
        raise ValueError("fp8 block dequantization needs a 2-D float8_e4m3fn weight")
    if dtype not in _FLOAT_DTYPES:
        raise NotImplementedError(f"dequantize_block_fp8 to {dtype} is not supported")
    scale = scale_inv.to(torch.float32)   # qparam-sized; float32 already in the checkpoints this converter targets
    args = SimpleNamespace(strategy="block", group_size=None, block_structure=[int(block_size[0]), int(block_size[1])])
    p = _resolve(weight, scale, None, args, None)
    # the block dequantization of `dequantize`, but in the requested dtype, which `dequantize` honours on the group path only
    return _call("ct_dequantize", N.OP_DEQUANTIZE, p, None, weight, weight.shape, dtype, None, None, weight.dtype, dtype, N.Q_INT, 8,
                 torch.float32)


def _awq(fn_name: str, src: torch.Tensor, out_shape, rows: int, n_out: int) -> torch.Tensor:
    if src.dtype != torch.int32 or src.ndim != 2:
        raise ValueError("AutoAWQ tensors are 2-D int32")
    return _simple(fn_name, src, out_shape, torch.int32,
                   lambda lib, a, o, i: getattr(lib, fn_name)(N.ptr(a), N.ptr(o), rows, n_out, i, N.stream_ptr(i)))


@torch.no_grad()
def awq_repack(qweight: torch.Tensor) -> torch.Tensor:
    """AutoAWQ GEMM qweight int32 [K, N/8] -> compressed-tensors weight_packed int32 [N, ceil(K/8)]
    (entrypoints/convert/converters/autoawq.py:120-126 with :179-262, one kernel)"""
    k, nw = qweight.shape
    return _awq("ct_awq_repack_int4", qweight, (nw * 8, (k + 7) // 8), k, nw * 8)


@torch.no_grad()
def awq_repack_zeros(qzeros: torch.Tensor) -> torch.Tensor:
    """AutoAWQ qzeros int32 [G, N/8] -> weight_zero_point int32 [N/8, G] (packed along dim 0, contiguous; autoawq.py:124-128)"""
    g, nw = qzeros.shape
    return _awq("ct_awq_repack_zeros_int4", qzeros, (nw, g), g, nw * 8)


def _tensor_observer_ok(xd: torch.Tensor) -> bool:
    return xd.dtype in _FLOAT_DTYPES and xd.is_contiguous() and xd.numel() > 0 and (xd.numel() * xd.element_size()) % 16 == 0 and xd.data_ptr() % 16 == 0


def _tensor_desc(xd: torch.Tensor, qtype: int, bits: int, q_dt=None, asym: bool = False) -> N.QuantDesc:
    cols = xd.shape[-1] if xd.ndim >= 1 else 1
    return _qdesc(xd.numel() // max(cols, 1), cols, N.INF, N.INF, 0, qtype, bits, x_dtype=xd.dtype, scale_dtype=xd.dtype,
                  compute_dtype=xd.dtype, zp_dtype=torch.int8 if asym else None, q_dtype=q_dt)


@torch.no_grad()
def observe_tensor_qparams(x: torch.Tensor, args) -> Tuple[torch.Tensor, Optional[torch.Tensor]]:
    """memoryless min-max observer + calculate_qparams (utils/helpers.py:50-137) for the TENSOR strategy, entirely on the device
    (`ct_observe_tensor`, kind 0): returns (scale [1] in x.dtype, zero point int8 [1] or None for symmetric schemes), both device
    tensors -- nothing is read back.  Raises NotImplementedError for what the kernel declines (callers fall back to torch reductions)."""
    qtype, bits = _qparams(args)
    symmetric = bool(getattr(args, "symmetric", True))
    idx = _dev_index(x)
    xd = _to_dev(x, idx)
    if not _tensor_observer_ok(xd) or qtype == N.Q_FP4 or (qtype == N.Q_FLOAT and not symmetric):
        raise NotImplementedError("per-tensor observer kernel: contiguous 16-byte aligned float tensor, int or symmetric fp8 scheme")
    scale = torch.empty((1,), dtype=x.dtype, device=xd.device)
    zp = None if symmetric else torch.empty((1,), dtype=torch.int8, device=xd.device)
    d = _tensor_desc(xd, qtype, bits, asym=not symmetric)
    N.check(N.lib().ct_observe_tensor(ctypes.byref(d), N.ptr(xd), 0, N.ptr(scale), N.ptr(zp), idx, N.stream_ptr(idx)), "observe_tensor_qparams")
    return scale, zp


@torch.no_grad()
def observe_tensor_gparam(x: torch.Tensor) -> torch.Tensor:
    """generate_gparam(x.min(), x.max()) (utils/helpers.py:308-337) on the device: the float32 [1] global scale of NVFP4"""
    idx = _dev_index(x)
    xd = _to_dev(x, idx)
    if not _tensor_observer_ok(xd):
        raise NotImplementedError("per-tensor observer kernel: contiguous 16-byte aligned float tensor")
    g = torch.empty((1,), dtype=torch.float32, device=xd.device)
    d = _tensor_desc(xd, N.Q_FP4, 4)
    N.check(N.lib().ct_observe_tensor(ctypes.byref(d), N.ptr(xd), 1, N.ptr(g), None, idx, N.stream_ptr(idx)), "observe_tensor_gparam")
    return g


# --------------------------------------------------------------------------------------------
# MSE weight observer: a shrink-grid search over each group's min / max (observer "mse" / "memoryless_mse")
# --------------------------------------------------------------------------------------------
_MSE_OBSERVERS = ("mse", "memoryless_mse")
_MSE_DEFAULTS = {"maxshrink": 0.20, "grid": 100.0, "patience": 5, "norm": 2.4}
_FLT_MAX = float(torch.finfo(torch.float32).max)


class _Mse(NamedTuple):
    steps: int
    patience: int
    norm: float
    shrink: tuple   # p_i = float32(1 - i / grid), i < steps


def _mse_params(args) -> Optional[_Mse]:
    """the search of an MSE observer from args.observer_kwargs, or None for every other observer"""
    if getattr(args, "observer", None) not in _MSE_OBSERVERS:
        return None
    kw = dict(getattr(args, "observer_kwargs", None) or {})
    unknown = sorted(set(kw) - set(_MSE_DEFAULTS))
    if unknown:
        raise ValueError(f"unknown MSE observer_kwargs {unknown}; expected a subset of {sorted(_MSE_DEFAULTS)}")
    p = {**_MSE_DEFAULTS, **kw}
    grid, maxshrink, norm = float(p["grid"]), float(p["maxshrink"]), float(p["norm"])
    steps = int(maxshrink * grid) if math.isfinite(maxshrink * grid) else 0
    if not 1 <= steps <= N.MSE_MAX_STEPS:
        raise ValueError(f"MSE observer: int(maxshrink * grid) = {steps} steps, expected 1..{N.MSE_MAX_STEPS}")
    patience = p["patience"]
    if isinstance(patience, bool) or not isinstance(patience, (int, float)) or patience != int(patience) or patience < 1:
        raise ValueError(f"MSE observer: patience must be an integer >= 1, got {patience!r}")
    patience = int(patience)
    if not math.isfinite(norm) or norm <= 0:
        raise ValueError(f"MSE observer: norm must be finite and > 0, got {p['norm']}")
    shrink = tuple(float(v) for v in torch.tensor([1 - i / grid for i in range(steps)], dtype=torch.float64).float())
    return _Mse(steps, patience, norm, shrink)


def _mse_choose(errors: torch.Tensor, mse: _Mse) -> Tuple[torch.Tensor, int]:
    """the search rule on an error table [n_groups, steps]: (chosen step of every group, stop step S).  Step i improves a group when
    its error is below min(FLT_MAX, every earlier error); S is the first step that ends `patience` steps in which no group of the
    weight improved (steps - 1 if none); a group takes its last improving step <= S, or 0"""
    e = errors.float().cpu()
    best = torch.full((e.shape[0],), _FLT_MAX)
    improved = torch.zeros(e.shape, dtype=torch.bool)
    for i in range(mse.steps):
        improved[:, i] = e[:, i] < best
        best = torch.where(improved[:, i], e[:, i], best)
    stop, run = mse.steps - 1, 0
    for i, a in enumerate(improved.any(0).tolist()):
        run = 0 if a else run + 1
        if run >= mse.patience:
            stop = i
            break
    idx = torch.arange(stop + 1)
    chosen = torch.where(improved[:, :stop + 1], idx, -1).amax(1).clamp(min=0) if e.shape[0] else torch.zeros(0, dtype=torch.int64)
    return chosen, stop


def _mse_record(errors: torch.Tensor) -> None:
    tables = getattr(_mode, "mse_tables", None)
    if tables is not None:
        tables.append(errors.float().cpu())


class _mse_error_tables:
    """test hook: every MSE search run inside the `with` appends its per-group error table [n_groups, steps] (float32, on the CPU) to
    the yielded list, the kernel's own errors included"""

    def __enter__(self) -> list:
        self.prev = getattr(_mode, "mse_tables", None)
        _mode.mse_tables = []
        return _mode.mse_tables

    def __exit__(self, *exc):
        _mode.mse_tables = self.prev


def _mse_aux(mse: _Mse, n_groups: int, device: torch.device):
    """the device block of an MSE descriptor (ct_mse_block) and the buffers it points to; keep the tuple alive over the call"""
    masks = torch.empty((n_groups,), dtype=torch.int64, device=device)
    errors = torch.empty((n_groups, mse.steps), dtype=torch.float32, device=device) if getattr(_mode, "mse_tables", None) is not None else None
    b = N.MseBlock(steps=mse.steps, patience=mse.patience, norm=mse.norm, any=0, masks=masks.data_ptr(),
                   errors=errors.data_ptr() if errors is not None else None)
    b.shrink[:mse.steps] = list(mse.shrink)
    blk = torch.frombuffer(bytearray(bytes(b)), dtype=torch.uint8).to(device)
    return blk, masks, errors


def _observe_mse(xd: torch.Tensor, args, mse: _Mse, kind: str, qdt=None, global_scale=None):
    """the MSE observer with torch ops on xd's device (any strategy, dtype or device): every candidate's qparams
    (calculate_qparams of the shrunk min / max), its fake-quantized weight and the per-group sum of |fq - x|^norm in float32, then
    the search rule and the min-max path's own output ops at each group's chosen candidate.
      kind "codes" / "pack": (codes or packed words, scale, zero point or None)   "nvfp4": (packed, fp8 scale, global scale)
      kind "mx": (codes or nibbles, E8M0 scale)"""
    from .quantization.utils.helpers import calculate_qparams

    strategy = _strategy_name(args)
    rows, cols = xd.shape
    if strategy in ("group", "tensor_group"):
        g = int(getattr(args, "group_size"))
        xr = xd.unflatten(-1, (-1, g))
        mn, mx = xr.amin(-1), xr.amax(-1)

        def gsum(e):
            return e.unflatten(-1, (-1, g)).sum(-1)
    elif strategy == "channel":
        mn, mx = xd.amin(-1, keepdim=True), xd.amax(-1, keepdim=True)

        def gsum(e):
            return e.sum(-1, keepdim=True)
    elif strategy == "tensor":
        mn, mx = (t.reshape(1) for t in torch.aminmax(xd))

        def gsum(e):
            return e.sum().reshape(1)
    elif strategy == "block":
        bs = getattr(args, "block_structure", None)
        if bs is None or len(bs) != 2:
            raise ValueError("block quantization needs a block_structure [rows, cols]")
        bh, bw = int(bs[0]), int(bs[1])
        nrb, ncb = -(-rows // bh), -(-cols // bw)

        def blocks(t):   # zero padding is neutral for min / max (the rule clamps min <= 0 <= max) and for the error sums
            return torch.nn.functional.pad(t, (0, ncb * bw - cols, 0, nrb * bh - rows)).reshape(nrb, bh, ncb, bw)
        mn, mx = blocks(xd).amin(dim=(1, 3)), blocks(xd).amax(dim=(1, 3))

        def gsum(e):
            return blocks(e).sum(dim=(1, 3))
    else:
        raise NotImplementedError(f"the MSE observer does not support strategy {strategy}")
    symmetric = bool(getattr(args, "symmetric", True))
    xf = xd.float()
    if kind == "nvfp4" and getattr(args, "scale_dtype", None) is None:
        # NVFP4 stores its group scales as float8_e4m3fn: every candidate is judged with the scale it would be stored with
        args = args.model_copy(update={"scale_dtype": torch.float8_e4m3fn})

    def qparams(p):   # calculate_qparams of min / max shrunk by p (torch's tensor * python float: float32 product, rounded to x's dtype)
        scale, zp = calculate_qparams((mn.float() * p).to(mn.dtype), (mx.float() * p).to(mx.dtype), args, global_scale=global_scale)
        return scale, (None if symmetric else zp)

    table = []
    for p in mse.shrink:
        scale, zp = qparams(p)
        d = (fake_quantize(xd, scale, zp, args, global_scale=global_scale).float() - xf).abs()
        table.append(gsum(d * d if mse.norm == 2.0 else d.pow(mse.norm)).reshape(-1))
    errors = torch.stack(table, 1)
    _mse_record(errors)
    chosen, _ = _mse_choose(errors, mse)
    p = torch.tensor(mse.shrink, dtype=torch.float32)[chosen].reshape(mn.shape).to(xd.device)
    scale, zp = qparams(p)
    if kind == "nvfp4":
        return quantize_pack_fp4(xd, scale, None, args, global_scale=global_scale), scale.to(torch.float8_e4m3fn), global_scale
    if kind == "mx":
        out = quantize_pack_fp4(xd, scale, None, args) if int(args.num_bits) == 4 else quantize(xd, scale, None, args, dtype=torch.float8_e4m3fn)
        return out, compress_mx_scale(scale, torch.uint8)
    out = quantize_pack(xd, scale, zp, args) if kind == "pack" else quantize(xd, scale, zp, args, dtype=qdt)
    return out, scale, zp


def _back_all(outs, x):
    return tuple(_back(t, x) if t is not None else None for t in outs)


@torch.no_grad()
def observe_quantize_pack(x: torch.Tensor, args) -> Tuple[torch.Tensor, torch.Tensor, Optional[torch.Tensor]]:
    """Memoryless min-max observer + quantize + pack in ONE pass over the weight (SURVEY 8(f) rank 1):
    returns (weight_packed int32, weight_scale in x.dtype [R, C/G], weight_zero_point int8 [R, C/G] or None).

    Equivalent to the reference flow  min/max per group -> calculate_qparams (utils/helpers.py:50-137)
    -> quantize(dtype=int8) -> pack_to_int32, bit for bit.  The fused kernel covers group quantization of
    bf16 / fp16 weights with group_size in {32, 64, 128, 256} and 4- or 8-bit codes; every other case runs
    the same three steps as separate GPU ops."""
    qtype, bits = _qparams(args)
    strategy = _strategy_name(args)
    symmetric = bool(getattr(args, "symmetric", True))
    if x.ndim != 2:
        raise ValueError("observe_quantize_pack expects a 2-D weight")
    rows, cols = x.shape
    idx = _dev_index(x)
    xd = _to_dev(x, idx)
    group = int(getattr(args, "group_size", 0) or 0)
    fused_ok = (qtype == N.Q_INT and strategy == "group" and group in (32, 64, 128, 256) and cols % group == 0
                and x.dtype in (torch.bfloat16, torch.float16) and bits in (4, 8) and (cols * bits) % 32 == 0
                and (rows * cols) % 32 == 0)
    mse = _mse_params(args) if x.numel() > 0 else None
    if fused_ok and (mse is None or idx != _CPU):
        ng = cols // group
        scale = torch.empty((rows, ng), dtype=x.dtype, device=xd.device)
        zp = None if symmetric else torch.empty((rows, ng), dtype=torch.int8, device=xd.device)
        packed = torch.empty((rows, cols * bits // 32), dtype=torch.int32, device=xd.device)
        d = _qdesc(rows, cols, 1, group, ng, qtype, bits, x_dtype=x.dtype, scale_dtype=x.dtype, compute_dtype=x.dtype,
                   zp_dtype=None if symmetric else torch.int8, q_dtype=torch.int8)
        aux = None
        if mse is not None:
            aux = _mse_aux(mse, rows * ng, xd.device)
            d.aux = aux[0].data_ptr()
        rc = N.lib().ct_observe_quantize_pack_int32(ctypes.byref(d), N.ptr(xd), N.ptr(scale), N.ptr(zp), N.ptr(packed), idx, N.stream_ptr(idx))
        if not (mse is not None and rc == N.CT_E_UNSUPPORTED):   # an MSE search the kernel declines runs with torch ops below
            N.check(rc, "observe_quantize_pack")
            if aux is not None and aux[2] is not None:
                _mse_record(aux[2])
            return _back(packed, x), _back(scale, x), (_back(zp, x) if zp is not None else None)
    if mse is not None:
        return _back_all(_observe_mse(xd, args, mse, "pack"), x)
    return _observe_unfused("observe_quantize_pack", x, xd, args, group, True, torch.int32)


def _observe_unfused(who: str, x, xd, args, group: int, pack: bool, qdt):
    """the observer with torch reductions on the device (min / max per group, channel or tensor -> calculate_qparams), then the
    quantize (pack: quantize + pack) kernel; returns (codes, scale, zero point or None) where x lives"""
    from .quantization.utils.helpers import calculate_qparams

    strategy = _strategy_name(args)
    if strategy == "group":
        xr = xd.unflatten(-1, (-1, group))
        mn, mx = xr.amin(-1), xr.amax(-1)
    elif strategy == "channel":
        mn, mx = xd.amin(-1, keepdim=True), xd.amax(-1, keepdim=True)
    elif strategy == "tensor":
        mn, mx = (t.reshape(1) for t in torch.aminmax(xd))
    else:
        raise NotImplementedError(f"{who} does not support strategy {strategy}")
    scale, zp = calculate_qparams(mn, mx, args)
    zp = None if bool(getattr(args, "symmetric", True)) else zp
    out = quantize_pack(xd, scale, zp, args) if pack else quantize(xd, scale, zp, args, dtype=qdt)
    return _back(out, x), _back(scale, x), (_back(zp, x) if zp is not None else None)


@torch.no_grad()
def observe_quantize_pack_nvfp4(x: torch.Tensor, args, global_scale: Optional[torch.Tensor] = None) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """NVFP4 "calibrate + compress" of one weight: returns (weight_packed uint8 [R, C/2], weight_scale float8_e4m3fn [R, C/16],
    weight_global_scale float32 [1]) -- what the reference produces with
        global_scale = generate_gparam(w.min(), w.max())                                   (utils/helpers.py:308-337)
        scale, _     = calculate_qparams(group min, group max, args, global_scale)         (utils/helpers.py:50-137)
        NVFP4PackedCompressor.compress({"weight", "weight_scale", "weight_global_scale"})  (compressors/nvfp4/base.py:73-93)
    The global scale needs the whole tensor first (one torch min/max reduction unless it is given); everything per group --
    max |x|, the fp8 scale, quantize, nibble packing -- is ONE more pass (`ct_observe_quantize_pack_nvfp4`): the weight is read twice
    instead of three times and neither the float scale tensor nor the unpacked fp4 values ever exist."""
    from .quantization.utils.helpers import calculate_qparams, generate_gparam

    qtype, bits = _qparams(args)
    group = int(getattr(args, "group_size", 0) or 0)
    if qtype != N.Q_FP4 or _strategy_name(args) != "tensor_group" or group != 16:
        raise ValueError("observe_quantize_pack_nvfp4 needs NVFP4 args (float, 4 bits, tensor_group, group_size 16)")
    if x.ndim != 2:
        raise ValueError("observe_quantize_pack_nvfp4 expects a 2-D weight")
    rows, cols = x.shape
    idx = _dev_index(x)
    xd = _to_dev(x, idx).contiguous()
    if global_scale is not None:
        gs = _to_dev(global_scale, idx)
    elif _tensor_observer_ok(xd):
        gs = observe_tensor_gparam(xd)                       # grid-wide max |x| -> generate_gparam on the device, no torch reduction
    else:
        gs = generate_gparam(xd.min(), xd.max())
    gs = gs.reshape(1).to(torch.float32).contiguous()
    mse = _mse_params(args) if x.numel() > 0 else None
    if x.dtype in (torch.bfloat16, torch.float16) and cols % 32 == 0 and rows > 0 and (mse is None or idx != _CPU):
        scale = torch.empty((rows, cols // 16), dtype=torch.float8_e4m3fn, device=xd.device)
        packed = torch.empty((rows, cols // 2), dtype=torch.uint8, device=xd.device)
        d = _nvfp4_observe_desc(rows, cols, x.dtype, gs.data_ptr())
        aux = _mse_aux(mse, rows * cols // 16, xd.device) if mse is not None else None
        if aux is not None:
            d.aux = aux[0].data_ptr()
        rc = N.lib().ct_observe_quantize_pack_nvfp4(ctypes.byref(d), N.ptr(xd), N.ptr(scale), N.ptr(packed), idx, N.stream_ptr(idx))
        if not (mse is not None and rc == N.CT_E_UNSUPPORTED):   # an MSE search the kernel declines runs with torch ops below
            N.check(rc, "observe_quantize_pack_nvfp4")
            if aux is not None and aux[2] is not None:
                _mse_record(aux[2])
            return _back(packed, x), _back(scale, x), _back(gs, x)
    if mse is not None:
        return _back_all(_observe_mse(xd, args, mse, "nvfp4", global_scale=gs), x)
    g = xd.unflatten(-1, (-1, 16))
    scale, _ = calculate_qparams(g.amin(-1), g.amax(-1), args, global_scale=gs)
    packed = quantize_pack_fp4(xd, scale, None, args, global_scale=gs)
    return _back(packed, x), _back(scale.to(torch.float8_e4m3fn), x), _back(gs, x)


def _nvfp4_observe_desc(rows: int, cols: int, x_dtype: torch.dtype, global_scale) -> N.QuantDesc:
    """descriptor of `ct_observe_quantize_pack_nvfp4` / batched op OP_OBSERVE_QUANTIZE_PACK_FP4: float8_e4m3fn scales written per
    group of 16, a float32 global scale at `global_scale`"""
    return _qdesc(rows, cols, 1, 16, cols // 16, N.Q_FP4, 4, global_scale, x_dtype=x_dtype, scale_dtype=torch.float8_e4m3fn,
                  compute_dtype=torch.float32, q_dtype=x_dtype, seff_dtype=torch.float32)


def _block_desc(rows: int, cols: int, bh: int, bw: int, x_dtype: torch.dtype) -> N.QuantDesc:
    """descriptor of `ct_observe_quantize_block` / batched op OP_OBSERVE_QUANTIZE_BLOCK for an fp8 weight [rows, cols] in blocks [bh, bw]"""
    return _qdesc(rows, cols, bh, bw, -(-cols // bw), N.Q_FLOAT, 8, x_dtype=x_dtype, scale_dtype=x_dtype, compute_dtype=x_dtype,
                  q_dtype=torch.float8_e4m3fn)


def _mx_desc(rows: int, cols: int, bits: int, x_dtype: torch.dtype) -> N.QuantDesc:
    """descriptor of `ct_observe_quantize_mx` / batched op OP_OBSERVE_QUANTIZE_MX: MXFP4 (bits 4) or MXFP8 (bits 8), groups of 32"""
    qtype, bits, q_dt = (N.Q_FP4, 4, torch.uint8) if bits == 4 else (N.Q_FLOAT, 8, torch.float8_e4m3fn)
    return _qdesc(rows, cols, 1, 32, cols // 32, qtype, bits, x_dtype=x_dtype, compute_dtype=x_dtype, scale_dtype=N.DT_E8M0, q_dtype=q_dt)


def _aligned(*tensors: torch.Tensor) -> bool:
    return all(t.data_ptr() % 16 == 0 for t in tensors)


def _observe_quantize_block(x: torch.Tensor, args, qtype: int, bits: int, symmetric: bool):
    """observe_quantize for the BLOCK strategy: the fused kernel for symmetric fp8 codes of bf16 / fp16 weights whose rows and block
    width are a multiple of 8 elements; otherwise torch block min / max -> calculate_qparams -> quantize, with identical results"""
    from .quantization.utils.helpers import calculate_qparams

    bs = getattr(args, "block_structure", None)
    if bs is None or len(bs) != 2:
        raise ValueError("block quantization needs a block_structure [rows, cols]")
    bh, bw = int(bs[0]), int(bs[1])
    rows, cols = x.shape
    nrb, ncb = -(-rows // bh), -(-cols // bw)
    qdt = torch.float8_e4m3fn if qtype == N.Q_FLOAT else torch.int8
    if x.device.type == "meta":
        zp = None if symmetric else torch.empty((nrb, ncb), dtype=qdt if qtype == N.Q_FLOAT else torch.int8, device="meta")
        return (torch.empty((rows, cols), dtype=qdt, device="meta"), torch.empty((nrb, ncb), dtype=x.dtype, device="meta"), zp)
    idx = _dev_index(x)
    xd = _to_dev(x, idx).contiguous()
    mse = _mse_params(args) if x.numel() > 0 else None
    if mse is not None:
        return _back_all(_observe_mse(xd, args, mse, "codes", qdt), x)
    if (idx != _CPU and qtype == N.Q_FLOAT and bits == 8 and symmetric and x.dtype in (torch.bfloat16, torch.float16)
            and cols % 8 == 0 and bw % 8 == 0 and rows * cols > 0 and _aligned(xd)):
        scale = torch.empty((nrb, ncb), dtype=x.dtype, device=xd.device)
        out = torch.empty((rows, cols), dtype=qdt, device=xd.device)
        d = _block_desc(rows, cols, bh, bw, x.dtype)
        rc = N.lib().ct_observe_quantize_block(ctypes.byref(d), N.ptr(xd), N.ptr(scale), N.ptr(out), idx, N.stream_ptr(idx))
        N.check(rc, "observe_quantize")
        return _back(out, x), _back(scale, x), None
    # unfused: min / max per block over the elements that exist (zero padding is neutral: the rule clamps min <= 0 <= max)
    xp = torch.nn.functional.pad(xd, (0, ncb * bw - cols, 0, nrb * bh - rows)).reshape(nrb, bh, ncb, bw)
    scale, zp = calculate_qparams(xp.amin(dim=(1, 3)), xp.amax(dim=(1, 3)), args)
    zp = None if symmetric else zp
    out = quantize(xd, scale, zp, args, dtype=qdt)
    return _back(out, x), _back(scale, x), (_back(zp, x) if zp is not None else None)


def _is_mx(args) -> bool:
    return (_type_name(args) == "float" and int(getattr(args, "num_bits", 0)) in (4, 8) and _strategy_name(args) == "group"
            and int(getattr(args, "group_size", 0) or 0) == 32 and getattr(args, "scale_dtype", None) == torch.uint8)


@torch.no_grad()
def observe_quantize_mx(x: torch.Tensor, args) -> Tuple[torch.Tensor, torch.Tensor]:
    """MXFP4 / MXFP8 "calibrate + compress" of one weight x [R, C] (bf16 / fp16): returns the compressor's tensors
        MXFP4: (weight_packed uint8 [R, C/2], weight_scale uint8 [R, C/32])
        MXFP8: (weight float8_e4m3fn [R, C],   weight_scale uint8 [R, C/32])
    -- what the reference produces with
        scale, _ = calculate_qparams(group min, group max, args)     (utils/helpers.py:50-137: generate_mx_scales and
                                                                      maybe_convert_from_mx_exp, quantization/utils/mxfp_utils.py)
        MXFP4PackedCompressor.compress / MXFP8QuantizationCompressor.compress({"weight", "weight_scale"})
                                                                     (quantize, pack_fp4_to_uint8 for MXFP4, compress_mx_scale)
    bit for bit, in ONE pass over the weight (`ct_observe_quantize_mx`): max |x| per group of 32, the power-of-two scale, its E8M0
    exponent and the codes come out of registers.  Weights the kernel does not take (fp32, C % 32 != 0, no CUDA device) run the same
    steps unfused: torch min / max per group, calculate_qparams, quantize(_pack_fp4), compress_mx_scale."""
    from .quantization.utils.helpers import calculate_qparams

    if not _is_mx(args):
        raise ValueError("observe_quantize_mx needs MX args (float, 4 or 8 bits, group, group_size 32, scale_dtype uint8)")
    if not bool(getattr(args, "symmetric", True)):
        raise NotImplementedError("MX formats are symmetric")
    if x.ndim != 2:
        raise ValueError("observe_quantize_mx expects a 2-D weight")
    bits = int(args.num_bits)
    rows, cols = x.shape
    if cols % 32 != 0:
        raise ValueError(f"tensor column shape must be divisble by the given group_size 32 but got {cols}")
    q_shape, q_dt = ((rows, cols // 2), torch.uint8) if bits == 4 else ((rows, cols), torch.float8_e4m3fn)
    if x.device.type == "meta":
        return torch.empty(q_shape, dtype=q_dt, device="meta"), torch.empty((rows, cols // 32), dtype=torch.uint8, device="meta")
    idx = _dev_index(x)
    xd = _to_dev(x, idx).contiguous()
    mse = _mse_params(args) if x.numel() > 0 else None
    if mse is not None:
        return _back_all(_observe_mse(xd, args, mse, "mx"), x)
    if idx != _CPU and x.dtype in (torch.bfloat16, torch.float16) and rows * cols > 0 and _aligned(xd):
        scale = torch.empty((rows, cols // 32), dtype=torch.uint8, device=xd.device)
        out = torch.empty(q_shape, dtype=q_dt, device=xd.device)
        d = _mx_desc(rows, cols, bits, x.dtype)
        rc = N.lib().ct_observe_quantize_mx(ctypes.byref(d), N.ptr(xd), N.ptr(scale), N.ptr(out), idx, N.stream_ptr(idx))
        N.check(rc, "observe_quantize_mx")
        return _back(out, x), _back(scale, x)
    g = xd.unflatten(-1, (-1, 32))
    scale, _ = calculate_qparams(g.amin(-1), g.amax(-1), args)
    out = quantize_pack_fp4(xd, scale, None, args) if bits == 4 else quantize(xd, scale, None, args, dtype=torch.float8_e4m3fn)
    return _back(out, x), _back(compress_mx_scale(scale, torch.uint8), x)


@torch.no_grad()
def observe_quantize(x: torch.Tensor, args, pack: bool = False) -> Tuple[torch.Tensor, torch.Tensor, Optional[torch.Tensor]]:
    """Memoryless min-max observer + quantize (+ pack_to_int32 when `pack`) in ONE pass over the weight, for the strategies with a
    fused kernel; returns (codes or packed words, scale, zero point or None) exactly as the reference's
    min/max -> calculate_qparams (utils/helpers.py:50-137) -> quantize(dtype=args.pytorch_dtype()) [-> pack_to_int32] flow does.

      CHANNEL (one scale per row): bf16 / fp16, cols % 8 == 0 -> `ct_observe_quantize_channel` (int8 codes, float8_e4m3fn codes,
                                   or 4- / 8-bit packed int32); one CTA per row up to 16384 columns, one thread-block cluster per row
                                   up to 131072; wider rows are declined by the kernel and take the unfused path below
      TENSOR (one scale)         : `ct_observe_quantize_tensor` -- grid-wide min / max, calculate_qparams by the last CTA, then the
                                   streaming quantize kernel with the device-resident scale; no host round trip (the FP8 preset)
      GROUP + pack               : `observe_quantize_pack`
      BLOCK (FP8_BLOCK)          : `ct_observe_quantize_block` -- one CTA per block: min / max, calculate_qparams, fp8 codes; returns
                                   (float8_e4m3fn [R, C], scale in x.dtype [ceil(R / bh), ceil(C / bw)], None)
    Everything else runs the observer with torch reductions on the device and then the quantize kernel.
    args.observer "mse" / "memoryless_mse" runs the MSE shrink-grid search instead: fused into the GROUP + pack kernel and the per-row
    CHANNEL kernel (rows up to 16384 columns), torch ops on the device (`_observe_mse`) for everything else."""
    qtype, bits = _qparams(args)
    strategy = _strategy_name(args)
    symmetric = bool(getattr(args, "symmetric", True))
    if x.ndim != 2:
        raise ValueError("observe_quantize expects a 2-D weight")
    if pack and qtype != N.Q_INT:
        raise ValueError("pack-quantized compression needs integer quantization")
    if strategy == "group" and pack:
        return observe_quantize_pack(x, args)
    if strategy == "block" and not pack:
        return _observe_quantize_block(x, args, qtype, bits, symmetric)
    rows, cols = x.shape
    idx = _dev_index(x)
    xd = _to_dev(x, idx).contiguous()
    qdt = torch.int32 if pack else (torch.float8_e4m3fn if qtype == N.Q_FLOAT else torch.int8)
    mse = _mse_params(args) if x.numel() > 0 else None
    fused_ok = (strategy == "channel" and x.dtype in (torch.bfloat16, torch.float16) and cols % 8 == 0 and cols > 0 and rows > 0
                and qtype in (N.Q_INT, N.Q_FLOAT) and (bits in (4, 8) if pack else bits == 8) and (symmetric or qtype == N.Q_INT))
    if fused_ok and (mse is None or idx != _CPU):
        scale = torch.empty((rows, 1), dtype=x.dtype, device=xd.device)
        zp = None if symmetric else torch.empty((rows, 1), dtype=torch.int8, device=xd.device)
        out = torch.empty((rows, cols * bits // 32) if pack else (rows, cols), dtype=qdt, device=xd.device)
        d = _qdesc(rows, cols, 1, N.INF, 1, qtype, bits, x_dtype=x.dtype, scale_dtype=x.dtype, compute_dtype=x.dtype,
                   zp_dtype=None if symmetric else torch.int8, q_dtype=qdt)
        aux = _mse_aux(mse, rows, xd.device) if mse is not None else None
        if aux is not None:
            d.aux = aux[0].data_ptr()
        rc = N.lib().ct_observe_quantize_channel(ctypes.byref(d), N.ptr(xd), N.ptr(scale), N.ptr(zp), N.ptr(out), idx, N.stream_ptr(idx))
        if rc != N.CT_E_UNSUPPORTED:   # declined (a row wider than the kernel holds): the unfused path below
            N.check(rc, "observe_quantize")
            if aux is not None and aux[2] is not None:
                _mse_record(aux[2])
            return _back(out, x), _back(scale, x), (_back(zp, x) if zp is not None else None)
    if mse is not None:
        return _back_all(_observe_mse(xd, args, mse, "pack" if pack else "codes", qdt), x)
    if (strategy == "tensor" and _tensor_observer_ok(xd) and qtype in (N.Q_INT, N.Q_FLOAT) and (symmetric or qtype == N.Q_INT)
            and (bits in (4, 8) if pack else bits == 8) and (not pack or (cols * bits) % 32 == 0)):
        # ONE call: grid-wide min / max -> calculate_qparams on the device -> quantize (or quantize + pack) with the device-resident scale
        scale = torch.empty((1,), dtype=x.dtype, device=xd.device)
        zp = None if symmetric else torch.empty((1,), dtype=torch.int8, device=xd.device)
        out = torch.empty((rows, cols * bits // 32) if pack else (rows, cols), dtype=qdt, device=xd.device)
        d = _tensor_desc(xd, qtype, bits, q_dt=qdt, asym=not symmetric)
        rc = N.lib().ct_observe_quantize_tensor(ctypes.byref(d), N.ptr(xd), N.ptr(scale), N.ptr(zp), N.ptr(out), idx, N.stream_ptr(idx))
        N.check(rc, "observe_quantize")
        return _back(out, x), _back(scale, x), (_back(zp, x) if zp is not None else None)
    group = int(getattr(args, "group_size")) if strategy == "group" else 0
    return _observe_unfused("observe_quantize", x, xd, args, group, pack, qdt)


# --------------------------------------------------------------------------------------------
# multi-tensor launch (the module loop of ModelCompressor.compress_model in one kernel)
# --------------------------------------------------------------------------------------------
def _scale_count(d: N.QuantDesc) -> int:
    """elements of the scale / zero-point tensor that the addressing  sidx = (r / rdiv) * s_row_stride + c / cdiv  can reach"""
    row_scaled = d.rdiv != N.INF
    row_blocks = -(-d.rows // d.rdiv) if row_scaled else 1
    per_row = 1 if d.cdiv == N.INF else -(-d.cols // d.cdiv)
    return row_blocks * d.s_row_stride if (row_scaled and d.s_row_stride > 0) else per_row


def _validate_problem(op: int, i: int, prob, on_cuda: Optional[int]) -> None:
    """A caller-built descriptor is trusted by the kernels: rows * cols that do not match the tensors are an out-of-bounds access on
    the device.  Cheap host-side check of every (desc, in, scale, zp, out): element counts, element sizes, placement, contiguity."""
    d, tin, sc, zp, out = prob

    def bad(msg):
        raise ValueError(f"batched: tensor {i}: {msg}")

    rows, cols, bits = int(d.rows), int(d.cols), int(d.num_bits)
    if rows < 0 or cols < 0:
        bad("negative shape in the descriptor")
    n = rows * cols
    words = rows * (-(-cols * bits // 32)) if bits > 0 else 0
    # (input elements, input bytes/elem, output elements, output bytes/elem); None = not checked for this op
    if op in (N.OP_QUANTIZE_PACK, N.OP_OBSERVE_QUANTIZE_PACK):
        want = (n, N.DT_SIZE.get(d.x_dtype), words, 4)
    elif op == N.OP_UNPACK_DEQUANTIZE:
        want = (words, 4, n, N.DT_SIZE.get(d.out_dtype))
    elif op == N.OP_QUANTIZE:
        want = (n, N.DT_SIZE.get(d.x_dtype), n, N.DT_SIZE.get(d.q_dtype))
    elif op == N.OP_DEQUANTIZE:
        want = (n, N.DT_SIZE.get(d.q_dtype), n, N.DT_SIZE.get(d.out_dtype))
    elif op == N.OP_FAKE_QUANTIZE:
        want = (n, N.DT_SIZE.get(d.x_dtype), n, N.DT_SIZE.get(d.out_dtype))
    elif op == N.OP_PACK_INT32:
        want = (n, 1, words, 4)
    elif op == N.OP_UNPACK_INT32:
        want = (words, 4, n, 1)
    elif op in (N.OP_QUANTIZE_PACK_FP4, N.OP_OBSERVE_QUANTIZE_PACK_FP4):
        want = (n, N.DT_SIZE.get(d.x_dtype), n // 2, 1)
    elif op == N.OP_UNPACK_DEQUANTIZE_FP4:
        want = (n // 2, 1, n, N.DT_SIZE.get(d.out_dtype))
    elif op == N.OP_OBSERVE_QUANTIZE_BLOCK:
        want = (n, N.DT_SIZE.get(d.x_dtype), n, 1)
    elif op == N.OP_OBSERVE_QUANTIZE_MX:
        want = (n, N.DT_SIZE.get(d.x_dtype), n // 2 if d.qtype == N.Q_FP4 else n, 1)
    elif op == N.OP_SPARSE24_QUANTIZE_PACK:          # kept codes [rows, cols/2] as a 4-bit stream; the bitmask (d.aux) is the caller's business
        want = (n, N.DT_SIZE.get(d.x_dtype), rows * (-(-(cols // 2) * bits // 32)), 4)
    elif op == N.OP_SPARSE24_UNPACK_DEQUANTIZE:
        want = (rows * (-(-(cols // 2) * bits // 32)), 4, n, N.DT_SIZE.get(d.out_dtype))
    else:
        bad(f"unknown op {op}")
    for what, t, numel, size in (("input", tin, want[0], want[1]), ("output", out, want[2], want[3])):
        if t is None:
            bad(f"{what} tensor is missing")
        if size is None:
            bad(f"the descriptor names no valid dtype for the {what}")
        if t.numel() != numel or t.element_size() != size:
            bad(f"{what} holds {t.numel()} elements of {t.element_size()} bytes, the descriptor ({rows} x {cols}, {bits} bits) needs {numel} of {size}")
    tensors = [("input", tin), ("output", out)]
    if op not in (N.OP_PACK_INT32, N.OP_UNPACK_INT32):
        if sc is None:
            bad("scale tensor is missing")
        ssize = N.DT_SIZE.get(d.scale_dtype)
        need = _scale_count(d)
        if ssize is None or sc.element_size() != ssize or sc.numel() < need:
            bad(f"scale holds {sc.numel()} elements of {sc.element_size()} bytes, the descriptor addresses {need} of {ssize}")
        tensors.append(("scale", sc))
        if zp is not None:
            zsize = N.DT_SIZE.get(d.zp_dtype)
            if zsize is None or zp.element_size() != zsize or zp.numel() < need:
                bad(f"zero point holds {zp.numel()} elements of {zp.element_size()} bytes, the descriptor addresses {need} of {zsize}")
            tensors.append(("zero point", zp))
    for what, t in tensors:
        if not t.is_contiguous():
            bad(f"{what} is not contiguous")
        if on_cuda is not None and (not t.is_cuda or t.device.index != on_cuda):
            bad(f"{what} lives on {t.device}, the launch runs on cuda:{on_cuda}")
        if on_cuda is None and t.is_cuda:
            bad(f"{what} lives on {t.device}, host_batched expects CPU tensors")


def _tables(problems):
    """the ctypes tables of a job list: descriptors, then the in / scale / zp / out pointers (0 for an absent tensor)"""
    n = max(len(problems), 1)
    vp = ctypes.c_void_p * n
    ptrs = [vp(*[(p[k].data_ptr() if p[k] is not None else 0) for p in problems]) for k in (1, 2, 3, 4)]
    return ((N.QuantDesc * n)(*[p[0] for p in problems]), *ptrs)


class BatchedPlan:
    """A validated multi-tensor launch that can be enqueued any number of times (`run()`): the descriptors are checked against their
    tensors once, the pointer tables are built once, and `run()` is a single ct_batched call on the current stream.  The plan keeps
    the tensors alive.  What a caller that compresses the same buffers repeatedly (benchmarks, double-buffered checkpoint
    writers) should hold instead of calling `batched` every time."""

    __slots__ = ("op", "n", "idx", "_keep", "_descs", "_ins", "_scs", "_zps", "_outs")

    def __init__(self, op: int, problems, device_index: Optional[int] = None):
        self.op, self.n = int(op), len(problems)
        self.idx = device_index if device_index is not None else (_dev_index(problems[0][1]) if problems else 0)
        for i, p in enumerate(problems):
            _validate_problem(self.op, i, p, self.idx)
        self._keep = list(problems)
        self._descs, self._ins, self._scs, self._zps, self._outs = _tables(problems)

    def run(self) -> None:
        if self.n == 0:
            return
        rc = N.lib().ct_batched(self.op, self.n, self._descs, ctypes.cast(self._ins, ctypes.c_void_p), ctypes.cast(self._scs, ctypes.c_void_p),
                                ctypes.cast(self._zps, ctypes.c_void_p), ctypes.cast(self._outs, ctypes.c_void_p), self.idx, N.stream_ptr(self.idx))
        N.check(rc, "ct_batched")


@torch.no_grad()
def batched(op: int, problems: Sequence[Tuple[N.QuantDesc, torch.Tensor, torch.Tensor, Optional[torch.Tensor], torch.Tensor]],
            device_index: Optional[int] = None) -> None:
    """problems: (desc, in, scale, zp, out) with every tensor already on the same CUDA device.  Every descriptor is checked against
    its tensors first (ValueError, nothing launched)."""
    if len(problems):
        BatchedPlan(op, problems, device_index).run()


@torch.no_grad()
def host_batched(op: int, problems: Sequence[Tuple[N.QuantDesc, torch.Tensor, torch.Tensor, Optional[torch.Tensor], torch.Tensor]],
                 device_index: Optional[int] = None) -> None:
    """like `batched` but every tensor lives in HOST memory (pinned for full PCIe rate): one pipelined
    H2D -> kernel -> D2H queue across all tensors (ct_host_run_many).  Blocking."""
    n = len(problems)
    if n == 0:
        return
    for i, p in enumerate(problems):
        _validate_problem(int(op), i, p, None)
    idx = device_index if device_index is not None else N.require_device(None)
    descs, ins, scs, zps, outs = _tables(problems)
    rc = N.lib().ct_host_run_many(int(op), n, descs, ctypes.cast(ins, ctypes.c_void_p), ctypes.cast(scs, ctypes.c_void_p),
                                  ctypes.cast(zps, ctypes.c_void_p), ctypes.cast(outs, ctypes.c_void_p), idx)
    N.check(rc, "ct_host_run_many")


# --------------------------------------------------------------------------------------------
# bitmasks and sparse formats
# --------------------------------------------------------------------------------------------
def pack_bitmasks(bytemasks: torch.Tensor) -> torch.Tensor:
    """reference: utils/helpers.py:306-317 (numpy.packbits, axis=-1, bitorder='little')"""
    cols = bytemasks.shape[-1]
    nb = (cols + 7) // 8
    out_shape = tuple(bytemasks.shape[:-1]) + (nb,)
    if bytemasks.numel() == 0:
        return torch.empty(out_shape, dtype=torch.uint8, device=bytemasks.device)
    idx = _dev_index(bytemasks)
    bm = _to_dev(bytemasks.to(torch.uint8) if bytemasks.dtype != torch.bool else bytemasks.view(torch.uint8), idx)
    rows = bm.numel() // cols
    out = torch.empty(out_shape, dtype=torch.uint8, device=bm.device)
    N.check(N.lib().ct_pack_bitmasks(N.ptr(bm), N.ptr(out), rows, cols, idx, N.stream_ptr(idx)), "pack_bitmasks")
    return _back(out, bytemasks)


def unpack_bitmasks(packed_bitmasks: torch.Tensor, original_shape: Sequence[int]) -> torch.Tensor:
    """reference: utils/helpers.py:320-343"""
    original_shape = tuple(int(s) for s in original_shape)
    cols = original_shape[-1]
    rows = math.prod(original_shape[:-1]) if len(original_shape) > 1 else 1
    if rows * cols == 0:
        return torch.empty(original_shape, dtype=torch.bool, device=packed_bitmasks.device)
    idx = _dev_index(packed_bitmasks)
    pk = _to_dev(packed_bitmasks, idx)
    out = torch.empty(original_shape, dtype=torch.uint8, device=pk.device)
    N.check(N.lib().ct_unpack_bitmasks(N.ptr(pk), N.ptr(out), rows, cols, idx, N.stream_ptr(idx)), "unpack_bitmasks")
    return _back(out.view(torch.bool), packed_bitmasks)


def sparse24_compress(x: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """2:4 bitmask compression of a 2-D tensor -> (values [R, C/2], bitmask uint8 [R, ceil(C/8)])"""
    if x.ndim != 2:
        raise ValueError("sparse24 compression expects a 2-D tensor")
    rows, cols = x.shape
    if cols % 4 != 0:
        raise ValueError(f"2:4 compression needs the column count to be a multiple of 4, got {cols}")
    idx = _dev_index(x)
    xd = _to_dev(x, idx)
    values = torch.empty((rows, cols // 2), dtype=x.dtype, device=xd.device)
    bitmask = torch.empty((rows, (cols + 7) // 8), dtype=torch.uint8, device=xd.device)
    rc = N.lib().ct_sparse24_compress(N.ptr(xd), N.DT[x.dtype], N.ptr(values), N.ptr(bitmask), rows, cols, idx, N.stream_ptr(idx))
    N.check(rc, "sparse24_compress")
    return _back(values, x), _back(bitmask, x)


def sparse24_decompress(values: torch.Tensor, bitmask: torch.Tensor, shape: Sequence[int]) -> torch.Tensor:
    rows, cols = int(shape[0]), int(shape[1])
    idx = _dev_index(values)
    v, b = _to_dev(values, idx), _to_dev(bitmask, idx)
    out = torch.empty((rows, cols), dtype=values.dtype, device=v.device)
    rc = N.lib().ct_sparse24_decompress(N.ptr(v), N.DT[values.dtype], N.ptr(b), N.ptr(out), rows, cols, idx, N.stream_ptr(idx))
    N.check(rc, "sparse24_decompress")
    return _back(out, values)


def bitmask_compress(x: torch.Tensor, exact: bool = True):
    """unstructured bitmask compression -> (values [nnz], bitmask uint8 [R, ceil(C/8)], row_offsets int64 [R])

    One ABI call, the dense tensor is read once (ct_bitmask_compress_onepass): the kernel writes into a buffer of capacity numel and
    leaves nnz on the device.  `exact=True` (the storage format: `compressed` holds exactly nnz elements) reads nnz back at the END
    and returns the slice; `exact=False` never synchronises and returns (values with capacity numel, bitmask, row_offsets, nnz) with
    nnz a 1-element int64 tensor on the device -- for callers that keep going on the stream (checkpoint writers that size the file
    record later)."""
    if x.ndim != 2:
        raise ValueError("bitmask compression expects a 2-D tensor")
    rows, cols = x.shape
    idx = _dev_index(x)
    xd = _to_dev(x, idx)
    bitmask = torch.empty((rows, (cols + 7) // 8), dtype=torch.uint8, device=xd.device)
    row_offsets = torch.empty((rows,), dtype=torch.int64, device=xd.device)
    nnz = torch.empty((1,), dtype=torch.int64, device=xd.device)
    values = torch.empty((rows * cols,), dtype=x.dtype, device=xd.device)
    N.check(N.lib().ct_bitmask_compress_onepass(N.ptr(xd), N.DT[x.dtype], N.ptr(values), N.ptr(bitmask), N.ptr(row_offsets), N.ptr(nnz),
                                                rows, cols, idx, N.stream_ptr(idx)), "bitmask_compress")
    if not exact:
        return _back(values, x), _back(bitmask, x), _back(row_offsets, x), _back(nnz, x)
    values = values[: int(nnz.item())].clone()      # the only host read, after all device work has been enqueued
    return _back(values, x), _back(bitmask, x), _back(row_offsets, x)


def bitmask_decompress(values: torch.Tensor, bitmask: torch.Tensor, row_offsets: torch.Tensor, shape: Sequence[int]) -> torch.Tensor:
    rows, cols = int(shape[0]), int(shape[1])
    idx = _dev_index(values, bitmask)
    v, b, ro = _to_dev(values, idx), _to_dev(bitmask, idx), _to_dev(row_offsets, idx)
    out = torch.empty((rows, cols), dtype=values.dtype, device=b.device)
    N.check(N.lib().ct_bitmask_decompress(N.ptr(v), N.DT[values.dtype], N.ptr(b), N.ptr(ro), N.ptr(out), rows, cols,
                                          idx, N.stream_ptr(idx)), "bitmask_decompress")
    return _back(out, bitmask)


# --------------------------------------------------------------------------------------------
# BASELINE config 4: "Sparse24BitMask + int4" (2:4 selection + pack-quantized) fused
# --------------------------------------------------------------------------------------------
@torch.no_grad()
def sparse24_quantize_pack(x: torch.Tensor, scale: torch.Tensor, zero_point: Optional[torch.Tensor], args) -> Tuple[torch.Tensor, torch.Tensor]:
    """2:4 compress + int4 quantize + pack in ONE pass over the dense weight:
        mask    = keep the 2 of largest |x| in every 4 consecutive columns (ties: lower column), as `sparse24_compress`
        codes   = quantize(x, scale, zero_point, args, dtype=int8)[mask].view(R, C/2)      (forward.py:36-73 on the kept columns)
        returns (pack_to_int32(codes, num_bits) int32 [R, C * bits / 64], pack_bitmasks(mask) uint8 [R, C/8])
    The fused kernel covers bf16 / fp16 weights, 4-bit integer codes, cols % 32 == 0 and scales with full rows; every other case
    composes the unfused kernels (same bits).  PARITY UNPINNED as a composite: quantize, the bitstream and the mask bit order are
    pinned by the reference's goldens, the selection rule and the composition are restated (SURVEY 8 a12 / a14)."""
    if x.ndim != 2:
        raise ValueError("sparse24_quantize_pack expects a 2-D weight")
    rows, cols = x.shape
    if cols % 4 != 0:
        raise ValueError(f"2:4 compression needs the column count to be a multiple of 4, got {cols}")
    _check_float(x, "input")
    _check_float(scale, "scale")
    qtype, bits = _qparams(args)
    if qtype != N.Q_INT:
        raise ValueError("pack-quantized compression needs integer quantization")
    p = _resolve(x, scale, zero_point, args, None)
    idx = _dev_index(x, p.scale)
    xd, sc, zp = _to_dev(x, idx), _to_dev(p.scale, idx), _to_dev(p.zp, idx)
    cd = torch.result_type(x, scale)
    packed = torch.empty((rows, -(-(cols // 2) * bits // 32)), dtype=torch.int32, device=xd.device)
    bitmask = torch.empty((rows, (cols + 7) // 8), dtype=torch.uint8, device=xd.device)
    d = _desc(p, x.dtype, sc.dtype, zp.dtype if zp is not None else None, cd, torch.int8, None, qtype, bits)
    rc = N.lib().ct_sparse24_quantize_pack_int4(ctypes.byref(d), N.ptr(xd), N.ptr(sc), N.ptr(zp), N.ptr(packed), N.ptr(bitmask), idx, N.stream_ptr(idx))
    if rc == N.CT_E_UNSUPPORTED:
        # unfused composition of the same kernels: 2:4 mask, dense codes, gather of the kept codes, bit packing
        _, bitmask = sparse24_compress(xd)
        q = quantize(xd, p.scale.to(xd.device), p.zp.to(xd.device) if p.zp is not None else None, args, dtype=torch.int8)
        kept = q[unpack_bitmasks(bitmask, (rows, cols))].view(rows, cols // 2)
        packed = pack_to_int32(kept.contiguous(), bits)
    else:
        N.check(rc, "sparse24_quantize_pack")
    return _back(packed, x), _back(bitmask, x)


@torch.no_grad()
def sparse24_unpack_dequantize(packed: torch.Tensor, bitmask: torch.Tensor, scale: torch.Tensor, zero_point: Optional[torch.Tensor],
                               num_bits: int, shape: Sequence[int], dtype: Optional[torch.dtype] = None) -> torch.Tensor:
    """inverse of `sparse24_quantize_pack`: kept codes back to their columns and dequantized (strategy inferred from the scale shape
    like forward.py:99-130), dropped columns = +0; returns `dtype` (default scale.dtype) [R, C]"""
    shape = tuple(int(v) for v in shape)
    rows, cols = shape
    if packed.dtype is not torch.int32:
        raise ValueError(f"Expected {torch.int32} but got {packed.dtype}, Aborting unpack.")
    _check_float(scale, "scale")
    like = torch.empty(shape, dtype=torch.int8, device="meta")
    args = _infer_dequant_args(like, scale)
    out_dtype = (dtype or scale.dtype) if _strategy_name(args) in ("group", "tensor_group") else scale.dtype
    p = _resolve(like, scale, zero_point, args, None)
    idx = _dev_index(packed, bitmask)
    pk, bm, sc, zp = _to_dev(packed, idx), _to_dev(bitmask, idx), _to_dev(p.scale, idx), _to_dev(p.zp, idx)
    out = torch.empty(shape, dtype=out_dtype, device=pk.device)
    d = _desc(p, None, sc.dtype, zp.dtype if zp is not None else None, None, torch.int8, out_dtype, N.Q_INT, int(num_bits))
    rc = N.lib().ct_sparse24_unpack_dequantize_int4(ctypes.byref(d), N.ptr(pk), N.ptr(bm), N.ptr(sc), N.ptr(zp), N.ptr(out), idx, N.stream_ptr(idx))
    if rc == N.CT_E_UNSUPPORTED:
        kept = unpack_from_int32(pk, int(num_bits), (rows, cols // 2))
        mask = unpack_bitmasks(bm, shape)
        q = torch.zeros(shape, dtype=torch.int8, device=pk.device)
        q[mask] = kept.reshape(-1)
        out = dequantize(q, p.scale.to(pk.device), p.zp.to(pk.device) if p.zp is not None else None, args, dtype=out_dtype)
        out = torch.where(mask, out, torch.zeros_like(out))
    else:
        N.check(rc, "sparse24_unpack_dequantize")
    return _back(out, packed)


# --------------------------------------------------------------------------------------------
# ImplBackend wiring (reference utils/impl_backend.py:23-134): the seven per-tensor hot-path ops and hadamard_transform are entrypoints.
#   backend "<op>_sm100": the CUDA kernels; req = a CUDA device is usable (CPU tensors are then staged through it, as before)
#   eager body "<op>_eager": the library's own host code (device = -1 twins, csrc/cpu_twin.cu) -- what a GPU-less host and
#                            CT_ENFORCE_EAGER=1 get.  Results are bit-identical (same per-element source as the generic kernels).
# --------------------------------------------------------------------------------------------
def _cuda_usable(*args, **kwargs) -> bool:
    return torch.cuda.is_available()


def _wire_impl_backend():
    from .utils.impl_backend import ImplBackend

    for name in ("pack_to_int32", "unpack_from_int32", "quantize", "dequantize", "fake_quantize", "quantize_pack", "unpack_dequantize",
                 "hadamard_transform"):
        fn = globals()[name]

        def cuda_fn(*a, _fn=fn, **k):
            return _fn(*a, **k)

        def eager_fn(*a, _fn=fn, **k):
            prev = getattr(_mode, "cpu", False)
            _mode.cpu = True
            try:
                return _fn(*a, **k)
            finally:
                _mode.cpu = prev

        functools.update_wrapper(cuda_fn, fn)
        functools.update_wrapper(eager_fn, fn)
        cuda_fn.__name__, eager_fn.__name__ = f"{name}_sm100", f"{name}_eager"
        ImplBackend.register(name, req=_cuda_usable, priority=0)(cuda_fn)
        globals()[name] = ImplBackend.entrypoint(name)(eager_fn)


_wire_impl_backend()
