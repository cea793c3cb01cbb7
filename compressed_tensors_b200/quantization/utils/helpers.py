"""
Quantization helpers on the host side of the path: ranges, the min/max -> (scale, zero point)
rule, dynamic qparams, block padding.  Mirror of quantization/utils/helpers.py:50-249, :374-428.

These operate on QPARAM-sized tensors (one value per tensor / channel / group / block): they are
host plumbing around the hot path, written with torch ops on whatever device the data lives on.
The min/max reduction over the full tensor and its fusion in front of quantize+pack is the
"next" row (f)1 of SURVEY.md section 8.
"""
from __future__ import annotations

import math

import torch
from torch import Tensor
from torch.nn import Module

from ..quant_args import FP4_E2M1_DATA, FP8_E4M3_DATA, QuantizationArgs, QuantizationStrategy, QuantizationType, round_to_quantized_type_dtype

__all__ = [
    "calculate_range",
    "calculate_qparams",
    "compute_dynamic_scales_and_zp",
    "is_module_quantized",
    "strategy_cdiv",
    "generate_gparam",
    "calculate_block_padding",
    "maybe_pad_tensor_for_block_quant",
    "is_model_quantized",
    "module_type",
    "get_torch_bit_depth",
    "can_quantize",
    "KV_CACHE_TARGETS",
]

# nominal targets of the scheme a `kv_cache_scheme` becomes on attention modules (apply_quantization_config never matches them)
KV_CACHE_TARGETS = ["re:.*(self_attn|attention)$"]


def calculate_range(quantization_args: QuantizationArgs, device) -> tuple[Tensor, Tensor]:
    """(q_min, q_max) as 0-dim fp32 tensors (helpers.py:198-226)"""
    if quantization_args.type == QuantizationType.INT:
        span = 2.0 ** quantization_args.num_bits
        lo, hi = -span / 2, span / 2 - 1
    elif quantization_args.type == QuantizationType.FLOAT:
        if quantization_args.num_bits == 8:
            lo, hi = FP8_E4M3_DATA.min, FP8_E4M3_DATA.max
        elif quantization_args.num_bits == 4:
            lo, hi = FP4_E2M1_DATA.min, FP4_E2M1_DATA.max
        else:
            raise NotImplementedError("Range calculation only supported for 4 and 8 bits")
    else:
        raise ValueError(f"Invalid quantization type {quantization_args.type}")
    return torch.tensor(lo, device=device), torch.tensor(hi, device=device)


def _divisor(value: float, like: Tensor) -> Tensor:
    """the Python-float divisor of the reference's formulas as a 0-dim tensor of `like`'s dtype ON ITS DEVICE: the result dtype
    is the one a Python scalar gives (also when `like` is 0-dim itself, the TENSOR strategy), the value is rounded to that
    dtype as the CPU kernels do with a scalar, and torch's CUDA kernels then perform a true IEEE division -- with a Python
    scalar they multiply by its reciprocal, which differs from the CPU result (the pinned one) by an ulp now and then"""
    return torch.tensor(value, dtype=like.dtype, device=like.device)


def calculate_qparams(min_vals: Tensor, max_vals: Tensor, quantization_args: QuantizationArgs,
                      global_scale: Tensor | None = None) -> tuple[Tensor, Tensor]:
    """observer rule of the reference (helpers.py:50-137), same op order so the scales agree bit for bit.

    CONTRACT: the result equals the reference's CPU result on every device.  The reference divides by a Python float; ATen's CUDA
    kernels turn that into a multiplication by the reciprocal, so the reference ITSELF differs between CPU and CUDA by an ulp
    now and then.  This engine pins the CPU value (the one the goldens and the reference's tests hold) and gets it on CUDA too by
    dividing by a 0-dim tensor (`_divisor`), which keeps true IEEE division; tests/test_gpu_observe.py checks CUDA == CPU golden."""
    from .mxfp_utils import generate_mx_scales, maybe_convert_from_mx_exp, should_generate_mx_scales

    min_vals = torch.min(min_vals, torch.zeros_like(min_vals))
    max_vals = torch.max(max_vals, torch.zeros_like(max_vals))
    device = min_vals.device
    bit_min, bit_max = calculate_range(quantization_args, device)
    bit_range = bit_max - bit_min
    if quantization_args.symmetric:
        max_val_pos = torch.max(torch.abs(min_vals), torch.abs(max_vals))
        if should_generate_mx_scales(quantization_args):
            scales = generate_mx_scales(x=max_val_pos, num_bits=quantization_args.num_bits)
        else:
            scales = max_val_pos / _divisor(float(bit_range) / 2, max_val_pos)
        zero_points = torch.zeros(scales.shape, device=device, dtype=min_vals.dtype)
    else:
        if quantization_args.num_bits == 4 and quantization_args.type == QuantizationType.FLOAT:
            raise NotImplementedError("Asymmetric Quantization is not supported for FP4")
        scales = (max_vals - min_vals) / _divisor(float(bit_range), max_vals)
        zero_points = bit_min - (min_vals / scales)
        zero_points = torch.clamp(zero_points, bit_min, bit_max)
    if global_scale is not None:
        scales = global_scale * scales
    if quantization_args.scale_dtype is not None:
        scales = round_to_quantized_type_dtype(scales, dtype=quantization_args.scale_dtype)
    scales = maybe_convert_from_mx_exp(quantization_args, scales)
    eps_dtype = quantization_args.scale_dtype if quantization_args.scale_dtype is not None else scales.dtype
    if eps_dtype == FP8_E4M3_DATA.dtype:
        eps = 0.125
    else:
        eps = torch.finfo(eps_dtype).eps if eps_dtype.is_floating_point else 1
    scales = torch.where(scales == 0, torch.tensor(eps, dtype=scales.dtype, device=device), scales)
    zero_points = round_to_quantized_type_dtype(zero_points, dtype=quantization_args.zp_dtype, cast_to_original_dtype=False)
    if scales.ndim == 0:
        scales, zero_points = scales.reshape(1), zero_points.reshape(1)
    return scales, zero_points


def generate_gparam(updated_min_val: Tensor, updated_max_val: Tensor, scale_data=FP8_E4M3_DATA, quant_data=FP4_E2M1_DATA,
                    dtype: torch.dtype | None = torch.float32) -> Tensor:
    """global scale of a tensor: maps its max |x| onto (max of the local-scale dtype) x (max of the element dtype), so
    that NVFP4's fp8 group scales use their whole range (helpers.py:308-337); NaN / inf results become 1.0"""
    lo = torch.min(updated_min_val, torch.zeros_like(updated_min_val))
    hi = torch.max(updated_max_val, torch.zeros_like(updated_max_val))
    top = torch.max(torch.abs(lo), torch.abs(hi))
    top = torch.clamp(top, min=torch.finfo(top.dtype).tiny)
    # Python float / tensor is Tensor.__rtruediv__ = top.reciprocal() * float: the reciprocal is rounded to top's dtype before the
    # product (2688 / 1.745 -> 1541 in fp16, where a correctly rounded quotient is 1540).  The value is pinned by the reference's
    # behaviour (fuzz_host_mirror.py); ct_observe_tensor (kind 1) restates exactly these two roundings.
    g = (scale_data.max * quant_data.max) / top
    g = torch.nan_to_num(g, nan=1.0, posinf=1.0, neginf=1.0)
    return g.to(dtype).reshape([1])


def compute_dynamic_scales_and_zp(value: Tensor, args: QuantizationArgs, module: Module = None, global_scale: Tensor | None = None):
    """min/max over the strategy's reduction dims, then calculate_qparams (helpers.py:140-195)"""
    keep = True
    if args.strategy == QuantizationStrategy.TOKEN:
        dims = tuple(i for i in range(value.ndim) if i not in (0, 1))
    elif args.strategy == QuantizationStrategy.TENSOR:
        dims = None
    elif args.strategy in (QuantizationStrategy.TENSOR_GROUP, QuantizationStrategy.GROUP):
        dims, keep = -1, False
        value = value.unflatten(-1, (math.ceil(value.shape[-1] / args.group_size), args.group_size))
    else:
        ok = (QuantizationStrategy.TOKEN, QuantizationStrategy.TENSOR, QuantizationStrategy.TENSOR_GROUP, QuantizationStrategy.GROUP)
        raise ValueError(f"Dynamic quantization is only supported for {ok}")
    if not dims:
        mn, mx = torch.aminmax(value)
    else:
        mn = torch.amin(value, dim=dims, keepdims=keep)
        mx = torch.amax(value, dim=dims, keepdims=keep)
    return calculate_qparams(mn, mx, args, global_scale=global_scale)


def is_module_quantized(module: Module) -> bool:
    """a module is quantized when its scheme has any of weights / input / output args (helpers.py:229-249)"""
    scheme = getattr(module, "quantization_scheme", None)
    if scheme is None:
        return False
    return any(getattr(scheme, k, None) is not None for k in ("weights", "input_activations", "output_activations"))


def strategy_cdiv(value: int, divisor: int, strategy=None, strict: bool = False) -> int:
    """ceil-division used for scale shapes; complains (or raises when strict) on a ragged last group"""
    out = math.ceil(value / divisor)
    if out * divisor != value and strict:
        raise ValueError(f"{strategy} quantization strategy requires strict division of weight/activation size {value} "
                         f"and group/block size {divisor}.")
    return out


def calculate_block_padding(shape, block_structure) -> tuple[int, int]:
    """(rows, cols) of zero padding that make the last two dims multiples of the block (helpers.py:374-397)"""
    if len(shape) < 2:
        raise ValueError(f"Tensor must be at least 2D, got shape {shape}")
    bh, bw = block_structure
    return (-shape[-2]) % bh, (-shape[-1]) % bw


def maybe_pad_tensor_for_block_quant(tensor: Tensor, block_structure: tuple[int, int]) -> Tensor:
    """zero-pad the last two dims up to multiples of the block (helpers.py:400-428)"""
    pr, pc = calculate_block_padding(tensor.shape, block_structure)
    if pr == 0 and pc == 0:
        return tensor
    return torch.nn.functional.pad(tensor, (0, pc, 0, pr), mode="constant", value=0)


def is_model_quantized(model: Module) -> bool:
    """some module of the model carries a non-empty quantization scheme (helpers.py:252-260)"""
    return any(is_module_quantized(m) for m in model.modules())


def module_type(module: Module) -> str:
    """class name of the module, the string "targets" are matched against (helpers.py:263-270)"""
    return type(module).__name__


def get_torch_bit_depth(value: Tensor) -> int:
    """bits per element of the tensor's dtype (helpers.py:273-285)"""
    dt = value.dtype
    return torch.finfo(dt).bits if dt.is_floating_point else torch.iinfo(dt).bits


def can_quantize(value: Tensor, quant_args: QuantizationArgs) -> bool:
    """the tensor is wider than the requested quantization (helpers.py:288-305); warns when it is narrower"""
    depth = get_torch_bit_depth(value)
    if depth < quant_args.num_bits:
        import logging

        logging.getLogger(__name__).warning(f"Can't quantize tensor with bit depth {depth} to {quant_args.num_bits}."
                                            "The QuantizationArgs provided are not compatible with the input tensor.")
    return depth > quant_args.num_bits
