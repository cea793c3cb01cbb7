"""
quantize / dequantize / fake_quantize and the module forward wrapper -- the public per-tensor API
of the reference (quantization/lifecycle/forward.py:36-329), here dispatching to the sm_90a
kernels.  Argument names, defaults, strategy inference and the dtype quirks are the reference's;
the bodies of _process_quantization / _process_group / _process_block / _quantize / _dequantize /
_quantize_dequantize (forward.py:184-241, forward_helpers.py:19-215, :523-572) are one fused CUDA
kernel each (compressed_tensors_b200/ops.py -> include/ct_b200.h).
"""
from __future__ import annotations

from functools import wraps

import torch
from torch.nn import Module

from ... import ops
from ...offload.cache import OffloadCache
from ..quant_args import DynamicType, QuantizationArgs
from ..quant_config import QuantizationStatus
from ..quant_scheme import QuantizationScheme
from ..utils.helpers import compute_dynamic_scales_and_zp

__all__ = ["quantize", "dequantize", "fake_quantize", "set_forward_quantized", "forward_quantize", "_process_quantization"]


@torch.no_grad()
def _process_quantization(x: torch.Tensor, scale: torch.Tensor, zero_point: torch.Tensor, args: QuantizationArgs,
                          g_idx: torch.Tensor | None = None, dtype: torch.dtype | None = None, do_quantize: bool = True,
                          do_dequantize: bool = True, global_scale: torch.Tensor | None = None) -> torch.Tensor:
    """the dispatcher behind quantize / dequantize / fake_quantize (forward.py:184-241): one CUDA kernel per combination"""
    if do_quantize and do_dequantize:
        return ops.fake_quantize(x, scale, zero_point, args, g_idx=g_idx, global_scale=global_scale)
    if do_quantize:
        return ops.quantize(x, scale, zero_point, args, dtype=dtype, g_idx=g_idx, global_scale=global_scale)
    return ops.dequantize(x, scale, zero_point, args=args, dtype=dtype, g_idx=g_idx, global_scale=global_scale)


@torch.no_grad()
def quantize(x: torch.Tensor, scale: torch.Tensor, zero_point: torch.Tensor, args: QuantizationArgs,
             dtype: torch.dtype | None = None, g_idx: torch.Tensor | None = None,
             global_scale: torch.Tensor | None = None) -> torch.Tensor:
    """x -> clamp(round(x / scale + zero_point)) per the strategy in args (forward.py:36-73)"""
    return ops.quantize(x, scale, zero_point, args, dtype=dtype, g_idx=g_idx, global_scale=global_scale)


@torch.no_grad()
def dequantize(x_q: torch.Tensor, scale: torch.Tensor, zero_point: torch.Tensor | None = None,
               args: QuantizationArgs | None = None, dtype: torch.dtype | None = None,
               g_idx: torch.Tensor | None = None, global_scale: torch.Tensor | None = None) -> torch.Tensor:
    """(x_q - zero_point) * scale; strategy inferred from the scale shape when args is None (forward.py:76-145)"""
    return ops.dequantize(x_q, scale, zero_point, args=args, dtype=dtype, g_idx=g_idx, global_scale=global_scale)


@torch.no_grad()
def fake_quantize(x: torch.Tensor, scale: torch.Tensor, zero_point: torch.Tensor, args: QuantizationArgs,
                  g_idx: torch.Tensor | None = None, global_scale: torch.Tensor | None = None) -> torch.Tensor:
    """quantize then dequantize in one pass (forward.py:148-181)"""
    return ops.fake_quantize(x, scale, zero_point, args, g_idx=g_idx, global_scale=global_scale)


def forward_quantize(module: Module, value: torch.Tensor, base_name: str, args: QuantizationArgs) -> torch.Tensor:
    """fake-quantize `value` with the module's static qparams or dynamic ones (forward.py:292-329)"""
    if getattr(module, "quantization_status", None) is not None and module.quantization_status >= QuantizationStatus.COMPRESSED and base_name == "weight":
        return value
    if value.numel() == 0:
        return value
    g_idx = getattr(module, "weight_g_idx", None)
    global_scale = getattr(module, f"{base_name}_global_scale", None)
    if args.dynamic in (True, DynamicType.LOCAL):
        # observer and fake quantization in one pass on the device (bit-identical); CPU, strided or g_idx inputs and whatever the kernel
        # declines take the two steps below, so their results and errors are the reference's
        if g_idx is None and value.is_cuda and value.is_contiguous():
            fused = ops.dynamic_fake_quantize(value, args, global_scale=global_scale)
            if fused is not None:
                return fused[0]
        scale, zero_point = compute_dynamic_scales_and_zp(value=value, args=args, module=module, global_scale=global_scale)
    else:
        scale = getattr(module, f"{base_name}_scale")
        zero_point = getattr(module, f"{base_name}_zero_point", None)
    return fake_quantize(x=value, scale=scale, zero_point=zero_point, args=args, g_idx=g_idx, global_scale=global_scale)


def set_forward_quantized(module: torch.nn.Linear | torch.nn.Embedding):
    """wrap module.forward with input / weight / output fake quantization (forward.py:244-289)"""
    original = module.forward.__func__ if hasattr(module.forward, "__func__") else type(module).forward

    @wraps(original)
    def quantized_forward(self, input: torch.Tensor) -> torch.Tensor:
        if isinstance(self._parameters, OffloadCache) and not OffloadCache.offloading_disabled:
            # an offloaded weight is onloaded anew on every read: keep the first onloaded copy for the whole call, so that the
            # layer's own forward reads the fake-quantized data patched into it (the reference loses it here)
            with OffloadCache.disable_offloading():
                return quantized_forward(self, input)
        scheme: QuantizationScheme | None = getattr(self, "quantization_scheme", None)
        status: QuantizationStatus | None = getattr(self, "quantization_status", None)
        enabled = getattr(self, "quantization_enabled", True) and scheme is not None and status is not None
        weight = self.weight
        weight_data = weight.data
        if enabled and scheme.input_activations:
            input = forward_quantize(self, input, "input", scheme.input_activations)
        if enabled and scheme.weights and status < QuantizationStatus.COMPRESSED:
            weight_data = forward_quantize(self, weight_data, "weight", scheme.weights)
        saved = weight.data
        weight.data = weight_data
        try:
            output = type(self).forward(self, input)
        finally:
            weight.data = saved
        if enabled and scheme.output_activations:
            output = forward_quantize(self, output, "output", scheme.output_activations)
        return output

    module.forward = quantized_forward.__get__(module)
