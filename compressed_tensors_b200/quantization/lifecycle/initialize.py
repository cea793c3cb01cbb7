"""
Attach quantization parameters to a module (mirror of quantization/lifecycle/initialize.py:46-276
for Linear / Embedding modules): `weight_scale`, `weight_zero_point`, `weight_g_idx`,
`input_scale`, ... with the shapes each strategy implies and the dtypes the kernels expect
(scale in the weight dtype, zero point in args.zp_dtype).
"""
from __future__ import annotations

import inspect
import logging
import math

import torch
from torch.nn import Module, Parameter

from ...offload import OffloadCache, get_execution_device, unwrap_offload_forward
from ...utils.helpers import deprecated, get_head_dim, get_num_attn_heads, get_num_kv_heads
from ..quant_args import ActivationOrdering, DynamicType, QuantizationArgs, QuantizationStrategy
from ..quant_config import QuantizationStatus
from ..quant_scheme import QuantizationScheme
from ..utils.helpers import strategy_cdiv
from .forward import set_forward_quantized

__all__ = ["initialize_module_for_quantization", "initialize_qparams", "initialize_attn_qparams", "is_cached_attention_module",
           "is_attention_module", "QPARAM_SUFFIXES"]

_LOGGER = logging.getLogger(__name__)

QPARAM_SUFFIXES = ("_scale", "_zero_point", "_global_scale", "_g_idx")
_BASE_NAMES = ("weight", "input", "output", "q", "k", "v")


def _clear_qparams(module: Module):
    for base in _BASE_NAMES:
        for suffix in QPARAM_SUFFIXES:
            name = base + suffix
            if name in module._parameters or name in module._buffers:
                delattr(module, name)


def initialize_module_for_quantization(module: Module, scheme: QuantizationScheme | None = None, force_zero_point: bool = True):
    scheme = scheme or getattr(module, "quantization_scheme", None)
    if scheme is None:
        return
    _clear_qparams(module)
    if is_cached_attention_module(module):
        initialize_attn_qparams(module, scheme, force_zero_point)
    elif isinstance(module, (torch.nn.Linear, torch.nn.Embedding)):
        weight = module.weight
        if scheme.input_activations is not None:
            initialize_qparams(module, "input", scheme.input_activations, weight.shape[-1:], weight.dtype, force_zero_point)
        if scheme.weights is not None:
            initialize_qparams(module, "weight", scheme.weights, weight.shape, weight.dtype, force_zero_point)
        if scheme.output_activations is not None:
            initialize_qparams(module, "output", scheme.output_activations, weight.shape[:-1], weight.dtype, force_zero_point)
        with unwrap_offload_forward(module):   # an offloaded module keeps moving its inputs to the onload device
            set_forward_quantized(module)
    else:
        raise ValueError(f"Quantization of module type {type(module)} is not supported")
    module.quantization_scheme = scheme
    module.quantization_status = QuantizationStatus.INITIALIZED


def _is_attention_module(module: Module) -> bool:
    """class name contains "attention" and the module owns one of the K / V projections (initialize.py:123-130 of the reference)"""
    return "attention" in module.__class__.__name__.lower() and any(
        hasattr(module, n) for n in ("k_proj", "v_proj", "qkv_proj", "kv_b_proj"))


@deprecated("is_cached_attention_module")
def is_attention_module(module: Module) -> bool:
    return _is_attention_module(module)


def is_cached_attention_module(module: Module) -> bool:
    """an attention module whose forward takes a KV cache (`past_key_values`, or `past_key_value` before transformers#39956): the
    modules that K / V quantization hooks can attach to"""
    if not _is_attention_module(module):
        return False
    try:
        parameters = inspect.signature(module.forward).parameters
    except (TypeError, ValueError):
        _LOGGER.warning("Unable to inspect an attention module's forward signature; skipping KV cache quantization for uninspectable modules")
        return False
    return "past_key_value" in parameters or "past_key_values" in parameters


def _validate_attention_scheme(scheme: QuantizationScheme) -> None:
    if scheme.weights is not None:
        raise ValueError("Cannot apply weight quantization to attention. Instead, target the (q|k|v)_proj submodule layers of attention")
    if scheme.input_activations is None:
        raise ValueError("Cannot apply attention quantization without specifying input activations")
    if scheme.output_activations is not None:
        raise ValueError("Cannot apply output quantization to attention")


def initialize_attn_qparams(module: Module, scheme: QuantizationScheme, force_zero_point: bool) -> None:
    """`q_*` (when the module carries a QuantizedAttentionImpl) and `k_*` / `v_*` (QuantizedKVCache) qparams of an attention module,
    shaped for states [batch, heads, seq, head_dim] of the decoder config the cache holds"""
    from ...modeling import IMPL_ATTR, KV_CACHE_ATTR

    impl = getattr(module, IMPL_ATTR, None)
    kv_cache = getattr(module, KV_CACHE_ATTR, None)
    if impl is None and kv_cache is None:
        raise ValueError(f"Attention module has quantization scheme but no {IMPL_ATTR} or {KV_CACHE_ATTR} attributes. Please ensure that "
                         "these attributes are initialized using `apply_quantization_config`.")
    _validate_attention_scheme(scheme)
    config = kv_cache.config
    head_dim = get_head_dim(config)
    dtype = next(module.parameters()).dtype
    args = scheme.input_activations
    if impl is not None:
        initialize_qparams(module, "q", args, (get_num_attn_heads(config), None, head_dim), dtype, force_zero_point)
    if kv_cache is not None:
        kv_shape = (get_num_kv_heads(config), None, head_dim)
        initialize_qparams(module, "k", args, kv_shape, dtype, force_zero_point)
        initialize_qparams(module, "v", args, kv_shape, dtype, force_zero_point)


def initialize_qparams(module: Module, base_name: str, quantization_args: QuantizationArgs, observed_shape, observed_dtype: torch.dtype,
                       force_zero_point: bool = True):
    strategy, dynamic = quantization_args.strategy, quantization_args.dynamic
    if isinstance(module._parameters, OffloadCache):
        device = get_execution_device(module)   # created where the module runs, then offloaded by its cache
    elif getattr(module, "weight", None) is not None:
        device = module.weight.device
    else:   # attention modules: the device of their projections
        device = next(module.parameters(), torch.empty(0)).device
    if dynamic is True:
        return
    if strategy == QuantizationStrategy.TENSOR_GROUP:
        module.register_parameter(f"{base_name}_global_scale", Parameter(torch.empty(1, dtype=torch.float32, device=device), requires_grad=False))
    if dynamic == DynamicType.LOCAL:
        return

    if strategy == QuantizationStrategy.TENSOR:
        shape = (1,)
    elif strategy == QuantizationStrategy.TOKEN:
        raise ValueError("Cannot perform static token quantization")
    elif strategy == QuantizationStrategy.CHANNEL:
        if len(observed_shape) < 2:
            raise ValueError("Channel quant requires at least 2 observed dimensions")
        shape = (observed_shape[-2], 1)
    elif strategy in (QuantizationStrategy.GROUP, QuantizationStrategy.TENSOR_GROUP):
        if len(observed_shape) < 1:
            raise ValueError("Group quant requires at least 1 observed dimension")
        groups = strategy_cdiv(observed_shape[-1], quantization_args.group_size, strategy)
        shape = (*observed_shape[:-1], groups)
        if quantization_args.actorder == ActivationOrdering.GROUP:
            module.register_parameter(f"{base_name}_g_idx", Parameter(
                torch.full((observed_shape[-1],), -1, device=device, dtype=torch.int), requires_grad=False))
    elif strategy == QuantizationStrategy.BLOCK:
        if len(observed_shape) < 2:
            raise ValueError("Block quant requires at least 2 observed dimensions")
        bh, bw = quantization_args.block_structure
        shape = (math.ceil(observed_shape[-2] / bh), strategy_cdiv(observed_shape[-1], bw, strategy))
    elif strategy == QuantizationStrategy.ATTN_HEAD:
        if len(observed_shape) < 3:
            raise ValueError("Attention quant requires at least 3 observed dimensions")
        shape = (observed_shape[-3], 1, 1)
    else:
        raise AssertionError(f"Unknown strategy {strategy}")

    scale_dtype = observed_dtype if observed_dtype in (torch.float16, torch.bfloat16, torch.float32, torch.float64) else torch.float16
    module.register_parameter(f"{base_name}_scale", Parameter(torch.empty(shape, dtype=scale_dtype, device=device), requires_grad=False))
    if force_zero_point or not quantization_args.symmetric:
        module.register_parameter(f"{base_name}_zero_point", Parameter(
            torch.zeros(shape, device=device, dtype=quantization_args.zp_dtype), requires_grad=False))
