"""
KV-cache quantization hooks (the reference's modeling/kvcache.py): a `QuantizedKVCache` submodule stands in for the
`past_key_values` argument of an attention module, so that every key / value pair the attention writes to its cache passes through a
`torch.nn.Module` -- where it is fake-quantized with the module's `k_*` / `v_*` qparams and where calibration code can hook it --
before it reaches the original cache object.

transformers is imported only by callers that need a model; this module itself runs without it.
"""
from __future__ import annotations

import inspect
from typing import Any, Callable, Optional, Sequence
from weakref import ref

import torch
from torch import Tensor
from torch.nn import Module
from torch.utils.hooks import RemovableHandle

from .. import ops
from ..quantization.quant_args import QuantizationStrategy
from ..utils.helpers import getattr_chain
from ..utils.internal import InternalModule

__all__ = ["QuantizedKVCache", "initialize_hooked_kv_cache", "register_key_hook", "register_value_hook", "KV_CACHE_ATTR"]

KV_CACHE_ATTR = "kv_cache"

_FUSED_STRATEGIES = (QuantizationStrategy.TENSOR, QuantizationStrategy.ATTN_HEAD)


def _fusable(module: Module, base_names: Sequence[str], args, states: Sequence[Tensor]) -> bool:
    """static per-tensor / per-head qparams on CUDA states: what ops.fake_quantize_heads covers in one launch"""
    return (args.dynamic is False and args.strategy in _FUSED_STRATEGIES and all(s.is_cuda for s in states)
            and all(hasattr(module, f"{b}_scale") and getattr(module, f"{b}_global_scale", None) is None for b in base_names))


def quantize_attention_states(module: Module, base_names: Sequence[str], states: Sequence[Tensor]) -> tuple:
    """fake-quantize q / k / v states with the attention module's qparams (`{base}_scale`, `{base}_zero_point`), as
    forward_quantize does, all in one launch when the scheme allows it"""
    from ..quantization.lifecycle.forward import forward_quantize

    args = getattr_chain(module, "quantization_scheme.input_activations", None)
    if args is None or not getattr(module, "quantization_enabled", True):
        return tuple(states)
    if _fusable(module, base_names, args, states):
        scales = [getattr(module, f"{b}_scale") for b in base_names]
        zero_points = [getattr(module, f"{b}_zero_point", None) for b in base_names]
        return tuple(ops.fake_quantize_heads(states, scales, zero_points, args))
    return tuple(forward_quantize(module, s, b, args) for b, s in zip(base_names, states))


class QuantizedKVCache(InternalModule):
    """
    Takes the place of the attention module's cache argument for one forward call: `update(key, value, ...)` fake-quantizes the new
    key and value states with the parent attention module's qparams and hands them to the original cache (held by weak reference,
    so layer-specific behaviour such as sliding windows is kept), or returns them when there is no cache.
    """

    def __init__(self, config, attn_module: Module):
        super().__init__()
        self.config = config
        self.attn_module = ref(attn_module)   # a strong reference would make a cycle parent -> child -> parent
        self.past_key_values = None

    def update(self, *args, **kwargs):
        return self(*args, **kwargs)

    def forward(self, key_states: Tensor, value_states: Tensor, *args, **kwargs):
        key_states, value_states = quantize_attention_states(self.attn_module(), ("k", "v"), (key_states, value_states))
        cache = self.past_key_values() if self.past_key_values is not None else None
        self.past_key_values = None
        if cache is None:
            return key_states, value_states
        return cache.update(key_states, value_states, *args, **kwargs)

    def add_past_key_values(self, past_key_values) -> None:
        self.past_key_values = ref(past_key_values) if past_key_values is not None else None


def _cache_kwarg(module: Module) -> str:
    # transformers renamed the argument to `past_key_values` (huggingface/transformers#39956)
    return "past_key_values" if "past_key_values" in inspect.signature(module.forward).parameters else "past_key_value"


def _swap_in_cache(module: Module, args: tuple, kwargs: dict[str, Any]):
    """forward pre-hook of a hooked attention module: its cache argument becomes the module's QuantizedKVCache"""
    name = _cache_kwarg(module)
    cache: QuantizedKVCache = getattr(module, KV_CACHE_ATTR)
    cache.add_past_key_values(kwargs.get(name, None))
    kwargs[name] = cache
    return args, kwargs


def initialize_hooked_kv_cache(model: Module, module: Module) -> None:
    """attach a QuantizedKVCache to the attention `module` of `model` (once; calling it again changes nothing)"""
    if hasattr(module, KV_CACHE_ATTR):
        return
    config = model.config.get_text_config(decoder=True)
    module.register_module(KV_CACHE_ATTR, QuantizedKVCache(config, module))
    module.register_forward_pre_hook(_swap_in_cache, with_kwargs=True)


def _register_state_hook(module: Module, submodule: Module, argument: str, hook: Callable[[Module, Tensor], Optional[Tensor]]) -> RemovableHandle:
    """pre-hook on `submodule` that passes its `argument` to hook(module, tensor) and replaces it with a non-None result"""
    signature = inspect.signature(submodule.forward)

    def _pre_hook(_sub: Module, args: tuple, kwargs: dict):
        bound = signature.bind(*args, **kwargs)
        result = hook(module, bound.arguments[argument])
        if result is not None:
            bound.arguments[argument] = result
        return bound.args, bound.kwargs

    return submodule.register_forward_pre_hook(_pre_hook, with_kwargs=True)


def register_key_hook(module: Module, hook: Callable[[Module, Tensor], Optional[Tensor]]) -> RemovableHandle:
    """hook(module, key_states) runs on the post-RoPE key states before they are quantized; a returned tensor replaces them"""
    return _register_state_hook(module, getattr(module, KV_CACHE_ATTR), "key_states", hook)


def register_value_hook(module: Module, hook: Callable[[Module, Tensor], Optional[Tensor]]) -> RemovableHandle:
    """hook(module, value_states) runs on the value states before they are quantized; a returned tensor replaces them"""
    return _register_state_hook(module, getattr(module, KV_CACHE_ATTR), "value_states", hook)
