"""
Attention (query) quantization hooks (the reference's modeling/attention.py): a `QuantizedAttentionImpl` submodule is called in place
of the model's attention function, through an implementation registered with transformers under the name `ct_hooked_attention`.  It
fake-quantizes the query states with the module's `q_*` qparams, then runs the model's original attention function.  Key and value
states are quantized by the module's QuantizedKVCache (kvcache.py), which `initialize_hooked_attention` attaches as well.
"""
from __future__ import annotations

from typing import Callable, Optional

from torch import Tensor
from torch.nn import Module
from torch.utils.hooks import RemovableHandle

from ..utils.internal import InternalModule
from .kvcache import _register_state_hook, initialize_hooked_kv_cache, quantize_attention_states

__all__ = ["QuantizedAttentionImpl", "initialize_hooked_attention", "register_query_hook", "IMPL_ATTR"]

IMPL_ATTR = "impl"
HOOKED_ATTENTION_NAME = "ct_hooked_attention"


class QuantizedAttentionImpl(InternalModule):
    """
    The attention function of a hooked model as a module: forward(module, query, key, value, ...) quantizes `query` and calls the
    attention implementation the model used before it was hooked (`_original_impl`, shared by all hooked modules: one hooked model
    at a time).
    """

    _original_impl = "eager"

    def __init__(self, config):
        super().__init__()
        self.config = config

    def forward(self, module: Module, query: Tensor, key: Tensor, value: Tensor, *args, **kwargs):
        from transformers.modeling_utils import ALL_ATTENTION_FUNCTIONS

        (query,) = quantize_attention_states(module, ("q",), (query,))
        return ALL_ATTENTION_FUNCTIONS[QuantizedAttentionImpl._original_impl](module, query, key, value, *args, **kwargs)


def _hooked_attention(module: Module, *args, **kwargs):
    impl = getattr(module, IMPL_ATTR, None)
    if impl is None:
        raise RuntimeError(f"the model runs the {HOOKED_ATTENTION_NAME} attention implementation, but this attention module has no "
                           f"`{IMPL_ATTR}` submodule: initialize it with initialize_hooked_attention")
    return impl(module, *args, **kwargs)


def initialize_hooked_attention(model: Module, module: Module) -> None:
    """
    Attach a QuantizedAttentionImpl and a QuantizedKVCache to the attention `module` and switch `model` to the hooked attention
    implementation (registered with transformers' attention and mask function tables; the mask function stays the original one).
    Calling it again changes nothing.
    """
    from transformers.masking_utils import ALL_MASK_ATTENTION_FUNCTIONS
    from transformers.modeling_utils import ALL_ATTENTION_FUNCTIONS

    if not hasattr(module, IMPL_ATTR):
        module.register_module(IMPL_ATTR, QuantizedAttentionImpl(model.config))
    original = model.config._attn_implementation
    if original != HOOKED_ATTENTION_NAME:
        QuantizedAttentionImpl._original_impl = original
        ALL_ATTENTION_FUNCTIONS.register(HOOKED_ATTENTION_NAME, _hooked_attention)
        ALL_MASK_ATTENTION_FUNCTIONS.register(HOOKED_ATTENTION_NAME, ALL_MASK_ATTENTION_FUNCTIONS[original])
        model.set_attn_implementation(HOOKED_ATTENTION_NAME)
        if model.config._attn_implementation != HOOKED_ATTENTION_NAME:
            raise RuntimeError(f"transformers did not switch the model to the {HOOKED_ATTENTION_NAME} attention implementation")
    initialize_hooked_kv_cache(model, module)


def register_query_hook(module: Module, hook: Callable[[Module, Tensor], Optional[Tensor]]) -> RemovableHandle:
    """hook(module, query) runs on the post-RoPE query states before they are quantized; a returned tensor replaces them"""
    return _register_state_hook(module, getattr(module, IMPL_ATTR), "query", hook)
