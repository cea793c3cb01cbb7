"""
apply_quantization_config: walk a model, match module names / class names against the config's
targets and ignore list, attach schemes and qparams (mirror of quantization/lifecycle/apply.py:100-169
for Linear / Embedding targets, attention modules and the KV cache -- the last two through the hooks of `modeling/`).

Target syntax (utils/match.py of the reference): a target matches a module when it equals the
module name, equals the class name, or is "re:<regex>" matching either.
"""
from __future__ import annotations

import logging
from collections import OrderedDict
from copy import deepcopy

import torch
from torch.nn import Module

from ...utils.match import is_match, is_narrow_match, match_named_modules, match_targets
from ..quant_args import QuantizationArgs
from ..quant_config import QuantizationConfig, QuantizationStatus
from ..quant_scheme import QuantizationScheme
from ..utils.helpers import KV_CACHE_TARGETS
from .initialize import initialize_module_for_quantization, is_cached_attention_module

__all__ = ["apply_quantization_config", "is_match", "match_named_modules", "load_pretrained_quantization_parameters"]

_LOGGER = logging.getLogger(__name__)


def apply_quantization_config(model: Module, config: QuantizationConfig | None, run_compressed: bool = False, show_progress: bool = False):
    """quantization/lifecycle/apply.py:100-192.  A module that matches several targets takes the scheme of the most specific one
    (`match_targets`: exact name, then regex on the name, then class name -- apply.py:149-151, :258-265), not the first in config
    order.  A `kv_cache_scheme` is applied to every cached attention module first; a config group that narrowly targets a cached
    attention module hooks its query, key and value states (modeling/).  Unlike the reference, a `kv_cache_scheme` that no module
    of the model can take raises instead of being dropped."""
    config = deepcopy(config)
    if config is None:
        return dict()
    force_zero_point = config.quantization_status < QuantizationStatus.COMPRESSED
    if getattr(config, "kv_cache_scheme", None) is not None:
        _apply_kv_cache_scheme(model, config.kv_cache_scheme, config.quantization_status)
    target_to_scheme = OrderedDict()
    for scheme in config.config_groups.values():
        for target in scheme.targets:
            target_to_scheme[target] = scheme
    for name, module in match_named_modules(model, target_to_scheme, config.ignore, warn_on_fail=True):
        scheme = target_to_scheme[match_targets(name, module, target_to_scheme)[0]]
        if is_cached_attention_module(module) and is_narrow_match(model, scheme.targets, name):
            from ...modeling import initialize_hooked_attention

            module.quantization_scheme = scheme
            initialize_hooked_attention(model, module)
            initialize_module_for_quantization(module, force_zero_point=force_zero_point)
            module.quantization_status = config.quantization_status
        elif isinstance(module, (torch.nn.Linear, torch.nn.Embedding)):
            module.quantization_scheme = scheme
            initialize_module_for_quantization(module, force_zero_point=force_zero_point)
            module.quantization_status = config.quantization_status


def _apply_kv_cache_scheme(model: Module, kv_cache_scheme: QuantizationArgs, status: QuantizationStatus) -> None:
    """k / v qparams and a QuantizedKVCache on every cached attention module (apply.py:172-192).  Runs before the config groups, so
    that an attention target initialised afterwards keeps its own q / k / v qparams."""
    if not kv_cache_scheme.symmetric:
        _LOGGER.warning("vLLM does not support asymmetric kv cache quantization")
    from ...modeling import initialize_hooked_kv_cache

    scheme = QuantizationScheme(targets=list(KV_CACHE_TARGETS), input_activations=kv_cache_scheme)
    modules = [m for m in model.modules() if is_cached_attention_module(m)]
    if not modules:
        raise NotImplementedError(
            "KV-cache quantization: the config has a `kv_cache_scheme`, but no attention module of this model could take it (an "
            "attention module whose forward takes `past_key_values`); refusing to drop the scheme silently")
    for module in modules:
        module.quantization_scheme = scheme
        initialize_hooked_kv_cache(model, module)
        initialize_module_for_quantization(module, force_zero_point=False)
        module.quantization_status = status


def load_pretrained_quantization_parameters(model: Module, model_name_or_path: str | None = None, load_weight_qparams: bool = False) -> None:
    """Copy the quantization parameters stored in a saved checkpoint into a model that `apply_quantization_config` has already
    initialised (apply.py:49-97, :195-236): input / output scales, zero points and g_idx always, the weight ones when asked.  A scale
    without a stored zero point (symmetric schemes) gets zeros.  `model_name_or_path` is a local checkpoint directory (or one
    .safetensors file): this engine has no download path."""
    from safetensors import safe_open

    from ...offload import update_offload_parameter
    from ...utils.safetensors_load import get_quantization_parameter_to_path_mapping
    from ..utils.helpers import is_module_quantized

    mapping = get_quantization_parameter_to_path_mapping(str(model_name_or_path))

    def read(full_name: str):
        path = mapping.get(full_name)
        if path is None:
            return None
        with safe_open(path, framework="pt", device="cpu") as f:
            return f.get_tensor(full_name)

    for name, module in model.named_modules():
        if not is_module_quantized(module):
            continue
        scheme = module.quantization_scheme
        bases = [b for b, on in (("input", scheme.input_activations is not None), ("output", scheme.output_activations is not None),
                                 ("weight", load_weight_qparams and scheme.weights is not None)) if on]
        for base in bases:
            g_idx = read(f"{name}.{base}_g_idx")
            if g_idx is not None:
                update_offload_parameter(module, f"{base}_g_idx", g_idx)
            scale = read(f"{name}.{base}_scale")
            if scale is None:
                continue
            update_offload_parameter(module, f"{base}_scale", scale)
            zp = read(f"{name}.{base}_zero_point")
            update_offload_parameter(module, f"{base}_zero_point", zp if zp is not None else torch.zeros_like(scale, device="cpu"))
