"""apply_transform_config (the reference's transform/apply.py)"""
from __future__ import annotations

import torch

from ..offload import disable_onloading
from . import TransformConfig
from .factory.base import TransformBase, TransformFactory

__all__ = ["apply_transform_config"]

TRANSFORM_CONFIG_NAME = "transform_config"


def apply_transform_config(model: torch.nn.Module, config: TransformConfig):
    """
    Apply a transform config to a model: weight transforms are fused into the weights, activation transforms are attached as
    submodules and run from hooks.  The config is attached to the model as `transform_config` for compression and serialization.

    :param model: model to apply the config to
    :param config: transform config to apply
    """
    for name, scheme in config.config_groups.items():
        TransformFactory.from_scheme(scheme, name=name).apply_to_model(model)
    _register_tied_transform_weights(model)
    setattr(model, TRANSFORM_CONFIG_NAME, config)


def _register_tied_transform_weights(model: torch.nn.Module):
    """
    Declare parameters that several transform submodules share as tied weights (`_tied_weights_keys` of every module after the
    first that holds them, mapping its key to the first full name), so that `save_pretrained` writes each shared tensor once.
    """
    first_seen: dict[int, str] = {}
    with disable_onloading():
        for module_name, module in model.named_modules():
            if not isinstance(module, TransformBase):
                continue
            tied_keys: dict[str, str] = {}
            for key in getattr(module, "_dynamic_tied_weights_keys", []):
                param = getattr(module, key, None)
                if param is None:
                    continue
                full_key = f"{module_name}.{key}" if module_name else key
                if id(param) not in first_seen:
                    first_seen[id(param)] = full_key
                else:
                    tied_keys[key] = first_seen[id(param)]
            if tied_keys:
                module._tied_weights_keys = tied_keys
