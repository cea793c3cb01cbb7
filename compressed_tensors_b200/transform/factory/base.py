"""
Transform factories and the transform modules they attach (the reference's transform/factory/base.py).

A factory builds one transform module per (module, TransformArgs) of its scheme and applies it at the args' location:
  input / output          forward pre-hook / forward hook on the module
  weight_input / output   fused into the weight (and, for weight_output, the bias) once; the transform submodule is then dropped,
                          unless the scheme `requires_grad`, where it stays as a parametrization of the weight
  q_attn / k_cache        query / key hooks of modeling/ (transformers is imported only for these)
"""
from __future__ import annotations

from abc import ABC, abstractmethod

import torch
import torch.nn.utils.parametrize as P
from torch import Tensor
from torch.nn import Module, Parameter

from ...distributed import is_distributed
from ...modeling.attention import initialize_hooked_attention, register_query_hook
from ...modeling.kvcache import initialize_hooked_kv_cache, register_key_hook
from ...offload import OffloadCache, align_module_device, register_offload_module, update_offload_parameter
from ...registry.registry import RegistryMixin
from ...utils.helpers import patch_attr
from ...utils.internal import InternalModule
from ...utils.match import match_named_modules
from .. import TransformArgs, TransformLocation, TransformScheme

__all__ = ["TransformFactory", "TransformBase"]


class TransformFactory(RegistryMixin, ABC):
    """
    Abstract factory of the transforms of one scheme

    :param name: name of the scheme's group (the transform submodules are named `{name}_{location}`)
    :param scheme: how the transforms are created and where they apply
    :param seed: seed of the generator that randomized transforms draw from
    """

    transforms: list["TransformBase"]

    def __init__(self, name: str, scheme: TransformScheme, seed: int | None = None):
        self.name = name
        self.scheme = scheme
        self.generator = torch.Generator()
        if seed is not None:
            self.generator.manual_seed(seed)

    @classmethod
    def from_scheme(cls, scheme: TransformScheme, **kwargs) -> "TransformFactory":
        """the registered factory of `scheme.type`, constructed with `scheme` and `kwargs`"""
        constructor = cls.get_value_from_registry(name=scheme.type)
        return constructor(scheme=scheme, **kwargs)

    @abstractmethod
    def create_transform(self, module: Module, args: TransformArgs) -> "TransformBase":
        """the transform that applies to `module` as `args` says (factories may share weights between transforms)"""
        raise NotImplementedError()

    def apply_to_model(self, model: Module, use_tqdm=True):
        """create the scheme's transforms for every matching module of `model` and apply them"""
        modules_args = [(module, arg) for arg in self.scheme.apply for _, module in match_named_modules(model, arg.targets, arg.ignore)]
        if use_tqdm:
            import tqdm
            import torch.distributed as dist

            modules_args = tqdm.tqdm(modules_args, desc=f"Applying {self.name} transforms",
                                     position=(dist.get_rank() if is_distributed() else 0))
        for module, arg in modules_args:
            self._apply_to_module(model, module, arg)

    def _apply_to_module(self, model: Module, module: Module, args: TransformArgs):
        """create the transform of `module` for `args` and apply it at its location"""
        transform_name = f"{self.name}_{args.location}"
        transform = self.create_transform(module, args)
        register_offload_module(module, transform_name, transform)   # offloaded like `module` when it is offloaded

        if args.location == TransformLocation.INPUT:

            def input_hook(_, args):
                return transform(args[0])

            module.register_forward_pre_hook(input_hook, prepend=True)

        elif args.location in (TransformLocation.WEIGHT_INPUT, TransformLocation.WEIGHT_OUTPUT):
            assert hasattr(module, "weight")
            # an offloaded module's weight is onloaded once, fused on the onload device and written back to its cache
            with torch.no_grad(), align_module_device(module):
                update_offload_parameter(module, "weight", transform(module.weight))
                # y' = R (W x + b) = (R W) x + R b: a rotated output needs the rotated bias too
                if args.location == TransformLocation.WEIGHT_OUTPUT and getattr(module, "bias", None) is not None:
                    update_offload_parameter(module, "bias", transform(module.bias.unsqueeze(-1)).squeeze(-1))

            if self.scheme.requires_grad:
                # training: the weight is recomputed from the transform on every forward, so gradients reach the transform
                if isinstance(module._parameters, OffloadCache):
                    raise ValueError("Offloaded training is not supported")
                P.register_parametrization(module, "weight", transform)
            else:
                delattr(module, transform_name)   # fused; unfusing is not supported

        elif args.location == TransformLocation.OUTPUT:

            def output_hook(_, _input, output):
                return transform(output)

            module.register_forward_hook(output_hook)

        elif args.location == TransformLocation.Q_ATTN:
            _require_pretrained(model)

            def query_hook(_, query_states):
                return transform(query_states)

            initialize_hooked_attention(model, module)
            register_query_hook(module, query_hook)

        elif args.location == TransformLocation.K_CACHE:
            _require_pretrained(model)

            def key_hook(_, key_states):
                return transform(key_states)

            initialize_hooked_kv_cache(model, module)
            register_key_hook(module, key_hook)

        else:
            raise NotImplementedError()


def _require_pretrained(model: Module) -> None:
    from transformers import PreTrainedModel

    if not isinstance(model, PreTrainedModel):
        raise ValueError(f"Cannot hook attention of model: {model}")


class TransformBase(InternalModule, ABC):
    """the application of one transform according to its TransformArgs"""

    args: TransformArgs
    weight: Parameter
    _dynamic_tied_weights_keys: list[str] = ["weight"]

    @abstractmethod
    def forward(self, value: Tensor) -> Tensor:
        raise NotImplementedError()

    def right_inverse(self, value: Tensor) -> Tensor:
        with patch_attr(self.args, "inverse", not self.args.inverse):
            return self.forward(value)

    def __repr__(self):
        return f"{self.__class__.__name__}(inverse={self.args.inverse})"
