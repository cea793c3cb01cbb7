"""
The `random-matrix` factory (the reference's transform/factory/matrix_multiply.py): a dense random matrix and its inverse.  A general
matrix product is a GEMM, so these transforms stay dense products through torch.
"""
from __future__ import annotations

import torch
from torch import Tensor, device, dtype
from torch.nn import Module, Parameter

from ...offload import get_execution_device
from ...utils.helpers import ParameterizedDefaultDict
from .. import TransformArgs, TransformScheme
from ..utils.matrix import apply_transform_weight, get_transform_size
from .base import TransformBase, TransformFactory

__all__ = ["RandomMatrixFactory", "RandomMatrixTransform"]


@TransformFactory.register("random-matrix")
class RandomMatrixFactory(TransformFactory):
    """
    Factory of random matrix transforms

    :param name: name of the scheme's group
    :param scheme: how the transforms are created and where they apply
    :param seed: seed of the generator the matrices are drawn from
    """

    def __init__(self, name: str, scheme: TransformScheme, seed: int | None = None):
        super().__init__(name, scheme, seed)
        self.weights = ParameterizedDefaultDict(self._create_weight)
        self.inverses = ParameterizedDefaultDict(self._create_inverse)

    def create_transform(self, module: Module, args: TransformArgs):
        """a RandomMatrixTransform for `module` (holding the inverse matrix when `args.inverse`); shared per size and precision"""
        size = get_transform_size(module, args.location, self.scheme.head_dim)
        precision = self.scheme.precision if args.is_online() else torch.float64
        weight = self.weights.get(size, factory_kwargs={"device": get_execution_device(module), "precision": precision})
        if args.inverse:
            weight = self.inverses[weight]
        return RandomMatrixTransform(weight, self.scheme, args, type(module))

    def _create_weight(self, size: int, device: device, precision: dtype) -> Parameter:
        data = torch.rand((size, size), generator=self.generator, dtype=precision, device=self.generator.device).to(device)
        return Parameter(data, requires_grad=self.scheme.requires_grad)

    def _create_inverse(self, weight: Parameter) -> Parameter:
        return Parameter(high_precision_invert(weight.data).contiguous(), requires_grad=False)


class RandomMatrixTransform(TransformBase):
    def __init__(self, weight: Tensor, scheme: TransformScheme, args: TransformArgs, module_type: type[torch.nn.Module]):
        super().__init__()
        self.weight = weight   # the inverse when args.inverse
        self.scheme = scheme
        self.args = args
        self.module_type = module_type

    def forward(self, value: Tensor) -> Tensor:
        return apply_transform_weight(self.weight.to(device=value.device), value.to(dtype=self.weight.dtype), self.args.location,
                                      self.module_type).to(value.dtype)

    def right_inverse(self, value: Tensor) -> Tensor:
        inverse = high_precision_invert(self.weight)
        return apply_transform_weight(inverse.to(device=value.device), value.to(dtype=inverse.dtype), self.args.location,
                                      self.module_type).to(value.dtype)


def high_precision_invert(weight: Tensor) -> Tensor:
    """inverse of `weight` computed in float64, returned in weight's dtype and device"""
    return torch.linalg.inv(weight.to(dtype=torch.float64)).to(dtype=weight.dtype)
