"""The `random-hadamard` factory (the reference's transform/factory/random_hadamard.py): Hadamard transforms with random signs"""
from __future__ import annotations

from torch import device, dtype
from torch.nn import Parameter

from ..utils.hadamard import random_hadamard_matrix
from .base import TransformFactory
from .hadamard import HadamardFactory

__all__ = ["RandomHadamardFactory"]


@TransformFactory.register("random-hadamard")
class RandomHadamardFactory(HadamardFactory):
    """
    Factory of random Hadamard transforms: diag(Q) . H with Q drawn from the factory's generator

    :param name: name of the scheme's group
    :param scheme: how the transforms are created and where they apply
    :param seed: seed of the generator that signs and permutations are drawn from
    """

    def _create_weight(self, size: int, device: device, construct_device: device, precision: dtype) -> Parameter:
        data = random_hadamard_matrix(size, precision, construct_device, self.generator).to(device=device)
        return Parameter(data, requires_grad=self.scheme.requires_grad)
