"""
Size and dense application of a transform matrix at a module location (the reference's transform/utils/matrix.py).

With x the input activation, y = x W^T the output of a Linear, V / U transform matrices on the input / output side and Vi the
inverse of V:  x' = x V,  W' = U^T W Vi^T,  y' = y U  keep  y' = x' W'^T.  An Embedding (y = x W) is handled the same way with
W in place of W^T.  A matrix smaller than the dimension it multiplies is applied block-diagonally (one block per head).
"""
from __future__ import annotations

import torch

from .. import TransformLocation

__all__ = ["get_transform_size", "apply_transform_weight"]


def get_transform_size(module: torch.nn.Module, location: TransformLocation, head_dim: int | None = None) -> int:
    """order of the transform matrix of `module` at `location` (`head_dim` when given; it must divide the dimension)"""
    size = None
    on_input = location in (TransformLocation.INPUT, TransformLocation.WEIGHT_INPUT)
    if isinstance(module, torch.nn.Linear):
        size = module.in_features if on_input else module.out_features
    elif isinstance(module, torch.nn.Embedding):
        size = module.num_embeddings if on_input else module.embedding_dim
    elif head_dim is None:
        raise NotImplementedError(f"Transforms on {type(module)} are not supported without head_dim")

    if head_dim is not None:
        if size is not None and size % head_dim != 0:
            raise ValueError(f"{head_dim} must divide {size} for {type(module)} at {location}")
        size = head_dim
    return size


def apply_transform_weight(transform_weight: torch.Tensor, value: torch.Tensor, location: TransformLocation,
                           module_type: type[torch.nn.Module]) -> torch.Tensor:
    """`value` with `transform_weight` applied as `location` of a module of type `module_type` requires (see the module docstring)"""
    assert transform_weight.shape[0] == transform_weight.shape[1]
    if TransformLocation(location).is_online():
        return _multihead_matmul(value, transform_weight)
    if module_type == torch.nn.Linear:
        if location == TransformLocation.WEIGHT_INPUT:
            return _multihead_matmul(value, transform_weight.T)
        if location == TransformLocation.WEIGHT_OUTPUT:
            return _multihead_matmul(transform_weight.T, value)
    elif module_type == torch.nn.Embedding:
        if location == TransformLocation.WEIGHT_INPUT:
            return _multihead_matmul(transform_weight, value)
        if location == TransformLocation.WEIGHT_OUTPUT:
            return _multihead_matmul(value, transform_weight)
    raise NotImplementedError(f"Applying transforms to {module_type} {location} is not supported")


def _multihead_matmul(A: torch.Tensor, B: torch.Tensor) -> torch.Tensor:
    """A @ B where the smaller of A's last and B's second-to-last dimension repeats block-diagonally to the larger one"""
    k_a, k_b = A.shape[-1], B.shape[-2]
    if k_a > k_b:
        return (A.unflatten(-1, (k_a // k_b, k_b)) @ B).flatten(-2, -1)
    if k_a < k_b:
        return (A @ B.unflatten(-2, (k_b // k_a, k_a))).flatten(-3, -2)
    return A @ B
