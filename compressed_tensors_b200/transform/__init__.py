"""
Transforms of the reference's transform/ package: the config schema (mirror of transform_args.py, transform_scheme.py,
transform_config.py; `ModelCompressor.update_config` carries a model's transform_config through to config.json), the three factories
(`hadamard`, `random-hadamard`, `random-matrix`, factory/) and `apply_transform_config` (apply.py).  Weight locations are fused into
the weights, online locations run as hooks; the two Hadamard factories run on the Walsh-Hadamard kernel (`ops.hadamard_transform`)
whenever their matrices have the structured form (DESIGN.md section 5).
"""
from __future__ import annotations

from enum import Enum

import torch
from pydantic import BaseModel, ConfigDict, Field, field_validator

from ..quantization.quant_args import TorchDtype

__all__ = [
    "TransformLocation", "TransformArgs", "TransformScheme", "TransformConfig",
    "TransformFactory", "TransformBase", "HadamardFactory", "HadamardTransform", "RandomHadamardFactory", "RandomMatrixFactory",
    "RandomMatrixTransform", "apply_transform_config",
]


class TransformLocation(str, Enum):
    INPUT = "input"
    WEIGHT_INPUT = "weight_input"
    WEIGHT_OUTPUT = "weight_output"
    OUTPUT = "output"
    K_CACHE = "k_cache"
    Q_ATTN = "q_attn"

    def is_online(self) -> bool:
        """applied to activations at run time (everything except the two weight locations)"""
        return self not in (TransformLocation.WEIGHT_INPUT, TransformLocation.WEIGHT_OUTPUT)


class TransformArgs(BaseModel, use_enum_values=True):
    targets: list[str]
    location: TransformLocation
    inverse: bool = Field(default=False)
    ignore: list[str] = Field(default_factory=list)

    @field_validator("targets", "ignore", mode="before")
    @classmethod
    def _wrap(cls, v):
        return [v] if isinstance(v, str) else v

    def is_online(self) -> bool:
        return TransformLocation(self.location).is_online()

    model_config = ConfigDict(extra="forbid")


class TransformScheme(BaseModel):
    type: str
    apply: list[TransformArgs] = Field(default_factory=list)
    randomize: bool = Field(default=False)
    requires_grad: bool = Field(default=False)
    head_dim: int | None = Field(default=None)
    precision: TorchDtype = Field(default=torch.float32)

    model_config = ConfigDict(extra="forbid")


class TransformConfig(BaseModel):
    config_groups: dict[str, TransformScheme]

    model_config = ConfigDict(extra="forbid")

    def merge(self, other: "TransformConfig") -> None:
        """append the other config's groups under keys that do not collide"""
        for key, scheme in other.config_groups.items():
            name, i = key, 0
            while name in self.config_groups:
                i += 1
                name = f"{key}_{i}"
            self.config_groups[name] = scheme


# the factories and apply_transform_config import the schema above (same order as the reference's transform/__init__.py)
from .factory.base import TransformBase, TransformFactory  # noqa: E402
from .factory.hadamard import HadamardFactory, HadamardTransform  # noqa: E402
from .factory.matrix_multiply import RandomMatrixFactory, RandomMatrixTransform  # noqa: E402
from .factory.random_hadamard import RandomHadamardFactory  # noqa: E402
from .apply import apply_transform_config  # noqa: E402
