"""
QuantizationStatus / QuantizationConfig -- mirror of quantization/quant_config.py:56-367 for what
the compress/decompress path reads and writes (the config.json `quantization_config` block).
"""
from __future__ import annotations

from collections import defaultdict
from enum import Enum
from typing import Annotated, Any

from pydantic import BaseModel, ConfigDict, Field
from torch.nn import Module

from ..config import CompressionFormat
from .quant_args import DynamicType, QuantizationArgs
from .quant_scheme import QuantizationScheme, preset_name_to_scheme

__all__ = ["QuantizationStatus", "QuantizationConfig", "LIFECYCLE_ORDER", "DEFAULT_QUANTIZATION_METHOD", "DEFAULT_QUANTIZATION_FORMAT"]


class QuantizationStatus(str, Enum):
    """ordered life cycle of a quantized module: initialized < calibration < frozen < compressed < decompressed"""

    INITIALIZED = "initialized"
    CALIBRATION = "calibration"
    FROZEN = "frozen"
    COMPRESSED = "compressed"
    DECOMPRESSED = "decompressed"

    @classmethod
    def lifecycle_order(cls) -> list:
        """the statuses in life-cycle order (the reference's method of this name returns None, quant_config.py:79-84; the list is what
        its docstring promises and what `LIFECYCLE_ORDER` holds)"""
        return list(LIFECYCLE_ORDER)

    def _rank(self) -> int:
        return LIFECYCLE_ORDER.index(self)

    def _other(self, other):
        if not isinstance(other, QuantizationStatus):
            raise NotImplementedError
        return other._rank()

    def __ge__(self, other):
        return True if other is None else self._rank() >= self._other(other)

    def __gt__(self, other):
        return True if other is None else self._rank() > self._other(other)

    def __lt__(self, other):
        return False if other is None else self._rank() < self._other(other)

    def __le__(self, other):
        return False if other is None else self._rank() <= self._other(other)


LIFECYCLE_ORDER = [
    QuantizationStatus.INITIALIZED,
    QuantizationStatus.CALIBRATION,
    QuantizationStatus.FROZEN,
    QuantizationStatus.COMPRESSED,
    QuantizationStatus.DECOMPRESSED,
]

DEFAULT_QUANTIZATION_METHOD = "compressed-tensors"
DEFAULT_QUANTIZATION_FORMAT = "fakequant"


def _map_to_checkpoint_names(model: Module, ignore_list: list) -> list:
    """HF module names -> checkpoint names for the ignore list: transformers v5 may rename weight keys on load
    (`model._weight_conversions`); the same reverse mapping save_pretrained applies to weights (quant_config.py:31-53)"""
    conversions = getattr(model, "_weight_conversions", None)
    if not conversions:
        return ignore_list
    inverted = [c.reverse_transform() for c in reversed(conversions)]
    out = []
    for name in ignore_list:
        for rev in inverted:
            renamed, matched = rev.rename_source_key(name)
            if matched is not None:
                name = renamed
        out.append(name)
    return out


def _vllm_module_type(name: str) -> str:
    """MoE router / gate layers are matched as 'Linear' when configs are loaded (quant_config.py:370-382)"""
    if "ExpertMLP" not in name and any(k in name for k in ("Router", "Gate", "Gating")):
        return "Linear"
    return name


get_vllm_module_type = _vllm_module_type   # the reference's public name


class QuantizationConfig(BaseModel):
    """model-level quantization description; groups may be given as preset names -> target lists"""

    config_groups: dict[str, QuantizationScheme | list[str]]
    quant_method: str = DEFAULT_QUANTIZATION_METHOD
    kv_cache_scheme: QuantizationArgs | None = None
    format: str = DEFAULT_QUANTIZATION_FORMAT
    quantization_status: QuantizationStatus = QuantizationStatus.INITIALIZED
    global_compression_ratio: float | None = None
    ignore: list[str] | None = Field(default_factory=list)
    run_compressed: Annotated[Any, Field(exclude=True)] = None  # unused, kept for old configs

    model_config = ConfigDict(extra="ignore")

    def model_post_init(self, __context):
        for name, value in list(self.config_groups.items()):
            if not isinstance(value, QuantizationScheme):
                self.config_groups[name] = preset_name_to_scheme(name=name, targets=value)

    def to_dict(self):
        return self.model_dump()

    @staticmethod
    def from_pretrained(model: Module, format: str | list | None = None) -> "QuantizationConfig | None":
        """rebuild the config from the `quantization_scheme` attached to each module (quant_config.py:186-289).  A quantized cached
        attention module gives the `kv_cache_scheme`; it also forms a config group when its query is hooked (an attention target)."""
        from ..modeling import IMPL_ATTR
        from .lifecycle.initialize import is_cached_attention_module
        from .utils.helpers import is_module_quantized

        schemes: list[QuantizationScheme] = []
        status = None
        kv_cache_scheme: QuantizationArgs | None = None
        quantized_types: set[str] = set()
        unquantized: dict[str, list[str]] = defaultdict(list)
        for name, sub in model.named_modules():
            kind = _vllm_module_type(type(sub).__name__)
            quantized = is_module_quantized(sub)
            cached_attention = quantized and is_cached_attention_module(sub)
            if quantized and (not cached_attention or hasattr(sub, IMPL_ATTR)):
                status = getattr(sub, "quantization_status", status)
                quantized_types.add(kind)
                if sub.quantization_scheme not in schemes:
                    schemes.append(sub.quantization_scheme)
            else:
                unquantized[kind].append(name)
            if cached_attention:
                status = getattr(sub, "quantization_status", status)
                kv_cache_scheme = sub.quantization_scheme.input_activations
        if not schemes and kv_cache_scheme is None:
            return None
        ignore = [n for kind, names in unquantized.items() if kind in quantized_types for n in names]
        groups = {f"group_{i}": s for i, s in enumerate(schemes)}
        if format is None:
            format = (CompressionFormat.int_quantized.value if status == QuantizationStatus.COMPRESSED
                      else CompressionFormat.dense.value)
        elif isinstance(format, list):
            format = CompressionFormat.mixed_precision.value if len(format) > 1 else format[0]
        ignore = _map_to_checkpoint_names(model, ignore)
        return QuantizationConfig(config_groups=groups, quantization_status=status, kv_cache_scheme=kv_cache_scheme,
                                  global_compression_ratio=None, format=format, ignore=ignore)

    def requires_calibration_data(self) -> bool:
        if self.kv_cache_scheme is not None:
            return True
        for scheme in self.config_groups.values():
            if scheme.weights is not None and scheme.weights.observer == "imatrix_mse":
                return True
            if scheme.input_activations is not None and scheme.input_activations.dynamic in (False, DynamicType.LOCAL):
                return True
            if scheme.output_activations is not None and not scheme.output_activations.dynamic:
                return True
        return False

    def merge(self, config: "QuantizationConfig") -> None:
        """
        Fold another config into this one, in place (quant_config.py:308-363): its groups are appended under non-colliding names
        (this config keeps precedence), plain names in `ignore` that the new groups target are dropped (regex entries stay), the
        format becomes mixed-precision when the groups disagree, the status becomes the later of the two.
        """
        import warnings

        from ..utils.helpers import find_unique_name
        from ..utils.match import match_name

        warnings.warn("Attempting to merge quantization configs. This is not a straightforward task and can lead to quantization configs "
                      "that fail to load. For best results, use complex targets lists instead of complex ingore lists")
        new_targets = [t for scheme in config.config_groups.values() for t in scheme.targets]
        self.ignore = [i for i in (self.ignore or []) if i.startswith("re:") or not any(match_name(i, t) for t in new_targets)]
        for name, scheme in config.config_groups.items():
            self.config_groups[find_unique_name(name, self.config_groups.keys())] = scheme
        formats = set(scheme.format for scheme in self.config_groups.values())
        self.format = next(iter(formats)) if len(formats) == 1 else CompressionFormat.mixed_precision.value
        if config.quantization_status > self.quantization_status:
            self.quantization_status = config.quantization_status
