"""
CompressedTensorsQuantizer: a dense bf16 / fp16 checkpoint, or an FP8-block one (float8_e4m3fn weights with a float32
`weight_scale_inv` per 128 x 128 block, as DeepSeek-V3 / Kimi-K2 / Qwen3-FP8 ship them) -> a compressed-tensors checkpoint, shard by
shard, without building the model.  Each targeted weight is calibrated with the memoryless min-max observer and compressed by ONE
fused observer kernel on the job's device; the tensors written are exactly those the compressor of the inferred format writes
(ModelCompressor.compress_model after calculate_qparams on the same min / max).  A scheme whose weights name observer "mse" /
"memoryless_mse" is calibrated with the MSE shrink-grid search over each group's min / max instead (`ops.observe_*`; fused into the
group, NVFP4 and per-row channel observer kernels, torch ops on the device otherwise), with the scheme's `observer_kwargs`; the
NVFP4 global scale stays the min-max one, so fused siblings still share it.  The config records `observer` and `observer_kwargs`.

NVFP4 siblings that a serving engine runs as one GEMM (q / k / v, gate / up, w1 / w3) share one weight_global_scale: the smallest
of their per-tensor global scales, computed on the device.  `get_dependencies` makes the first member of each group (q_proj,
gate_proj, w1) depend on the others, so every group is loaded into one job even when it spans shards.
"""
from __future__ import annotations

import threading
from typing import Iterable, Optional, Union

import torch

from .... import ops
from ....compressors.format import infer_module_format
from ....config import CompressionFormat
from ....quantization import QuantizationConfig, QuantizationScheme, QuantizationStatus, preset_name_to_scheme
from ....utils.match import match_name, match_quantizable_tensors

__all__ = ["CompressedTensorsQuantizer"]

FUSED_GROUPS = (("q_proj", "k_proj", "v_proj"), ("gate_proj", "up_proj"), ("w1", "w3"))   # leader first
FP8_BLOCK = (128, 128)


def _value(v):
    return getattr(v, "value", v)


_WRITABLE = (CompressionFormat.nvfp4_pack_quantized, CompressionFormat.mxfp4_pack_quantized, CompressionFormat.mxfp8_quantized,
             CompressionFormat.pack_quantized, CompressionFormat.int_quantized, CompressionFormat.float_quantized,
             CompressionFormat.naive_quantized)


def _per_element(scale: torch.Tensor, shape) -> torch.Tensor:
    """a per-channel / per-group / per-block / per-tensor scale repeated to one value per weight element"""
    s = scale.reshape(1, 1) if scale.numel() == 1 else scale
    for d in (0, 1):
        s = s.repeat_interleave(-(-shape[d] // s.shape[d]), dim=d).narrow(d, 0, shape[d])
    return s


def _positive_zero(codes: torch.Tensor, w: torch.Tensor, scale: torch.Tensor) -> torch.Tensor:
    """float8_e4m3fn codes with +0 where the reference writes +0: its compressors compute x / scale in x's dtype and then add the
    (all-zero) zero point every weight carries until it is compressed, so a quotient that is -0 in x's dtype (a -0.0 weight, or a
    negative one whose quotient underflows) becomes +0; a negative quotient that only rounds to zero in float8 stays -0"""
    b = codes.view(torch.uint8)
    zero_quotient = (w / _per_element(scale.to(w.dtype), w.shape)) == 0
    return b.masked_fill_(zero_quotient & (b == 0x80), 0).view(torch.float8_e4m3fn)


class CompressedTensorsQuantizer:
    """
    :param scheme: a preset name ("W4A16", "FP8_DYNAMIC", "NVFP4A16", "MXFP4", ...) or a QuantizationScheme; its weights are
        quantized, its activations must be dynamic (nothing about them can be learned from the weights)
    :param targets: modules to quantize, as in the other converters (empty or "Linear": every module with a `weight`)
    :param ignore: modules to leave dense
    :param dtype: None for a dense checkpoint; for an FP8-block checkpoint, the dtype its weights are dequantized to before they are
        observed (what FP8BlockDequantizer(dtype=...) would write)
    :param fused_groups: for NVFP4, the sibling modules (last name component, first member leading) that share one global scale.
        Every member named here must exist next to its leader: planning fails with "Dependency weight ... not found" otherwise
        (e.g. MLA attention, with q_proj but no k_proj / v_proj).  Pass () to give every weight its own global scale.
    """

    def __init__(self, scheme: Union[str, QuantizationScheme], targets: Iterable[str] = ("Linear",), ignore: Iterable[str] = tuple(),
                 dtype: Optional[torch.dtype] = None, fused_groups: Iterable[Iterable[str]] = FUSED_GROUPS):
        self.targets, self.ignore, self.dtype = list(targets), list(ignore), dtype
        self.fused_groups = tuple(tuple(g) for g in fused_groups)
        self.scheme_name = scheme if isinstance(scheme, str) else None
        scheme = preset_name_to_scheme(scheme, ["Linear"]) if isinstance(scheme, str) else scheme.model_copy(deep=True)
        if scheme.weights is None:
            raise ValueError(f"scheme {self.scheme_name or scheme} quantizes no weights")
        self.scheme = scheme
        self.format = CompressionFormat(scheme.format) if scheme.format is not None else infer_module_format(torch.nn.Linear, scheme)
        if self.format not in _WRITABLE:
            raise ValueError(f"CompressedTensorsQuantizer cannot write format {self.format.value}")
        self.scheme.format = self.format.value
        args = scheme.weights
        self._nvfp4 = _value(args.type) == "float" and args.num_bits == 4 and _value(args.strategy) == "tensor_group"
        self._lock = threading.Lock()
        self._quantized: set[str] = set()

    # ------------------------------------------------------------------ planning
    def _targeted(self, module_name: str) -> bool:
        return any(True for _ in match_quantizable_tensors({f"{module_name}.weight": None}, self.ignore, self.targets))

    def get_dependencies(self, weight_name: str) -> set[str]:
        module_name, _, param = weight_name.rpartition(".")
        if param != "weight" or not self._targeted(module_name):
            return set()
        deps = {f"{module_name}.weight_scale_inv"} if self.dtype is not None else set()
        if self._nvfp4:
            parent, _, leaf = module_name.rpartition(".")
            prefix = f"{parent}." if parent else ""
            for group in self.fused_groups:
                if leaf == group[0]:
                    deps |= {f"{prefix}{m}.weight" for m in group[1:] if self._targeted(f"{prefix}{m}")}
        return deps

    # ------------------------------------------------------------------ validation (meta tensors, whole checkpoint)
    def _check_scheme(self):
        name = self.scheme_name or "the scheme"
        for kind in ("input_activations", "output_activations"):
            a = getattr(self.scheme, kind)
            if a is not None and a.dynamic is not True:
                raise ValueError(f"{name}: {kind} need static calibration (dynamic={_value(a.dynamic)!r}); a model-free conversion can only "
                                 "write schemes whose activations are quantized dynamically")
        if self.scheme.weights.actorder is not None:
            raise ValueError(f"{name}: activation ordering needs calibration data")
        if self.scheme.weights.dynamic is not False:
            raise ValueError(f"{name}: weights must be quantized statically")
        ops._mse_params(self.scheme.weights)   # an MSE observer's kwargs are checked before any shard is written

    def validate(self, tensors: dict[str, torch.Tensor]):
        self._check_scheme()
        args = self.scheme.weights
        targeted = {n for _, n in match_quantizable_tensors(tensors, self.ignore, self.targets, param_targets=["weight", "weight_scale_inv"])}
        quantized = set()
        for name, t in tensors.items():
            module_name, _, param = name.rpartition(".")
            if param == "weight_scale_inv":
                if name not in targeted and not any(match_name(module_name, i) for i in self.ignore):
                    raise ValueError(f"Found unexpected non-targeted tensor {name}")
                if f"{module_name}.weight" not in tensors:
                    raise ValueError(f"Found weight_scale_inv without corresponding weight {name}")
                continue
            if param != "weight":
                continue
            if name not in targeted:
                continue
            if t.ndim != 2 or not t.is_floating_point():
                raise ValueError(f"{name}: targeted tensor is not a 2-D floating-point weight (shape {tuple(t.shape)}, {t.dtype})")
            has_inv = f"{module_name}.weight_scale_inv" in tensors
            if self.dtype is not None and not has_inv:
                raise ValueError(f"Found weight without corresponding weight_scale_inv {name}")
            if has_inv and self.dtype is None:
                raise ValueError(f"{name} has a weight_scale_inv: pass the dtype to dequantize FP8-block weights to")
            if has_inv:
                inv = tensors[f"{module_name}.weight_scale_inv"]
                grid = tuple(-(-s // b) for s, b in zip(t.shape, FP8_BLOCK))
                if t.dtype != torch.float8_e4m3fn or tuple(inv.shape) != grid:
                    raise ValueError(f"{name}: expected float8_e4m3fn with a weight_scale_inv of shape {grid}, got {t.dtype} and "
                                     f"{tuple(inv.shape)}")
            elif t.dtype not in (torch.bfloat16, torch.float16, torch.float32):
                raise ValueError(f"{name}: cannot quantize a {t.dtype} weight without a weight_scale_inv")
            gsz = args.group_size if _value(args.strategy) in ("group", "tensor_group") else None
            if gsz and t.shape[1] % gsz != 0:
                raise ValueError(f"{name}: {t.shape[1]} columns are not a multiple of the group size {gsz}")
            quantized.add(module_name)
        with self._lock:
            self._quantized |= quantized

    # ------------------------------------------------------------------ conversion
    def _compress(self, w: torch.Tensor, global_scale: Optional[torch.Tensor]) -> dict[str, torch.Tensor]:
        args, fmt = self.scheme.weights, self.format
        if fmt == CompressionFormat.nvfp4_pack_quantized:
            packed, scale, gs = ops.observe_quantize_pack_nvfp4(w, args, global_scale=global_scale)
            return {"weight_packed": packed, "weight_scale": scale, "weight_global_scale": gs}
        if fmt == CompressionFormat.mxfp4_pack_quantized:
            packed, scale = ops.observe_quantize_mx(w, args)
            return {"weight_packed": packed, "weight_scale": scale}
        if fmt == CompressionFormat.mxfp8_quantized:
            q, scale = ops.observe_quantize_mx(w, args)
            return {"weight": _positive_zero(q, w, ops.decompress_mx_scale(scale)), "weight_scale": scale}
        if fmt == CompressionFormat.pack_quantized:
            packed, scale, zp = ops.observe_quantize(w, args, pack=True)
            out = {"weight_packed": packed, "weight_scale": scale, "weight_shape": torch.tensor(w.shape)}
            if zp is not None:   # asymmetric group / channel zero points are packed along dim 0, as the compressor packs them
                out["weight_zero_point"] = ops.pack_to_int32(zp, args.num_bits, packed_dim=0) if _value(args.strategy) in ("group", "channel") else zp
            return out
        if fmt in (CompressionFormat.int_quantized, CompressionFormat.float_quantized, CompressionFormat.naive_quantized):
            q, scale, zp = ops.observe_quantize(w, args)
            out = {"weight": _positive_zero(q, w, scale) if q.dtype == torch.float8_e4m3fn else q, "weight_scale": scale}
            if zp is not None:
                out["weight_zero_point"] = zp
            return out
        raise AssertionError(fmt)   # __init__ admits only the formats above

    def process(self, tensors: dict[str, torch.Tensor]) -> dict[str, torch.Tensor]:
        weights = {}
        for module_name, name in match_quantizable_tensors(tensors, self.ignore, self.targets):
            w = tensors.pop(name)
            inv = tensors.pop(f"{module_name}.weight_scale_inv", None)
            weights[module_name] = ops.dequantize_block_fp8(w, inv, FP8_BLOCK, self.dtype) if inv is not None else w
        shared = {}
        if self._nvfp4:   # one global scale per fused group: the smallest member scale (largest amax), never leaving the device
            for module_name in weights:
                parent, _, leaf = module_name.rpartition(".")
                prefix = f"{parent}." if parent else ""
                for group in self.fused_groups:
                    if leaf == group[0]:
                        members = [f"{prefix}{m}" for m in group if f"{prefix}{m}" in weights]
                        gs = torch.stack([ops.observe_tensor_gparam(weights[m]).reshape(()) for m in members]).amin().reshape(1)
                        shared.update({m: gs.clone() for m in members})   # one tensor each: safetensors refuses shared storage
        out = {}
        for module_name, w in weights.items():
            out.update({f"{module_name}.{k}": v for k, v in self._compress(w, shared.get(module_name)).items()})
        out.update(tensors)   # untargeted tensors pass through unchanged
        return out

    def create_config(self) -> QuantizationConfig:
        """the scheme on exactly the modules the validated checkpoint had quantized, by name: tensor names cannot tell a Linear from an
        Embedding or a router, so applying the config to the model built from the checkpoint marks exactly those modules"""
        scheme = self.scheme.model_copy(deep=True)
        scheme.targets = sorted(self._quantized)
        return QuantizationConfig(config_groups={"group_0": scheme}, ignore=[], format=self.format.value,
                                  quantization_status=QuantizationStatus.COMPRESSED.value)
