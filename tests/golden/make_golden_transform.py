#!/usr/bin/env python
"""
Golden vectors for transforms (the reference's transform/ package), recorded by importing the reference exactly like make_golden.py
does.  Needs transformers.

    python tests/golden/make_golden_transform.py   ->  tests/golden/transform.pt.gz

Factory level ("factory" cases), for every type x randomize x location x head_dim in {None, 8} x bf16 / fp16 / fp32, on a seeded
Linear(16, 64) with bias: the transform's `weight` and `perm` (factory seed FACTORY_SEED), its output on a seeded input (online
locations) or the fused weight and bias (weight locations).

Model level ("model" cases), on the seeded 2-layer Llama of make_golden_kv.py (bf16): a SpinQuant-like config (R1 hidden size via
weight_output / weight_input, R2 per head on v / o, R3 on q_attn / k_cache, R4 on the down_proj input) and a QuIP-like
random-hadamard config, each alone and followed by W4A16 (group 64) with an FP8 per-tensor kv_cache_scheme (weight scales from the
per-group min / max, Q / K / V scales fixed): logits, parameter names / shapes / dtypes, the tied-weight keys of every transform module
and the transform_config ModelCompressor.update_config writes.
"""
import json
import os
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as mg  # noqa: E402  (imports the reference from a temp copy)
import make_golden_kv as mgkv  # noqa: E402

from compressed_tensors.compressors import ModelCompressor  # noqa: E402
from compressed_tensors.quantization import QuantizationConfig, apply_quantization_config  # noqa: E402
from compressed_tensors.quantization.utils import calculate_qparams  # noqa: E402
from compressed_tensors.transform import (  # noqa: E402
    TransformArgs,
    TransformBase,
    TransformConfig,
    TransformFactory,
    TransformScheme,
    apply_transform_config,
)

FACTORY_SEED = 42
TYPES = ("hadamard", "random-hadamard", "random-matrix")
LOCATIONS = ("input", "weight_input", "weight_output", "output")
DTYPES = (torch.bfloat16, torch.float16, torch.float32)


def factory_cases():
    out = []
    for type_ in TYPES:
        for randomize in (False, True):
            for location in LOCATIONS:
                for head_dim in (None, 8):
                    for dtype in DTYPES:
                        torch.manual_seed(7)
                        module = torch.nn.Linear(16, 64, bias=True).to(dtype)
                        scheme = TransformScheme(type=type_, randomize=randomize, head_dim=head_dim)
                        factory = TransformFactory.from_scheme(scheme, name="", seed=FACTORY_SEED)
                        args = TransformArgs(targets="Linear", location=location)
                        tfm = factory.create_transform(module, args)
                        case = dict(type=type_, randomize=randomize, location=location, head_dim=head_dim, dtype=str(dtype),
                                    weight=tfm.weight.detach().clone(), perm=getattr(tfm, "perm", None),
                                    module_weight=module.weight.detach().clone(), module_bias=module.bias.detach().clone())
                        if case["perm"] is not None:
                            case["perm"] = case["perm"].detach().clone()
                        with torch.no_grad():
                            if args.is_online():
                                width = 16 if location == "input" else 64
                                x = torch.randn(3, 5, width, generator=torch.Generator().manual_seed(11)).to(dtype)
                                case["x"], case["y"] = x, tfm(x)
                            else:
                                case["fused_weight"] = tfm(module.weight)
                                if location == "weight_output":
                                    case["fused_bias"] = tfm(module.bias.unsqueeze(-1)).squeeze(-1)
                        out.append(case)
    return out


HIDDEN = ["re:.*q_proj$", "re:.*k_proj$", "re:.*v_proj$", "re:.*up_proj$", "re:.*gate_proj$", "lm_head"]
SPINQUANT = dict(config_groups={
    "R1": dict(type="hadamard", apply=[
        dict(targets=["re:.*embed_tokens$", "re:.*o_proj$", "re:.*down_proj$"], location="weight_output"),
        dict(targets=HIDDEN, location="weight_input", inverse=True)]),
    "R2": dict(type="hadamard", head_dim=64, apply=[
        dict(targets=["re:.*v_proj$"], location="weight_output"),
        dict(targets=["re:.*o_proj$"], location="weight_input", inverse=True)]),
    "R3": dict(type="hadamard", head_dim=64, apply=[
        dict(targets=["re:.*self_attn$"], location="q_attn"),
        dict(targets=["re:.*self_attn$"], location="k_cache")]),
    "R4": dict(type="hadamard", apply=[
        dict(targets=["re:.*down_proj$"], location="input"),
        dict(targets=["re:.*down_proj$"], location="weight_input", inverse=True)]),
})
QUIP = dict(config_groups={
    "v": dict(type="random-hadamard", randomize=True, apply=[
        dict(targets=["Linear"], ignore=["lm_head"], location="input"),
        dict(targets=["Linear"], ignore=["lm_head"], location="weight_input", inverse=True)]),
    "u": dict(type="random-hadamard", apply=[
        dict(targets=["Linear"], ignore=["lm_head"], location="weight_output"),
        dict(targets=["Linear"], ignore=["lm_head"], location="output", inverse=True)]),
})
W4A16_KV = dict(config_groups={"w": dict(targets=["Linear"], weights=dict(num_bits=4, type="int", symmetric=True, strategy="group",
                                                                          group_size=64, dynamic=False))},
                ignore=["lm_head"], kv_cache_scheme=mgkv.FP8_TENSOR)
KV_SCALE = 0.0625


def calibrate(model):
    """weight scales from the per-group min / max, Q / K / V scales fixed: every scale is set, none is left as allocated"""
    for m in model.modules():
        scheme = getattr(m, "quantization_scheme", None)
        if scheme is None:
            continue
        if scheme.weights is not None and hasattr(m, "weight_scale"):
            g = scheme.weights.group_size
            w = m.weight.detach().reshape(m.weight.shape[0], -1, g)
            scale, zp = calculate_qparams(w.amin(-1), w.amax(-1), scheme.weights)
            m.weight_scale.data.copy_(scale.reshape(m.weight_scale.shape))
            m.weight_zero_point.data.copy_(zp.reshape(m.weight_zero_point.shape))
        for base in ("q", "k", "v"):   # the query too: R3 on q_attn makes the kv_cache_scheme quantize Q
            if hasattr(m, f"{base}_scale"):
                getattr(m, f"{base}_scale").data.fill_(KV_SCALE)


def model_case(name, tcfg, quant):
    model = mgkv.build_model(torch.bfloat16)
    config = TransformConfig(**tcfg)
    apply_transform_config(model, config)
    if quant:
        apply_quantization_config(model, QuantizationConfig(**W4A16_KV))
        calibrate(model)
    ids = torch.randint(0, mgkv.MODEL["vocab_size"], (1, 8), generator=torch.Generator().manual_seed(mgkv.SEED + 1))
    with torch.no_grad():
        logits = model(ids, use_cache=False).logits
    params = [(n, tuple(p.shape), str(p.dtype)) for n, p in model.named_parameters()]
    tied = {n: dict(getattr(m, "_tied_weights_keys", None) or {}) for n, m in model.named_modules() if isinstance(m, TransformBase)}
    compressor = ModelCompressor.from_pretrained_model(model)
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "config.json"), "w") as f:
            json.dump({}, f)
        compressor.update_config(d)
        with open(os.path.join(d, "config.json")) as f:
            written = json.load(f)
    return dict(name=name, quant=quant, config=tcfg, ids=ids, logits=logits, params=params, tied=tied, written=written)


def main():
    out = dict(factory=factory_cases(), model=[model_case(n, c, q) for n, c in (("spinquant", SPINQUANT), ("quip", QUIP))
                                              for q in (False, True)])
    mg.save("transform.pt", out)


if __name__ == "__main__":
    main()
