#!/usr/bin/env python
"""
Golden vectors for CompressedTensorsQuantizer, produced with the reference's public API only (imported like make_golden.py):

  1. the seeded one-layer Llama checkpoints of quantizer_checkpoint.py (bf16, fp16, and FP8-block dequantized to bf16 by the
     reference's FP8BlockDequantizer), loaded into transformers' LlamaForCausalLM;
  2. apply_quantization_config with each preset on ["Linear"], ignoring lm_head (and embed_tokens, which is no Linear anyway);
  3. the memoryless min-max calibration: calculate_qparams on each group's / channel's / block's / tensor's min and max, and for NVFP4
     generate_gparam of every weight with q / k / v and gate / up sharing the smallest of their global scales;
  4. ModelCompressor.from_pretrained_model(model).compress_model(model)

and records every tensor of the compressed state dict (a digest, and the tensor itself up to 1024 elements) and the
quantization_config.

    python tests/golden/make_golden_quantizer.py   ->  tests/golden/quantizer.pt.gz
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as mg  # noqa: E402  (imports the reference from a temp copy)
import quantizer_checkpoint as qc  # noqa: E402

from compressed_tensors.compressors import ModelCompressor  # noqa: E402
from compressed_tensors.entrypoints.convert import FP8BlockDequantizer  # noqa: E402
from compressed_tensors.quantization import QuantizationConfig, apply_quantization_config, preset_name_to_scheme  # noqa: E402
from compressed_tensors.quantization.utils import calculate_qparams, generate_gparam  # noqa: E402

FULL_MAX = 1024
FUSED = (("q_proj", "k_proj", "v_proj"), ("gate_proj", "up_proj"))


def build_model(tensors: dict, dtype: torch.dtype):
    from transformers import LlamaConfig, LlamaForCausalLM

    cfg = qc.config_dict(dtype)
    cfg.pop("architectures"), cfg.pop("model_type"), cfg.pop("torch_dtype")
    with torch.device("meta"):
        model = LlamaForCausalLM(LlamaConfig(**cfg))
    model.load_state_dict(tensors, assign=True, strict=True)
    return model.to(dtype)


def _min_max_strategy(args) -> str:
    return getattr(args.strategy, "value", args.strategy)


def _min_max(w: torch.Tensor, args):
    s = _min_max_strategy(args)
    if s in ("group", "tensor_group"):
        g = w.unflatten(-1, (-1, args.group_size))
        return g.amin(-1), g.amax(-1)
    if s == "channel":
        return w.amin(-1, keepdim=True), w.amax(-1, keepdim=True)
    if s == "tensor":
        return w.amin().reshape(1), w.amax().reshape(1)
    if s == "block":
        bh, bw = args.block_structure
        r, c = w.shape
        p = torch.nn.functional.pad(w, (0, -(-c // bw) * bw - c, 0, -(-r // bh) * bh - r)).reshape(-(-r // bh), bh, -(-c // bw), bw)
        return p.amin(dim=(1, 3)), p.amax(dim=(1, 3))
    raise NotImplementedError(s)


@torch.no_grad()
def calibrate(model):
    mods = {n: m for n, m in model.named_modules() if getattr(m, "quantization_scheme", None) is not None}
    gscales = {}
    for name, m in mods.items():
        if _min_max_strategy(m.quantization_scheme.weights) == "tensor_group":
            gscales[name] = generate_gparam(m.weight.min(), m.weight.max())
    for name in list(gscales):
        parent, _, leaf = name.rpartition(".")
        for group in FUSED:
            if leaf == group[0]:
                members = [f"{parent}.{g}" for g in group if f"{parent}.{g}" in gscales]
                shared = torch.stack([gscales[n] for n in members]).amin(0)
                for n in members:
                    gscales[n] = shared
    for name, m in mods.items():
        args = m.quantization_scheme.weights
        gs = gscales.get(name)
        if gs is not None:
            m.weight_global_scale.data.copy_(gs)
        mn, mx = _min_max(m.weight, args)
        scale, zp = calculate_qparams(mn, mx, args, global_scale=gs)
        m.weight_scale.data.copy_(scale.reshape(m.weight_scale.shape))
        if hasattr(m, "weight_zero_point"):
            m.weight_zero_point.data.copy_(zp.reshape(m.weight_zero_point.shape))


def run(tensors: dict, dtype: torch.dtype, preset: str) -> dict:
    model = build_model(tensors, dtype)
    config = QuantizationConfig(config_groups={"group_0": preset_name_to_scheme(preset, ["Linear"])}, ignore=list(qc.IGNORE))
    apply_quantization_config(model, config)
    calibrate(model)
    compressor = ModelCompressor.from_pretrained_model(model)
    compressor.compress_model(model)
    state = {}
    for k, v in model.state_dict().items():
        v = v.detach().cpu()
        state[k] = dict(digest=qc.digest(v), dtype=str(v.dtype), shape=list(v.shape), full=v.clone() if v.numel() <= FULL_MAX else None)
    quantized = sorted(n for n, m in model.named_modules() if getattr(m, "quantization_scheme", None) is not None)
    return dict(state={k: {a: b for a, b in d.items() if b is not None} for k, d in state.items()},
                config=compressor.quantization_config.model_dump(mode="json"), quantized=quantized)


def main():
    out = {"sources": {}, "cases": []}
    sources = {"bf16": (qc.dense_tensors(torch.bfloat16), torch.bfloat16), "fp16": (qc.dense_tensors(torch.float16), torch.float16)}
    fp8 = qc.fp8_block_tensors()
    dense_from_fp8 = FP8BlockDequantizer(targets=["Linear"], ignore=list(qc.IGNORE), dtype=torch.bfloat16).process(dict(fp8))
    sources["fp8_block"] = (dense_from_fp8, torch.bfloat16)
    out["sources"]["fp8_block"] = {n: qc.digest(t) for n, t in fp8.items()}
    out["sources"]["fp8_block_dequantized"] = {n: qc.digest(t) for n, t in dense_from_fp8.items()}
    for src in ("bf16", "fp16"):
        out["sources"][src] = {n: qc.digest(t) for n, t in sources[src][0].items()}
    for src, (tensors, dtype) in sources.items():
        for preset in qc.PRESETS:
            out["cases"].append(dict(source=src, preset=preset, **run(tensors, dtype, preset)))
            print(src, preset, flush=True)
    mg.save("quantizer.pt", out)


if __name__ == "__main__":
    main()
