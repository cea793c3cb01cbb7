"""
The seeded checkpoints behind tests/golden/quantizer.pt.gz: a one-layer Llama whose `down_proj` is 16512 columns wide (wider than one
CTA of the channel observer holds) and whose q / k / v and gate / up sit in different shards, in bf16 and fp16, and the same model as an
FP8-block checkpoint (float8_e4m3fn weights with one float32 `weight_scale_inv` per 128 x 128 block, as DeepSeek-V3 ships them).
Shared by the golden generator (which runs the reference) and the tests (which run the converter), so both see the same tensors;
the golden stores a digest of every input tensor to prove it.
"""
import hashlib
import json
import os

import torch

HIDDEN, INTERMEDIATE, HEADS, KV_HEADS, HEAD_DIM, VOCAB = 128, 16512, 2, 1, 64, 256
PRESETS = ("W4A16", "W4A16_ASYM", "W8A16", "W4A8", "W4AFP8", "W8A8", "INT8", "FP8_DYNAMIC", "FP8_BLOCK", "NVFP4A16", "MXFP4A16", "MXFP4",
           "MXFP8A16", "MXFP8")
IGNORE = ("lm_head", "re:.*embed_tokens$")   # the model-free flow cannot tell an Embedding from a Linear: name it
SHARDS = {   # shard file -> tensors in it; q / k / v and gate / up are split across shards on purpose
    "model-00001-of-00003.safetensors": ("model.embed_tokens.weight", "model.layers.0.input_layernorm.weight", "model.layers.0.self_attn.q_proj.weight"),
    "model-00002-of-00003.safetensors": ("model.layers.0.self_attn.k_proj.weight", "model.layers.0.self_attn.o_proj.weight",
                                         "model.layers.0.mlp.gate_proj.weight", "model.layers.0.post_attention_layernorm.weight"),
    "model-00003-of-00003.safetensors": ("model.layers.0.self_attn.v_proj.weight", "model.layers.0.mlp.up_proj.weight",
                                         "model.layers.0.mlp.down_proj.weight", "model.norm.weight", "lm_head.weight"),
}
LINEARS = ("self_attn.q_proj", "self_attn.k_proj", "self_attn.v_proj", "self_attn.o_proj", "mlp.gate_proj", "mlp.up_proj", "mlp.down_proj")


def config_dict(dtype: torch.dtype) -> dict:
    return dict(architectures=["LlamaForCausalLM"], model_type="llama", hidden_size=HIDDEN, intermediate_size=INTERMEDIATE,
                num_hidden_layers=1, num_attention_heads=HEADS, num_key_value_heads=KV_HEADS, head_dim=HEAD_DIM, vocab_size=VOCAB,
                max_position_embeddings=64, tie_word_embeddings=False, torch_dtype=str(dtype).split(".")[-1])


def _shape(name: str):
    if "layernorm" in name or name == "model.norm.weight":
        return (HIDDEN,)
    if "embed_tokens" in name or name.startswith("lm_head"):
        return (VOCAB, HIDDEN)
    out, inp = {"q_proj": (HEADS * HEAD_DIM, HIDDEN), "k_proj": (KV_HEADS * HEAD_DIM, HIDDEN), "v_proj": (KV_HEADS * HEAD_DIM, HIDDEN),
                "o_proj": (HIDDEN, HEADS * HEAD_DIM), "gate_proj": (INTERMEDIATE, HIDDEN), "up_proj": (INTERMEDIATE, HIDDEN),
                "down_proj": (HIDDEN, INTERMEDIATE)}[name.split(".")[-2]]
    return (out, inp)


def dense_tensors(dtype: torch.dtype) -> dict:
    """the dense checkpoint: Gaussian weights with per-row spread (so channels differ), a few outliers, one all-zero row in
    down_proj and in v_proj (the scale that replaces a zero one), and an o_proj row whose tiny negative weights divide to -0"""
    g = torch.Generator().manual_seed(20261017)
    out = {}
    for shard in SHARDS.values():
        for name in shard:
            shp = _shape(name)
            if len(shp) == 1:
                out[name] = (1 + 0.1 * torch.randn(shp, generator=g)).to(dtype)
                continue
            w = torch.randn(shp, generator=g) * (0.02 * (0.25 + torch.rand(shp[0], 1, generator=g) * 2))
            idx = torch.randint(0, w.numel(), (8,), generator=g)
            w.view(-1)[idx] *= 40
            if name.endswith(("down_proj.weight", "v_proj.weight")):
                w[3] = 0
            if name.endswith("o_proj.weight"):   # large row max + the smallest negative subnormals: x / scale underflows to -0
                w[5, 0] = 1000
                w[5, 1:9] = -(2.0 ** -24 if dtype == torch.float16 else 2.0 ** -133)
            out[name] = w.to(dtype)
    return out


def fp8_block_tensors() -> dict:
    """the FP8-block checkpoint: every Linear weight as float8_e4m3fn codes plus a float32 weight_scale_inv [ceil(R/128), ceil(C/128)];
    embeddings, norms and lm_head in bf16"""
    g = torch.Generator().manual_seed(7171)
    out = {}
    for name, t in dense_tensors(torch.bfloat16).items():
        if any(name.endswith(f"{m}.weight") for m in LINEARS):
            r, c = t.shape
            out[name] = (torch.randn(r, c, generator=g) * 64).clamp(-448, 448).to(torch.float8_e4m3fn)
            out[name[: -len("weight")] + "weight_scale_inv"] = torch.rand(-(-r // 128), -(-c // 128), generator=g) * 1e-3 + 1e-5
        else:
            out[name] = t
    return out


def write_checkpoint(directory: str, tensors: dict, dtype: torch.dtype) -> None:
    """safetensors shards + index + config.json, with every weight_scale_inv in its weight's shard except q_proj's (in the last one)"""
    from safetensors.torch import save_file

    os.makedirs(directory, exist_ok=True)
    placement = {n: f for f, names in SHARDS.items() for n in names}
    for n in tensors:
        if n.endswith("weight_scale_inv"):
            placement[n] = list(SHARDS)[-1] if "q_proj" in n else placement[n[: -len("_scale_inv")]]
    weight_map = {}
    for f in SHARDS:
        part = {n: t.contiguous() for n, t in tensors.items() if placement[n] == f}
        save_file(part, os.path.join(directory, f))
        weight_map.update({n: f for n in part})
    with open(os.path.join(directory, "model.safetensors.index.json"), "w") as fh:
        json.dump({"metadata": {"total_size": sum(t.nbytes for t in tensors.values())}, "weight_map": weight_map}, fh)
    with open(os.path.join(directory, "config.json"), "w") as fh:
        json.dump(config_dict(dtype), fh)


def digest(t: torch.Tensor) -> str:
    """sha256 over dtype, shape and the raw bytes"""
    h = hashlib.sha256(f"{t.dtype}{tuple(t.shape)}".encode())
    if t.numel():
        dense = torch.empty((t.numel(),), dtype=t.dtype).copy_(t.detach().cpu().reshape(-1))   # fresh standard strides
        h.update(dense.view(torch.uint8).numpy().tobytes())
    return h.hexdigest()
