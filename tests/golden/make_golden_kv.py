#!/usr/bin/env python
"""
Golden vectors for KV-cache and attention quantization (the reference's modeling/ hooks, `_apply_kv_cache_scheme` and the attention
branch of apply_quantization_config), recorded on a small seeded LlamaForCausalLM built from a LlamaConfig, by importing the reference
exactly like make_golden.py does.  Needs transformers.

    python tests/golden/make_golden_kv.py   ->  tests/golden/kv.pt.gz

Per (case, dtype): the model seed and config, the input ids, per layer the pre-quantization Q / K / V (register_*_hook) and the
post-quantization ones (forward hooks on the QuantizedKVCache; the query as the original attention function receives it), the
logits (use_cache=False), name / shape / dtype of every parameter after apply, the attention implementation,
QuantizationConfig.from_pretrained(model).model_dump() and the attention modules' own tensors after ModelCompressor.compress_model and then decompress_model.
Scales are set from a first, unquantized pass: the observer's min / max over the tensor (TENSOR) or per head (ATTN_HEAD) through
calculate_qparams.
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as mg  # noqa: E402  (imports the reference from a temp copy)

from compressed_tensors.compressors import ModelCompressor  # noqa: E402
from compressed_tensors.modeling import (  # noqa: E402
    IMPL_ATTR,
    KV_CACHE_ATTR,
    QuantizedAttentionImpl,
    register_key_hook,
    register_query_hook,
    register_value_hook,
)
from compressed_tensors.quantization import QuantizationArgs, QuantizationConfig, apply_quantization_config  # noqa: E402
from compressed_tensors.quantization.utils import calculate_qparams  # noqa: E402
from transformers import LlamaConfig, LlamaForCausalLM  # noqa: E402
from transformers.modeling_utils import ALL_ATTENTION_FUNCTIONS  # noqa: E402

MODEL = dict(num_hidden_layers=2, hidden_size=256, num_attention_heads=4, num_key_value_heads=2, head_dim=64, vocab_size=256,
             intermediate_size=512, max_position_embeddings=128)
SEED = 1234
FP8_TENSOR = dict(num_bits=8, type="float", symmetric=True, strategy="tensor", dynamic=False)
CASES = {
    "kv_fp8_tensor": dict(config_groups={}, kv_cache_scheme=FP8_TENSOR),
    "kv_int8_head_asym": dict(config_groups={}, kv_cache_scheme=dict(num_bits=8, type="int", symmetric=False, strategy="attn_head", dynamic=False)),
    "attn_fp8_tensor": dict(config_groups={"attn": dict(targets=["re:.*self_attn$"], input_activations=FP8_TENSOR)}),
    "kv_int8_token_dynamic": dict(config_groups={}, kv_cache_scheme=dict(num_bits=8, type="int", symmetric=True, strategy="token", dynamic=True)),
}


def build_model(dtype):
    torch.manual_seed(SEED)
    return LlamaForCausalLM(LlamaConfig(**MODEL)).to(dtype).eval()


def attention_modules(model):
    return [m for m in model.modules() if hasattr(m, KV_CACHE_ATTR)]


def capture_pre(model, store):
    """pre-quantization states per layer through the register_*_hook API"""
    handles = []
    for i, m in enumerate(attention_modules(model)):
        def rec(name, i=i):
            def hook(_module, t):
                store.setdefault(i, {})[name] = t.detach().clone()
            return hook
        handles.append(register_key_hook(m, rec("k")))
        handles.append(register_value_hook(m, rec("v")))
        if hasattr(m, IMPL_ATTR):
            handles.append(register_query_hook(m, rec("q")))
    return handles


def capture_post(model, store):
    """post-quantization K / V: outputs of each QuantizedKVCache (use_cache=False -> the quantized pair)"""
    handles = []
    for i, m in enumerate(attention_modules(model)):
        def hook(_cache, _args, out, i=i):
            store.setdefault(i, {})["k"], store[i]["v"] = out[0].detach().clone(), out[1].detach().clone()
        handles.append(getattr(m, KV_CACHE_ATTR).register_forward_hook(hook))
    return handles


def observe(args, t):
    """min / max of the observer for the qparams shape of the strategy: [1] (TENSOR) or [H, 1, 1] (ATTN_HEAD)"""
    if args.strategy == "attn_head":
        h = t.shape[1]
        return t.amin((0, 2, 3)).reshape(h, 1, 1), t.amax((0, 2, 3)).reshape(h, 1, 1)
    return t.amin().reshape(1), t.amax().reshape(1)


def record(case, cfg, dtype):
    model = build_model(dtype)
    config = QuantizationConfig(**cfg)
    apply_quantization_config(model, config)
    params = [(n, tuple(p.shape), str(p.dtype)) for n, p in model.named_parameters()]
    ids = torch.randint(0, MODEL["vocab_size"], (1, 8), generator=torch.Generator().manual_seed(SEED + 1))
    mods = attention_modules(model)
    args = getattr(mods[0].quantization_scheme, "input_activations")

    # pass 1, quantization disabled: per-layer ranges -> qparams
    if not args.dynamic:
        calib = {}
        hs = capture_pre(model, calib)
        for m in mods:
            m.quantization_enabled = False
        with torch.no_grad():
            model(ids, use_cache=False)
        for m in mods:
            del m.quantization_enabled
        for h in hs:
            h.remove()
        for i, m in enumerate(mods):
            for base, t in calib[i].items():
                scale, zp = calculate_qparams(*observe(args, t), args)
                getattr(m, f"{base}_scale").data.copy_(scale.reshape(getattr(m, f"{base}_scale").shape))
                if hasattr(m, f"{base}_zero_point"):
                    getattr(m, f"{base}_zero_point").data.copy_(zp.reshape(getattr(m, f"{base}_zero_point").shape))

    # pass 2: pre / post states and logits
    pre, post, queries = {}, {}, []
    hs = capture_pre(model, pre) + capture_post(model, post)
    original = QuantizedAttentionImpl._original_impl
    if any(hasattr(m, IMPL_ATTR) for m in mods):
        def recording_attention(module, query, key, value, *a, **k):
            queries.append(query.detach().clone())
            return ALL_ATTENTION_FUNCTIONS[original](module, query, key, value, *a, **k)
        ALL_ATTENTION_FUNCTIONS.register("golden_record", recording_attention)
        QuantizedAttentionImpl._original_impl = "golden_record"
    with torch.no_grad():
        logits = model(ids, use_cache=False).logits
    QuantizedAttentionImpl._original_impl = original
    for h in hs:
        h.remove()
    for i, q in enumerate(queries):
        post[i]["q"] = q

    qparams = [{k: v.detach().clone() for k, v in m.named_parameters(recurse=False)} for m in mods]
    dump = QuantizationConfig.from_pretrained(model).model_dump(mode="json")
    compressor = ModelCompressor.from_pretrained_model(model)
    compressor.compress_model(model)
    compressed = [{k: v.detach().clone() for k, v in m.state_dict().items() if "." not in k} for m in mods]
    compressor.decompress_model(model)
    decompressed = [{k: v.detach().clone() for k, v in m.state_dict().items() if "." not in k} for m in mods]
    return dict(case=case, dtype=str(dtype), seed=SEED, model=MODEL, config=cfg, ids=ids, params=params, qparams=qparams,
                attn_implementation=model.config._attn_implementation, pre=[pre[i] for i in range(len(mods))],
                post=[post[i] for i in range(len(mods))], logits=logits, from_pretrained=dump, compressed=compressed,
                decompressed=decompressed, status_after_decompress=str(mods[0].quantization_status.value))


def main():
    out = []
    for dtype in (torch.bfloat16, torch.float32):
        for case, cfg in CASES.items():
            out.append(record(case, cfg, dtype))
    mg.save("kv.pt", out)


if __name__ == "__main__":
    main()
