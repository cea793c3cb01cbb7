"""
KV-cache and attention quantization on the host: `kv_cache_scheme` and attention targets through apply_quantization_config, the
modeling/ hooks, QuantizationConfig.from_pretrained and ModelCompressor.compress_model, against tests/golden/kv.pt.gz (recorded from
the reference on a seeded 2-layer LlamaForCausalLM, tests/golden/make_golden_kv.py).  Needs transformers.
"""
import pytest
import torch

transformers = pytest.importorskip("transformers")

import oracle  # noqa: E402
from tests import golden  # noqa: E402
from tests.util import same  # noqa: E402

CASES = golden.load("kv")
IDS = [f"{c['case']}-{c['dtype'].split('.')[-1]}" for c in CASES]
DTYPES = {"torch.bfloat16": torch.bfloat16, "torch.float32": torch.float32}
# logits of the replay: bit-identical on the machine that recorded them; elsewhere the unquantized parts of the model (sdpa, matmuls)
# may reorder floating-point sums.  Bounds: a few units in the last place of each dtype at logits of magnitude ~1.
LOGIT_TOL = {torch.float32: dict(rtol=1e-5, atol=1e-5), torch.bfloat16: dict(rtol=2e-2, atol=2e-2)}


def build(case, device="cpu"):
    from compressed_tensors_b200.quantization import QuantizationConfig, apply_quantization_config

    torch.manual_seed(case["seed"])
    model = transformers.LlamaForCausalLM(transformers.LlamaConfig(**case["model"])).to(DTYPES[case["dtype"]]).eval()
    apply_quantization_config(model, QuantizationConfig(**case["config"]))
    model.to(device)
    return model


def attention_modules(model):
    from compressed_tensors_b200.modeling import KV_CACHE_ATTR

    return [m for m in model.modules() if hasattr(m, KV_CACHE_ATTR)]


def replay(case, device="cpu"):
    """run a golden case on this engine: the golden qparams, the pre- / post-quantization states per layer and the logits"""
    from compressed_tensors_b200.modeling import (IMPL_ATTR, QuantizedAttentionImpl, register_key_hook, register_query_hook,
                                                  register_value_hook)
    from transformers.modeling_utils import ALL_ATTENTION_FUNCTIONS

    model = build(case, device)
    mods = attention_modules(model)
    for m, qp in zip(mods, case["qparams"]):
        for name, t in qp.items():
            getattr(m, name).data.copy_(t)
    pre, post, queries, handles = {}, {}, [], []
    for i, m in enumerate(mods):
        def rec(name, i=i):
            def hook(_module, t):
                pre.setdefault(i, {})[name] = t.detach().clone()
            return hook

        def out_hook(_cache, _args, out, i=i):
            post.setdefault(i, {})["k"], post[i]["v"] = out[0].detach().clone(), out[1].detach().clone()
        handles += [register_key_hook(m, rec("k")), register_value_hook(m, rec("v")), m.kv_cache.register_forward_hook(out_hook)]
        if hasattr(m, IMPL_ATTR):
            handles.append(register_query_hook(m, rec("q")))
    original = QuantizedAttentionImpl._original_impl
    if any(hasattr(m, IMPL_ATTR) for m in mods):
        def recording_attention(module, query, key, value, *a, **k):
            queries.append(query.detach().clone())
            return ALL_ATTENTION_FUNCTIONS[original](module, query, key, value, *a, **k)
        ALL_ATTENTION_FUNCTIONS.register("kv_test_record", recording_attention)
        QuantizedAttentionImpl._original_impl = "kv_test_record"
    try:
        with torch.no_grad():
            logits = model(case["ids"].to(device), use_cache=False).logits
    finally:
        QuantizedAttentionImpl._original_impl = original
        for h in handles:
            h.remove()
    for i, q in enumerate(queries):
        post[i]["q"] = q
    return model, [pre[i] for i in range(len(mods))], [post[i] for i in range(len(mods))], logits


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_apply_structure_and_config_match_reference(case):
    from compressed_tensors_b200.quantization import QuantizationConfig

    model = build(case)
    assert [(n, tuple(p.shape), str(p.dtype)) for n, p in model.named_parameters()] == [tuple(p) for p in case["params"]]
    assert model.config._attn_implementation == case["attn_implementation"]
    assert QuantizationConfig.from_pretrained(model).model_dump(mode="json") == case["from_pretrained"]


@pytest.mark.parametrize("case", [c for c in CASES if not c["config"].get("kv_cache_scheme", {}).get("dynamic")],
                         ids=[i for c, i in zip(CASES, IDS) if not c["config"].get("kv_cache_scheme", {}).get("dynamic")])
def test_reference_post_states_equal_oracle_fake_quantize(case):
    """the reference's post-quantization states are the oracle's fake_quantize of its pre-quantization states, bit for bit"""
    from compressed_tensors_b200.quantization import QuantizationConfig

    cfg = QuantizationConfig(**case["config"])
    args = cfg.kv_cache_scheme or next(iter(cfg.config_groups.values())).input_activations
    for layer, (pre, post, qp) in enumerate(zip(case["pre"], case["post"], case["qparams"])):
        assert set(post) == set(pre)
        for base, x in pre.items():
            want = oracle.fake_quantize(x, qp[f"{base}_scale"], qp.get(f"{base}_zero_point"), strategy=str(getattr(args.strategy, "value", args.strategy)),
                                        num_bits=args.num_bits, qtype=str(getattr(args.type, "value", args.type)))
            same(post[base], want, f"layer {layer} {base}: ")


@pytest.mark.parametrize("case", CASES, ids=IDS)
def test_hooks_reproduce_reference_states_and_logits(case):
    _, pre, post, logits = replay(case)
    for layer, (got, want) in enumerate(zip(post, case["post"])):
        assert set(got) == set(want)
        for base in want:
            same(got[base], want[base], f"layer {layer} post {base}: ")
    assert [set(p) for p in pre] == [set(p) for p in case["pre"]]
    torch.testing.assert_close(logits, case["logits"], **LOGIT_TOL[DTYPES[case["dtype"]]])


@pytest.mark.parametrize("case", [c for c in CASES if c["dtype"] == "torch.float32"], ids=[i for c, i in zip(CASES, IDS) if c["dtype"] == "torch.float32"])
def test_compress_and_decompress_model_keep_the_reference_attention_tensors(case):
    from compressed_tensors_b200.compressors import ModelCompressor

    model, *_ = replay(case)
    compressor = ModelCompressor.from_pretrained_model(model)
    for step in ("compressed", "decompressed"):
        getattr(compressor, "compress_model" if step == "compressed" else "decompress_model")(model)
        for m, want in zip(attention_modules(model), case[step]):
            got = {k: v for k, v in m.state_dict().items() if "." not in k}
            assert sorted(got) == sorted(want), step
            for k in want:
                same(got[k], want[k], f"{step} {k}: ")
    assert all(m.quantization_status.value == case["status_after_decompress"] for m in attention_modules(model))


def test_update_config_writes_the_kv_cache_scheme(tmp_path):
    import json

    from compressed_tensors_b200.compressors import ModelCompressor

    case = next(c for c in CASES if c["case"] == "kv_fp8_tensor")
    model, *_ = replay(case)
    compressor = ModelCompressor.from_pretrained_model(model)
    compressor.compress_model(model)
    compressor.update_config(str(tmp_path))
    written = json.loads((tmp_path / "config.json").read_text())["quantization_config"]
    assert written["kv_cache_scheme"] == case["from_pretrained"]["kv_cache_scheme"]


def test_hooks_fire_once_per_layer_and_reinitialising_is_a_no_op():
    """the reference's test_attention_and_cache.py, on the local model: one query / key / value call per layer and forward, and a
    second initialisation attaches nothing new"""
    from compressed_tensors_b200.modeling import (IMPL_ATTR, KV_CACHE_ATTR, initialize_hooked_attention, initialize_hooked_kv_cache,
                                                  register_key_hook, register_query_hook, register_value_hook)

    case = next(c for c in CASES if c["case"] == "attn_fp8_tensor" and c["dtype"] == "torch.float32")
    model = build(case)
    mods = attention_modules(model)
    calls = {"q": 0, "k": 0, "v": 0}

    def count(name):
        def hook(_module, t):
            calls[name] += 1
        return hook
    for m in mods:
        register_query_hook(m, count("q"))
        register_key_hook(m, count("k"))
        register_value_hook(m, count("v"))
    impls = [getattr(m, IMPL_ATTR) for m in mods]
    caches = [getattr(m, KV_CACHE_ATTR) for m in mods]
    n_pre_hooks = [len(m._forward_pre_hooks) for m in mods]
    for m in mods:
        initialize_hooked_attention(model, m)
        initialize_hooked_kv_cache(model, m)
    assert [getattr(m, IMPL_ATTR) for m in mods] == impls and [getattr(m, KV_CACHE_ATTR) for m in mods] == caches
    assert [len(m._forward_pre_hooks) for m in mods] == n_pre_hooks
    with torch.no_grad():
        model(case["ids"], use_cache=False)
    assert calls == {"q": len(mods), "k": len(mods), "v": len(mods)}
    with torch.no_grad():
        model(case["ids"])   # with a DynamicCache: the QuantizedKVCache hands the states on to it
    assert calls == {"q": 2 * len(mods), "k": 2 * len(mods), "v": 2 * len(mods)}


def test_kv_cache_scheme_skips_attention_without_a_cache_argument():
    """apply.py:172-192 only hooks attention modules whose forward takes a KV cache (the reference's
    test_apply_kv_cache_skips_non_cache_attention, re-expressed)"""
    from types import SimpleNamespace

    from compressed_tensors_b200.quantization import QuantizationArgs, QuantizationConfig, apply_quantization_config

    class TextAttention(torch.nn.Module):
        def __init__(self):
            super().__init__()
            self.k_proj = torch.nn.Linear(4, 4)

        def forward(self, hidden_states, past_key_value=None):
            return hidden_states

    class VisionAttention(TextAttention):
        def forward(self, hidden_states, **kwargs):
            return hidden_states

    class Config:
        text_config = SimpleNamespace(num_attention_heads=2, num_key_value_heads=1, head_dim=2)

        def get_text_config(self, decoder=False):
            return self.text_config

    model = torch.nn.Module()
    model.config = Config()
    model.text_attention, model.vision_attention = TextAttention(), VisionAttention()
    args = QuantizationArgs(num_bits=8, type="float", strategy="tensor")
    apply_quantization_config(model, QuantizationConfig(config_groups={}, kv_cache_scheme=args))
    assert model.text_attention.kv_cache.config is model.config.text_config
    assert hasattr(model.text_attention, "k_scale") and hasattr(model.text_attention, "v_scale")
    assert not any(hasattr(model.vision_attention, n) for n in ("quantization_scheme", "kv_cache", "k_scale", "v_scale"))


def test_attention_scheme_validation():
    from compressed_tensors_b200.quantization import QuantizationConfig, apply_quantization_config

    case = next(c for c in CASES if c["case"] == "attn_fp8_tensor")
    torch.manual_seed(case["seed"])
    model = transformers.LlamaForCausalLM(transformers.LlamaConfig(**case["model"]))
    bad = {"attn": dict(targets=["re:.*self_attn$"], weights=dict(num_bits=8), input_activations=dict(num_bits=8))}
    with pytest.raises(ValueError, match="weight quantization to attention"):
        apply_quantization_config(model, QuantizationConfig(config_groups=bad))


def test_modelopt_nvfp4_kv_cache_config_loads_and_runs():
    """ModelOptNvfp4Converter emits a kv_cache_scheme; the engine now applies it, takes the converted k_scale / v_scale and runs"""
    from compressed_tensors_b200.entrypoints.convert import ModelOptNvfp4Converter
    from compressed_tensors_b200.quantization import QuantizationArgs, QuantizationStatus, apply_quantization_config

    kv = QuantizationArgs(num_bits=8, type="float", strategy="tensor", dynamic=False)
    conv = ModelOptNvfp4Converter(targets=[r"re:.*mlp\.down_proj$"], kv_cache_scheme=kv)
    case = next(c for c in CASES if c["case"] == "kv_fp8_tensor" and c["dtype"] == "torch.float32")
    torch.manual_seed(case["seed"])
    model = transformers.LlamaForCausalLM(transformers.LlamaConfig(**case["model"])).eval()
    config = conv.create_config()
    config.config_groups = {}          # the NVFP4 weight groups need a compressed checkpoint; this test is about the KV cache
    config.quantization_status = QuantizationStatus.FROZEN
    apply_quantization_config(model, config)
    n = case["model"]["num_hidden_layers"]
    stored = {f"model.layers.{i}.self_attn.{p}": torch.tensor([0.05 + 0.01 * i], dtype=torch.float32) for i in range(n) for p in ("k_scale", "v_scale")}
    converted = conv.process(dict(stored))
    for name, t in converted.items():
        module_name, _, param = name.rpartition(".")
        getattr(model.get_submodule(module_name), param).data.copy_(t)
    got = model.model.layers[1].self_attn.k_scale
    assert got.dtype == torch.float32 and float(got) == pytest.approx(0.06)
    with torch.no_grad():
        logits = model(case["ids"], use_cache=False).logits
    assert torch.isfinite(logits).all()


def test_no_cached_attention_module_still_refuses_the_kv_cache_scheme():
    from compressed_tensors_b200.quantization import QuantizationConfig, apply_quantization_config

    cfg = QuantizationConfig(config_groups={}, kv_cache_scheme={"num_bits": 8, "type": "float", "symmetric": True})
    with pytest.raises(NotImplementedError, match="no attention module"):
        apply_quantization_config(torch.nn.Sequential(torch.nn.Linear(32, 32)), cfg)


@pytest.mark.parametrize("symmetric", [True, False], ids=["sym", "asym"])
def test_fake_quantize_heads_without_the_strided_kernel_keeps_per_head_scales(symmetric):
    """tensors the strided kernel does not take (here: CPU tensors) go through fake_quantize with the [H, 1, 1] ATTN_HEAD scales as
    given, one per head, not flattened into a scale along D"""
    from compressed_tensors_b200 import ops
    from compressed_tensors_b200.quantization import QuantizationArgs
    from compressed_tensors_b200.quantization.utils import calculate_qparams

    args = QuantizationArgs(num_bits=8, type="int", symmetric=symmetric, strategy="attn_head")
    gen = torch.Generator().manual_seed(11)
    xs = [torch.randn(2, 16, 4, 64, generator=gen).transpose(1, 2).to(torch.bfloat16) for _ in range(2)]
    scales, zps = [], []
    for x in xs:
        scale, zp = calculate_qparams(x.amin((0, 2, 3)).reshape(4, 1, 1), x.amax((0, 2, 3)).reshape(4, 1, 1), args)
        scales.append(scale)
        zps.append(None if symmetric else zp)
    got = ops.fake_quantize_heads(xs, scales, zps, args)
    for x, s, z, g in zip(xs, scales, zps, got):
        want = oracle.fake_quantize(x, s, z, strategy="attn_head", num_bits=8, qtype="int")
        same(g, want)
