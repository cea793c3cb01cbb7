"""
Host side of CompressedTensorsQuantizer (no GPU): the converter's planning, validation, tensor naming and config logic, run over the
whole model-free flow (convert_checkpoint on the CPU) with the tensor-level ops backed by the CPU oracle and the fused observers
restated as their unfused reference flow (min / max -> calculate_qparams -> quantize), against golden vectors that the reference's
own apply_quantization_config + calculate_qparams + ModelCompressor.compress_model produced (tests/golden/make_golden_quantizer.py).
The kernels under the same flow are covered by tests/test_gpu_quantizer.py.
"""
import json
import os
import sys

import pytest
import torch

import compressed_tensors_b200.ops as ops
from compressed_tensors_b200.entrypoints.convert import CompressedTensorsQuantizer, build_inverse_weight_maps, convert_checkpoint
from compressed_tensors_b200.quantization.utils.helpers import calculate_qparams, generate_gparam
from compressed_tensors_b200.utils.safetensors_load import get_checkpoint_files, get_weight_map
from tests.golden import load
from tests.golden import quantizer_checkpoint as qc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G = load("quantizer")
CASES = [(c["source"], c["preset"]) for c in G["cases"]]


def _strategy(args):
    return getattr(args.strategy, "value", args.strategy)


def _min_max(x, args):
    s = _strategy(args)
    if s in ("group", "tensor_group"):
        g = x.unflatten(-1, (-1, args.group_size))
        return g.amin(-1), g.amax(-1)
    if s == "channel":
        return x.amin(-1, keepdim=True), x.amax(-1, keepdim=True)
    if s == "tensor":
        return x.amin().reshape(1), x.amax().reshape(1)
    bh, bw = args.block_structure
    r, c = x.shape
    p = torch.nn.functional.pad(x, (0, -(-c // bw) * bw - c, 0, -(-r // bh) * bh - r)).reshape(-(-r // bh), bh, -(-c // bw), bw)
    return p.amin(dim=(1, 3)), p.amax(dim=(1, 3))


def _observe_quantize(x, args, pack=False):
    scale, zp = calculate_qparams(*_min_max(x, args), args)
    zp = None if args.symmetric else zp
    if pack:
        return ops.quantize_pack(x, scale, zp, args), scale, zp
    return ops.quantize(x, scale, zp, args, dtype=args.pytorch_dtype()), scale, zp


def _observe_quantize_pack_nvfp4(x, args, global_scale=None):
    gs = generate_gparam(x.min(), x.max()) if global_scale is None else global_scale
    scale, _ = calculate_qparams(*_min_max(x, args), args, global_scale=gs)
    return ops.quantize_pack_fp4(x, scale, None, args, global_scale=gs), scale.to(torch.float8_e4m3fn), gs


def _observe_quantize_mx(x, args):
    scale, _ = calculate_qparams(*_min_max(x, args), args)
    q = ops.quantize_pack_fp4(x, scale, None, args) if args.num_bits == 4 else ops.quantize(x, scale, None, args, dtype=torch.float8_e4m3fn)
    return q, ops.compress_mx_scale(scale, torch.uint8)


@pytest.fixture
def oracle_ops():
    """ops -> CPU oracle, observers -> their unfused reference flow, for the duration of one test"""
    sys.path.insert(0, os.path.join(ROOT, "tests", "reference_compat"))
    import oracle_patch

    saved = {n: getattr(ops, n) for n in dir(ops) if not n.startswith("__")}
    bound = {(name, fn): getattr(mod, fn) for name, mod in list(sys.modules.items())
             if name.startswith("compressed_tensors_b200.") and mod is not None and mod is not ops
             for fn in ("pack_to_int32", "unpack_from_int32", "pack_fp4_to_uint8", "unpack_fp4_from_uint8", "pack_bitmasks", "unpack_bitmasks")
             if hasattr(mod, fn)}
    oracle_patch.apply("compressed_tensors_b200")
    ops.observe_quantize, ops.observe_quantize_pack_nvfp4, ops.observe_quantize_mx = _observe_quantize, _observe_quantize_pack_nvfp4, _observe_quantize_mx
    ops.observe_tensor_gparam = lambda x: generate_gparam(x.min(), x.max())
    try:
        yield
    finally:
        for n, v in saved.items():
            setattr(ops, n, v)
        for (name, fn), v in bound.items():
            setattr(sys.modules[name], fn, v)


def _source(source):
    if source == "fp8_block":
        return qc.fp8_block_tensors(), torch.bfloat16, torch.bfloat16
    dt = torch.bfloat16 if source == "bf16" else torch.float16
    return qc.dense_tensors(dt), dt, None


def _read_all(directory):
    from safetensors.torch import load_file

    out = {}
    for f in sorted(os.listdir(directory)):
        if f.endswith(".safetensors"):
            out.update(load_file(os.path.join(directory, f)))
    return out


def _check_against_golden(out: dict, case: dict):
    assert set(out) == set(case["state"]), f"names differ: {sorted(set(out) ^ set(case['state']))}"
    for name, ref in case["state"].items():
        t = out[name]
        assert str(t.dtype) == ref["dtype"] and list(t.shape) == ref["shape"], f"{name}: {t.dtype} {list(t.shape)} vs {ref['dtype']} {ref['shape']}"
        assert qc.digest(t) == ref["digest"], f"{name}: bits differ from the reference" + (f" ({t} vs {ref['full']})" if "full" in ref else "")


def _case(source, preset):
    return next(c for c in G["cases"] if c["source"] == source and c["preset"] == preset)


def test_sources_match_golden():
    for source in ("bf16", "fp16"):
        assert {n: qc.digest(t) for n, t in qc.dense_tensors(torch.bfloat16 if source == "bf16" else torch.float16).items()} == G["sources"][source]
    assert {n: qc.digest(t) for n, t in qc.fp8_block_tensors().items()} == G["sources"]["fp8_block"]


@pytest.mark.parametrize("source,preset", CASES)
def test_convert_checkpoint_matches_reference(tmp_path, oracle_ops, source, preset):
    tensors, dt, deq = _source(source)
    qc.write_checkpoint(str(tmp_path / "in"), tensors, dt)
    conv = CompressedTensorsQuantizer(preset, ignore=list(qc.IGNORE), dtype=deq)
    convert_checkpoint(str(tmp_path / "in"), str(tmp_path / "out"), conv, device="cpu")
    case = _case(source, preset)
    _check_against_golden(_read_all(str(tmp_path / "out")), case)
    with open(tmp_path / "out" / "config.json") as f:
        written = json.load(f)["quantization_config"]
    ref = case["config"]
    assert written["format"] == ref["format"] and written["quantization_status"] == "compressed"
    for kind in ("weights", "input_activations", "output_activations"):
        assert written["config_groups"]["group_0"][kind] == ref["config_groups"]["group_0"][kind], kind


@pytest.mark.parametrize("preset", ["W8A8", "FP8_DYNAMIC"])
def test_wide_row_channel_on_oracle(oracle_ops, preset):
    """the 16512-column down_proj with one scale per row, through the oracle, equals the reference's compress_model bit for bit"""
    tensors = qc.dense_tensors(torch.bfloat16)
    name = "model.layers.0.mlp.down_proj"
    out = CompressedTensorsQuantizer(preset).process({f"{name}.weight": tensors[f"{name}.weight"]})
    ref = _case("bf16", preset)["state"]
    assert out[f"{name}.weight"].shape[1] == qc.INTERMEDIATE > 16384
    for k in ("weight", "weight_scale"):
        assert qc.digest(out[f"{name}.{k}"]) == ref[f"{name}.{k}"]["digest"], k


def test_process_fp8_source_equals_dequantizer_then_quantizer(oracle_ops):
    from compressed_tensors_b200.entrypoints.convert import FP8BlockDequantizer

    src = qc.fp8_block_tensors()
    direct = CompressedTensorsQuantizer("NVFP4A16", ignore=list(qc.IGNORE), dtype=torch.bfloat16).process(dict(src))
    dense = FP8BlockDequantizer(targets=["re:.*proj$"], dtype=torch.bfloat16).process(dict(src))
    two_step = CompressedTensorsQuantizer("NVFP4A16", ignore=list(qc.IGNORE)).process(dense)
    assert set(direct) == set(two_step)
    for k in direct:
        assert qc.digest(direct[k]) == qc.digest(two_step[k]), k


def _meta(tensors):
    return {k: torch.empty(v.shape, dtype=v.dtype, device="meta") for k, v in tensors.items()}


@pytest.mark.parametrize("preset", ["FP8", "NVFP4"])
def test_validate_refuses_static_activation_schemes(preset):
    with pytest.raises(ValueError, match=preset):
        CompressedTensorsQuantizer(preset).validate({"a.weight": torch.empty(8, 32, device="meta")})


@pytest.mark.parametrize("preset", ["W8A8", "FP8_DYNAMIC", "MXFP4", "W4A16", "NVFP4A16"])
def test_validate_accepts_dynamic_activation_schemes(preset):
    CompressedTensorsQuantizer(preset).validate({"a.weight": torch.empty(8, 128, dtype=torch.bfloat16, device="meta")})


def test_validate_refusals():
    q = CompressedTensorsQuantizer("W8A8")
    with pytest.raises(ValueError, match="experts.weight"):
        q.validate({"experts.weight": torch.empty(2, 8, 8, device="meta")})
    with pytest.raises(ValueError, match="a.weight"):
        q.validate({"a.weight": torch.empty(8, 8, dtype=torch.int8, device="meta")})
    with pytest.raises(ValueError, match="weight_scale_inv without corresponding weight"):
        q.validate({"a.weight_scale_inv": torch.empty(1, 1, device="meta")})
    with pytest.raises(ValueError, match="pass the dtype"):
        q.validate({"a.weight": torch.empty(8, 8, dtype=torch.float8_e4m3fn, device="meta"), "a.weight_scale_inv": torch.empty(1, 1, device="meta")})
    fp8 = CompressedTensorsQuantizer("W8A8", ignore=list(qc.IGNORE), dtype=torch.bfloat16)
    with pytest.raises(ValueError, match="weight without corresponding weight_scale_inv"):
        fp8.validate({"a.weight": torch.empty(8, 8, dtype=torch.float8_e4m3fn, device="meta")})
    with pytest.raises(ValueError, match="weight_scale_inv of shape"):
        fp8.validate({"a.weight": torch.empty(256, 8, dtype=torch.float8_e4m3fn, device="meta"), "a.weight_scale_inv": torch.empty(1, 1, device="meta")})
    with pytest.raises(ValueError, match="group size"):
        CompressedTensorsQuantizer("W4A16").validate({"a.weight": torch.empty(8, 96, dtype=torch.bfloat16, device="meta")})
    ok = _meta(qc.fp8_block_tensors())
    fp8.validate(ok)


@pytest.mark.parametrize("source", ["bf16", "fp8_block"])
def test_fused_groups_load_into_one_job(tmp_path, source):
    tensors, dt, deq = _source(source)
    qc.write_checkpoint(str(tmp_path), tensors, dt)
    files = get_checkpoint_files(str(tmp_path))
    wm = get_weight_map(files)
    plans = build_inverse_weight_maps(wm, files, [CompressedTensorsQuantizer("NVFP4A16", ignore=list(qc.IGNORE), dtype=deq)])
    jobs = [sorted(n for names in plan.values() for n in names) for plan in plans.values()]
    loaded = [n for job in jobs for n in job]
    assert sorted(loaded) == sorted(wm), "every tensor is loaded by exactly one job"
    attn = "model.layers.0.self_attn."
    mlp = "model.layers.0.mlp."
    for group in ((f"{attn}q_proj", f"{attn}k_proj", f"{attn}v_proj"), (f"{mlp}gate_proj", f"{mlp}up_proj")):
        job = next(j for j in jobs if f"{group[0]}.weight" in j)
        assert all(f"{m}.weight" in job for m in group)
        if deq is not None:
            assert all(f"{m}.weight_scale_inv" in job for m in group)
    assert len({wm[f"{attn}{m}_proj.weight"] for m in "qkv"}) == 3, "the fixture splits q / k / v over three shards"
    # schemes without a global scale keep one job per weight
    plans = build_inverse_weight_maps(wm, files, [CompressedTensorsQuantizer("W4A16", ignore=list(qc.IGNORE), dtype=deq)])
    job = next(sorted(n for names in p.values() for n in names) for p in plans.values() if any(f"{attn}q_proj.weight" in v for v in p.values()))
    assert f"{attn}k_proj.weight" not in job


@pytest.mark.parametrize("preset,ignore", [("W4A16_ASYM", qc.IGNORE), ("NVFP4A16", qc.IGNORE), ("FP8_BLOCK", qc.IGNORE), ("W8A8", ())])
def test_written_config_loads_back(tmp_path, oracle_ops, preset, ignore):
    """config.json -> ModelCompressor.from_compression_config + apply_quantization_config on the checkpoint's own model: exactly the
    modules the converter quantized are quantized, with the names and shapes of the compressed parameters the converter wrote"""
    from transformers import LlamaConfig, LlamaForCausalLM

    from compressed_tensors_b200.compressors import ModelCompressor
    from compressed_tensors_b200.quantization import apply_quantization_config
    from compressed_tensors_b200.quantization.utils.helpers import is_module_quantized

    tensors, dt, deq = _source("bf16")
    qc.write_checkpoint(str(tmp_path / "in"), tensors, dt)
    convert_checkpoint(str(tmp_path / "in"), str(tmp_path / "out"), CompressedTensorsQuantizer(preset, ignore=list(ignore)), device="cpu")
    with open(tmp_path / "out" / "config.json") as f:
        cfg = json.load(f)
    compressor = ModelCompressor.from_compression_config(cfg)
    kw = {k: v for k, v in cfg.items() if k not in ("architectures", "model_type", "torch_dtype", "quantization_config")}
    with torch.device("meta"):
        model = LlamaForCausalLM(LlamaConfig(**kw))
    apply_quantization_config(model, compressor.quantization_config)
    quantized = sorted(n for n, m in model.named_modules() if is_module_quantized(m))
    # with nothing ignored, the embedding and lm_head are quantized too, and the config names them, so the load still matches
    extra = [] if ignore else ["lm_head", "model.embed_tokens"]
    assert quantized == sorted(_case("bf16", preset)["quantized"] + extra)
    compressor.compress_model(model)   # what transformers does on load: the compressed parameters, shape only on meta
    state = {k: v for k, v in model.state_dict().items()}
    written = _read_all(str(tmp_path / "out"))
    assert set(state) == set(written)
    for k, v in written.items():
        assert tuple(state[k].shape) == tuple(v.shape), k


def test_fused_groups_can_be_turned_off(tmp_path):
    """MLA attention has q_proj but no k_proj / v_proj: the default grouping names missing siblings, fused_groups=() plans it"""
    from safetensors.torch import save_file

    t = {"model.layers.0.self_attn.q_proj.weight": torch.zeros(64, 64, dtype=torch.bfloat16),
         "model.layers.0.self_attn.kv_a_proj_with_mqa.weight": torch.zeros(32, 64, dtype=torch.bfloat16)}
    save_file(t, str(tmp_path / "model.safetensors"))
    files = get_checkpoint_files(str(tmp_path))
    wm = get_weight_map(files)
    with pytest.raises(ValueError, match=r"[kv]_proj\.weight not found"):
        build_inverse_weight_maps(wm, files, [CompressedTensorsQuantizer("NVFP4A16")])
    plans = build_inverse_weight_maps(wm, files, [CompressedTensorsQuantizer("NVFP4A16", fused_groups=())])
    assert sorted(n for p in plans.values() for names in p.values() for n in names) == sorted(t)


def test_unwritable_format_is_refused_up_front():
    from compressed_tensors_b200.quantization import preset_name_to_scheme

    scheme = preset_name_to_scheme("W4A16", ["Linear"])
    scheme.format = "dense"
    with pytest.raises(ValueError, match="cannot write format dense"):
        CompressedTensorsQuantizer(scheme)
