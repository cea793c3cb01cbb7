"""
Transforms on the H100: ct_hadamard_transform against its CPU twin bit for bit (every order 2^1 .. 2^15, dtype, precision, matrix
form, inverse, head blocking, strided [B, H, S, D] views), fp64 weight fusion against the reference's goldens, the model-level goldens
of tests/golden/transform.pt.gz (make_golden_transform.py) including compress_model -> decompress_model, and the dense path for a
weight that is not a verified Hadamard matrix.
"""
import json
import os
import tempfile

import pytest
import torch

from compressed_tensors_b200 import _native as N
from compressed_tensors_b200 import ops
from tests import golden

gpu = pytest.mark.gpu
DTYPES = (torch.bfloat16, torch.float16, torch.float32)


def _eager(*args):
    from compressed_tensors_b200.utils import ImplBackend

    return ImplBackend.call("hadamard_transform_eager", *args)


def run_model_case(case, device):
    """build the seeded Llama of make_golden_kv.py, apply the case's configs on `device`, and return what the golden records"""
    from transformers import LlamaConfig, LlamaForCausalLM

    from compressed_tensors_b200.compressors import ModelCompressor
    from compressed_tensors_b200.quantization import QuantizationConfig, apply_quantization_config
    from compressed_tensors_b200.quantization.utils import calculate_qparams
    from compressed_tensors_b200.transform import TransformBase, TransformConfig, apply_transform_config

    torch.manual_seed(1234)
    model_cfg = dict(num_hidden_layers=2, hidden_size=256, num_attention_heads=4, num_key_value_heads=2, head_dim=64, vocab_size=256,
                     intermediate_size=512, max_position_embeddings=128)
    model = LlamaForCausalLM(LlamaConfig(**model_cfg)).to(torch.bfloat16).eval().to(device)
    apply_transform_config(model, TransformConfig(**case["config"]))
    if case["quant"]:
        fp8 = dict(num_bits=8, type="float", symmetric=True, strategy="tensor", dynamic=False)
        apply_quantization_config(model, QuantizationConfig(
            config_groups={"w": dict(targets=["Linear"], weights=dict(num_bits=4, type="int", symmetric=True, strategy="group",
                                                                      group_size=64, dynamic=False))},
            ignore=["lm_head"], kv_cache_scheme=fp8))
        for m in model.modules():
            scheme = getattr(m, "quantization_scheme", None)
            if scheme is None:
                continue
            if scheme.weights is not None and hasattr(m, "weight_scale"):
                w = m.weight.detach().reshape(m.weight.shape[0], -1, scheme.weights.group_size)
                scale, zp = calculate_qparams(w.amin(-1), w.amax(-1), scheme.weights)
                m.weight_scale.data.copy_(scale.reshape(m.weight_scale.shape))
                m.weight_zero_point.data.copy_(zp.reshape(m.weight_zero_point.shape))
            for base in ("q", "k", "v"):   # the query too: R3 on q_attn makes the kv_cache_scheme quantize Q
                if hasattr(m, f"{base}_scale"):
                    getattr(m, f"{base}_scale").data.fill_(0.0625)
    with torch.no_grad():
        logits = model(case["ids"].to(device), use_cache=False).logits.cpu()
    params = [(n, tuple(p.shape), str(p.dtype)) for n, p in model.named_parameters()]
    tied = {n: dict(getattr(m, "_tied_weights_keys", None) or {}) for n, m in model.named_modules() if isinstance(m, TransformBase)}
    compressor = ModelCompressor.from_pretrained_model(model)
    with tempfile.TemporaryDirectory() as d:
        with open(os.path.join(d, "config.json"), "w") as f:
            json.dump({}, f)
        compressor.update_config(d)
        with open(os.path.join(d, "config.json")) as f:
            written = json.load(f)
    return dict(model=model, compressor=compressor, logits=logits, params=params, tied=tied, written=written)


def _without_version(written: dict) -> dict:
    """config.json contents without the package version (the reference's differs)"""
    return {k: {kk: vv for kk, vv in v.items() if kk != "version"} if isinstance(v, dict) else v for k, v in written.items()}


@gpu
@pytest.mark.parametrize("precision", (torch.float32, torch.float64))
@pytest.mark.parametrize("dtype", DTYPES)
def test_kernel_equals_cpu_twin_every_order(dtype, precision):
    gen = torch.Generator().manual_seed(3)
    for log2_n in range(1, 16):
        n = 1 << log2_n
        heads = 3 if n <= 4096 else 1
        x = torch.randn(5, heads * n, generator=gen).to(dtype)
        q = (torch.randint(0, 2, (n,), generator=gen) * 2 - 1).to(torch.int8)
        perm = torch.randperm(n, generator=gen)
        xd = x.cuda()
        for sign in (None, q):
            for p in (None, perm):
                for inverse in (False, True):
                    want = _eager(x, n, sign, p, inverse, precision)
                    got = ops.hadamard_transform(xd, n, None if sign is None else sign.cuda(), None if p is None else p.cuda(),
                                                 inverse, precision)
                    assert torch.equal(got.cpu(), want), (n, sign is None, p is None, inverse)


@gpu
@pytest.mark.parametrize("dtype", DTYPES)
def test_strided_attention_views_keep_strides(dtype):
    gen = torch.Generator().manual_seed(4)
    for B, H, S, D in ((1, 32, 256, 128), (4, 8, 1, 128), (2, 8, 33, 64)):
        base = torch.randn(B, S, H, D, generator=gen).to(dtype).cuda()
        x = base.transpose(1, 2)                       # [B, H, S, D] view, rows not contiguous
        q = (torch.randint(0, 2, (D,), generator=gen) * 2 - 1).to(torch.int8)
        perm = torch.randperm(D, generator=gen)
        launches = N.launch_count()
        y = ops.hadamard_transform(x, D, q.cuda(), perm.cuda())
        assert N.launch_count() - launches == 1
        assert all(a == b for a, b, size in zip(y.stride(), x.stride(), x.shape) if size > 1)
        assert torch.equal(y.cpu(), _eager(x.cpu().contiguous(), D, q, perm, False, torch.float32))
    odd = torch.randn(6, 40, 16, generator=gen).to(dtype).cuda()[:, 1:33, :]   # a slice: 16-element rows at odd offsets
    assert torch.equal(ops.hadamard_transform(odd, 16).cpu(), _eager(odd.cpu().contiguous(), 16, None, None, False, torch.float32))


@gpu
def test_cpu_tensor_is_staged_through_the_gpu():
    x = torch.randn(64, 512, dtype=torch.bfloat16)
    y = ops.hadamard_transform(x, 128)
    assert y.device.type == "cpu" and torch.equal(y, _eager(x, 128, None, None, False, torch.float32))


GOLD = golden.load("transform")


def _factory_id(c):
    return f"{c['type']}-{'rand' if c['randomize'] else 'fixed'}-{c['location']}-hd{c['head_dim']}-{c['dtype'].split('.')[-1]}"


@gpu
@pytest.mark.parametrize("case", [c for c in GOLD["factory"] if c["type"] != "random-matrix" and c["location"].startswith("weight")],
                         ids=_factory_id)
def test_fp64_weight_fusion_equals_golden(case):
    from compressed_tensors_b200.transform import TransformArgs, TransformFactory, TransformScheme

    dtype = getattr(torch, case["dtype"].split(".")[-1])
    module = torch.nn.Linear(16, 64, bias=True).to(dtype).cuda()
    with torch.no_grad():
        module.weight.copy_(case["module_weight"])
        module.bias.copy_(case["module_bias"])
    tfm = TransformFactory.from_scheme(TransformScheme(type=case["type"], randomize=case["randomize"], head_dim=case["head_dim"]),
                                       name="", seed=42).create_transform(module, TransformArgs(targets="Linear", location=case["location"]))
    launches = N.launch_count()
    with torch.no_grad():
        fused = tfm(module.weight)
    assert N.launch_count() > launches              # the kernel, not the dense product
    assert torch.equal(fused.cpu(), case["fused_weight"])
    if case["location"] == "weight_output":
        with torch.no_grad():
            assert torch.equal(tfm(module.bias.unsqueeze(-1)).squeeze(-1).cpu(), case["fused_bias"])


@gpu
@pytest.mark.parametrize("case", GOLD["model"], ids=lambda c: f"{c['name']}{'-w4a16-kvfp8' if c['quant'] else ''}")
def test_model_golden_on_gpu(case):
    pytest.importorskip("transformers")
    got = run_model_case(case, "cuda")
    assert got["params"] == case["params"]
    assert got["tied"] == case["tied"]
    assert _without_version(got["written"]) == _without_version(case["written"])
    # online rotations may differ from the reference's by one bf16 ulp per element (DESIGN.md section 3), and the GPU's bf16 GEMMs
    # sum in another order than the CPU's the golden was recorded on: two ulps of the top of the logit range (|logit| < 2), twice the
    # largest difference seen on an H100 (2^-7)
    assert torch.allclose(got["logits"].float(), case["logits"].float(), atol=2.0 ** -6, rtol=0.0), \
        float((got["logits"].float() - case["logits"].float()).abs().max())
    if case["quant"]:
        model, compressor = got["model"], got["compressor"]
        compressor.compress_model(model)
        assert any(n.endswith("weight_packed") for n, _ in model.named_parameters())
        compressor.decompress_model(model)
        with torch.no_grad():
            again = model(case["ids"].cuda(), use_cache=False).logits.cpu()
        assert torch.equal(again, got["logits"])       # the decompressed weights are the fake-quantized ones


@gpu
def test_non_hadamard_weight_takes_the_dense_path():
    from compressed_tensors_b200.transform import TransformArgs, TransformFactory, TransformScheme

    module = torch.nn.Linear(64, 64, bias=False).cuda()
    tfm = TransformFactory.from_scheme(TransformScheme(type="hadamard"), name="").create_transform(
        module, TransformArgs(targets="Linear", location="input"))
    x = torch.randn(8, 64, device="cuda")
    launches = N.launch_count()
    tfm(x)
    assert N.launch_count() - launches == 1
    with torch.no_grad():
        tfm.weight[0, 0] = 0.5
    launches = N.launch_count()
    y = tfm(x)
    assert N.launch_count() == launches
    assert torch.equal(y, tfm._dense(x))
