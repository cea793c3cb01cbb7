"""
Transforms on the H100: ct_hadamard_transform against its CPU twin bit for bit and against the float64 reference of
test_transform_host.py (every order 2^1 .. 2^15, dtype, precision, matrix form, inverse, partial last tiles, the fp64 2^15 tile loop,
head blocking, strided [B, H, S, D] views, unaligned rows, overflow, subnormals, inf / NaN), fp64 weight fusion against the reference's
goldens, the model-level goldens of tests/golden/transform.pt.gz (make_golden_transform.py) including compress_model ->
decompress_model and R3 + FP8 KV per layer, the dense path for a weight that is not a verified Hadamard matrix, and which writes to
the weight and permutation the transform follows.
"""
import json
import os
import tempfile

import pytest
import torch

from compressed_tensors_b200 import _native as N
from compressed_tensors_b200 import ops
from tests import golden
from tests.test_transform_host import (
    assert_fp64_result,
    assert_online_bound,
    check_data_writes_keep_the_verified_snapshot,
    check_tracked_writes_are_followed,
    structured_reference,
    transform_cases,
)
from tests.util import same, same_nan

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


def _run(x, n, sign, perm, inverse, precision):
    dev = x.device
    return ops.hadamard_transform(x, n, None if sign is None else sign.to(dev), None if perm is None else perm.to(dev), inverse, precision)


def assert_matches_reference(got, x, n, sign, perm, inverse, precision):
    """fp32: the online bound of DESIGN.md section 3; fp64: bit for bit (16-bit inputs) or half an fp32 ulp (fp32 inputs)"""
    ref = structured_reference(x, n, sign, perm, inverse)
    (assert_fp64_result if precision == torch.float64 else assert_online_bound)(got, ref, x, n)


@gpu
@pytest.mark.parametrize("precision", (torch.float32, torch.float64))
@pytest.mark.parametrize("dtype", DTYPES)
def test_kernel_equals_cpu_twin_every_order(dtype, precision):
    """every order, form and inverse, against the twin bit for bit and the float64 reference; rows of 3 blocks, and for n < 4096
    one row more than a 4096-element tile holds (a one-row partial last tile)"""
    gen = torch.Generator().manual_seed(3)
    for log2_n in range(1, 16):
        n = 1 << log2_n
        heads = 3 if n <= 4096 else 1
        shapes = [(5, heads * n)] + ([(4096 // n + 1, n)] if n < 4096 else [])
        for shape in shapes:
            x = torch.randn(*shape, generator=gen).to(dtype)
            xd = x.cuda()
            for sign, p, inverse in transform_cases(n, gen):
                got = _run(xd, n, sign, p, inverse, precision)
                assert torch.equal(got.cpu(), _eager(x, n, sign, p, inverse, precision)), (n, shape, sign is None, p is None, inverse)
                assert_matches_reference(got, xd, n, sign, p, inverse, precision)


@gpu
@pytest.mark.parametrize("dtype", DTYPES)
def test_fp64_order_2_15_loops_over_more_tiles_than_its_grid(dtype):
    """fp64 at n = 2^15 keeps each tile in a global scratch slice per CTA, on a grid of 2 x SMs: 2 x SMs + 7 rows make 7 CTAs take
    a second tile in the same slice"""
    n = 1 << 15
    rows = 2 * torch.cuda.get_device_properties(0).multi_processor_count + 7
    gen = torch.Generator().manual_seed(30)
    x = torch.randn(rows, n, generator=gen).to(dtype).cuda()
    for sign, p, inverse in transform_cases(n, gen):
        assert_matches_reference(_run(x, n, sign, p, inverse, torch.float64), x, n, sign, p, inverse, torch.float64)


@gpu
@pytest.mark.parametrize("dtype", DTYPES)
def test_strided_attention_views_keep_strides(dtype):
    gen = torch.Generator().manual_seed(4)
    # [B, H, S, D] and the order n: one block per row, head blocking (D = 256 in blocks of 64), decode (S = 1)
    for B, H, S, D, n in ((1, 32, 256, 128, 128), (4, 8, 1, 128, 128), (2, 8, 33, 64, 64), (2, 4, 17, 256, 64), (3, 8, 1, 256, 64)):
        base = torch.randn(B, S, H, D, generator=gen).to(dtype).cuda()
        x = base.transpose(1, 2)                       # [B, H, S, D] view, rows not contiguous
        q = (torch.randint(0, 2, (n,), generator=gen) * 2 - 1).to(torch.int8)
        perm = torch.randperm(n, generator=gen)
        for precision in (torch.float32, torch.float64):
            launches = N.launch_count()
            y = ops.hadamard_transform(x, n, q.cuda(), perm.cuda(), False, precision)
            assert N.launch_count() - launches == 1
            assert all(a == b for a, b, size in zip(y.stride(), x.stride(), x.shape) if size > 1)
            assert torch.equal(y.cpu(), _eager(x.cpu().contiguous(), n, q, perm, False, precision))
            assert_matches_reference(y, x, n, q, perm, False, precision)
    odd = torch.randn(6, 40, 16, generator=gen).to(dtype).cuda()[:, 1:33, :]   # a slice: 16-element rows at odd offsets
    assert torch.equal(ops.hadamard_transform(odd, 16).cpu(), _eager(odd.cpu().contiguous(), 16, None, None, False, torch.float32))


@gpu
@pytest.mark.parametrize("dtype", DTYPES)
def test_rows_one_element_off_alignment_take_element_loads(dtype):
    """a dense tensor that starts one element past a 16-byte boundary is read and written element by element (no 16-byte accesses),
    with every form and both precisions"""
    gen = torch.Generator().manual_seed(31)
    for n in (2, 16, 128, 4096):
        x = torch.randn(3 * 2 * n + 1, generator=gen).to(dtype).cuda()[1:].view(3, 2 * n)
        assert x.data_ptr() % 16 != 0
        for sign, p, inverse in transform_cases(n, gen):
            for precision in (torch.float32, torch.float64):
                got = _run(x, n, sign, p, inverse, precision)
                assert torch.equal(got.cpu(), _eager(x.cpu(), n, sign, p, inverse, precision)), (n, sign is None, p is None, inverse)
                assert_matches_reference(got, x, n, sign, p, inverse, precision)


@gpu
def test_fp16_overflow_gives_inf_where_the_reference_does():
    """rows of +-60000 at n = 16: every output is 15000 times an even sum of signs, so exactly representable (0, +-30000,
    +-60000) or past the fp16 range (+-90000 and beyond), and both precisions must give the float64 value rounded through fp32"""
    n = 16
    gen = torch.Generator().manual_seed(32)
    x = ((torch.randint(0, 2, (64, 2 * n), generator=gen) * 2 - 1) * 60000.0).half().cuda()
    for sign, p, inverse in transform_cases(n, gen):
        want = structured_reference(x, n, sign, p, inverse).float().half()
        assert bool(want.isinf().any()) and bool(want.isfinite().any())
        for precision in (torch.float32, torch.float64):
            assert torch.equal(_run(x, n, sign, p, inverse, precision), want), (sign is None, p is None, inverse, precision)


@gpu
@pytest.mark.parametrize("dtype", DTYPES)
def test_subnormal_and_signed_zero_inputs(dtype):
    """small multiples of the dtype's smallest subnormal and +-0; at orders with sqrt(n) a power of two the sums and the division
    are exact in either precision, so both must equal the float64 reference rounded through fp32 (compared by value)"""
    gen = torch.Generator().manual_seed(33)
    step = torch.finfo(dtype).tiny * torch.finfo(dtype).eps
    for n in (4, 16, 64):
        sub = (torch.randint(-100, 101, (4, 2 * n), generator=gen).double() * step)
        zeros = torch.zeros(2, 2 * n, dtype=torch.float64) * (torch.randint(0, 2, (2, 2 * n), generator=gen) * 2 - 1)
        x = torch.cat((sub, zeros)).to(dtype).cuda()
        assert bool((x[:4] != 0).any()) and bool((x[:4].abs() < torch.finfo(dtype).tiny).all())
        for sign, p, inverse in transform_cases(n, gen):
            want = structured_reference(x, n, sign, p, inverse).float().to(dtype)
            for precision in (torch.float32, torch.float64):
                assert torch.equal(_run(x, n, sign, p, inverse, precision), want), (n, sign is None, p is None, inverse, precision)


@gpu
@pytest.mark.parametrize("dtype", DTYPES)
def test_rows_with_inf_and_nan_equal_the_twin(dtype):
    """non-finite inputs propagate as the twin's butterfly order makes them: NaN positions and every other bit equal, payloads free"""
    gen = torch.Generator().manual_seed(34)
    for n in (8, 256):
        x = torch.randn(6, 2 * n, generator=gen)
        x[0, 3], x[1, 1], x[1, n + 2], x[2, 0], x[3, 5], x[3, 6] = float("inf"), float("-inf"), float("inf"), float("nan"), float("inf"), float("-inf")
        x = x.to(dtype)
        for sign, p, inverse in transform_cases(n, gen):
            for precision in (torch.float32, torch.float64):
                got = _run(x.cuda(), n, sign, p, inverse, precision).cpu()
                same_nan(got, _eager(x, n, sign, p, inverse, precision), f"n={n} sign={sign is not None} perm={p is not None} inv={inverse}")


@gpu
def test_tracked_writes_are_followed_on_gpu():
    check_tracked_writes_are_followed("cuda")


@gpu
def test_data_writes_keep_the_verified_snapshot_on_gpu():
    check_data_writes_keep_the_verified_snapshot("cuda")


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
def test_r3_rotation_then_fp8_kv_quantization_is_exact_per_layer():
    """SpinQuant-like golden with W4A16 + FP8 KV: per layer, the quantized Q and K the attention receives equal the oracle's
    fake_quantize of the twin's R3 rotation of the states that reach the hooks (the twin gives the kernel's bits)"""
    pytest.importorskip("transformers")
    import inspect

    import oracle
    from compressed_tensors_b200.modeling import IMPL_ATTR, KV_CACHE_ATTR, QuantizedAttentionImpl
    from transformers.modeling_utils import ALL_ATTENTION_FUNCTIONS

    case = next(c for c in GOLD["model"] if c["name"] == "spinquant" and c["quant"])
    model = run_model_case(case, "cuda")["model"]
    mods = [m for m in model.modules() if hasattr(m, KV_CACHE_ATTR)]
    assert mods and all(hasattr(m, IMPL_ATTR) for m in mods)
    pre, post, handles = [{} for _ in mods], [{} for _ in mods], []

    def capture(store, base, sub):
        signature = inspect.signature(sub.forward)

        def hook(_sub, args, kwargs):
            store[base] = signature.bind(*args, **kwargs).arguments["query" if base == "q" else "key_states"].detach().clone()
        return sub.register_forward_pre_hook(hook, with_kwargs=True, prepend=True)

    for i, m in enumerate(mods):
        def post_k(_cache, _args, out, i=i):
            post[i]["k"] = out[0].detach().clone()
        handles += [capture(pre[i], "k", getattr(m, KV_CACHE_ATTR)), capture(pre[i], "q", getattr(m, IMPL_ATTR)),
                    getattr(m, KV_CACHE_ATTR).register_forward_hook(post_k)]
    original, queries = QuantizedAttentionImpl._original_impl, []

    def recording_attention(module, query, key, value, *a, **k):
        queries.append(query.detach().clone())
        return ALL_ATTENTION_FUNCTIONS[original](module, query, key, value, *a, **k)

    ALL_ATTENTION_FUNCTIONS["r3_test_record"] = recording_attention     # this instance only, removed below
    QuantizedAttentionImpl._original_impl = "r3_test_record"
    try:
        with torch.no_grad():
            model(case["ids"].cuda(), use_cache=False)
    finally:
        QuantizedAttentionImpl._original_impl = original
        del ALL_ATTENTION_FUNCTIONS["r3_test_record"]
        for h in handles:
            h.remove()
    assert len(queries) == len(mods)
    for i, m in enumerate(mods):
        post[i]["q"] = queries[i]
        for base, location in (("q", "q_attn"), ("k", "k_cache")):
            t = getattr(m, f"R3_{location}")
            n, perm = t.weight.shape[0], getattr(t, "perm", None)
            x = pre[i][base]
            rotated = _eager(x.cpu().contiguous(), n, t.weight[:, 0].cpu(), None if perm is None else perm.cpu(), bool(t.args.inverse),
                             t.weight.dtype)
            zp = getattr(m, f"{base}_zero_point", None)
            want = oracle.fake_quantize(rotated, getattr(m, f"{base}_scale").cpu(), zp.cpu() if zp is not None else None,
                                        strategy="tensor", num_bits=8, qtype="float")
            assert not torch.equal(rotated, x.cpu())
            same(post[i][base].cpu(), want, f"layer {i} {base}")


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
