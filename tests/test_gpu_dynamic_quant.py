"""
ops.dynamic_fake_quantize (ct_dynamic_fake_quantize: the dynamic activation observer fused with fake_quantize) on the GPU:
  * every case of tests/golden/dynamic.pt.gz: output, scale and zero point bit-identical to the reference's, and to the two-step GPU
    path (compute_dynamic_scales_and_zp + ops.fake_quantize) in the same process
  * inputs outside the fused path (fp32, non-contiguous, g_idx, ragged groups, cols % 8 != 0) give what the two steps give
  * the fake-quantized inputs of every quantized Linear of a seeded 2-layer Llama equal the two-step path's
  * the fused op is enqueue-only: it can be captured in a CUDA graph
"""
import pytest
import torch

from compressed_tensors_b200 import _native as N
from compressed_tensors_b200 import ops
from tests.test_dynamic_quant_host import CASES, INPUTS, args_of, case_id, module_for
from tests.util import same

pytestmark = pytest.mark.gpu
DEV = "cuda"


def two_step(x, args, gs=None, g_idx=None):
    from compressed_tensors_b200.quantization.utils import compute_dynamic_scales_and_zp

    scale, zp = compute_dynamic_scales_and_zp(value=x, args=args, module=None, global_scale=gs)
    return ops.fake_quantize(x, scale, zp, args, g_idx=g_idx, global_scale=gs), scale, zp


def without_fused(monkeypatch):
    monkeypatch.setattr(ops, "dynamic_fake_quantize", lambda *a, **k: None)


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_golden_cases_are_bit_identical(case):
    args, x = args_of(case), INPUTS[case["input"]].to(DEV)
    gs = case["global_scale"].to(DEV) if case["global_scale"] is not None else None
    n0 = N.launch_count()
    res = ops.dynamic_fake_quantize(x, args, global_scale=gs)
    assert res is not None, N.last_error()
    strategy = args.strategy.value if hasattr(args.strategy, "value") else args.strategy
    one_scale = strategy == "tensor" or (strategy == "token" and x.ndim <= 2)
    assert N.launch_count() - n0 == (2 if one_scale else 1)
    out, scale, zp = res
    same(out.cpu(), case["out"], "out vs golden")
    same(scale.cpu(), case["scale"], "scale vs golden")
    same(zp.cpu(), case["zero_point"], "zero point vs golden")
    ref_out, ref_scale, ref_zp = two_step(x, args, gs)
    same(out, ref_out, "out vs two-step")
    same(scale, ref_scale, "scale vs two-step")
    same(zp, ref_zp, "zero point vs two-step")
    # forward_quantize takes the fused path and returns the same
    from compressed_tensors_b200.quantization.lifecycle.forward import forward_quantize

    m = module_for(case)
    if gs is not None:
        m.input_global_scale = gs
    same(forward_quantize(m, x, "input", args), ref_out, "forward_quantize")


def _args(**kw):
    from compressed_tensors_b200.quantization import QuantizationArgs

    base = dict(num_bits=8, type="int", strategy="token", symmetric=True, dynamic=True)
    base.update(kw)
    return QuantizationArgs(**base)


def _outcome(fn):
    try:
        return fn()
    except Exception as e:   # noqa: BLE001 -- the exception type and message are what is compared
        return (type(e), str(e))


@pytest.mark.parametrize("what", ["fp32", "non_contiguous", "g_idx", "ragged_group", "cols_not_8", "group_256", "wider_than_32768",
                                  "asym_fp8", "int4_token_fp16"])
def test_inputs_outside_the_fused_path_behave_as_before(what, monkeypatch):
    from compressed_tensors_b200.quantization.lifecycle.forward import forward_quantize

    gen = torch.Generator().manual_seed(7)
    x = torch.randn(3, 5, 256, generator=gen).to(torch.bfloat16).to(DEV)
    args = _args()
    m = torch.nn.Module()
    if what == "fp32":
        x = x.float()
    elif what == "non_contiguous":
        x = x.transpose(0, 1)
    elif what == "g_idx":
        args = _args(strategy="group", group_size=64)
        m.weight_g_idx = torch.randperm(256, generator=gen).div(64, rounding_mode="floor").to(torch.int32).to(DEV)
    elif what == "ragged_group":
        args, x = _args(strategy="group", group_size=128), x[..., :192].contiguous()
    elif what == "cols_not_8":
        x = x[..., :252].contiguous()
    elif what == "group_256":
        args = _args(strategy="group", group_size=256)
    elif what == "wider_than_32768":
        x = torch.randn(1, 2, 32768 + 512, generator=gen).to(torch.bfloat16).to(DEV)
    elif what == "asym_fp8":
        args = _args(type="float", symmetric=False)
    else:
        args, x = _args(num_bits=4), x.half()
    got = _outcome(lambda: forward_quantize(m, x, "input", args))
    with monkeypatch.context() as mp:
        without_fused(mp)
        want = _outcome(lambda: forward_quantize(m, x, "input", args))
    if isinstance(want, tuple):
        assert got == want
    else:
        same(got, want, what)
    if what in ("group_256", "int4_token_fp16"):   # inside the fused path after all: the fused op must agree too
        res = ops.dynamic_fake_quantize(x, args)
        if res is not None:
            same(res[0], want, what)


def test_widest_rows_and_ragged_row_counts():
    """TOKEN rows of 28672 / 29568 / 32768 columns (the 512-thread CTA) and group counts that are not a multiple of the tile"""
    gen = torch.Generator().manual_seed(11)
    for cols, rows, args in ((28672, 3, _args()), (29568, 5, _args(type="float")), (32768, 2, _args(symmetric=False)),
                             (4104, 7, _args()), (1040, 33, _args(strategy="group", group_size=16, type="float")),
                             (160, 1001, _args(strategy="group", group_size=32, type="float", scale_dtype=torch.uint8, zp_dtype=torch.uint8))):
        x = (torch.randn(1, rows, cols, generator=gen) * 3).to(torch.bfloat16).to(DEV)
        res = ops.dynamic_fake_quantize(x, args)
        assert res is not None, (cols, N.last_error())
        want = two_step(x, args)
        for a, b, what in zip(res, want, ("out", "scale", "zero point")):
            same(a, b, f"{cols}x{rows} {what}")


def test_llama_linear_inputs_match_the_two_step_path(monkeypatch):
    transformers = pytest.importorskip("transformers")
    from compressed_tensors_b200.quantization import QuantizationConfig, QuantizationScheme, apply_quantization_config, preset_name_to_scheme

    cfg = transformers.LlamaConfig(num_hidden_layers=2, hidden_size=256, num_attention_heads=4, num_key_value_heads=2, head_dim=64,
                                   vocab_size=256, intermediate_size=512, max_position_embeddings=128)
    ids = torch.randint(0, 256, (2, 48), generator=torch.Generator().manual_seed(5)).to(DEV)
    for preset in ("FP8_DYNAMIC", "W8A8", "NVFP4", "MXFP4"):
        torch.manual_seed(1234)
        model = transformers.LlamaForCausalLM(cfg).to(torch.bfloat16).to(DEV).eval()
        acts = preset_name_to_scheme(preset, ["Linear"]).input_activations
        apply_quantization_config(model, QuantizationConfig(config_groups={"g": QuantizationScheme(targets=["Linear"], input_activations=acts)}))
        for name, p in model.named_parameters():
            if name.endswith("input_global_scale"):
                p.data.fill_(64.0)
        linears = {m: n for n, m in model.named_modules() if isinstance(m, torch.nn.Linear) and getattr(m, "quantization_scheme", None)}
        assert linears

        def run():
            seen = {}
            orig = torch.nn.Linear.forward

            def record(self, input):
                if self in linears:
                    seen[linears[self]] = input.clone()
                return orig(self, input)

            with monkeypatch.context() as mp:
                mp.setattr(torch.nn.Linear, "forward", record)
                with torch.no_grad():
                    model(ids)
            return seen

        fused_calls = []
        real = ops.dynamic_fake_quantize
        with monkeypatch.context() as mp:
            mp.setattr(ops, "dynamic_fake_quantize", lambda *a, **k: fused_calls.append(1) or real(*a, **k))
            fused = run()
        with monkeypatch.context() as mp:
            without_fused(mp)
            ref = run()
        assert fused_calls and set(fused) == set(ref) == set(linears.values())
        for n in ref:
            same(fused[n], ref[n], f"{preset} {n}")


def test_fused_op_is_capturable_in_a_cuda_graph():
    gen = torch.Generator().manual_seed(3)
    cases = [(_args(), (4, 16, 4096)), (_args(strategy="group", group_size=128, type="float"), (2, 8, 1024)),
             (_args(strategy="tensor", symmetric=False), (4, 1024))]
    for args, shape in cases:
        x = torch.randn(shape, generator=gen).to(torch.bfloat16).to(DEV)
        ops.dynamic_fake_quantize(x, args)   # warm-up outside the capture
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        g = torch.cuda.CUDAGraph()
        with torch.cuda.stream(s):
            with torch.cuda.graph(g, stream=s):
                res = ops.dynamic_fake_quantize(x, args)
        torch.cuda.current_stream().wait_stream(s)
        x.copy_(torch.randn(shape, generator=gen).to(torch.bfloat16))
        g.replay()
        torch.cuda.synchronize()
        want = two_step(x, args)
        for a, b in zip(res, want):
            same(a, b, f"graph replay {shape}")
