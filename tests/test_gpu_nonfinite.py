"""
NaN and infinite inputs and scales on the GPU, against tests/golden/nonfinite.pt.gz (the reference) and the oracle.  Fake-quantized
values and scales must put NaN where the reference does (any payload) and match everywhere else bit for bit; zero points are compared
where the reference did not cast a NaN to int8.  Integer and fp8 codes made from NaN are undefined in the reference and not compared.
  * static fake_quantize: the streaming kernel (bf16, fp16, fp32) and the generic one (NVFP4: global scale, fp4), and all 65536 bf16 /
    fp16 bit patterns through int4, int8 with a zero point and fp8 at scales 2^-7, 1, 37.5 and inf against the oracle
  * dynamic activations: ops.dynamic_fake_quantize and forward_quantize against the golden and the two-step path, with the launch
    counts of finite inputs
  * fake_quantize_heads on transposed [B, H, S, D] views
  * the tensor, channel and group observers and the NVFP4 global scale
"""
import pytest
import torch

import oracle
from compressed_tensors_b200 import _native as N
from compressed_tensors_b200 import ops
from tests.test_dynamic_quant_host import args_of, module_for
from tests.test_gpu_dynamic_quant import two_step
from tests.test_nonfinite_host import DYNAMIC, HEADS, QPARAMS, STATIC, STATIC_INPUTS, INPUTS, dynamic_id, qparams_id, same_zp, \
    static_args, static_id
from tests.util import same_nan

pytestmark = pytest.mark.gpu
DEV = "cuda"


def dev(t):
    return None if t is None else t.to(DEV)


# ---------------------------------------------------------------------------------------------------------------------------------
# (A) static fake_quantize
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", STATIC, ids=static_id)
def test_static_fake_quantize_matches_the_golden(case):
    x = STATIC_INPUTS[case["x"]].to(DEV)
    out = ops.fake_quantize(x, dev(case["scale"]), dev(case["zero_point"]), static_args(case), global_scale=dev(case["global_scale"]))
    same_nan(out.cpu(), case["out"], "fake_quantize")


SWEEP = {"int4": (4, "int", False), "int8_zp": (8, "int", True), "fp8": (8, "float", False)}


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("scheme", list(SWEEP))
@pytest.mark.parametrize("scale", [2.0 ** -7, 1.0, 37.5, float("inf")], ids=["2^-7", "1", "37.5", "inf"])
def test_every_bit_pattern_matches_the_oracle(dtype, scheme, scale):
    from compressed_tensors_b200.quantization import QuantizationArgs

    bits, qtype, zp = SWEEP[scheme]
    x = torch.arange(-32768, 32768, dtype=torch.int32).to(torch.int16).view(dtype).reshape(-1, 64)
    s = torch.tensor([scale], dtype=dtype)
    z = torch.tensor([-5], dtype=torch.int8) if zp else None
    want = oracle.fake_quantize(x, s, z, strategy="tensor", num_bits=bits, qtype=qtype)
    assert bool(want.isnan().any())
    args = QuantizationArgs(num_bits=bits, type=qtype, symmetric=not zp, strategy="tensor")
    same_nan(ops.fake_quantize(x.to(DEV), s.to(DEV), dev(z), args).cpu(), want, f"{scheme} scale {scale}")


# ---------------------------------------------------------------------------------------------------------------------------------
# (B) dynamic activations
# ---------------------------------------------------------------------------------------------------------------------------------
def nan_free_groups(args, x):
    """None, or for MX schemes the groups of 32 that hold no NaN.  The reference's MX scale of a group with a NaN depends on the NaN
    bits torch's CPU reductions return, which vary with the NaN's position in the group (tests/golden/nonfinite.pt.gz has both
    outcomes); those groups are left out, every other group (inf ones included) is compared"""
    if args.scale_dtype != torch.uint8:
        return None
    return ~x.cpu().reshape(-1, 32).isnan().any(1)


def same_groups(got, want, keep, what):
    if keep is None:
        same_nan(got.cpu(), want.cpu(), what)
    elif got.numel() == keep.numel():
        same_nan(got.cpu().reshape(-1)[keep], want.cpu().reshape(-1)[keep], what)
    else:
        same_nan(got.cpu().reshape(-1, 32)[keep], want.cpu().reshape(-1, 32)[keep], what)


@pytest.mark.parametrize("case", DYNAMIC, ids=dynamic_id)
def test_dynamic_fake_quantize_matches_the_golden_and_the_two_steps(case):
    from compressed_tensors_b200.quantization.lifecycle.forward import forward_quantize

    args, x = args_of(case), INPUTS[case["input"]].to(DEV)
    gs = dev(case["global_scale"])
    defined = case["zp_defined"]
    keep = nan_free_groups(args, x)
    n0 = N.launch_count()
    res = ops.dynamic_fake_quantize(x, args, global_scale=gs)
    assert res is not None, N.last_error()
    strategy = args.strategy.value if hasattr(args.strategy, "value") else args.strategy
    one_scale = strategy == "tensor" or (strategy == "token" and x.ndim <= 2)
    assert N.launch_count() - n0 == (2 if one_scale else 1)   # as for finite inputs: NaN handling adds no launch
    out, scale, zp = res
    same_groups(out, case["out"], keep, "out vs golden")
    same_groups(scale, case["scale"], keep, "scale vs golden")
    same_zp(zp.cpu(), case["zero_point"], defined, "zero point vs golden")
    ref_out, ref_scale, ref_zp = two_step(x, args, gs)
    same_groups(ref_scale, case["scale"], keep, "two-step scale vs golden")
    same_groups(scale, ref_scale, keep, "scale vs two-step")
    same_zp(zp.cpu(), ref_zp.cpu(), defined, "zero point vs two-step")
    if bool(defined.all()):   # the two steps use the zero point they cast; the fused op's values behind an undefined one are NaN
        same_groups(out, ref_out, keep, "out vs two-step")
    m = module_for(case)
    if gs is not None:
        m.input_global_scale = gs
    same_groups(forward_quantize(m, x, "input", args), case["out"], keep, "forward_quantize vs golden")


# ---------------------------------------------------------------------------------------------------------------------------------
# (C) KV heads
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", HEADS, ids=lambda c: f"{c['args']['strategy']}-{str(c['x'].dtype)[6:]}-nan_scale{bool(c['scale'].isnan().any())}")
def test_fake_quantize_heads_on_transposed_views(case):
    from compressed_tensors_b200.quantization import QuantizationArgs

    x = case["x"]
    view = x.transpose(1, 2).contiguous().to(DEV).transpose(1, 2)   # [B, S, H, D] storage seen as [B, H, S, D], as transformers hands it over
    assert not view.is_contiguous()
    n0 = N.launch_count()
    (out,) = ops.fake_quantize_heads([view], [dev(case["scale"])], [dev(case["zero_point"])], QuantizationArgs(**case["args"]))
    assert N.launch_count() - n0 == 1
    same_nan(out.cpu(), case["out"], "fake_quantize_heads")


# ---------------------------------------------------------------------------------------------------------------------------------
# (D) observers
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", QPARAMS, ids=qparams_id)
def test_observers_match_the_reference_qparams(case):
    from compressed_tensors_b200.quantization import QuantizationArgs

    a, w = case["args"], case["x"].to(DEV)
    args = QuantizationArgs(**a)
    defined = case["zp_defined"]
    if a["strategy"] == "tensor":
        scale, zp = ops.observe_tensor_qparams(w, args)
        same_nan(scale.cpu(), case["scale"], "observe_tensor_qparams scale")
        if zp is not None:
            same_zp(zp.cpu(), case["zero_point"], defined, "observe_tensor_qparams zero point")
        same_nan(ops.observe_tensor_gparam(w).cpu(), case["gparam"], "observe_tensor_gparam")
    if a["strategy"] == "group":
        _, scale, zp = ops.observe_quantize_pack(w, args)
    else:
        _, scale, zp = ops.observe_quantize(w, args)
    same_nan(scale.cpu().reshape(case["scale"].shape), case["scale"], "observe_quantize scale")
    if zp is not None:
        same_zp(zp.cpu(), case["zero_point"], defined, "observe_quantize zero point")
