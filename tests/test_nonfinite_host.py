"""
CPU checks of NaN and infinite inputs and scales against tests/golden/nonfinite.pt.gz (recorded from the reference by
make_golden_nonfinite.py).  Fake-quantized values and scales are floats with defined values: NaN must land where the reference puts
it (any payload), everything else bit for bit.  A zero point is compared only where the reference did not cast a NaN to int8.
  * the golden agrees with the oracle (oracle.fake_quantize, oracle.qparams.calculate_qparams), which the GPU tests compare against
  * fake_quantize, compute_dynamic_scales_and_zp and forward_quantize on CPU tensors (the CPU twins) reproduce the golden
"""
import pytest
import torch

import oracle
from oracle.qparams import calculate_qparams as oracle_qparams
from tests import golden
from tests.test_dynamic_quant_host import args_of, module_for, observe, two_d
from tests.util import same, same_nan

GOLDEN = golden.load("nonfinite")
STATIC_INPUTS = GOLDEN["static_inputs"]
STATIC = GOLDEN["static"]
INPUTS = GOLDEN["inputs"]
DYNAMIC = GOLDEN["dynamic"]
HEADS = GOLDEN["heads"]
QPARAMS = GOLDEN["qparams"]


def static_id(c):
    x = STATIC_INPUTS[c["x"]]
    s = c["scale"]
    sv = f"{s.flatten()[0].item():g}" if s.numel() == 1 or c["args"]["strategy"] == "tensor_group" else f"{c['args']['strategy']}"
    return f"{c['scheme']}-{str(x.dtype)[6:]}-{sv}"


def dynamic_id(c):
    x = INPUTS[c["input"]]
    gs = "" if c["global_scale"] is None else f"-gs{c['global_scale'].item():g}"
    return f"{c['scheme']}-{str(x.dtype)[6:]}-{'x'.join(map(str, x.shape))}{gs}"


def qparams_id(c):
    return f"{c['scheme']}-{c['args']['strategy']}-{str(c['x'].dtype)[6:]}-{c['plant']}"


def static_args(c):
    from compressed_tensors_b200.quantization import QuantizationArgs

    return QuantizationArgs(**c["args"])


def oracle_static(c, x=None):
    a = c["args"]
    x = STATIC_INPUTS[c["x"]] if x is None else x
    return oracle.fake_quantize(x, c["scale"], c["zero_point"], strategy=a["strategy"], group_size=a.get("group_size"),
                                num_bits=a["num_bits"], qtype=a["type"], global_scale=c["global_scale"])


def observe_w(w, strategy, group):
    """the observer's min / max of a 2-D weight for TENSOR ([1]), CHANNEL ([R, 1]) or GROUP ([R, C / group])"""
    if strategy == "tensor":
        return w.amin().reshape(1), w.amax().reshape(1)
    if strategy == "channel":
        return w.amin(dim=1, keepdim=True), w.amax(dim=1, keepdim=True)
    g = w.unflatten(-1, (w.shape[1] // group, group))
    return g.amin(dim=-1), g.amax(dim=-1)


def same_zp(got, want, defined, what):
    same(got.reshape(want.shape)[defined], want[defined], what)


# ---------------------------------------------------------------------------------------------------------------------------------
# (A) static fake_quantize
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", STATIC, ids=static_id)
def test_static_golden_agrees_with_the_oracle(case):
    same_nan(oracle_static(case), case["out"], "oracle fake_quantize")


@pytest.mark.parametrize("case", STATIC, ids=static_id)
def test_static_cpu_twin_reproduces_the_golden(case):
    from compressed_tensors_b200 import ops

    x = STATIC_INPUTS[case["x"]]
    if case["scheme"] == "nvfp4":
        with pytest.raises(NotImplementedError, match="CPU twins"):   # the CPU twins have no FP4 arithmetic
            ops.fake_quantize(x, case["scale"], case["zero_point"], static_args(case), global_scale=case["global_scale"])
        return
    same_nan(ops.fake_quantize(x, case["scale"], case["zero_point"], static_args(case), global_scale=case["global_scale"]), case["out"],
             "fake_quantize (CPU twin)")


def test_static_golden_covers_every_pattern_at_every_lane():
    per_tensor = sorted({c["x"] for c in STATIC if c["args"]["strategy"] == "tensor"})
    assert [STATIC_INPUTS[i].dtype for i in per_tensor] == [torch.bfloat16, torch.float16, torch.float32]
    for x in (STATIC_INPUTS[i] for i in per_tensor[:2]):
        bits = x.flatten().view(torch.int16).to(torch.int32) & 0xFFFF
        mant = 7 if x.dtype == torch.bfloat16 else 10
        exp_all = ((1 << (15 - mant)) - 1) << mant
        lanes = torch.arange(bits.numel()) % 8
        special = (bits & exp_all) == exp_all
        seen = torch.zeros(1 << 16, 8, dtype=torch.bool)
        seen[bits[special], lanes[special]] = True
        assert int(seen.any(1).sum()) == 2 << mant and bool(seen[seen.any(1)].all())   # every NaN / inf pattern at all 8 lanes
        assert bool((~special).any())
    scales = {float(c["scale"].flatten()[0]) for c in STATIC if c["args"]["strategy"] == "tensor"}
    assert scales == {2.0 ** -7, 1.0, 37.5, float("inf")}


# ---------------------------------------------------------------------------------------------------------------------------------
# (B) dynamic activations
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", DYNAMIC, ids=dynamic_id)
def test_dynamic_golden_agrees_with_the_oracle(case):
    args = args_of(case)
    x = INPUTS[case["input"]]
    x2, s2, z2, strategy = two_d(x, case["scale"], case["zero_point"], args)
    qtype = args.type.value if hasattr(args.type, "value") else args.type
    if not (args.num_bits == 4 and qtype == "float") and args.scale_dtype is None and case["global_scale"] is None:
        mn, mx = observe(x2, strategy, args.group_size)
        s, z = oracle_qparams(mn, mx, num_bits=args.num_bits, qtype=qtype, symmetric=args.symmetric)
        same_nan(s.reshape(s2.shape), s2, "scale")
        same_zp(z, case["zero_point"], case["zp_defined"], "zero point")
    z2 = torch.where(case["zp_defined"], case["zero_point"], torch.zeros_like(case["zero_point"])).reshape(z2.shape) \
        if case["zero_point"].dtype == torch.int8 else z2
    out = oracle.fake_quantize(x2, s2, z2, strategy=strategy, group_size=args.group_size, num_bits=args.num_bits, qtype=qtype,
                               global_scale=case["global_scale"])
    same_nan(out.reshape(x.shape), case["out"], "fake-quantized values")


@pytest.mark.parametrize("case", DYNAMIC, ids=dynamic_id)
def test_dynamic_cpu_path_reproduces_the_golden(case):
    from compressed_tensors_b200.quantization.lifecycle.forward import forward_quantize
    from compressed_tensors_b200.quantization.utils import compute_dynamic_scales_and_zp

    args, x, m = args_of(case), INPUTS[case["input"]], module_for(case)
    scale, zp = compute_dynamic_scales_and_zp(value=x, args=args, module=m, global_scale=case["global_scale"])
    same_nan(scale, case["scale"], "scale")
    same_zp(zp, case["zero_point"], case["zp_defined"], "zero point")
    if args.num_bits == 4 and args.type == "float":
        return   # the CPU twins have no FP4 arithmetic (test_dynamic_quant_host.py checks that they say so)
    if not bool(case["zp_defined"].all()):
        return   # the CPU twin casts the undefined zero point its own way; the values behind it are NaN in any case
    same_nan(forward_quantize(m, x, "input", args), case["out"], "forward_quantize")


def test_dynamic_golden_holds_the_planted_values():
    """NaN at lane 0 / lane 7 / the end of a row / a whole row / the tail, +-inf, fp16 overflow, and NaN, inf and finite scales"""
    for x in INPUTS:
        assert bool(x.isnan().any()) and bool(x.isfinite().any())
    assert any(bool(x.isposinf().any()) and bool(x.isneginf().any()) for x in INPUTS if x.dtype == torch.float16)
    assert any(INPUTS[c["input"]].shape[-1] == 32768 for c in DYNAMIC)
    for scheme in ("W8A8", "FP8_DYNAMIC", "MXFP4", "NVFP4"):
        scales = torch.cat([c["scale"].float().flatten() for c in DYNAMIC if c["scheme"] == scheme])
        assert bool(scales.isnan().any() or scales.isinf().any()) and bool(scales.isfinite().any()), scheme
    assert not all(bool(c["zp_defined"].all()) for c in DYNAMIC)


# ---------------------------------------------------------------------------------------------------------------------------------
# (C) KV heads, (D) observer qparams
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", HEADS, ids=lambda c: f"{c['args']['strategy']}-{str(c['x'].dtype)[6:]}-nan_scale{bool(c['scale'].isnan().any())}")
def test_heads_golden_agrees_with_the_oracle(case):
    a = case["args"]
    got = oracle.fake_quantize(case["x"], case["scale"], case["zero_point"], strategy=a["strategy"], num_bits=a["num_bits"], qtype=a["type"])
    same_nan(got, case["out"], "oracle fake_quantize")


@pytest.mark.parametrize("case", QPARAMS, ids=qparams_id)
def test_qparams_golden_agrees_with_the_oracle(case):
    a = case["args"]
    mn, mx = observe_w(case["x"], a["strategy"], a.get("group_size"))
    s, z = oracle_qparams(mn, mx, num_bits=a["num_bits"], qtype=a["type"], symmetric=a["symmetric"])
    same_nan(s.reshape(case["scale"].shape), case["scale"], "scale")
    same_zp(z, case["zero_point"], case["zp_defined"], "zero point")


@pytest.mark.parametrize("case", QPARAMS, ids=qparams_id)
def test_qparams_host_rule_reproduces_the_golden(case):
    from compressed_tensors_b200.quantization import QuantizationArgs
    from compressed_tensors_b200.quantization.utils import calculate_qparams, generate_gparam

    a, w = case["args"], case["x"]
    mn, mx = observe_w(w, a["strategy"], a.get("group_size"))
    s, z = calculate_qparams(mn, mx, QuantizationArgs(**a))
    same_nan(s, case["scale"], "scale")
    same_zp(z, case["zero_point"], case["zp_defined"], "zero point")
    same_nan(generate_gparam(w.amin(), w.amax()), case["gparam"], "generate_gparam")
