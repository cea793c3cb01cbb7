"""
CPU checks of dynamic activation quantization against tests/golden/dynamic.pt.gz (recorded from the reference by
make_golden_dynamic.py):
  * the golden agrees with the CPU oracle composed as min / max -> oracle calculate_qparams -> oracle fake_quantize, wherever the
    oracle covers the scheme (int / fp8 qparams; the fake quantization of every scheme, FP4 and MX included, with the golden qparams)
  * compute_dynamic_scales_and_zp and forward_quantize on CPU tensors (the CPU twins) reproduce the golden, so the CPU / eager path
    is unchanged
  * the dispatch of forward_quantize and ops.dynamic_fake_quantize: which inputs take the fused kernel and which the two steps, and
    what descriptor reaches the native entry, checked with a stub of the native call (no CUDA needed)
"""
import math

import pytest
import torch

import oracle
from oracle.qparams import calculate_qparams as oracle_qparams
from tests import golden
from tests.util import same

GOLDEN = golden.load("dynamic")
INPUTS = GOLDEN["inputs"]
CASES = GOLDEN["cases"]


def args_of(case):
    from compressed_tensors_b200.quantization import QuantizationArgs, preset_name_to_scheme

    if case["args"]:
        return QuantizationArgs(**case["args"])
    return preset_name_to_scheme(case["scheme"], ["Linear"]).input_activations


def case_id(case):
    x = INPUTS[case["input"]]
    gs = "" if case["global_scale"] is None else f"-gs{case['global_scale'].item():g}"
    return f"{case['scheme']}-{str(x.dtype)[6:]}-{'x'.join(map(str, x.shape))}{gs}"


def module_for(case):
    m = torch.nn.Module()
    if case["global_scale"] is not None:
        m.input_global_scale = case["global_scale"]
    return m


def two_d(x, scale, zp, args):
    """x and its qparams as the 2-D problem fake_quantize solves: rows of a token / group, or the whole tensor"""
    strategy = args.strategy.value if hasattr(args.strategy, "value") else args.strategy
    if strategy == "token" and x.ndim > 2:
        rows = x.shape[0] * x.shape[1]
        return x.reshape(rows, -1), scale.reshape(rows, 1), zp.reshape(rows, 1), "channel"
    if strategy in ("group", "tensor_group"):
        x2 = x.reshape(-1, x.shape[-1])
        return x2, scale.reshape(x2.shape[0], -1), zp.reshape(x2.shape[0], -1), "group"
    return x.reshape(-1, x.shape[-1]), scale, zp, "tensor"


def observe(x2, strategy, group_size):
    if strategy == "channel":
        return x2.amin(dim=1, keepdim=True), x2.amax(dim=1, keepdim=True)
    if strategy == "group":
        g = x2.unflatten(-1, (x2.shape[-1] // group_size, group_size))
        return g.amin(dim=-1), g.amax(dim=-1)
    return torch.aminmax(x2)


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_golden_agrees_with_the_oracle(case):
    args = args_of(case)
    x = INPUTS[case["input"]]
    x2, s2, z2, strategy = two_d(x, case["scale"], case["zero_point"], args)
    qtype = args.type.value if hasattr(args.type, "value") else args.type
    fp4_or_scaled = args.num_bits == 4 or args.scale_dtype is not None or case["global_scale"] is not None
    if not fp4_or_scaled:
        mn, mx = observe(x2, strategy, args.group_size)
        s, z = oracle_qparams(mn, mx, num_bits=args.num_bits, qtype=qtype, symmetric=args.symmetric)
        same(s.reshape(s2.shape), s2, "scale")
        same(z.reshape(z2.shape), z2, "zero point")
    out = oracle.fake_quantize(x2, s2, z2, strategy=strategy, group_size=args.group_size, num_bits=args.num_bits, qtype=qtype,
                               global_scale=case["global_scale"])
    same(out.reshape(x.shape), case["out"], "fake-quantized values")


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_cpu_path_reproduces_the_golden(case):
    from compressed_tensors_b200.quantization.lifecycle.forward import forward_quantize
    from compressed_tensors_b200.quantization.utils import compute_dynamic_scales_and_zp

    args, x, m = args_of(case), INPUTS[case["input"]], module_for(case)
    scale, zp = compute_dynamic_scales_and_zp(value=x, args=args, module=m, global_scale=case["global_scale"])
    same(scale, case["scale"], "scale")
    same(zp, case["zero_point"], "zero point")
    if args.num_bits == 4 and args.type == "float":
        with pytest.raises(NotImplementedError, match="CPU twins"):   # the CPU twins have no FP4 arithmetic
            forward_quantize(m, x, "input", args)
        return
    same(forward_quantize(m, x, "input", args), case["out"], "forward_quantize")


# ---------------------------------------------------------------------------------------------------------------------------
# dispatch, with the native call stubbed
# ---------------------------------------------------------------------------------------------------------------------------
class _OnDevice(torch.Tensor):
    """a CPU tensor that reports itself as a CUDA tensor, so that the dispatch can be exercised without one"""

    @property
    def is_cuda(self):
        return True


class _StubLib:
    def __init__(self, rc=0):
        self.rc, self.calls = rc, []

    def ct_dynamic_fake_quantize(self, dref, asym, scale_round, x, out, scale, zp, idx, stream):
        d = dref._obj   # the QuantDesc behind ctypes.byref
        self.calls.append(dict(rows=d.rows, cols=d.cols, rdiv=d.rdiv, cdiv=d.cdiv, srs=d.s_row_stride, x_dtype=d.x_dtype, scale_dtype=d.scale_dtype,
                               zp_dtype=d.zp_dtype, compute_dtype=d.compute_dtype, seff_dtype=d.seff_dtype, qtype=d.qtype, bits=d.num_bits,
                               gs=bool(d.global_scale), asym=asym, scale_round=scale_round))
        return self.rc


@pytest.fixture
def stub(monkeypatch):
    from compressed_tensors_b200 import _native as N

    lib = _StubLib()
    monkeypatch.setattr(N, "lib", lambda: lib)
    monkeypatch.setattr(N, "stream_ptr", lambda idx: None)
    return lib


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_fused_op_builds_the_reference_qparam_shapes_and_descriptor(case, stub):
    from compressed_tensors_b200 import _native as N
    from compressed_tensors_b200 import ops

    args, x = args_of(case), INPUTS[case["input"]]
    res = ops.dynamic_fake_quantize(x.as_subclass(_OnDevice), args, global_scale=case["global_scale"])
    assert res is not None and len(stub.calls) == 1
    out, scale, zp = res
    assert out.shape == x.shape and out.dtype == x.dtype
    assert scale.shape == case["scale"].shape and scale.dtype == case["scale"].dtype
    assert zp.shape == case["zero_point"].shape and zp.dtype == case["zero_point"].dtype
    c = stub.calls[0]
    strategy = args.strategy.value if hasattr(args.strategy, "value") else args.strategy
    assert c["rows"] * c["cols"] == x.numel() and c["x_dtype"] == N.DT[x.dtype] and c["scale_dtype"] == N.DT[scale.dtype]
    if strategy == "token" and x.ndim > 2:
        assert (c["rows"], c["rdiv"], c["cdiv"], c["srs"]) == (x.shape[0] * x.shape[1], 1, N.INF, 1)
    elif strategy in ("token", "tensor"):
        assert (c["rdiv"], c["cdiv"], c["srs"]) == (N.INF, N.INF, 0)   # a 2-D value under TOKEN reduces over the whole tensor
    else:
        assert (c["cols"], c["rdiv"], c["cdiv"], c["srs"]) == (x.shape[-1], 1, args.group_size, x.shape[-1] // args.group_size)
    assert c["asym"] == (0 if args.symmetric else 1) and c["gs"] == (case["global_scale"] is not None)
    assert c["scale_round"] == {None: N.DT_NONE, torch.float8_e4m3fn: N.DT[torch.float8_e4m3fn], torch.uint8: N.DT_E8M0}[args.scale_dtype]
    # compute / effective scale dtypes are those fake_quantize derives from the returned scale
    assert c["seff_dtype"] == N.DT[scale.dtype] and c["compute_dtype"] == N.DT[torch.promote_types(x.dtype, scale.dtype)]


def _args(**kw):
    from compressed_tensors_b200.quantization import QuantizationArgs

    base = dict(num_bits=8, type="int", strategy="token", symmetric=True, dynamic=True)
    base.update(kw)
    return QuantizationArgs(**base)


@pytest.mark.parametrize("what", ["cpu", "fp32", "cols_not_8", "ragged_group", "zero_dim", "channel", "float16_bits"])
def test_fused_op_declines_without_calling_the_library(what, stub):
    from compressed_tensors_b200 import ops

    x, args = torch.randn(4, 6, 64, dtype=torch.bfloat16).as_subclass(_OnDevice), _args()
    if what == "cpu":
        x = torch.randn(4, 6, 64, dtype=torch.bfloat16)
    elif what == "fp32":
        x = torch.randn(4, 6, 64).as_subclass(_OnDevice)
    elif what == "cols_not_8":
        x = torch.randn(4, 6, 60, dtype=torch.bfloat16).as_subclass(_OnDevice)
    elif what == "ragged_group":
        args = _args(strategy="group", group_size=128, type="float")
    elif what == "zero_dim":
        x = torch.tensor(1.0, dtype=torch.bfloat16).as_subclass(_OnDevice)
    elif what == "channel":
        args = _args(strategy="channel", dynamic=False)
    else:
        args = _args(num_bits=16)
    assert ops.dynamic_fake_quantize(x, args) is None
    assert stub.calls == []


def test_fused_op_declines_non_contiguous_values_and_unsupported_answers(stub):
    from compressed_tensors_b200 import _native as N
    from compressed_tensors_b200 import ops

    x = torch.randn(4, 64, 6, dtype=torch.bfloat16).transpose(1, 2).as_subclass(_OnDevice)
    assert ops.dynamic_fake_quantize(x, _args()) is None and stub.calls == []
    stub.rc = N.CT_E_UNSUPPORTED
    assert ops.dynamic_fake_quantize(torch.randn(4, 6, 64, dtype=torch.bfloat16).as_subclass(_OnDevice), _args()) is None
    assert len(stub.calls) == 1


@pytest.mark.parametrize("what", ["fused", "cpu", "g_idx", "non_contiguous", "declined", "static", "empty"])
def test_forward_quantize_dispatch(what, monkeypatch):
    from compressed_tensors_b200.quantization.lifecycle import forward as F

    calls = []
    sentinel = torch.zeros(1)

    def fused(value, args, global_scale=None):
        calls.append(("fused", global_scale))
        return None if what == "declined" else (sentinel, None, None)

    monkeypatch.setattr(F.ops, "dynamic_fake_quantize", fused)
    monkeypatch.setattr(F, "compute_dynamic_scales_and_zp", lambda **k: calls.append("observe") or (torch.ones(1), torch.zeros(1, dtype=torch.int8)))
    monkeypatch.setattr(F, "fake_quantize", lambda **k: calls.append(("fake_quantize", k["g_idx"])) or k["x"])
    m = torch.nn.Module()
    m.input_global_scale = torch.ones(1)
    x = torch.randn(2, 3, 64, dtype=torch.bfloat16)
    args = _args()
    if what != "cpu":
        x = x.as_subclass(_OnDevice)
    if what == "g_idx":
        m.weight_g_idx = torch.zeros(64, dtype=torch.int32)
    if what == "non_contiguous":
        x = torch.randn(2, 64, 3, dtype=torch.bfloat16).transpose(1, 2).as_subclass(_OnDevice)
    if what == "static":
        args = _args(strategy="tensor", dynamic=False)
        m.input_scale, m.input_zero_point = torch.ones(1), torch.zeros(1, dtype=torch.int8)
    if what == "empty":
        x = torch.empty(0, 64, dtype=torch.bfloat16).as_subclass(_OnDevice)
    r = F.forward_quantize(m, x, "input", args)
    if what == "fused":
        assert r is sentinel and calls == [("fused", m.input_global_scale)]
    elif what == "declined":
        assert calls == [("fused", m.input_global_scale), "observe", ("fake_quantize", None)]
    elif what == "empty":
        assert r is x and calls == []
    elif what == "static":
        assert calls == [("fake_quantize", None)]
    elif what == "g_idx":
        assert calls == ["observe", ("fake_quantize", m.weight_g_idx)]
    else:
        assert calls == ["observe", ("fake_quantize", None)]


def test_golden_covers_the_issue_edge_cases():
    """the fixture holds the edge cases the kernels must reproduce: eps scales of all-zero rows / groups, fp16 MX scales that
    underflowed to 0 and became 1, 32768-wide rows and -0.0 inputs"""
    mx16 = [c for c in CASES if c["scheme"] == "MXFP4" and INPUTS[c["input"]].dtype == torch.float16]
    assert any(bool((c["scale"] == 1).any()) for c in mx16)
    assert any(INPUTS[c["input"]].shape[-1] == 32768 for c in CASES)
    assert any(bool((INPUTS[c["input"]] == 0).all(dim=-1).any()) for c in CASES)
    assert any(bool(torch.signbit(INPUTS[c["input"]][INPUTS[c["input"]] == 0]).any()) for c in CASES)
    assert not any(bool(INPUTS[c["input"]].isnan().any()) for c in CASES)
    assert math.isfinite(sum(float(c["out"].float().abs().sum()) for c in CASES))
