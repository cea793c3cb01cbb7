"""
The fused BLOCK / MX weight observers without a GPU: the CPU oracle reproduces every golden case of the reference (block scales and fp8
codes; MX float scales, E8M0 exponents, E2M1 bytes and fp8 codes), the argument checks and meta shapes of ops.observe_quantize (BLOCK)
and ops.observe_quantize_mx, the batched descriptor checks of the two new ops, and the ABI they add.
"""
import ctypes
import math
import os
import re
from types import SimpleNamespace

import pytest
import torch

import oracle
from compressed_tensors_b200 import _native as N
from compressed_tensors_b200 import ops
from compressed_tensors_b200.quantization import QuantizationArgs, calculate_qparams, preset_name_to_scheme
from oracle.qparams import calculate_qparams as orc_qparams
from tests.golden import load
from tests.util import same, same_nan

_G = load("observe_block_mx")
_BLOCK = [i for i, c in enumerate(_G) if c["kind"] == "block"]
_MX = [i for i, c in enumerate(_G) if c["kind"] == "mx"]
_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def block_minmax(x: torch.Tensor, bh: int, bw: int):
    """min / max of every [bh, bw] block over the elements that exist (zero padding: the rule clamps min <= 0 <= max)"""
    rows, cols = x.shape
    nrb, ncb = math.ceil(rows / bh), math.ceil(cols / bw)
    xp = torch.nn.functional.pad(x, (0, ncb * bw - cols, 0, nrb * bh - rows)).reshape(nrb, bh, ncb, bw)
    return xp.amin(dim=(1, 3)), xp.amax(dim=(1, 3))


def nan_block_mask(scale: torch.Tensor, shape, bh: int, bw: int) -> torch.Tensor:
    """elements whose block scale is NaN: their codes are not part of the bit-exact contract"""
    m = scale.isnan().repeat_interleave(bh, 0).repeat_interleave(bw, 1)
    return m[: shape[0], : shape[1]]


def nan_quotient_mask(x: torch.Tensor, scale: torch.Tensor) -> torch.Tensor:
    """MX elements whose quotient x / scale is NaN (an inf in a group whose scale is inf): the codes made from a NaN are not part of
    the bit-exact contract (E2M1 has no NaN, and the reference, the oracle and the kernels each map it to a different code)"""
    return (x.float() / scale.float().repeat_interleave(32, 1)).isnan()


def test_golden_covers_the_cases():
    assert len(_BLOCK) >= 12 and len(_MX) >= 16
    assert {c["x"].dtype for c in _G} == {torch.bfloat16, torch.float16}
    assert any(c["x"].shape[0] % c["block"][0] or c["x"].shape[1] % c["block"][1] for c in (_G[i] for i in _BLOCK))
    assert any(c["block"][0] != c["block"][1] for c in (_G[i] for i in _BLOCK))
    assert any(c["scale"].isnan().any() for c in (_G[i] for i in _BLOCK))
    assert {_G[i]["num_bits"] for i in _MX} == {4, 8}


@pytest.mark.parametrize("i", _BLOCK)
def test_oracle_block_golden(i):
    c = _G[i]
    x, (bh, bw) = c["x"], c["block"]
    mn, mx = block_minmax(x, bh, bw)
    scale, _ = orc_qparams(mn, mx, num_bits=8, qtype="float", symmetric=True)
    same_nan(scale, c["scale"], "oracle block scale")
    q = oracle.quantize(x, c["scale"], None, strategy="block", block_structure=[bh, bw], num_bits=8, qtype="float", dtype=torch.float8_e4m3fn)
    keep = ~nan_block_mask(c["scale"], x.shape, bh, bw)
    same(q.view(torch.uint8)[keep], c["weight"].view(torch.uint8)[keep], "oracle block codes")


@pytest.mark.parametrize("i", _MX)
def test_oracle_mx_golden(i):
    c = _G[i]
    x, bits = c["x"], c["num_bits"]
    args = preset_name_to_scheme(c["preset"], ["Linear"]).weights
    g = x.unflatten(-1, (-1, 32))
    scale, _ = calculate_qparams(g.amin(-1), g.amax(-1), args)       # the host mirror of the MX exponent rule
    same(scale, c["scale_float"], "MX scale")
    same(oracle.compress_mx_scale(scale), c["scale"], "E8M0 exponents")
    keep = ~nan_quotient_mask(x, scale)
    if bits == 4:
        v = oracle.quantize(x, scale, None, strategy="group", group_size=32, num_bits=4, qtype="float")
        keep = keep[:, 0::2] & keep[:, 1::2]
        same(oracle.pack_fp4_to_uint8(v)[keep], c["q"][keep], "E2M1 bytes")
    else:
        q = oracle.quantize(x, scale, None, strategy="group", group_size=32, num_bits=8, qtype="float", dtype=torch.float8_e4m3fn)
        same(q.view(torch.uint8)[keep], c["q"].view(torch.uint8)[keep], "fp8 codes")


def _block_args(bh=128, bw=128, **kw):
    return QuantizationArgs(**{**dict(num_bits=8, type="float", strategy="block", symmetric=True, dynamic=False, block_structure=[bh, bw]), **kw})


@pytest.mark.parametrize("shape,block", [((300, 200), (128, 128)), ((4096, 14336), (128, 128)), ((257, 96), (64, 32))])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_block_meta_shapes(shape, block, dtype):
    q, s, z = ops.observe_quantize(torch.empty(shape, dtype=dtype, device="meta"), _block_args(*block))
    assert q.device.type == "meta" and q.dtype == torch.float8_e4m3fn and tuple(q.shape) == shape
    assert s.dtype == dtype and tuple(s.shape) == (math.ceil(shape[0] / block[0]), math.ceil(shape[1] / block[1]))
    assert z is None


@pytest.mark.parametrize("preset,bits", [("MXFP4", 4), ("MXFP4A16", 4), ("MXFP8", 8), ("MXFP8A16", 8)])
@pytest.mark.parametrize("shape", [(257, 96), (4096, 14336)])
def test_mx_meta_shapes(preset, bits, shape):
    args = preset_name_to_scheme(preset, ["Linear"]).weights
    q, s = ops.observe_quantize_mx(torch.empty(shape, dtype=torch.bfloat16, device="meta"), args)
    assert q.device.type == "meta" and s.device.type == "meta"
    assert s.dtype == torch.uint8 and tuple(s.shape) == (shape[0], shape[1] // 32)
    if bits == 4:
        assert q.dtype == torch.uint8 and tuple(q.shape) == (shape[0], shape[1] // 2)
    else:
        assert q.dtype == torch.float8_e4m3fn and tuple(q.shape) == shape


def test_mx_argument_checks():
    mx4 = preset_name_to_scheme("MXFP4", ["Linear"]).weights
    meta = torch.empty((64, 256), dtype=torch.bfloat16, device="meta")
    for bad in (preset_name_to_scheme("NVFP4", ["Linear"]).weights, preset_name_to_scheme("FP8_BLOCK", ["Linear"]).weights,
                preset_name_to_scheme("W4A16", ["Linear"]).weights, mx4.model_copy(update={"group_size": 16}),
                mx4.model_copy(update={"scale_dtype": None})):
        with pytest.raises(ValueError):
            ops.observe_quantize_mx(meta, bad)
    with pytest.raises(ValueError, match="2-D"):
        ops.observe_quantize_mx(torch.empty((2, 64, 256), dtype=torch.bfloat16, device="meta"), mx4)
    with pytest.raises(ValueError, match="divisble"):
        ops.observe_quantize_mx(torch.empty((64, 48), dtype=torch.bfloat16, device="meta"), mx4)
    with pytest.raises(NotImplementedError):
        ops.observe_quantize_mx(meta, mx4.model_copy(update={"symmetric": False}))


def test_block_argument_checks():
    meta = torch.empty((256, 256), dtype=torch.bfloat16, device="meta")
    ns = SimpleNamespace(strategy="block", block_structure=None, num_bits=8, type="float", symmetric=True, group_size=None)
    with pytest.raises(ValueError, match="block_structure"):
        ops.observe_quantize(meta, ns)
    with pytest.raises(ValueError, match="2-D"):
        ops.observe_quantize(torch.empty((2, 256, 256), dtype=torch.bfloat16, device="meta"), _block_args())


def _problem(op, d, x_dt, out_numel, out_dt, scale_numel, scale_dt):
    n = int(d.rows) * int(d.cols)
    return (d, torch.empty(n, dtype=x_dt), torch.empty(scale_numel, dtype=scale_dt), None, torch.empty(out_numel, dtype=out_dt))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_batched_descriptor_checks(dtype):
    d = ops._block_desc(300, 200, 128, 128, dtype)
    assert (d.rdiv, d.cdiv, d.s_row_stride, d.scale_dtype, d.q_dtype) == (128, 128, 2, N.DT[dtype], N.DT[torch.float8_e4m3fn])
    ops._validate_problem(N.OP_OBSERVE_QUANTIZE_BLOCK, 0, _problem(0, d, dtype, 60000, torch.float8_e4m3fn, 6, dtype), None)
    with pytest.raises(ValueError, match="scale"):
        ops._validate_problem(N.OP_OBSERVE_QUANTIZE_BLOCK, 0, _problem(0, d, dtype, 60000, torch.float8_e4m3fn, 4, dtype), None)
    with pytest.raises(ValueError, match="output"):
        ops._validate_problem(N.OP_OBSERVE_QUANTIZE_BLOCK, 0, _problem(0, d, dtype, 30000, torch.uint8, 6, dtype), None)
    for bits, out_numel in ((4, 257 * 48), (8, 257 * 96)):
        d = ops._mx_desc(257, 96, bits, dtype)
        assert (d.rdiv, d.cdiv, d.s_row_stride, d.scale_dtype) == (1, 32, 3, N.DT_E8M0)
        ops._validate_problem(N.OP_OBSERVE_QUANTIZE_MX, 0, _problem(0, d, dtype, out_numel, torch.uint8, 257 * 3, torch.uint8), None)
        with pytest.raises(ValueError, match="output"):
            ops._validate_problem(N.OP_OBSERVE_QUANTIZE_MX, 0, _problem(0, d, dtype, out_numel * 2 + 2, torch.uint8, 257 * 3, torch.uint8), None)
        with pytest.raises(ValueError, match="scale"):
            ops._validate_problem(N.OP_OBSERVE_QUANTIZE_MX, 0, _problem(0, d, dtype, out_numel, torch.uint8, 257 * 3, dtype), None)


def test_abi():
    header = open(os.path.join(_ROOT, "include", "ct_b200.h")).read()
    for name in ("ct_observe_quantize_block", "ct_observe_quantize_mx"):
        assert re.search(rf"\bint {name}\(", header), name
        assert name in N.EXPORTED_SYMBOLS
    assert re.search(r"CT_OP_OBSERVE_QUANTIZE_BLOCK = (\d+)", header).group(1) == str(N.OP_OBSERVE_QUANTIZE_BLOCK) == "13"
    assert re.search(r"CT_OP_OBSERVE_QUANTIZE_MX = (\d+)", header).group(1) == str(N.OP_OBSERVE_QUANTIZE_MX) == "14"
    if os.path.exists(N.LIB_PATH):
        lib = ctypes.CDLL(N.LIB_PATH)
        assert hasattr(lib, "ct_observe_quantize_block") and hasattr(lib, "ct_observe_quantize_mx")
