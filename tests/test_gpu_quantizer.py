"""
CompressedTensorsQuantizer and the cluster-wide channel observer on the H100:
  - convert_checkpoint with the quantizer is bit-identical to the reference's apply_quantization_config + calculate_qparams +
    compress_model (tests/golden/quantizer.pt.gz) for every preset, from bf16, fp16 and FP8-block checkpoints, with 1 and 2 workers;
  - the written checkpoint loads and decompresses with ModelCompressor.decompress_model into fake_quantize of the source weights
    with the observed qparams;
  - ct_observe_quantize_channel on rows wider than 16384 columns (thread-block clusters) equals the unfused torch path bit for bit,
    and its codes equal the CPU oracle's for the same finite qparams, and declines rows wider than one cluster holds, where observe_quantize takes the unfused path.
"""
import ctypes
import json

import pytest
import torch

import oracle
from compressed_tensors_b200 import _native as N
from compressed_tensors_b200 import ops
from compressed_tensors_b200.entrypoints.convert import CompressedTensorsQuantizer, convert_checkpoint
from compressed_tensors_b200.quantization import QuantizationArgs
from compressed_tensors_b200.quantization.utils.helpers import calculate_qparams, generate_gparam
from tests.golden import quantizer_checkpoint as qc
from tests.test_quantizer_host import CASES, _case, _check_against_golden, _min_max, _read_all, _source

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("workers", [1, 2])
@pytest.mark.parametrize("source,preset", CASES)
def test_convert_checkpoint_on_device_matches_reference(tmp_path, source, preset, workers):
    tensors, dt, deq = _source(source)
    qc.write_checkpoint(str(tmp_path / "in"), tensors, dt)
    convert_checkpoint(str(tmp_path / "in"), str(tmp_path / "out"), CompressedTensorsQuantizer(preset, ignore=list(qc.IGNORE), dtype=deq),
                       max_workers=workers, device="cuda")
    _check_against_golden(_read_all(str(tmp_path / "out")), _case(source, preset))


FUSED = (("q_proj", "k_proj", "v_proj"), ("gate_proj", "up_proj"))


def _expected_fake_quantized(tensors: dict, name: str, args) -> torch.Tensor:
    """fake_quantize of the source weight with the memoryless min-max qparams (NVFP4: the fused group's smallest global scale)"""
    w = tensors[f"{name}.weight"].cuda()
    gs = None
    if getattr(args.strategy, "value", args.strategy) == "tensor_group":
        parent, _, leaf = name.rpartition(".")
        group = next((g for g in FUSED if leaf in g), (leaf,))
        gs = torch.stack([generate_gparam(tensors[f"{parent}.{m}.weight"].cuda().min(), tensors[f"{parent}.{m}.weight"].cuda().max())
                          for m in group]).amin(0)
    scale, zp = calculate_qparams(*_min_max(w, args), args, global_scale=gs)
    return ops.fake_quantize(w, scale, None if args.symmetric else zp, args, global_scale=gs)


# FP8_BLOCK is left out: gate_proj / up_proj are one 128-column block wide, and dequantize cannot tell their [129, 1] block scale
# from a channel scale by its shape
@pytest.mark.parametrize("preset", ["W4A16", "W4A16_ASYM", "W8A16", "W8A8", "FP8_DYNAMIC", "NVFP4A16", "MXFP4", "MXFP8"])
def test_output_decompresses_to_fake_quantize(tmp_path, preset):
    from transformers import LlamaConfig, LlamaForCausalLM

    from compressed_tensors_b200.compressors import ModelCompressor
    from compressed_tensors_b200.quantization import apply_quantization_config

    tensors = qc.dense_tensors(torch.bfloat16)
    qc.write_checkpoint(str(tmp_path / "in"), tensors, torch.bfloat16)
    convert_checkpoint(str(tmp_path / "in"), str(tmp_path / "out"), CompressedTensorsQuantizer(preset, ignore=list(qc.IGNORE)), device="cuda")
    with open(tmp_path / "out" / "config.json") as f:
        cfg = json.load(f)
    compressor = ModelCompressor.from_compression_config(cfg)
    kw = {k: v for k, v in cfg.items() if k not in ("architectures", "model_type", "torch_dtype", "quantization_config")}
    with torch.device("meta"):
        model = LlamaForCausalLM(LlamaConfig(**kw))
    apply_quantization_config(model, compressor.quantization_config)
    compressor.compress_model(model)                       # the compressed parameter layout (meta), as on load
    model.load_state_dict({k: v.cuda() for k, v in _read_all(str(tmp_path / "out")).items()}, assign=True, strict=True)
    compressor.decompress_model(model)
    args = compressor.quantization_config.config_groups["group_0"].weights
    for name in _case("bf16", preset)["quantized"]:
        got = model.get_submodule(name).weight
        want = _expected_fake_quantized(tensors, name, args)
        assert torch.equal(got, want), name   # by value: dequantizing a zero code gives +0 where fake_quantize keeps -0


# ------------------------------------------------------------------------------------------------ wide-row channel observer
def _args(kind: str, symmetric: bool) -> QuantizationArgs:
    if kind == "fp8":
        return QuantizationArgs(num_bits=8, type="float", strategy="channel", symmetric=True)
    return QuantizationArgs(num_bits=4 if kind == "pack4" else 8, type="int", strategy="channel", symmetric=symmetric)


def _rows(rows: int, cols: int, dtype: torch.dtype, at: int = 0) -> torch.Tensor:
    """random rows with the special ones at rows at .. at + 5"""
    g = torch.Generator().manual_seed(rows * 131 + cols)
    x = torch.randn(rows, cols, generator=g) * (0.5 + torch.rand(rows, 1, generator=g))
    x[at] = 0                                                                   # zero row: the eps scale
    x[at + 1] = torch.finfo(dtype).tiny * torch.rand(cols, generator=g) / 64    # subnormal row
    x[at + 2, cols // 3] = float("inf")
    x[at + 3, cols - 1] = float("-inf")
    x[at + 4, cols // 2] = float("nan")
    x[at + 5, 7] = -0.0
    x[at + 5] = torch.where(x[at + 5].abs() < 0.5, 0.0, x[at + 5])
    return x.to(dtype)


def _unfused(x: torch.Tensor, args, pack: bool):
    scale, zp = calculate_qparams(x.amin(-1, keepdim=True), x.amax(-1, keepdim=True), args)
    zp = None if args.symmetric else zp
    out = ops.quantize_pack(x, scale, zp, args) if pack else ops.quantize(x, scale, zp, args, dtype=args.pytorch_dtype())
    return out, scale, zp


def _oracle(x: torch.Tensor, args, pack: bool, scale: torch.Tensor, zp):
    """the CPU oracle's codes for the device's qparams (those are checked against the unfused path separately)"""
    t = getattr(args.type, "value", args.type)
    q = oracle.quantize(x.cpu(), scale.cpu(), None if zp is None else zp.cpu(), strategy="channel", group_size=None, block_structure=None,
                        num_bits=args.num_bits, qtype=t, dtype=torch.float8_e4m3fn if t == "float" else torch.int8)
    return oracle.pack_to_int32(q, args.num_bits) if pack else q


def _same(a, b, what):
    assert a is None and b is None or (a.dtype == b.dtype and a.shape == b.shape), what
    if a is not None:
        assert torch.equal(a.cpu().view(torch.uint8), b.cpu().view(torch.uint8)), what


WIDEST = 8 * 16384


@pytest.mark.parametrize("cols", [16392, 28672, 53248, WIDEST])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("kind,symmetric", [("int8", True), ("int8", False), ("fp8", True), ("pack4", True), ("pack4", False),
                                            ("pack8", True), ("pack8", False)])
def test_wide_row_channel_kernel_matches_fallback_and_oracle(cols, dtype, kind, symmetric):
    _check_wide(_rows(24, cols, dtype).cuda(), kind, symmetric)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("kind,symmetric", [("int8", True), ("int8", False), ("fp8", True), ("pack4", True), ("pack4", False),
                                            ("pack8", True), ("pack8", False)])
def test_wide_row_channel_kernel_loops_over_rows(dtype, kind, symmetric):
    """more rows than resident clusters: each cluster strides over rows with the next row in flight and reuses its shared memory;
    the special rows sit in a later pass"""
    _check_wide(_rows(2048, 28672, dtype, at=1600).cuda(), kind, symmetric)


def _check_wide(x: torch.Tensor, kind: str, symmetric: bool):
    args, pack = _args(kind, symmetric), kind.startswith("pack")
    got = ops.observe_quantize(x, args, pack=pack)
    want = _unfused(x, args, pack)
    for i, what in enumerate(("codes", "scale", "zero point")):
        _same(got[i], want[i], f"{what} vs the unfused path")
    finite = torch.isfinite(got[1].float()).flatten().cpu()   # rows with an inf / NaN scale: the device's codes follow ops.quantize's
    _same(got[0].cpu()[finite], _oracle(x, args, pack, got[1], got[2])[finite], "codes vs the oracle")   # rule, not the oracle's


def test_channel_kernel_declines_rows_wider_than_one_cluster():
    cols = WIDEST + 8
    x = _rows(8, cols, torch.bfloat16).cuda()
    args = _args("int8", False)
    d = N.QuantDesc()
    d.rows, d.cols, d.rdiv, d.cdiv, d.s_row_stride = 8, cols, 1, N.INF, 1
    d.x_dtype = d.scale_dtype = d.compute_dtype = N.DT[torch.bfloat16]
    d.zp_dtype, d.q_dtype, d.out_dtype, d.qtype, d.num_bits = N.DT[torch.int8], N.DT[torch.int8], N.DT_NONE, N.Q_INT, 8
    scale = torch.empty(8, 1, dtype=torch.bfloat16, device="cuda")
    zp = torch.empty(8, 1, dtype=torch.int8, device="cuda")
    out = torch.empty(8, cols, dtype=torch.int8, device="cuda")
    idx = x.device.index
    rc = N.lib().ct_observe_quantize_channel(ctypes.byref(d), N.ptr(x), N.ptr(scale), N.ptr(zp), N.ptr(out), idx, N.stream_ptr(idx))
    assert rc == N.CT_E_UNSUPPORTED
    got = ops.observe_quantize(x, args)
    want = _unfused(x, args, False)
    for i in range(3):
        _same(got[i], want[i], "declined row: observe_quantize takes the unfused path")
