"""
The fused BLOCK (FP8_BLOCK) and MX (MXFP4 / MXFP8) weight observers on the device: the reference's golden cases, seeded weights of
Llama-3-8B / 70B shapes against the unfused path (torch min / max -> calculate_qparams -> quantize / quantize_pack_fp4 ->
compress_mx_scale) and the oracle, a whole layer set in one batched launch, the declines, a weight past 2^31 elements, and
ModelCompressor.compress_model on models calibrated either way.  Codes made from a NaN quotient are not compared (their scale is NaN,
or an inf met an inf scale): E2M1 has no NaN, and fp8 NaN payloads are not part of the contract.
"""
import copy
import ctypes
import math

import pytest
import torch

import oracle
from compressed_tensors_b200 import _native as N
from compressed_tensors_b200 import ops
from compressed_tensors_b200.quantization import QuantizationArgs, calculate_qparams, preset_name_to_scheme
from oracle.qparams import calculate_qparams as orc_qparams
from tests.golden import load
from tests.util import same, same_nan

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
F8 = torch.float8_e4m3fn

LLAMA_8B = [(4096, 4096), (1024, 4096), (14336, 4096), (4096, 14336)]
LLAMA_70B = [(8192, 8192), (1024, 8192), (28672, 8192), (8192, 28672)]


def block_args(bh=128, bw=128, **kw):
    return QuantizationArgs(**{**dict(num_bits=8, type="float", strategy="block", symmetric=True, dynamic=False, block_structure=[bh, bw]), **kw})


def mx_args(bits):
    return preset_name_to_scheme("MXFP4" if bits == 4 else "MXFP8", ["Linear"]).weights


def unfused_block(w, args):
    """torch block min / max -> calculate_qparams -> ops.quantize: the path observe_quantize takes where the kernel declines"""
    bh, bw = args.block_structure
    rows, cols = w.shape
    nrb, ncb = math.ceil(rows / bh), math.ceil(cols / bw)
    wp = torch.nn.functional.pad(w, (0, ncb * bw - cols, 0, nrb * bh - rows)).reshape(nrb, bh, ncb, bw)
    scale, _ = calculate_qparams(wp.amin(dim=(1, 3)), wp.amax(dim=(1, 3)), args)
    del wp
    return ops.quantize(w, scale, None, args, dtype=F8), scale


def unfused_mx(w, args):
    g = w.unflatten(-1, (-1, 32))
    scale, _ = calculate_qparams(g.amin(-1), g.amax(-1), args)
    q = ops.quantize_pack_fp4(w, scale, None, args) if args.num_bits == 4 else ops.quantize(w, scale, None, args, dtype=F8)
    return q, ops.compress_mx_scale(scale, torch.uint8), scale


def nan_quotient(w, scale, bh, bw):
    """elements whose x / scale is NaN (scale expanded over its [bh, bw] block)"""
    s = scale.float().repeat_interleave(bh, 0).repeat_interleave(bw, 1)[: w.shape[0], : w.shape[1]]
    return (w.float() / s).isnan()


def same_codes(got, want, keep, what):
    same(got.contiguous().view(torch.uint8)[keep], want.contiguous().view(torch.uint8)[keep], what)


def check_mx(got_q, got_s, want_q, want_s, w, scale, bits, what):
    same(got_s, want_s, what + " E8M0 scale")
    keep = ~nan_quotient(w, scale, 1, 32)
    if bits == 4:
        keep = keep[:, 0::2] & keep[:, 1::2]
    same_codes(got_q, want_q, keep, what + " codes")


# ---------------------------------------------------------------------------------------------------------------------
# golden cases of the reference
# ---------------------------------------------------------------------------------------------------------------------
_G = load("observe_block_mx")


@pytest.mark.parametrize("i", range(len(_G)))
def test_golden(i):
    c = _G[i]
    x = c["x"].to(DEV)
    if c["kind"] == "block":
        bh, bw = c["block"]
        q, s, z = ops.observe_quantize(x, block_args(bh, bw))
        assert z is None
        same_nan(s.cpu(), c["scale"], f"case {i} block scale")
        same_codes(q.cpu(), c["weight"], ~nan_quotient(c["x"], c["scale"], bh, bw), f"case {i} block codes")
    else:
        q, s = ops.observe_quantize_mx(x, mx_args(c["num_bits"]))
        check_mx(q.cpu(), s.cpu(), c["q"], c["scale"], c["x"], c["scale_float"], c["num_bits"], f"case {i}")


# ---------------------------------------------------------------------------------------------------------------------
# Llama-sized weights against the unfused path (and the oracle)
# ---------------------------------------------------------------------------------------------------------------------
def _weight(shape, dtype, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    w = torch.randn(shape, generator=g, device=DEV) * 0.02
    w = torch.where(torch.rand(shape, generator=g, device=DEV) < 0.001, w * 40, w)
    return w.to(dtype)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("shape", LLAMA_8B + LLAMA_70B + [(300, 200), (4097, 4104)])
def test_block_vs_unfused(shape, dtype):
    w = _weight(shape, dtype, shape[0] * 7 + shape[1])
    args = block_args()
    q, s, _ = ops.observe_quantize(w, args)
    wq, ws = unfused_block(w, args)
    same(s, ws, f"{shape} block scale")
    same_codes(q, wq, torch.ones_like(w, dtype=torch.bool), f"{shape} block codes")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("bits", [4, 8])
@pytest.mark.parametrize("shape", LLAMA_8B + LLAMA_70B + [(257, 96)])
def test_mx_vs_unfused(shape, bits, dtype):
    w = _weight(shape, dtype, shape[0] * 5 + shape[1] + bits)
    args = mx_args(bits)
    q, s = ops.observe_quantize_mx(w, args)
    wq, ws, _ = unfused_mx(w, args)
    same(s, ws, f"{shape} MX scale")
    same_codes(q, wq, torch.ones_like(wq, dtype=torch.bool), f"{shape} MX codes")


@pytest.mark.parametrize("kind", ["block", "mxfp4", "mxfp8"])
def test_large_vs_oracle(kind):
    w = _weight((4096, 14336), torch.bfloat16, 11)
    wc = w.cpu()
    if kind == "block":
        q, s, _ = ops.observe_quantize(w, block_args())
        wr = wc.reshape(32, 128, 112, 128)
        os_, _ = orc_qparams(wr.amin(dim=(1, 3)), wr.amax(dim=(1, 3)), num_bits=8, qtype="float", symmetric=True)
        same(s.cpu(), os_, "block scale vs oracle")
        oq = oracle.quantize(wc, os_, None, strategy="block", block_structure=[128, 128], num_bits=8, qtype="float", dtype=F8)
        same(q.cpu().view(torch.uint8), oq.view(torch.uint8), "block codes vs oracle")
        return
    bits = 4 if kind == "mxfp4" else 8
    args = mx_args(bits)
    q, s = ops.observe_quantize_mx(w, args)
    g = wc.unflatten(-1, (-1, 32))
    scale, _ = calculate_qparams(g.amin(-1), g.amax(-1), args)          # host mirror on the CPU (pinned by the goldens)
    same(s.cpu(), oracle.compress_mx_scale(scale), "E8M0 vs oracle")
    if bits == 4:
        v = oracle.quantize(wc, scale, None, strategy="group", group_size=32, num_bits=4, qtype="float")
        same(q.cpu(), oracle.pack_fp4_to_uint8(v), "E2M1 vs oracle")
    else:
        oq = oracle.quantize(wc, scale, None, strategy="group", group_size=32, num_bits=8, qtype="float", dtype=F8)
        same(q.cpu().view(torch.uint8), oq.view(torch.uint8), "fp8 vs oracle")


# ---------------------------------------------------------------------------------------------------------------------
# a whole layer set in one launch
# ---------------------------------------------------------------------------------------------------------------------
_LAYER = [(4096, 4096), (1024, 4096), (1024, 4096), (4096, 4096), (14336, 4096), (14336, 4096), (4096, 14336), (300, 224), (257, 96)]


@pytest.mark.parametrize("kind", ["block", "mxfp4", "mxfp8"])
def test_batched_one_launch(kind):
    ws = [_weight(s, torch.bfloat16 if i % 3 else torch.float16, 100 + i) for i, s in enumerate(_LAYER)]
    problems, want = [], []
    for w in ws:
        r, c = w.shape
        if kind == "block":
            q, s, _ = ops.observe_quantize(w, block_args())
            d = ops._block_desc(r, c, 128, 128, w.dtype)
            problems.append((d, w, torch.empty_like(s), None, torch.empty_like(q)))
        else:
            q, s = ops.observe_quantize_mx(w, mx_args(4 if kind == "mxfp4" else 8))
            d = ops._mx_desc(r, c, 4 if kind == "mxfp4" else 8, w.dtype)
            problems.append((d, w, torch.empty_like(s), None, torch.empty_like(q)))
        want.append((q, s))
    op = N.OP_OBSERVE_QUANTIZE_BLOCK if kind == "block" else N.OP_OBSERVE_QUANTIZE_MX
    plan = ops.BatchedPlan(op, problems)
    torch.cuda.synchronize()
    n0 = N.launch_count()
    plan.run()
    torch.cuda.synchronize()
    assert N.launch_count() - n0 == 1
    for i, ((_, _, s, _, q), (wq, wsc)) in enumerate(zip(problems, want)):
        same(s.view(torch.uint8), wsc.view(torch.uint8), f"tensor {i} scale")
        same(q.view(torch.uint8), wq.view(torch.uint8), f"tensor {i} codes")


@pytest.mark.parametrize("kind", ["block", "mxfp8"])
def test_batched_cuda_graph_capture(kind):
    """a whole-model call captured once (the job table goes up by upload kernels, 24 jobs each) and replayed on new data"""
    ws = [_weight(s, torch.bfloat16, 200 + i) for i, s in enumerate([(1024, 4096), (512, 1536), (300, 224)] * 10)]
    probs = []
    for w in ws:
        r, c = w.shape
        if kind == "block":
            d, s = ops._block_desc(r, c, 128, 128, w.dtype), torch.empty((math.ceil(r / 128), math.ceil(c / 128)), dtype=w.dtype, device=DEV)
        else:
            d, s = ops._mx_desc(r, c, 8, w.dtype), torch.empty((r, c // 32), dtype=torch.uint8, device=DEV)
        probs.append((d, w, s, None, torch.empty((r, c), dtype=F8, device=DEV)))
    plan = ops.BatchedPlan(N.OP_OBSERVE_QUANTIZE_BLOCK if kind == "block" else N.OP_OBSERVE_QUANTIZE_MX, probs)
    side = torch.cuda.Stream(device=DEV)
    side.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(side):
        plan.run()
        side.synchronize()
        with torch.cuda.graph(graph, stream=side):
            plan.run()
    for w in ws:
        w.mul_(-0.5)
    graph.replay()
    torch.cuda.synchronize()
    for i, (_, w, s, _, q) in enumerate(probs):
        wq, wsc = ops.observe_quantize(w, block_args())[:2] if kind == "block" else ops.observe_quantize_mx(w, mx_args(8))
        same(s.view(torch.uint8), wsc.view(torch.uint8), f"tensor {i} scale after replay")
        same(q.view(torch.uint8), wq.view(torch.uint8), f"tensor {i} codes after replay")


# ---------------------------------------------------------------------------------------------------------------------
# declines
# ---------------------------------------------------------------------------------------------------------------------
def _call(fn, d, x, s, q, device=0):
    return getattr(N.lib(), fn)(ctypes.byref(d), N.ptr(x), N.ptr(s), N.ptr(q), device, N.stream_ptr(0))


def test_native_declines():
    x = _weight((256, 256), torch.bfloat16, 1)
    s, q = torch.empty((2, 2), dtype=torch.bfloat16, device=DEV), torch.empty((256, 256), dtype=F8, device=DEV)
    cases = []
    d = ops._block_desc(256, 256, 128, 128, torch.bfloat16); d.x_dtype = d.scale_dtype = d.compute_dtype = N.DT[torch.float32]
    cases.append(("fp32", "ct_observe_quantize_block", d))
    d = ops._block_desc(256, 252, 128, 126, torch.bfloat16)
    cases.append(("unaligned rows", "ct_observe_quantize_block", d))
    d = ops._block_desc(256, 256, 128, 128, torch.bfloat16); d.zp_dtype = N.DT[F8]
    cases.append(("asymmetric fp8", "ct_observe_quantize_block", d))
    d = ops._mx_desc(256, 256, 4, torch.bfloat16); d.zp_dtype = N.DT[torch.uint8]
    cases.append(("asymmetric fp4", "ct_observe_quantize_mx", d))
    d = ops._mx_desc(256, 256, 4, torch.bfloat16); d.x_dtype = d.compute_dtype = N.DT[torch.float32]
    cases.append(("fp32 mx", "ct_observe_quantize_mx", d))
    for what, fn, d in cases:
        assert _call(fn, d, x, s, q) == N.CT_E_UNSUPPORTED, what
    for fn, d in (("ct_observe_quantize_block", ops._block_desc(256, 256, 128, 128, torch.bfloat16)),
                  ("ct_observe_quantize_mx", ops._mx_desc(256, 256, 8, torch.bfloat16))):
        xc, sc, qc = x.cpu(), torch.empty(64, dtype=torch.uint8), torch.empty((256, 256), dtype=torch.uint8)
        assert _call(fn, d, xc, sc, qc, device=-1) == N.CT_E_UNSUPPORTED, fn + " on the host"


@pytest.mark.parametrize("case", ["fp32", "cols % 8", "block width % 8"])
def test_block_decline_is_unfused(case):
    shape, args, dtype = (300, 200), block_args(), torch.bfloat16
    if case == "fp32":
        dtype = torch.float32
    elif case == "cols % 8":
        shape, args = (260, 130), block_args(128, 65)
    else:
        shape, args = (256, 240), block_args(64, 60)
    w = _weight(shape, dtype, 3)
    q, s, _ = ops.observe_quantize(w, args)
    wq, wsc = unfused_block(w, args)
    same(s, wsc, case + " scale")
    same_codes(q, wq, torch.ones_like(w, dtype=torch.bool), case + " codes")


@pytest.mark.parametrize("bits", [4, 8])
def test_mx_decline_is_unfused(bits):
    w = _weight((128, 512), torch.float32, 4)
    q, s = ops.observe_quantize_mx(w, mx_args(bits))
    wq, wsc, _ = unfused_mx(w, mx_args(bits))
    same(s, wsc, "fp32 MX scale")
    same_codes(q, wq, torch.ones_like(wq, dtype=torch.bool), "fp32 MX codes")


# ---------------------------------------------------------------------------------------------------------------------
# past 2^31 elements
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["block", "mxfp4"])
def test_past_2_31(kind):
    shape = (16385, 131072)
    assert shape[0] * shape[1] > 2 ** 31
    w = _weight(shape, torch.bfloat16, 31)
    if kind == "block":
        q, s, _ = ops.observe_quantize(w, block_args())
        wq, wsc = unfused_block(w, block_args())
    else:
        q, s = ops.observe_quantize_mx(w, mx_args(4))
        wq, wsc, _ = unfused_mx(w, mx_args(4))
    assert torch.equal(s.view(torch.uint8), wsc.view(torch.uint8)), kind + " scale"
    assert torch.equal(q.view(torch.uint8), wq.view(torch.uint8)), kind + " codes"


# ---------------------------------------------------------------------------------------------------------------------
# ModelCompressor.compress_model on models calibrated by the fused ops and by the unfused path
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("preset", ["FP8_BLOCK", "MXFP4A16", "MXFP8A16"])
def test_compress_model_fused_calibration(preset):
    from compressed_tensors_b200.compressors import ModelCompressor
    from compressed_tensors_b200.quantization import QuantizationConfig, QuantizationStatus, apply_quantization_config
    from compressed_tensors_b200.utils import get_direct_state_dict

    torch.manual_seed(5)
    base = torch.nn.Sequential(torch.nn.Linear(512, 384, bias=False), torch.nn.Linear(384, 1024, bias=False),
                               torch.nn.Linear(1024, 300, bias=False)).to(torch.bfloat16).to(DEV)
    models = []
    for fused in (False, True):
        model = copy.deepcopy(base)
        apply_quantization_config(model, QuantizationConfig(config_groups={preset: ["Linear"]}))
        for lin in model:
            a = lin.quantization_scheme.weights
            w = lin.weight.data
            if preset == "FP8_BLOCK":
                s = ops.observe_quantize(w, a)[1] if fused else unfused_block(w, a)[1]
            else:
                s = ops.decompress_mx_scale(ops.observe_quantize_mx(w, a)[1]) if fused else unfused_mx(w, a)[2]
            lin.weight_scale.data = s.to(w.dtype)
            lin.quantization_status = QuantizationStatus.FROZEN
        mc = ModelCompressor.from_pretrained_model(model)
        mc.compress_model(model)
        models.append(model)
    for i, (a, b) in enumerate(zip(*models)):
        sa, sb = get_direct_state_dict(a), get_direct_state_dict(b)
        assert sorted(sa) == sorted(sb)
        codes = "weight_packed" if preset == "MXFP4A16" else "weight"
        assert sb[codes].dtype == (torch.uint8 if preset == "MXFP4A16" else F8), f"{preset} layer {i} is not compressed"
        assert sb["weight_scale"].dtype == (torch.bfloat16 if preset == "FP8_BLOCK" else torch.uint8)
        for k in sa:
            if sa[k] is None or sb[k] is None:
                assert sa[k] is None and sb[k] is None, f"{preset} layer {i} {k}"
            elif sa[k].dtype.is_floating_point or sa[k].dtype == F8:
                same(sb[k].contiguous().view(torch.uint8), sa[k].contiguous().view(torch.uint8), f"{preset} layer {i} {k}")
            else:
                assert torch.equal(sb[k], sa[k]), f"{preset} layer {i} {k}"
