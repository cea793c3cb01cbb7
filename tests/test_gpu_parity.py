"""
GPU parity tests: the sm_90a kernels (through compressed_tensors_b200.ops -> C ABI) against
  (1) the golden vectors produced by running the reference (tests/golden),
  (2) the oracle on larger seeded inputs,
  (3) size-independent properties at BASELINE.json's full tensor sizes.
Bit-exact everywhere (integer codes, packed words, fp8 bytes AND dequantized floats: the
north star allows 1 ulp on floats, these tests demand 0).
"""
import ctypes
from types import SimpleNamespace

import pytest
import torch

import oracle
from compressed_tensors_b200 import _native as N
from compressed_tensors_b200 import ops
from tests.golden import load
from tests.util import bits_equal, diff_report, same, same_values

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def ns(**kw):
    d = dict(strategy="tensor", group_size=None, block_structure=None, num_bits=8, type="int", symmetric=True)
    d.update(kw)
    return SimpleNamespace(**d)


def cuda(t):
    return None if t is None else t.to(DEV)


# --------------------------------------------------------------------------------------------
# 0. the arithmetic proof the fast path rests on
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", [N.DT[torch.bfloat16], N.DT[torch.float16]])
def test_division_selftest_exhaustive(dt):
    mism = ctypes.c_uint64(123)
    N.check(N.lib().ct_selftest_division(dt, ctypes.byref(mism), 0))
    assert mism.value == 0


# --------------------------------------------------------------------------------------------
# 1. golden vectors
# --------------------------------------------------------------------------------------------
def test_pack_golden_gpu():
    for c in load("pack"):
        v = c["value"].to(DEV)
        got = ops.pack_to_int32(v, c["bits"], c["packed_dim"])
        assert got.is_cuda and got.dtype == torch.int32
        same_values(got.contiguous().cpu(), c["packed"], str((c["bits"], c["packed_dim"], tuple(v.shape))))
        if c["packed_dim"] == 0:
            assert list(got.shape) == c["view_shape"]
        if not c.get("out_of_range"):
            back = ops.unpack_from_int32(c["packed"].to(DEV), c["bits"], c["value"].shape, c["packed_dim"])
            same_values(back.cpu(), c["value"], "")


_Q = load("quant")


def _cid(c):
    a = c["args"]
    x = c["x"] if isinstance(c["x"], str) else "act"
    return f"{x}-{a['strategy']}-g{a.get('group_size')}-b{a['num_bits']}{a['type']}-{'sym' if a['symmetric'] else 'asym'}-{c['tag']}"


@pytest.mark.parametrize("c", _Q["cases"], ids=_cid)
def test_quant_golden_gpu(c):
    x = _Q["x"][c["x"]] if isinstance(c["x"], str) else c["x"]
    a = SimpleNamespace(**c["args"])
    xd, sd, zd, gd = cuda(x), cuda(c["scale"]), cuda(c["zp"]), cuda(c["g_idx"])
    q = ops.quantize(xd, sd, zd, a, dtype=c["q"].dtype, g_idx=gd)
    same(q.cpu(), c["q"], "quantize: ")
    qf = ops.quantize(xd, sd, zd, a, dtype=None, g_idx=gd)
    same(qf.cpu(), c["qf"], "quantize(dtype=None): ")
    dq = ops.dequantize(cuda(c["q"]), sd, zd, args=a, g_idx=gd)
    same(dq.cpu(), c["dq"], "dequantize: ")
    if c["dq_inferred"] is not None:
        dqi = ops.dequantize(cuda(c["q"]), sd, zd, g_idx=gd)
        same(dqi.cpu(), c["dq_inferred"], "dequantize(inferred): ")
    fq = ops.fake_quantize(xd, sd, zd, a, g_idx=gd)
    same(fq.cpu(), c["fq"], "fake_quantize: ")


def test_sweep_golden_gpu():
    """every bf16 / fp16 bit pattern x 4 scales, int4 / int8+zp / fp8 / fake-quant; every int8 and fp8 code"""
    sw = load("sweep")
    pat = torch.arange(65536, dtype=torch.int32).to(torch.uint16)
    n = 0
    for name, dt in (("bf16", torch.bfloat16), ("fp16", torch.float16)):
        x = pat.view(dt).reshape(256, 256).clone()
        x[x.isnan()] = 0
        xd = x.to(DEV)
        for sval in (2.0 ** -7, 0.01, 1.0, 37.5):
            s = torch.tensor([sval]).to(dt).to(DEV)
            key = f"{name}/s{sval}"
            got = ops.quantize(xd, s, None, ns(num_bits=4), dtype=torch.int8)
            same_values(got.cpu(), sw[key + "/int4"], str(key))
            zp = torch.tensor([3], dtype=torch.int8, device=DEV)
            got = ops.quantize(xd, s, zp, ns(num_bits=8, symmetric=False), dtype=torch.int8)
            same_values(got.cpu(), sw[key + "/int8zp3"], str(key))
            got = ops.quantize(xd, s, None, ns(type="float"), dtype=torch.float8_e4m3fn)
            same_values(got.cpu().view(torch.uint8), sw[key + "/fp8"], str(key))
            got = ops.fake_quantize(xd, s, None, ns(num_bits=4))
            same_values(got.cpu().view(torch.int16), sw[key + "/fq_int4"], str(key + " fq_int4 "))
            got = ops.fake_quantize(xd, s, None, ns(type="float"))
            same_values(got.cpu().view(torch.int16), sw[key + "/fq_fp8"], str(key + " fq_fp8 "))
            n += 5
    codes = torch.arange(-128, 128, dtype=torch.int8).reshape(1, 256).to(DEV)
    f8 = torch.arange(256, dtype=torch.int32).to(torch.uint8).view(torch.float8_e4m3fn).reshape(1, 256).to(DEV)
    for name, dt in (("bf16", torch.bfloat16), ("fp16", torch.float16), ("fp32", torch.float32)):
        for sval in (0.00731, 0.02, 1.0, 1.7):
            s = torch.tensor([sval]).to(dt).to(DEV)
            zp = torch.tensor([-5], dtype=torch.int8, device=DEV)
            same(ops.dequantize(codes, s, None).cpu(), sw[f"dq/{name}/s{sval}/int8"], "")
            same(ops.dequantize(codes, s, zp).cpu(), sw[f"dq/{name}/s{sval}/int8zp"], "")
            d = ops.dequantize(f8, s, None).cpu()
            d[d.isnan()] = 0
            same(d, sw[f"dq/{name}/s{sval}/fp8"], "")
            n += 3
    assert n == len(sw)


def test_bitmask_golden_gpu():
    sp = load("sparse")
    for c in sp["bitmask"]:
        got = ops.pack_bitmasks(c["mask"].to(DEV))
        same_values(got.cpu(), c["packed"], "")
        same_values(ops.unpack_bitmasks(c["packed"].to(DEV), list(c["mask"].shape)).cpu(), c["mask"], "")


# --------------------------------------------------------------------------------------------
# 2. seeded inputs vs the oracle, fast (streaming) path
# --------------------------------------------------------------------------------------------
def _weights(shape, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(shape, generator=g) * 0.02).to(dtype)


def _group_qparams(w, bits, group, sym, dtype):
    wf = w.float().unflatten(-1, (-1, group))
    mn, mx = wf.amin(-1).clamp(max=0), wf.amax(-1).clamp(min=0)
    qmax, qmin = 2 ** (bits - 1) - 1, -(2 ** (bits - 1))
    if sym:
        scale = torch.maximum(mn.abs(), mx.abs()) / ((qmax - qmin) / 2)
        zp = None
    else:
        scale = (mx - mn) / float(qmax - qmin)
        zp = (qmin - mn / scale).clamp(qmin, qmax).round().to(torch.int8)
    scale = scale.to(dtype)
    scale[scale == 0] = torch.finfo(dtype).eps
    return scale, zp


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("bits,sym", [(4, True), (4, False), (8, True), (8, False)])
def test_quantize_pack_vs_oracle(dtype, bits, sym):
    w = _weights((1024, 4096), dtype, 1000 + bits)
    scale, zp = _group_qparams(w, bits, 128, sym, dtype)
    a = ns(strategy="group", group_size=128, num_bits=bits, symmetric=sym)
    want_q = oracle.quantize(w, scale, zp, strategy="group", group_size=128, num_bits=bits, dtype=torch.int8)
    want = oracle.pack_to_int32(want_q, bits)
    launches = N.launch_count()
    got = ops.quantize_pack(w.to(DEV), scale.to(DEV), cuda(zp), a)
    assert N.launch_count() == launches + 1, "fused path must be a single kernel"
    same_values(got.cpu(), want, "")
    # decompress side: unpack + dequantize == oracle dequantize == oracle fake_quantize
    want_dq = oracle.dequantize(want_q, scale, zp)
    got_dq = ops.unpack_dequantize(got, scale.to(DEV), cuda(zp), bits, w.shape)
    same(got_dq.cpu(), want_dq, "")
    want_fq = oracle.fake_quantize(w, scale, zp, strategy="group", group_size=128, num_bits=bits)
    same_values(want_dq, want_fq, "oracle dq vs fq")
    got_fq = ops.fake_quantize(w.to(DEV), scale.to(DEV), cuda(zp), a)
    same(got_fq.cpu(), want_fq, "")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("strategy", ["tensor", "channel", "group"])
def test_fp8_quantize_dequantize_vs_oracle(dtype, strategy):
    w = _weights((1024, 4096), dtype, 77)
    if strategy == "tensor":
        scale = (w.float().abs().max() / 448).to(dtype).reshape(1)
        kw = dict(strategy="tensor")
    elif strategy == "channel":
        scale = (w.float().abs().amax(-1, keepdim=True) / 448).to(dtype)
        kw = dict(strategy="channel")
    else:
        scale = (w.float().unflatten(-1, (-1, 128)).abs().amax(-1) / 448).to(dtype)
        kw = dict(strategy="group", group_size=128)
    a = ns(type="float", **kw)
    want = oracle.quantize(w, scale, None, qtype="float", dtype=torch.float8_e4m3fn, **kw)
    got = ops.quantize(w.to(DEV), scale.to(DEV), None, a, dtype=torch.float8_e4m3fn)
    same_values(got.cpu().view(torch.uint8), want.view(torch.uint8), "")
    want_dq = oracle.dequantize(want, scale, None)
    got_dq = ops.dequantize(got, scale.to(DEV), None)
    same(got_dq.cpu(), want_dq, "")
    want_fq = oracle.fake_quantize(w, scale, None, qtype="float", **kw)
    got_fq = ops.fake_quantize(w.to(DEV), scale.to(DEV), None, a)
    same(got_fq.cpu(), want_fq, "")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("sym", [True, False])
def test_int8_channel_quantize_vs_oracle(dtype, sym):
    w = _weights((512, 4096), dtype, 5)
    wf = w.float()
    mn, mx = wf.amin(-1, keepdim=True).clamp(max=0), wf.amax(-1, keepdim=True).clamp(min=0)
    if sym:
        scale, zp = (torch.maximum(mn.abs(), mx.abs()) / 127.5).to(dtype), None
    else:
        scale = ((mx - mn) / 255.0).to(dtype)
        zp = (-128 - mn / scale.float()).clamp(-128, 127).round().to(torch.int8)
    a = ns(strategy="channel", num_bits=8, symmetric=sym)
    want = oracle.quantize(w, scale, zp, strategy="channel", num_bits=8, dtype=torch.int8)
    got = ops.quantize(w.to(DEV), scale.to(DEV), cuda(zp), a, dtype=torch.int8)
    same_values(got.cpu(), want, "")
    want_dq = oracle.dequantize(want, scale, zp)
    got_dq = ops.dequantize(got, scale.to(DEV), cuda(zp))
    same(got_dq.cpu(), want_dq, "")
    want_fq = oracle.fake_quantize(w, scale, zp, strategy="channel", num_bits=8)
    got_fq = ops.fake_quantize(w.to(DEV), scale.to(DEV), cuda(zp), a)
    same(got_fq.cpu(), want_fq, "")


def test_extreme_scales_take_the_ieee_division_path():
    """scales outside [2^-100, 2^100], zero, subnormal: the per-chunk slow path must still match"""
    g = torch.Generator().manual_seed(9)
    x = (torch.randn(64, 1024, generator=g)).bfloat16()
    x[0, :16] = torch.tensor([0.0, -0.0, 1e-38, -1e-38, 3e38, -3e38, 1e-30, 1.0] * 2).bfloat16()
    scales = torch.tensor([1e-38, 9e-41, 3e38, 2.0 ** -101, 2.0 ** 101, 2.0 ** -100, 2.0 ** 100, 1e-45] * 8).bfloat16().reshape(64, 1)
    scales[scales == 0] = 1e-40
    for a, kw in ((ns(strategy="channel", num_bits=4), dict(num_bits=4)), (ns(strategy="channel", type="float"), dict(qtype="float"))):
        dt = torch.int8 if a.type == "int" else torch.float8_e4m3fn
        want = oracle.quantize(x, scales, None, strategy="channel", dtype=dt, **kw)
        got = ops.quantize(x.to(DEV), scales.to(DEV), None, a, dtype=dt)
        same_values(got.cpu().view(torch.uint8), want.view(torch.uint8), "")


@pytest.mark.parametrize("bits", [1, 2, 3, 4, 5, 6, 7, 8])
@pytest.mark.parametrize("shape", [(64, 4096), (33, 100), (7, 1), (128, 33)])
def test_pack_unpack_vs_oracle(bits, shape):
    g = torch.Generator().manual_seed(bits * 7 + shape[1])
    q = torch.randint(-(1 << (bits - 1)), 1 << (bits - 1), shape, dtype=torch.int8, generator=g)
    for pd in (1, 0):
        want = oracle.pack_to_int32(q, bits, pd)
        got = ops.pack_to_int32(q.to(DEV), bits, pd)
        same_values(got.contiguous().cpu(), want, "")
        back = ops.unpack_from_int32(got, bits, q.shape, pd)
        same_values(back.cpu(), q, "")


def test_ragged_and_odd_bits_fused_vs_oracle():
    """generic kernels: rows not a multiple of 32 elements, 3/5/6/7-bit codes, g_idx, one-row scales"""
    w = _weights((50, 200), torch.bfloat16, 3)
    for bits in (2, 3, 5, 6, 7):
        scale = (w.float().abs().amax(-1, keepdim=True) / (2 ** (bits - 1) - 0.5)).bfloat16()
        a = ns(strategy="channel", num_bits=bits)
        want = oracle.pack_to_int32(oracle.quantize(w, scale, None, strategy="channel", num_bits=bits, dtype=torch.int8), bits)
        got = ops.quantize_pack(w.to(DEV), scale.to(DEV), None, a)
        same_values(got.cpu(), want, str(bits))
        dq = ops.unpack_dequantize(got, scale.to(DEV), None, bits, w.shape)
        want_dq = oracle.fake_quantize(w, scale, None, strategy="channel", num_bits=bits)
        same_values(dq.cpu(), want_dq, f"ragged dq bits={bits}")


# --------------------------------------------------------------------------------------------
# 3. BASELINE.json full sizes: properties that need no oracle pass over the whole tensor
# --------------------------------------------------------------------------------------------
LLAMA8B = [(4096, 4096), (1024, 4096), (14336, 4096), (4096, 14336)]


@pytest.mark.parametrize("shape", LLAMA8B)
def test_full_size_w4a16_properties(shape):
    R, C = shape
    g = torch.Generator(device=DEV).manual_seed(1000)
    w = (torch.randn(R, C, device=DEV, generator=g) * 0.02).bfloat16()
    scale = (w.float().unflatten(-1, (-1, 128)).abs().amax(-1) / 7.5).bfloat16()
    a = ns(strategy="group", group_size=128, num_bits=4)
    packed = ops.quantize_pack(w, scale, None, a)
    assert packed.shape == (R, C // 8) and packed.dtype == torch.int32
    # (a) fused == unfused composition, (b) pack/unpack round trip, (c) decompress == fake_quantize
    q = ops.quantize(w, scale, None, a, dtype=torch.int8)
    assert int(q.min()) >= -8 and int(q.max()) <= 7
    same_values(ops.pack_to_int32(q, 4), packed, "")
    same_values(ops.unpack_from_int32(packed, 4, w.shape), q, "")
    dq = ops.unpack_dequantize(packed, scale, None, 4, w.shape)
    same_values(dq, ops.fake_quantize(w, scale, None, a), "decompress == fake_quantize")
    same(dq, ops.dequantize(q, scale, None), "")
    # (d) idempotence: quantizing the dequantized tensor reproduces the codes
    same_values(ops.quantize_pack(dq, scale, None, a), packed, "")
    # (e) spot rows against the oracle
    rows = torch.tensor([0, 1, R // 2, R - 1])
    want = oracle.pack_to_int32(oracle.quantize(w[rows].cpu(), scale[rows].cpu(), None, strategy="group", group_size=128, num_bits=4, dtype=torch.int8), 4)
    same_values(packed[rows].cpu(), want, "")


@pytest.mark.parametrize("shape", LLAMA8B)
def test_full_size_fp8_properties(shape):
    R, C = shape
    g = torch.Generator(device=DEV).manual_seed(1001)
    w = (torch.randn(R, C, device=DEV, generator=g) * 0.02).bfloat16()
    scale = (w.float().abs().max() / 448).bfloat16().reshape(1)
    a = ns(type="float")
    q = ops.quantize(w, scale, None, a, dtype=torch.float8_e4m3fn)
    dq = ops.dequantize(q, scale, None)
    same_values(dq, ops.fake_quantize(w, scale, None, a), "decompress == fake_quantize")
    same_values(ops.quantize(dq, scale, None, a, dtype=torch.float8_e4m3fn).view(torch.uint8), q.view(torch.uint8), "")
    rows = torch.tensor([0, R // 3, R - 1])
    want = oracle.quantize(w[rows].cpu(), scale.cpu(), None, qtype="float", dtype=torch.float8_e4m3fn)
    same_values(q[rows].cpu().view(torch.uint8), want.view(torch.uint8), "")


LLAMA8B_LAYER = [(4096, 4096), (1024, 4096), (1024, 4096), (4096, 4096), (14336, 4096), (14336, 4096), (4096, 14336)]


@pytest.mark.parametrize("scheme", ["w4a16_sym", "w4a16_asym", "fp8_tensor"])
def test_full_layer_every_element_vs_oracle_through_batched(scheme):
    """BASELINE.json's full sizes against the ORACLE, every element: all 7 Linear weights of a Llama-3-8B layer (218 M elements) go
    through ONE multi-tensor launch (ct_batched, the entry point ModelCompressor and bench.py use) per direction, and every packed
    word / fp8 byte / dequantized bf16 value is compared with the CPU oracle's result for the whole tensor."""
    ws, scs, zps = [], [], []
    for i, (R, C) in enumerate(LLAMA8B_LAYER):
        g = torch.Generator(device=DEV).manual_seed(1000 + i)
        w = (torch.randn(R, C, device=DEV, generator=g) * 0.02).bfloat16()
        if scheme == "fp8_tensor":
            sc, zp = (w.abs().max().float() / 448).bfloat16().reshape(1), None
        else:
            sc, zp = _group_qparams(w, 4, 128, scheme == "w4a16_sym", torch.bfloat16)
        ws.append(w); scs.append(sc); zps.append(zp)
    if scheme == "fp8_tensor":
        a, op_c, op_d, qd = ns(type="float"), N.OP_QUANTIZE, N.OP_DEQUANTIZE, torch.float8_e4m3fn
        okw_ = dict(strategy="tensor", qtype="float", dtype=torch.float8_e4m3fn)
    else:
        a, op_c, op_d, qd = ns(strategy="group", group_size=128, num_bits=4, symmetric=scheme == "w4a16_sym"), N.OP_QUANTIZE_PACK, N.OP_UNPACK_DEQUANTIZE, torch.int8
        okw_ = dict(strategy="group", group_size=128, num_bits=4, dtype=torch.int8)
    comp, cprobs, dprobs, backs = [], [], [], []
    for w, sc, zp in zip(ws, scs, zps):
        R, C = w.shape
        p = ops._resolve(w, sc, zp, a, None)
        zdt = zp.dtype if zp is not None else None
        if scheme == "fp8_tensor":
            out = torch.empty(R, C, dtype=qd, device=DEV)
            d = ops._desc(p, w.dtype, sc.dtype, zdt, torch.bfloat16, qd, qd, N.Q_FLOAT, 8)
            d2 = ops._desc(p, None, sc.dtype, zdt, None, qd, torch.bfloat16, N.Q_INT, 8)
        else:
            out = torch.empty(R, C // 8, dtype=torch.int32, device=DEV)
            d = ops._desc(p, w.dtype, sc.dtype, zdt, torch.bfloat16, torch.int8, None, N.Q_INT, 4)
            d2 = ops._desc(p, None, sc.dtype, zdt, None, torch.int8, torch.bfloat16, N.Q_INT, 4)
        back = torch.empty(R, C, dtype=torch.bfloat16, device=DEV)
        cprobs.append((d, w, p.scale.contiguous(), p.zp.contiguous() if p.zp is not None else None, out))
        dprobs.append((d2, out, p.scale.contiguous(), p.zp.contiguous() if p.zp is not None else None, back))
        comp.append(out); backs.append(back)
    launches = N.launch_count()
    ops.batched(op_c, cprobs)
    ops.batched(op_d, dprobs)
    assert N.launch_count() - launches == 2, "one multi-tensor launch per direction"
    for i, (w, sc, zp, out, back) in enumerate(zip(ws, scs, zps, comp, backs)):
        wc, scc, zpc = w.cpu(), sc.cpu(), (zp.cpu() if zp is not None else None)
        q = oracle.quantize(wc, scc, zpc, **okw_)
        if scheme == "fp8_tensor":
            same_values(out.cpu().view(torch.uint8), q.view(torch.uint8), f"{scheme} tensor {i} {tuple(w.shape)} fp8 bytes")
        else:
            same_values(out.cpu(), oracle.pack_to_int32(q, 4), f"{scheme} tensor {i} {tuple(w.shape)} packed words")
        same(back.cpu(), oracle.dequantize(q, scc, zpc), f"{scheme} tensor {i} {tuple(w.shape)} dequantized")


def test_batched_rejects_descriptors_that_do_not_match_their_tensors():
    """a wrong descriptor would be an out-of-bounds access on the device: ops.batched checks sizes on the host and launches nothing"""
    a = ns(strategy="group", group_size=128, num_bits=4)
    w = _weights((64, 256), torch.bfloat16, 1).to(DEV)
    sc = (w.float().unflatten(-1, (-1, 128)).abs().amax(-1) / 7.5).bfloat16()
    out = torch.zeros(64, 32, dtype=torch.int32, device=DEV)
    p = ops._resolve(w, sc, None, a, None)
    d = ops._desc(p, w.dtype, sc.dtype, None, torch.bfloat16, torch.int8, None, N.Q_INT, 4)
    launches = N.launch_count()
    for bad in [(d, w[:32], sc, None, out), (d, w, sc[:, :1].contiguous(), None, out), (d, w, sc, None, out[:32]),
                (d, w.float(), sc, None, out), (d, w.t(), sc, None, out), (d, w.cpu(), sc, None, out), (d, w, sc, None, None)]:
        with pytest.raises(ValueError, match="batched: tensor 0"):
            ops.batched(N.OP_QUANTIZE_PACK, [bad])
    assert N.launch_count() == launches
    ops.batched(N.OP_QUANTIZE_PACK, [(d, w, sc, None, out)])
    same_values(out, ops.quantize_pack(w, sc, None, a), "valid problem still runs")


def test_batched_launch_equals_per_tensor():
    """one persistent launch over a table of tensors == per-tensor launches"""
    shapes = [(1024, 4096), (512, 1024), (4096, 512), (64, 128), (2048, 14336)]
    a = ns(strategy="group", group_size=128, num_bits=4)
    ws, scs, singles, outs, probs = [], [], [], [], []
    for i, (R, C) in enumerate(shapes):
        w = _weights((R, C), torch.bfloat16, 50 + i).to(DEV)
        sc = (w.float().unflatten(-1, (-1, 128)).abs().amax(-1) / 7.5).bfloat16()
        singles.append(ops.quantize_pack(w, sc, None, a))
        out = torch.zeros(R, C // 8, dtype=torch.int32, device=DEV)
        p = ops._resolve(w, sc, None, a, None)
        d = ops._desc(p, w.dtype, sc.dtype, None, torch.bfloat16, torch.int8, None, N.Q_INT, 4)
        probs.append((d, w, sc, None, out))
        ws.append(w); scs.append(sc); outs.append(out)
    launches = N.launch_count()
    ops.batched(N.OP_QUANTIZE_PACK, probs)
    assert N.launch_count() == launches + 1
    for s, o in zip(singles, outs):
        same_values(s, o, "")


def test_host_buffers_pipeline_equals_device_path():
    """CPU tensors go through ct_host_run_many (chunked H2D / kernel / D2H) and must give identical bytes"""
    w = _weights((12288, 4096), torch.bfloat16, 31)   # 96 MiB -> 3 chunks
    scale = (w.float().unflatten(-1, (-1, 128)).abs().amax(-1) / 7.5).bfloat16()
    a = ns(strategy="group", group_size=128, num_bits=4)
    dev = ops.quantize_pack(w.to(DEV), scale.to(DEV), None, a).cpu()
    host = ops.quantize_pack(w, scale, None, a)
    assert not host.is_cuda and torch.equal(host, dev)
    back_dev = ops.unpack_dequantize(dev.to(DEV), scale.to(DEV), None, 4, w.shape).cpu()
    back_host = ops.unpack_dequantize(host, scale, None, 4, w.shape)
    assert not back_host.is_cuda and bits_equal(back_host, back_dev)
    s8 = (w.float().abs().max() / 448).bfloat16().reshape(1)
    q_host = ops.quantize(w, s8, None, ns(type="float"), dtype=torch.float8_e4m3fn)
    q_dev = ops.quantize(w.to(DEV), s8.to(DEV), None, ns(type="float"), dtype=torch.float8_e4m3fn).cpu()
    same_values(q_host.view(torch.uint8), q_dev.view(torch.uint8), "")


# --------------------------------------------------------------------------------------------
# 4. sparse formats vs the restated oracle (parity unpinned, see oracle header)
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32, torch.int8])
@pytest.mark.parametrize("shape", [(128, 4096), (17, 40), (5, 12)])
def test_sparse24_vs_oracle(dtype, shape):
    g = torch.Generator().manual_seed(shape[1])
    x = torch.randn(shape, generator=g) * 10
    x = x.round().to(dtype) if dtype == torch.int8 else x.to(dtype)
    vals, bm = oracle.sparse24_compress(x)
    gv, gb = ops.sparse24_compress(x.to(DEV))
    same_values(gb.cpu(), bm, "")
    same(gv.cpu(), vals, "")
    dense = ops.sparse24_decompress(gv, gb, x.shape)
    same(dense.cpu(), oracle.sparse24_decompress(vals, bm, x.shape), "")


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32, torch.int8])
@pytest.mark.parametrize("shape", [(64, 4096), (9, 37), (300, 1000)])
def test_bitmask_compress_vs_oracle(dtype, shape):
    g = torch.Generator().manual_seed(shape[0])
    x = torch.randn(shape, generator=g) * 5
    x[torch.rand(shape, generator=g) < 0.7] = 0
    x = x.round().to(dtype) if dtype == torch.int8 else x.to(dtype)
    vals, bm, offs = oracle.bitmask_compress(x)
    gv, gb, go = ops.bitmask_compress(x.to(DEV))
    same_values(gb.cpu(), bm, "")
    same(gv.cpu(), vals, "")
    same_values(go.cpu(), offs, "row offsets")
    dense = ops.bitmask_decompress(gv, gb, go, x.shape)
    same(dense.cpu(), x.where(x != 0, torch.zeros_like(x)), "")


@pytest.mark.parametrize("shape", [(2, 128), (5, 16384), (3, 16512), (1, 8192), (37, 8192), (700, 4096), (150, 14336),
                                   (37, 4128), (5, 2080), (9, 1056)])
def test_bitmask_expand_rows_pipeline(shape, monkeypatch):
    """the pipelined row expansion (persistent CTAs, bulk-copy ring; csrc/sparse.cu bitmask_expand_rows_kernel) against the oracle:
    rows that are empty, full, and mixed; more rows than one CTA's ring holds; the last rows of the tensor (values fetched after the
    scan, because the run's 16-byte over-read would leave `values`); and the per-row kernel on the shapes the pipeline declines (one
    row, more than 2048 units per row, cols % 128 != 0 with 4, 2 and 1 segments per iteration)"""
    g = torch.Generator().manual_seed(shape[0] * 7 + shape[1])
    x = (torch.randn(shape, generator=g) * 3).bfloat16()
    x[torch.rand(shape, generator=g) < 0.5] = 0
    R = shape[0]
    if R >= 5:
        x[1] = 0                                             # an empty row
        x[2] = 1.5                                           # a full row
        x[R - 2] = 0                                         # the last row's predecessor is empty: its run ends where the last row starts
        x[R - 1, : shape[1] // 2] = 0
    vals, bm, offs = oracle.bitmask_compress(x)
    want = oracle.bitmask_decompress(vals, bm, x.shape)
    gv, gb, go = vals.to(DEV), bm.to(DEV), offs.to(DEV)
    launches = N.launch_count()
    dense = ops.bitmask_decompress(gv, gb, go, x.shape)
    assert N.launch_count() - launches == 1
    same(dense.cpu(), want, "row expand vs oracle")
    for pct in ("100", "400"):                              # ring of exactly one worst-case row (no prefetch at full density) / a deep one
        monkeypatch.setenv("CT_B200_BITMASK_RING_PCT", pct)
        same(ops.bitmask_decompress(gv, gb, go, x.shape), dense, f"ring {pct} %")


@pytest.mark.parametrize("density", [0.0, 0.03, 0.5, 0.97, 1.0])
@pytest.mark.parametrize("shape", [(8, 32), (64, 4096), (300, 1000), (1031, 2056), (4096, 14336)])
def test_bitmask_onepass_lookback_vs_oracle(shape, density):
    """the one-pass kernels (decoupled look-back scan, csrc/bitmask_onepass.cu): every output of the format -- values, mask bytes,
    row offsets, nnz -- against the restated oracle, the no-sync (`exact=False`) form included, for densities from empty to full, tiles
    that hold many rows and rows that span many tiles; the same bits as the two-phase ABI (count -> scan -> move); and the expansion
    without row_offsets, which recomputes the scan from the mask popcounts"""
    g = torch.Generator().manual_seed(shape[1] + int(density * 100))
    x = (torch.randn(shape, generator=g) * 3).bfloat16()
    x[torch.rand(shape, generator=g) >= density] = 0
    x[0, 0] = -0.0                                           # -0.0 is a zero of the format
    vals, bm, offs = oracle.bitmask_compress(x)
    xd = x.to(DEV)
    launches = N.launch_count()
    cap, gb, go, nnz = ops.bitmask_compress(xd, exact=False)
    onepass = (x.numel() // 8) % 4 == 0                      # otherwise: two-phase kernels behind the same call
    assert N.launch_count() - launches == (1 if onepass else 3), "one kernel: the dense tensor is read once"
    assert cap.numel() == x.numel() and nnz.is_cuda and int(nnz.item()) == vals.numel()
    same_values(gb.cpu(), bm, "mask bytes")
    same_values(go.cpu(), offs, "row offsets")
    same(cap[: vals.numel()].cpu(), vals, "values")
    gv, gb2, go2 = ops.bitmask_compress(xd)
    assert gv.numel() == vals.numel()
    same(gv.cpu(), vals, "values (exact)")
    launches = N.launch_count()
    dense = ops.bitmask_decompress(gv, gb, go, x.shape)
    assert N.launch_count() - launches == 1
    same(dense.cpu(), x.where(x != 0, torch.zeros_like(x)), "expand")
    same(dense.cpu(), oracle.bitmask_decompress(vals, bm, x.shape), "expand vs oracle")
    rows, cols = shape
    st = N.stream_ptr(0)
    tb = torch.empty_like(gb)
    to = torch.empty_like(go)
    tn = torch.empty(1, dtype=torch.int64, device=DEV)
    ws = torch.empty(N.lib().ct_bitmask_workspace_bytes(rows, cols), dtype=torch.uint8, device=DEV)
    N.check(N.lib().ct_bitmask_count(N.ptr(xd), N.DT[x.dtype], N.ptr(tb), N.ptr(to), N.ptr(tn), N.ptr(ws), rows, cols, 0, st))
    tv = torch.empty(int(tn.item()), dtype=x.dtype, device=DEV)
    N.check(N.lib().ct_bitmask_compress(N.ptr(xd), N.DT[x.dtype], N.ptr(tb), N.ptr(to), N.ptr(tv), rows, cols, 0, st))
    same(tv, gv, "two-phase values"); same_values(tb, gb, "two-phase mask"); same_values(to, go, "two-phase offsets")
    out = torch.empty_like(xd)
    rc = N.lib().ct_bitmask_decompress(N.ptr(cap), N.DT[x.dtype], N.ptr(gb), N.ptr(None), N.ptr(out), rows, cols, 0, st)
    if onepass:
        N.check(rc)
        same(out, dense, "look-back expand == row_offsets expand")
    else:
        assert rc == N.CT_E_UNSUPPORTED                      # without row_offsets only the look-back kernel can expand
