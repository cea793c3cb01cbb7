"""
Every bf16 / fp16 bit pattern through the FP4 (E2M1) and MX kernels, bit for bit against the CPU oracle (tests/test_fp4_sweep_host.py
proves the oracle equal to the reference's own outputs and to a float64 model on these ladders) and against
tests/golden/fp4_sweep.pt.gz.  Codes made from NaN quotients (NaN inputs, 0 / 0 under a zero scale, inf / inf under an infinite MX
scale) are undefined in the reference and not compared; fake-quantized and dequantized NaNs must sit where the oracle puts them.

Each encode and decode sweep runs three ways, so that both kernels are checked and the test knows which one ran:
  fast     a layout the streaming planner takes (cols % 32 == 0, 16-byte aligned);
  generic  the same data as a view 2 bytes past an aligned allocation, which the planner must send to the generic kernel;
  batched  one ops.batched call holding one entry of each, which must make exactly 2 launches (one per streaming kernel, one per generic
           tensor), proving the aligned entry took the streaming kernel and the offset one did not.

Kernel branches and the tests that reach them:
  Fp4NvQuantPackOp, scale in the x dtype (sel 1) and in float32 (sel 2)       test_nvfp4_every_pattern_every_e4m3_scale
  Fp4NvQuantPackOp::unit_slow, |scale / gs| across 2^10 and 2^-100             test_nvfp4_global_scales_across_the_division_range
  Fp4NvQuantPackOp, +0.0 under a negative scale (sent to unit_slow)              test_nvfp4_positive_zero_under_a_negative_scale
  Fp4NvQuantPackOp::unit_slow, +-0.0 with a -0.0 zero point                     test_nvfp4_negative_zero_zero_point_in_unit_slow
  NVFP4 zero points (fp8 +0.0, -0.0, values) on chunk_fast and unit_slow       test_nvfp4_zero_points
  Fp4MxQuantPackOp: every power of two, ScaleCtx.slow (other scales), zp     test_mxfp4_every_pattern_every_scale
  generic quantize / fake_quantize / dequantize / cast_to_fp4                 test_generic_fp4_ops_every_pattern
  Fp4UnpackDequantOp: fp8 scales (Fp4DqTile.fast across gs 2^+-60, recip_div across 2^-40 and 2^14), E8M0 (255 too), float scales
                                                                              test_unpack_dequantize_every_byte_*
  ct_observe_quantize_pack_nvfp4 on every max |x| (group max across 2^-40, 2^14; gs across 2^+-60)
                                                                              test_nvfp4_observer_every_group_max
  ct_observe_quantize_mx (MXFP4, MXFP8) on every max |x|                       test_mx_observer_every_group_max
  ct_dynamic_fake_quantize (NVFP4 with a global-scale ladder, MXFP4) on every max |x|
                                                                              test_dynamic_fake_quantize_every_group_max
  ct_host_run_many for OP_QUANTIZE_PACK_FP4 and OP_UNPACK_DEQUANTIZE_FP4        test_host_resident_fp4_ops
  compress_mx_scale / decompress_mx_scale on every input                        test_mx_scale_codes_every_pattern
"""
import numpy as np
import pytest
import torch

import oracle
from compressed_tensors_b200 import _native as N
from compressed_tensors_b200 import ops
from compressed_tensors_b200.quantization import QuantizationArgs
from tests import e2m1_model as M
from tests.golden import load
from tests.util import same, same_nan

pytestmark = pytest.mark.gpu
DEV = "cuda"
F8 = torch.float8_e4m3fn
TD = {"bf16": torch.bfloat16, "fp16": torch.float16}
GS_384 = 2688.0 / 7.0
NV = QuantizationArgs(num_bits=4, type="float", symmetric=True, strategy="tensor_group", group_size=16)
G = load("fp4_sweep")["cases"]


def mx_args(group=32, bits=4, **kw):
    return QuantizationArgs(num_bits=bits, type="float", symmetric=True, strategy="group", group_size=group, **kw)


def f32_next(v, toward):
    return float(np.nextafter(np.float32(v), np.float32(toward)))


def patterns(dt, reps=1):
    """every pattern of dt as [1024 * reps, 64]: block r of 1024 rows holds all 65536 patterns again"""
    x = torch.arange(65536, dtype=torch.int32).to(torch.int16).view(TD[dt]).reshape(1024, 64)
    return x.repeat(reps, 1)


def per_block(values, reps_rows, groups, dtype):
    """a [len(values) * reps_rows, groups] scale (or zero-point) tensor whose block i of rows holds values[i]"""
    return torch.tensor(values, dtype=torch.float64).repeat_interleave(reps_rows)[:, None].expand(-1, groups).to(dtype).contiguous()


def offset_view(t):
    """t copied to the device into a view 2 bytes past an aligned allocation"""
    k = max(1, 2 // t.element_size())
    base = torch.empty(t.numel() + k, dtype=t.dtype, device=DEV)
    v = base[k:k + t.numel()].view(t.shape)
    v.copy_(t.to(DEV))
    return v


def dev(t):
    return None if t is None else t.to(DEV)


def packed_want(q):
    """(the oracle's codes packed, the bytes to compare): a byte is compared when neither of its quotients is NaN -- a NaN input,
    0 / 0 under a zero scale, inf / inf under an infinite one -- since the reference's code of a NaN is undefined"""
    keep = ~q.isnan().reshape(q.shape[0], -1, 2).any(-1)
    return oracle.pack_fp4_to_uint8(torch.nan_to_num(q, nan=0.0)), keep


def same_codes(got, want, what):
    packed, keep = want
    same(got.cpu()[keep], packed[keep], what)


def first_finite_e4m3_bytes(stride=1):
    b = [i for i in range(256) if (i & 0x7F) != 0x7F]
    return b[::stride]


# ---------------------------------------------------------------------------------------------------------------------------------
# three ways through op 8 (quantize + pack to FP4) and op 9 (unpack + dequantize FP4)
# ---------------------------------------------------------------------------------------------------------------------------------
def qpack_problem(x, scale, zp, args, gs, xd):
    """(problem for ops.batched / ops.host_batched, output, global-scale tensor to keep alive); x, scale, zp on the CPU, xd = x where
    the kernel reads it"""
    sc, gsv, se = ops._global_scale(scale, gs)
    cd = torch.result_type(x, sc if gsv is None else ops._like(sc, se))
    p = ops._resolve(x, sc, zp, args, None)
    d = ops._desc(p, x.dtype, p.scale.dtype, zp.dtype if zp is not None else None, cd, x.dtype, None, N.Q_FP4, 4, se)
    where = xd.device
    keep = gsv.to(where).contiguous() if gsv is not None else None
    if keep is not None:
        d.global_scale = keep.data_ptr()
    out = torch.empty((x.shape[0], x.shape[1] // 2), dtype=torch.uint8, device=where)
    zz = p.zp.to(where).contiguous() if p.zp is not None else None
    return (d, xd, p.scale.to(where).contiguous(), zz, out), out, keep


def qpack_three_ways(x, scale, zp, args, gs, want, what):
    """quantize_pack_fp4 on the aligned layout, on a 2-byte-offset view, and both in one ops.batched call (2 launches)"""
    xa = x.to(DEV)
    xo = offset_view(x)
    same_codes(ops.quantize_pack_fp4(xa, dev(scale), dev(zp), args, global_scale=dev(gs)), want, f"{what} fast")
    same_codes(ops.quantize_pack_fp4(xo, dev(scale), dev(zp), args, global_scale=dev(gs)), want, f"{what} generic")
    pa, oa, ka = qpack_problem(x, scale, zp, args, gs, xa)
    po, oo, ko = qpack_problem(x, scale, zp, args, gs, xo)
    n0 = N.launch_count()
    ops.batched(N.OP_QUANTIZE_PACK_FP4, [pa, po])
    assert N.launch_count() - n0 == 2, "one streaming launch and one generic launch"
    torch.cuda.synchronize()
    same_codes(oa, want, f"{what} batched fast entry")
    same_codes(oo, want, f"{what} batched generic entry")


def nv_want(x, scale, zp, gs):
    return packed_want(oracle.quantize(x, scale, zp, strategy="tensor_group", group_size=16, num_bits=4, qtype="float", global_scale=gs))


def mx_want(x, scale, zp, group):
    return packed_want(oracle.quantize(x, scale, zp, strategy="group", group_size=group, num_bits=4, qtype="float"))


# ---------------------------------------------------------------------------------------------------------------------------------
# encode with a given scale
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dt", ["bf16", "fp16"])
@pytest.mark.parametrize("gs", [1.0, GS_384], ids=["gs1", "gs384"])
def test_nvfp4_every_pattern_every_e4m3_scale(dt, gs):
    """Fp4NvQuantPackOp (sel 1: scale in the x dtype; sel 2: float32 scale) and the generic quantize + pack: every pattern under every
    finite e4m3 scale byte of both signs"""
    bytes_ = first_finite_e4m3_bytes()
    svals = M.e4m3_decode(np.array(bytes_)).tolist()
    x = patterns(dt, len(bytes_))
    gst = torch.tensor([gs], dtype=torch.float32)
    s32 = per_block(svals, 1024, 4, torch.float32)
    want = nv_want(x, s32, None, gst)
    for sdt in (TD[dt], torch.float32):
        qpack_three_ways(x, s32.to(sdt), None, NV, gst, want, f"nvfp4 {dt} scale {sdt} gs {gs}")
    print(f"{x.numel()} elements x 2 scale dtypes x 3 ways")


def division_range_global_scales():
    """global scales that put |1.0 / gs| on 2^10 and 2^-100 and one ulp either side of each"""
    out = []
    for g in (2.0 ** -10, 2.0 ** 100):
        out += [g, f32_next(g, 0), f32_next(g, np.inf)]
    return out


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
@pytest.mark.parametrize("gs", division_range_global_scales(), ids=lambda g: f"{g:.9g}")
def test_nvfp4_global_scales_across_the_division_range(dt, gs):
    """Fp4NvQuantPackOp switches a unit to IEEE division (unit_slow) when |scale / gs| leaves [2^-100, 2^10]: scales of +-1.0 sit on,
    just inside and just outside each end, the other scale bytes on either side"""
    bytes_ = sorted(set(first_finite_e4m3_bytes(16) + [0x38, 0xB8, 0x7E, 0x01, 0x36, 0x4C]))
    svals = M.e4m3_decode(np.array(bytes_)).tolist()
    x = patterns(dt, len(bytes_))
    gst = torch.tensor([gs], dtype=torch.float32)
    s32 = per_block(svals, 1024, 4, torch.float32)
    want = nv_want(x, s32, None, gst)
    model = torch.from_numpy(M.pack_nibbles(np.nan_to_num(M.nvfp4_quantize(M.bits_to_float(x.view(torch.int16).numpy().view(np.uint16), dt),
                                                                           s32.double().numpy().repeat(16, 1), gs), nan=0.0)))
    same_codes(model, want, "model vs oracle")
    for sdt in (TD[dt], torch.float32):
        qpack_three_ways(x, s32.to(sdt), None, NV, gst, want, f"nvfp4 {dt} gs {gs!r}")
    print(f"{x.numel()} elements x 2 scale dtypes x 3 ways")


def test_nvfp4_positive_zero_under_a_negative_scale():
    """Fp4NvQuantPackOp: x = +0.0 under a negative scale quantizes to +0.0 (code 0) like the reference's torch.sign; the residual
    division step gave -0.0 (code 8) until negative scales were sent to unit_slow"""
    x = torch.zeros(1, 32, dtype=torch.bfloat16)
    x[0, 1::2] = -0.0
    s = torch.tensor([[-1.0, -448.0]])
    want = nv_want(x, s, None, torch.tensor([1.0]))
    assert bool((want[0] == 0).all())
    qpack_three_ways(x, s, None, NV, torch.tensor([1.0]), want, "+0.0 / negative scale")


def test_nvfp4_negative_zero_zero_point_in_unit_slow():
    """Fp4NvQuantPackOp::unit_slow: x = +-0.0 with an fp8 zero point of -0.0 (byte 0x80) quantizes to +0.0 (code 0) like the
    reference's torch.sign, under a scale the unit sends slow (2048 > 2^10) and under a negative one; it gave -0.0 (code 8) until
    unit_slow mapped a zero quotient to +0.0"""
    x = torch.zeros(2, 32, dtype=torch.bfloat16)
    x[:, 0::2] = -0.0
    s = torch.tensor([[2048.0, 2048.0], [-1.0, -1.0]])
    zp = torch.full((2, 2), -0.0).to(F8)
    assert bool((zp.view(torch.uint8) == 0x80).all())
    want = nv_want(x, s, zp, torch.tensor([1.0]))
    assert bool((want[0] == 0).all())
    qpack_three_ways(x, s, zp, NV, torch.tensor([1.0]), want, "+-0.0 with a -0.0 zero point")


ZP_VALUES = [0.0, -0.0, 0.5, -0.5, 1.0, -1.0, 1.5, -1.5, 2.0, -2.0, 3.0, -3.0, 4.0, -4.0]


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
@pytest.mark.parametrize("zp_mode", ["zeros", "negative_zeros", "values"])
@pytest.mark.parametrize("gs", [GS_384, 2.0 ** -10], ids=["gs384", "gs2^-10"])
def test_nvfp4_zero_points(dt, zp_mode, gs):
    """the zero-point add of Fp4NvQuantPackOp (chunk_fast and unit_slow) and of the generic kernel: fp8 +0.0, fp8 -0.0, and fp8
    values in {+-0, +-0.5 .. +-4}, one per group.  At gs 2^-10 every scale byte above 1.0 puts s_eff above 2^10: those units, and
    every negative scale, take unit_slow"""
    bytes_ = first_finite_e4m3_bytes(8)
    svals = M.e4m3_decode(np.array(bytes_)).tolist()
    x = patterns(dt, len(bytes_))
    gst = torch.tensor([gs], dtype=torch.float32)
    s = per_block(svals, 1024, 4, TD[dt])
    if zp_mode == "values":
        zp = torch.tensor(ZP_VALUES)[torch.arange(s.numel()) % len(ZP_VALUES)].reshape(s.shape).to(F8)
    else:
        zp = torch.full(s.shape, 0.0 if zp_mode == "zeros" else -0.0).to(F8)
    want = nv_want(x, s, zp, gst)
    qpack_three_ways(x, s, zp, NV, gst, want, f"nvfp4 {dt} zp {zp_mode} gs {gs}")
    print(f"{x.numel()} elements x 3 ways")


def mx_scales(dt):
    lo, hi = (-133, 127) if dt == "bf16" else (-24, 15)
    return [2.0 ** e for e in range(lo, hi + 1)], [0.3, 1.7, 3.0, 0.011, 100.0]


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
@pytest.mark.parametrize("zp_dt,group", [(None, 32), (torch.uint8, 32), (torch.int8, 32), (torch.uint8, 64), (torch.int8, 64), (None, 64)])
def test_mxfp4_every_pattern_every_scale(dt, zp_dt, group):
    """Fp4MxQuantPackOp (arithmetic in the x dtype): every pattern under every power of two the dtype holds and under scales that are
    not powers of two (ScaleCtx.slow); uint8 / int8 zero points of both signs and of 128 and more on every eighth power of two and on
    the other scales"""
    pows, other = mx_scales(dt)
    svals = (pows if zp_dt is None and group == 32 else pows[::8]) + other
    x = patterns(dt, len(svals))
    s = per_block(svals, 1024, 64 // group, TD[dt])
    zp = None
    if zp_dt is not None:
        # negative int8 values catch a missing sign extension, uint8 values of 128 and more a signed read
        vals = [0, 1, 3, 128, 200, 255] if zp_dt == torch.uint8 else [0, 1, -1, -3, 127, -128]
        zp = torch.tensor(vals, dtype=zp_dt)[torch.arange(s.numel()) % len(vals)].reshape(s.shape)
    want = mx_want(x, s, zp, group)
    qpack_three_ways(x, s, zp, mx_args(group), None, want, f"mxfp4 {dt} zp {zp_dt} group {group}")
    print(f"{x.numel()} elements x 3 ways")


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
@pytest.mark.parametrize("kind", ["nvfp4", "mxfp4"])
def test_generic_fp4_ops_every_pattern(dt, kind):
    """the generic quantize / fake_quantize / dequantize kernels with FP4 args, and cast_to_fp4, on every pattern"""
    if kind == "nvfp4":
        bytes_ = first_finite_e4m3_bytes(8)
        svals, args, gst, groups = M.e4m3_decode(np.array(bytes_)).tolist(), NV, torch.tensor([GS_384], dtype=torch.float32), 4
        okw = dict(strategy="tensor_group", group_size=16, global_scale=gst)
    else:
        pows, other = mx_scales(dt)
        svals, args, gst, groups = pows[::4] + other, mx_args(), None, 2
        okw = dict(strategy="group", group_size=32)
    x = patterns(dt, len(svals))
    s = per_block(svals, 1024, groups, TD[dt])
    q = oracle.quantize(x, s, None, num_bits=4, qtype="float", **okw)
    same_nan(ops.quantize(x.to(DEV), s.to(DEV), None, args, global_scale=dev(gst)).cpu(), q, "quantize")
    same_nan(ops.fake_quantize(x.to(DEV), s.to(DEV), None, args, global_scale=dev(gst)).cpu(),
             oracle.fake_quantize(x, s, None, num_bits=4, qtype="float", **okw), "fake_quantize")
    qc = torch.nan_to_num(q, nan=0.0)
    same_nan(ops.dequantize(qc.to(DEV), s.to(DEV), None, args, dtype=TD[dt], global_scale=dev(gst)).cpu(),
             oracle.dequantize(qc, s, None, dtype=TD[dt], **okw), "dequantize")
    xs = patterns(dt)
    same_nan(ops.cast_to_fp4(xs.to(DEV)).cpu(), oracle.cast_to_fp4(xs), "cast_to_fp4")
    print(f"{x.numel()} elements through three ops, 65536 through cast_to_fp4")


# ---------------------------------------------------------------------------------------------------------------------------------
# decode
# ---------------------------------------------------------------------------------------------------------------------------------
PACKED = torch.arange(256, dtype=torch.int32).to(torch.uint8).repeat(256, 1)       # row r: every packed byte, under scale byte r
ROWS = torch.arange(256, dtype=torch.int32).to(torch.uint8)


def udq_problem(packed, stored, code, odt, group, gs, pd):
    R, C = packed.shape[0], packed.shape[1] * 2
    se = torch.float32 if gs is not None else odt                 # every scale here is stored in, or decoded to, the output dtype
    like = torch.empty((R, C), dtype=torch.int8, device="meta")
    from types import SimpleNamespace
    p = ops._resolve(like, stored, None, SimpleNamespace(strategy="group", group_size=group, block_structure=None), None)
    d = ops._desc(p, None, torch.float32, None, None, None, odt, N.Q_FP4, 4, se)
    d.scale_dtype = code
    keep = gs.to(pd.device).contiguous() if gs is not None else None
    if keep is not None:
        d.global_scale = keep.data_ptr()
    out = torch.empty((R, C), dtype=odt, device=pd.device)
    return (d, pd, p.scale.to(pd.device).contiguous(), None, out), out, keep


def udq_three_ways(packed, stored, stored_kind, code, odt, group, gs, want, what):
    kw = dict(global_scale=dev(gs), dtype=odt, stored_scale=stored_kind)
    same_nan(ops.unpack_dequantize_fp4(packed.to(DEV), stored.to(DEV), **kw).cpu(), want, f"{what} fast")
    po_in = offset_view(packed)
    same_nan(ops.unpack_dequantize_fp4(po_in, stored.to(DEV), **kw).cpu(), want, f"{what} generic")
    pa, oa, ka = udq_problem(packed, stored, code, odt, group, gs, packed.to(DEV))
    po, oo, ko = udq_problem(packed, stored, code, odt, group, gs, po_in)
    n0 = N.launch_count()
    ops.batched(N.OP_UNPACK_DEQUANTIZE_FP4, [pa, po])
    assert N.launch_count() - n0 == 2, "one streaming launch and one generic launch"
    torch.cuda.synchronize()
    same_nan(oa.cpu(), want, f"{what} batched fast entry")
    same_nan(oo.cpu(), want, f"{what} batched generic entry")


def udq_want(packed, s_float, group, gs, odt):
    R, C = packed.shape[0], packed.shape[1] * 2
    return oracle.dequantize(oracle.unpack_fp4_from_uint8(packed, R, C, odt), s_float, None, strategy="group", group_size=group,
                             global_scale=gs, dtype=odt)


def fp8_global_scales():
    return [1.0, GS_384, 2.0 ** 60, f32_next(2.0 ** 60, np.inf), f32_next(2.0 ** 60, 0), 2.0 ** -60, f32_next(2.0 ** -60, 0),
            f32_next(2.0 ** -60, np.inf), 2.0 ** -10, 2.0 ** 31]


@pytest.mark.parametrize("odt", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("gs", fp8_global_scales(), ids=lambda g: f"{g:.9g}")
def test_unpack_dequantize_every_byte_fp8_scale(odt, gs):
    """Fp4UnpackDequantOp with stored e4m3 scales: every packed byte under every scale byte (NaN ones too); global scales at 2^+-60 and
    one ulp either side (Fp4DqTile.fast), and 2^-10 / 2^31, which carry scale / gs across 2^14 and 2^-40 (recip_div)"""
    stored = ROWS[:, None].repeat(1, 32).view(F8)
    gst = torch.tensor([gs], dtype=torch.float32)
    want = udq_want(PACKED, stored.to(odt), 16, gst, odt)
    model = M.fp4_dequantize(M.unpack_nibbles(PACKED.numpy()), M.rn(M.e4m3_decode(np.arange(256)), {torch.bfloat16: "bf16", torch.float16: "fp16"}[odt])[:, None], gs,
                             {torch.bfloat16: "bf16", torch.float16: "fp16"}[odt])
    same_nan(torch.from_numpy(model).to(odt), want, "model vs oracle")
    for c in G:
        if c["kind"] == "nvfp4_decompress" and c["global_scale"] == gs and odt == torch.bfloat16:
            same_nan(want, c["weight"], "oracle vs golden")
    udq_three_ways(PACKED, stored, "fp8", N.DT[F8], odt, 16, gst, want, f"fp8 scales gs {gs!r} -> {odt}")
    print(f"{want.numel()} elements x 3 ways")


@pytest.mark.parametrize("odt", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_unpack_dequantize_every_byte_e8m0_scale(odt):
    """Fp4UnpackDequantOp with stored E8M0 scales: every packed byte under every exponent byte, 255 (2^128 = inf) included"""
    stored = ROWS[:, None].repeat(1, 16).contiguous()
    want = udq_want(PACKED, oracle.decompress_mx_scale(stored).to(odt), 32, None, odt)
    if odt == torch.bfloat16:
        (c,) = [c for c in G if c["kind"] == "mxfp4_decompress"]
        same_nan(want, c["weight"], "oracle vs golden")
    udq_three_ways(PACKED, stored, "e8m0", N.DT_E8M0, odt, 32, None, want, f"e8m0 scales -> {odt}")
    print(f"{want.numel()} elements x 3 ways")


@pytest.mark.parametrize("odt", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("gs", [None, GS_384], ids=["no_gs", "gs384"])
def test_unpack_dequantize_every_float_scale(odt, gs):
    """Fp4UnpackDequantOp with a float scale in the output dtype: every finite pattern of it, each under all 16 codes"""
    s = torch.arange(65536, dtype=torch.int32).to(torch.int16).view(odt)
    s = s[s.isfinite()]
    s = s[: s.numel() // 2 * 2].reshape(-1, 2)
    row = torch.tensor([0x10, 0x32, 0x54, 0x76, 0x98, 0xBA, 0xDC, 0xFE], dtype=torch.uint8).repeat(2)
    packed = row.repeat(s.shape[0], 1)
    gst = None if gs is None else torch.tensor([gs], dtype=torch.float32)
    want = udq_want(packed, s, 16, gst, odt)
    udq_three_ways(packed, s, None, N.DT[odt], odt, 16, gst, want, f"float scales gs {gs} -> {odt}")
    print(f"{want.numel()} elements x 3 ways")


def test_unpack_fp4_from_uint8_every_byte():
    for odt in (torch.bfloat16, torch.float16, torch.float32):
        same(ops.unpack_fp4_from_uint8(PACKED.to(DEV), 256, 512, odt).cpu(), oracle.unpack_fp4_from_uint8(PACKED, 256, 512, odt), f"{odt}")


# ---------------------------------------------------------------------------------------------------------------------------------
# observers on every max |x|
# ---------------------------------------------------------------------------------------------------------------------------------
OBSERVER_GLOBAL_SCALES = [1.0, GS_384, 2.0 ** 40, 2.0 ** 60, f32_next(2.0 ** 60, np.inf), 2.0 ** -60, f32_next(2.0 ** -60, 0)]
T_TIES = [0.0, 0.25, 0.75, 1.25, 1.75, 2.5, 3.5, 5.0, -0.25, -0.75, -1.25, -1.75, -2.5, -3.5, -5.0]


def observer_input(dt, group):
    """group g: max |x| = the g-th positive finite pattern (then 0 and +inf), negated for every third group; the other elements
    RN(amax * t / 6) for t on the E2M1 ties, so that the quotients fall on or next to them"""
    bits = np.concatenate([np.arange(1, 0x7F80 if dt == "bf16" else 0x7C00), [0, 0x7F80 if dt == "bf16" else 0x7C00]]).astype(np.uint16)
    if bits.size % 4:
        bits = np.concatenate([bits, np.zeros(4 - bits.size % 4, dtype=np.uint16)])
    amax = torch.from_numpy(bits.view(np.int16)).view(TD[dt])
    t = torch.tensor((T_TIES * 3)[: group - 1], dtype=torch.float64) / 6.0
    rest = (amax.double()[:, None] * t[None, :]).to(TD[dt])
    rest = torch.where(amax[:, None].isinf(), torch.zeros_like(rest), rest)
    sign = torch.where(torch.arange(amax.numel()) % 3 == 2, -1.0, 1.0).to(TD[dt])
    x = torch.cat([(amax * sign)[:, None], rest], 1)
    return x.reshape(-1, 64), bits


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
@pytest.mark.parametrize("gs", OBSERVER_GLOBAL_SCALES + [-GS_384], ids=lambda g: f"{g:.9g}")
def test_nvfp4_observer_every_group_max(dt, gs):
    """ct_observe_quantize_pack_nvfp4 with an explicit global scale: one group per max |x| (crossing 2^-40 and 2^14 by construction),
    scale bytes against the golden's calculate_qparams (or the model where the golden has no such global scale), codes against the
    oracle given the returned scale.  A negative global scale gives negative effective scales, which must take the slow unit (x = +0.0
    stays +0.0)"""
    x, bits = observer_input(dt, 16)
    gst = torch.tensor([gs], dtype=torch.float32)
    packed, scale, gs_out = ops.observe_quantize_pack_nvfp4(x.to(DEV), NV, global_scale=gst.to(DEV))
    same(gs_out.cpu(), gst, "global scale")
    got = scale.cpu().view(torch.uint8).reshape(-1)
    want = torch.from_numpy(M.nvfp4_scale_code(M.bits_to_float(bits, dt), gs, dt))
    gold = [c for c in G if c["kind"] == "nvfp4_qparams" and c["dtype"] == dt and c["sided"] == "one" and c["global_scale"] == gs]
    if gold:
        same(want[: gold[0]["scale"].numel()], gold[0]["scale"], "model vs golden")
    same(got, want, "fp8 group scales")
    s = scale.cpu().float().reshape(x.shape[0], -1)
    same_codes(packed, nv_want(x, s, None, gst), "nibbles vs oracle")
    print(f"{x.numel()} elements, {got.numel()} groups")


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
@pytest.mark.parametrize("bits", [4, 8])
def test_mx_observer_every_group_max(dt, bits):
    """ct_observe_quantize_mx (MXFP4, MXFP8): one group of 32 per max |x|; E8M0 bytes against compress_mx_scale of the golden's
    calculate_qparams scale (MXFP4) or of the model's (MXFP8), codes against the oracle given that scale"""
    x, b = observer_input(dt, 32)
    args = mx_args(bits=bits, scale_dtype=torch.uint8)
    q, code = ops.observe_quantize_mx(x.to(DEV), args)
    s_t = torch.from_numpy(M.mx_scale(b, dt, bits)).to(TD[dt])
    if bits == 4:
        (gold,) = [c for c in G if c["kind"] == "mxfp4_qparams" and c["dtype"] == dt and c["sided"] == "one"]
        same(s_t[: gold["scale"].numel()], gold["scale"], "model vs golden")
    same(code.cpu().reshape(-1), oracle.compress_mx_scale(s_t), "E8M0 scale bytes")
    s = s_t.reshape(x.shape[0], -1)
    if bits == 4:
        same_codes(q, mx_want(x, s, None, 32), "nibbles vs oracle")
    else:
        want = oracle.quantize(x, s, None, strategy="group", group_size=32, num_bits=8, qtype="float", dtype=F8)
        k = ~oracle.quantize(x, s, None, strategy="group", group_size=32, num_bits=4, qtype="float").isnan()   # no code for NaN quotients
        same(q.cpu().view(torch.uint8)[k], want.view(torch.uint8)[k], "fp8 codes vs oracle")
    print(f"{x.numel()} elements, {code.numel()} groups")


def activation_args(preset):
    from compressed_tensors_b200.quantization import preset_name_to_scheme

    return preset_name_to_scheme(preset, ["Linear"]).input_activations


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
@pytest.mark.parametrize("preset,gs", [("NVFP4", g) for g in OBSERVER_GLOBAL_SCALES] + [("MXFP4", None)],
                         ids=lambda v: v if isinstance(v, str) else ("-" if v is None else f"{v:.9g}"))
def test_dynamic_fake_quantize_every_group_max(dt, preset, gs):
    """ct_dynamic_fake_quantize with the NVFP4 (group 16, float32 global scale) and MXFP4 (group 32, E8M0) activation args: one group
    per max |x|; scales against the model (and the golden's calculate_qparams where it has that global scale), the fake-quantized
    values against the oracle's fake_quantize given the returned scale and zero point, with NaN where the oracle puts it"""
    args = activation_args(preset)
    group = int(args.group_size)
    x, bits = observer_input(dt, group)
    gst = None if gs is None else torch.tensor([gs], dtype=torch.float32)
    n0 = N.launch_count()
    res = ops.dynamic_fake_quantize(x.to(DEV), args, global_scale=dev(gst))
    assert res is not None, N.last_error()
    assert N.launch_count() - n0 == 1
    out, scale, zp = (t.cpu() for t in res)
    if preset == "NVFP4":
        same(scale.to(F8).view(torch.uint8).reshape(-1), torch.from_numpy(M.nvfp4_scale_code(M.bits_to_float(bits, dt), gs, dt)), "scales vs model")
        assert bool((scale == scale.to(F8).float()).all()), "the float32 scale holds e4m3 values"
        gold = [c for c in G if c["kind"] == "nvfp4_qparams" and c["dtype"] == dt and c["sided"] == "one" and c["global_scale"] == gs]
        okw = dict(strategy="tensor_group", group_size=16, global_scale=gst)
    else:
        same(scale.reshape(-1), torch.from_numpy(M.mx_scale(bits, dt)).to(TD[dt]), "scales vs model")
        gold = [c for c in G if c["kind"] == "mxfp4_qparams" and c["dtype"] == dt and c["sided"] == "one"]
        okw = dict(strategy="group", group_size=32)
    if gold:
        n = gold[0]["scale"].numel()
        got = scale.to(F8).view(torch.uint8).reshape(-1)[:n] if preset == "NVFP4" else scale.reshape(-1)[:n]
        same(got, gold[0]["scale"], "scales vs golden")
    want = oracle.fake_quantize(x, scale, zp, num_bits=4, qtype="float", **okw)
    same_nan(out, want, "fake-quantized values vs oracle")
    print(f"{x.numel()} elements, {scale.numel()} groups")


# ---------------------------------------------------------------------------------------------------------------------------------
# host-resident tensors and the scale encodings
# ---------------------------------------------------------------------------------------------------------------------------------
def test_host_resident_fp4_ops():
    """ct_host_run_many (ops.host_batched, CPU tensors) for OP_QUANTIZE_PACK_FP4 and OP_UNPACK_DEQUANTIZE_FP4 on every pattern"""
    bytes_ = first_finite_e4m3_bytes(8)
    svals = M.e4m3_decode(np.array(bytes_)).tolist()
    x = patterns("bf16", len(bytes_))
    gst = torch.tensor([GS_384], dtype=torch.float32)
    s = per_block(svals, 1024, 4, torch.float32)
    pr, out, keep = qpack_problem(x, s, None, NV, gst, x)
    ops.host_batched(N.OP_QUANTIZE_PACK_FP4, [pr])
    same_codes(out, nv_want(x, s, None, gst), "host quantize_pack_fp4")
    stored = ROWS[:, None].repeat(1, 32).view(F8)
    pr, out, keep = udq_problem(PACKED, stored, N.DT[F8], torch.bfloat16, 16, gst, PACKED)
    ops.host_batched(N.OP_UNPACK_DEQUANTIZE_FP4, [pr])
    same_nan(out, udq_want(PACKED, stored.to(torch.bfloat16), 16, gst, torch.bfloat16), "host unpack_dequantize_fp4")


@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_mx_scale_codes_every_pattern(dt):
    """compress_mx_scale on all 65536 patterns and decompress_mx_scale on all 256 bytes, against the golden"""
    (c,) = [c for c in G if c["kind"] == "compress_mx_scale" and c["dtype"] == dt]
    x = patterns(dt).reshape(-1)
    same(ops.compress_mx_scale(x.to(DEV)).cpu(), c["code"], "compress_mx_scale")
    (d,) = [c for c in G if c["kind"] == "decompress_mx_scale"]
    same_nan(ops.decompress_mx_scale(ROWS.to(DEV)).cpu(), d["value"], "decompress_mx_scale")
