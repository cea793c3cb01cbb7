"""
Every bf16 / fp16 bit pattern, under a ladder of scales and zero points, through the integer and FP8 kernels, bit for bit against
the float64 model of tests/int_fp8_model.py (which tests/test_int_sweep_host.py proves equal to the reference's own outputs and to the
CPU oracle), evaluated on the device, and against the oracle on a sample of rows.  Codes made from NaN quotients are undefined in
the reference and not compared; fake-quantized and dequantized NaNs must sit where the model puts them.

Row r of an input holds all 65536 patterns of its dtype under one (scale, zero point).  The ladder: every binade of the scale dtype
(subnormals included) at two mantissas, every mantissa at three binades, the neighbours of 2^-100 and 2^100 where the kernels switch
from a reciprocal to IEEE division, +-0, infinities and negative scales; zero points cycle through every value of the code width, so
each meets a subset of the scales.  float32 inputs hold each code's half-way quotients and one ulp either side times the row's scale,
at every binade.  Scales are GROUP scales of group 8, 16 or 32 (one value per row), which caps the thread unit at 1, 2 or 4 chunks
(dispatch.cu plan_one's max_unit), or CHANNEL scales.

Each encode and decode runs three ways: fast (aligned), generic (a view 2 bytes past an aligned allocation) and batched (both in one
ops.batched call, which must make exactly 2 launches: one streaming, one generic).

Streaming leaves (fast_quant.cu, fast_pack.cu, fast_fake.cu) and the tests that reach them:
  QuantizeOp<P, KIND, ZP, 2>          test_quantize (16-bit dtypes, group >= 16), test_quantize_every_scale_pattern
  QuantizeOp<P, KIND, ZP, 1>          test_quantize (group 8, and every float32 input)
  DequantF32ScaleOp<P>                test_dequantize_fp8_with_f32_scales
  DequantizeOp<P, QF8, 0>             test_dequantize
  DequantizeOp<P, QF8, 1>             test_dequantize
  DequantizeOp<P, QF8, 2>             test_dequantize
  DequantizeOp<P, QI_WIDE, 0>         test_dequantize
  DequantizeOp<P, QI_WIDE, 1>         test_dequantize
  QuantPackOp<P, BITS, ZP, GMAX>      test_quantize_pack (group 32 for 4 bits, >= 16 for 8 bits)
  QuantPackOp<P, BITS, ZP, 1>         test_quantize_pack (group 8, and every float32 input)
  UnpackDequantOp<P, 4, 0>            test_unpack_dequantize
  UnpackDequantOp<P, 4, 1>            test_unpack_dequantize
  UnpackDequantOp<P, 8, 0>            test_unpack_dequantize
  UnpackDequantOp<P, 8, 1>            test_unpack_dequantize
  PackOp<4>                           test_pack_and_unpack_every_code
  PackOp<8>                           test_pack_and_unpack_every_code
  UnpackOp<4>                         test_pack_and_unpack_every_code
  UnpackOp<8>                         test_pack_and_unpack_every_code
  FakeQuantOp<P, QF8, 0>              test_fake_quantize
  FakeQuantOp<P, QF8, 1>              test_fake_quantize
  FakeQuantOp<P, QF8, 2>              test_fake_quantize, test_fake_quantize_heads
  FakeQuantOp<P, QI_WIDE, 0>          test_fake_quantize (bf16 8-bit codes, float32; fp16 has no code wider than its magic)
  FakeQuantOp<P, QI_WIDE, 1>          test_fake_quantize
  FakeQuantOp<P, QI_NARROW, 0>        test_fake_quantize (2-7 bits in bf16, 2-8 in fp16), test_fake_quantize_heads
  FakeQuantOp<P, QI_NARROW, 1>        test_fake_quantize
Also: ct_host_run_many (ops.host_batched, CPU tensors) in test_host_resident_ops.
"""
import os
import re

import numpy as np
import pytest
import torch

import oracle
from compressed_tensors_b200 import _native as N
from compressed_tensors_b200 import ops
from tests import int_fp8_model as M
from tests.util import same, same_nan

pytestmark = pytest.mark.gpu
DEV = "cuda"
F8 = torch.float8_e4m3fn
TD = {"bf16": torch.bfloat16, "fp16": torch.float16, "f32": torch.float32}
MANT = {"bf16": 7, "fp16": 10, "f32": 23}
EMIN = {"bf16": -133, "fp16": -24, "f32": -149}                 # smallest subnormal 2^EMIN
EMAX = {"bf16": 127, "fp16": 15, "f32": 127}
CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "compressed_tensors_b200", "csrc")


class Args:
    def __init__(self, kind, bits, zp, strategy="group", group_size=32):
        self.strategy, self.group_size, self.block_structure = strategy, group_size, None
        self.num_bits, self.type, self.symmetric = bits, "float" if kind == "fp8" else "int", zp is None


# ---------------------------------------------------------------------------------------------------------------------------------
# the ladder and the model on the device
# ---------------------------------------------------------------------------------------------------------------------------------
def ladder(dt):
    """scale values of dtype dt (float64 list, each exact in dt)"""
    m = MANT[dt]
    second = 1.0 + (0b1010101 << (m - 7)) / 2.0 ** m                # a mantissa with bits set all along
    out = []
    for e in range(EMIN[dt], EMAX[dt] + 1):
        for mant in (1.0, second):
            v = float(M.rn(np.ldexp(mant, e), dt))
            if v != 0 and np.isfinite(v):
                out.append(v)
    for e in (-8, 0, 5):
        out += [np.ldexp(1.0 + k / 2.0 ** m, e) for k in range(2 ** min(m, 10))][:: (1 if m <= 10 else 1)]
    if dt != "fp16":
        ulp = 2.0 ** -(m + 1)
        for e in (-100, 100):
            out += [np.ldexp(1.0 - ulp, e), np.ldexp(1.0, e), np.ldexp(1.0 + 2 * ulp, e)]
    out += [0.0, -0.0, float("inf"), -float("inf"), -1.0, -0.3, -(2.0 ** EMIN[dt]), -float(M.rn(0.01, dt))]
    return [float(M.rn(v, dt)) for v in out]


def zero_points(kind, bits, zp_kind, n):
    """n zero points cycling through every value of the width: int8 values in [qmin, qmax], or every finite e4m3 byte"""
    if zp_kind is None:
        return None
    if zp_kind == "fp8":
        b = np.array([i for i in range(256) if (i & 0x7F) != 0x7F])
        return torch.from_numpy(b[np.arange(n) % b.size].astype(np.uint8)).view(F8)
    lo, hi = (-128, 127) if kind == "fp8" else (-(1 << (bits - 1)), (1 << (bits - 1)) - 1)
    v = np.arange(lo, hi + 1)
    return torch.from_numpy(v[(np.arange(n) * 7) % v.size].astype(np.int8))


def rnd(v, tdt):
    """one ATen op in tdt on float64 device values (M.op): float32 first, then tdt"""
    return v.float().to(tdt).double()


def model_rounded(x, s, zp, kind, bits):
    """M.quantize on the device: x [R, C] of dtype T, s / zp [R] -> the rounded values (float64), NaN where the reference has NaN"""
    tdt = x.dtype
    t = rnd(x.double() / s.double()[:, None], tdt)
    if zp is not None:
        t = rnd(t + zp.double()[:, None], tdt)
    lo, hi = M.q_range(kind, bits)
    t = torch.clamp(t, lo, hi)
    return t.to(F8).double() if kind == "fp8" else torch.round(t)


def model_dequant(r, s, zp, tdt):
    """M.dequantize on the device: r [R, C] code values, s / zp [R] -> values of dtype tdt"""
    v = rnd(r, tdt)
    if zp is not None:
        v = rnd(v - zp.double()[:, None], tdt)
    return (v * s.double()[:, None]).float().to(tdt)


def check_model_sample(x, s, zp, kind, bits, rounded, fake=None):
    """the device formulas above against the numpy model on every 97th row"""
    tdt = {torch.bfloat16: "bf16", torch.float16: "fp16", torch.float32: "f32"}[x.dtype]
    for r in range(0, x.shape[0], 97):
        xr = x[r].cpu().double().numpy()
        z = None if zp is None else float(zp[r].double())
        want = M.quantize(xr, float(s[r].double()), tdt, kind, bits, z)
        got = rounded[r].cpu().numpy()
        ok = (np.isnan(got) & np.isnan(want)) | ((got == want) & (np.signbit(got) == np.signbit(want)))
        assert ok.all(), f"device model row {r}"
        if fake is not None:
            wf = M.fake_quantize(xr, float(s[r].double()), tdt, kind, bits, z)
            gf = fake[r].cpu().double().numpy()
            ok = (np.isnan(gf) & np.isnan(wf)) | ((gf == wf) & (np.signbit(gf) == np.signbit(wf)))
            assert ok.all(), f"device model fake row {r}"


def inputs(dt, kind, bits, zp_kind):
    """(x [R, C], per-row scales [R], per-row zero points [R] or None), on the device"""
    s = torch.tensor(ladder(dt), dtype=torch.float64).to(TD[dt])
    if dt == "f32":
        lo, hi = M.q_range(kind, bits)
        if kind == "int":
            ties = [k + 0.5 for k in range(int(lo) - 1, int(hi) + 1)]
        else:
            g = M.e4m3_decode(np.arange(127))
            ties = ((g[:-1] + g[1:]) / 2).tolist() + [448.0, 464.0, 480.0]
            ties += [-t for t in ties]
        t32 = np.array(ties, dtype=np.float32)
        q = np.concatenate([t32, np.nextafter(t32, np.float32(-np.inf)), np.nextafter(t32, np.float32(np.inf)), [0.0, -0.0, np.nan]])
        q = np.concatenate([q, np.zeros((-q.size) % 64)]).astype(np.float32)
        x = (torch.from_numpy(q).double().to(DEV)[None, :] * s.double().to(DEV)[:, None]).float()
    else:
        x = torch.arange(65536, dtype=torch.int32, device=DEV).to(torch.int16).view(TD[dt])[None, :].expand(s.numel(), -1).contiguous()
    zp = zero_points(kind, bits, zp_kind, s.numel())
    return x, s.to(DEV), (zp.to(DEV) if zp is not None else None)


def scale_tensor(s, cols, group):
    return s[:, None].expand(-1, cols // group).contiguous() if group else s[:, None].contiguous()


def zp_tensor(zp, cols, group):
    return None if zp is None else scale_tensor(zp, cols, group)


def args_for(kind, bits, zp, group):
    return Args(kind, bits, zp, "group" if group else "channel", group)


def offset_view(t):
    """t copied into a view 2 bytes past an aligned allocation"""
    k = max(1, 2 // t.element_size())
    base = torch.empty(t.numel() + k, dtype=t.dtype, device=DEV)
    v = base[k:k + t.numel()].view(t.shape)
    v.copy_(t)
    return v


def three_ways(recipe, src, rest, check, what):
    """recipe(src, *rest) -> ops._*_call: run it on the aligned source, on an offset copy, and both in one ops.batched call"""
    srco = offset_view(src)
    for name, s_ in (("fast", src), ("generic", srco)):
        check(ops._run(recipe(s_, *rest)), f"{what} {name}")
    calls = [recipe(src, *rest), recipe(srco, *rest)]
    outs = [torch.empty(c.out_shape, dtype=c.out_dtype, device=DEV) for c in calls]
    n0 = N.launch_count()
    ops.batched(calls[0].op, [(c.desc, c.src, c.p.scale, c.p.zp, o) for c, o in zip(calls, outs)])
    assert N.launch_count() - n0 == 2, "one streaming launch and one generic launch"
    torch.cuda.synchronize()
    for o, name in zip(outs, ("batched fast entry", "batched generic entry")):
        check(o, f"{what} {name}")


def code_checker(rounded, kind):
    keep = ~rounded.isnan()
    want = torch.nan_to_num(rounded, nan=0.0).to(F8).view(torch.uint8) if kind == "fp8" else torch.nan_to_num(rounded, nan=0.0).to(torch.int8)

    def check(got, what):
        g = got.reshape(want.shape)
        g = g.view(torch.uint8) if g.dtype == F8 else g
        bad = int(((g != want) & keep).sum())
        assert bad == 0, f"{what}: {bad} of {int(keep.sum())} codes differ"
    return check


def oracle_rows(x, s, zp, kind, bits, fn="quantize"):
    """the oracle on every 61st row (CHANNEL scales), on the CPU"""
    rows = torch.arange(0, x.shape[0], 61, device=x.device)
    xs, ss = x[rows].cpu(), s[rows].cpu()[:, None]
    zs = None if zp is None else zp[rows].cpu()[:, None]
    kw = dict(strategy="channel", num_bits=bits, qtype="float" if kind == "fp8" else "int")
    if fn == "quantize":
        return rows, oracle.quantize(xs, ss, zs, dtype=F8 if kind == "fp8" else torch.int8, **kw)
    return rows, oracle.fake_quantize(xs, ss, zs, **kw)


GROUPS = [8, 16, 32, None]


# ---------------------------------------------------------------------------------------------------------------------------------
# encode
# ---------------------------------------------------------------------------------------------------------------------------------
QUANT_CFGS = [("int", 8, None), ("int", 8, "int8"), ("int", 4, None), ("int", 4, "int8"), ("fp8", 8, None), ("fp8", 8, "int8"),
              ("fp8", 8, "fp8")]


@pytest.mark.parametrize("group", GROUPS, ids=lambda g: f"g{g}" if g else "channel")
@pytest.mark.parametrize("cfg", QUANT_CFGS, ids=lambda c: f"{c[0]}{c[1]}-zp{c[2]}")
@pytest.mark.parametrize("dt", ["bf16", "fp16", "f32"])
def test_quantize(dt, cfg, group):
    """QuantizeOp (int8 / e4m3 codes): every pattern under every scale of the ladder"""
    kind, bits, zpk = cfg
    x, s, zp = inputs(dt, kind, bits, zpk)
    rounded = model_rounded(x, s, zp, kind, bits)
    check_model_sample(x, s, zp, kind, bits, rounded)
    rows, want = oracle_rows(x, s, zp, kind, bits)
    code_checker(rounded[rows].cpu(), kind)(want, "oracle vs model")
    C = x.shape[1]
    sc, zt = scale_tensor(s, C, group), zp_tensor(zp, C, group)
    a = args_for(kind, bits, zpk, group)
    q_dt = F8 if kind == "fp8" else torch.int8
    three_ways(lambda src: ops._quantize_call(src, sc, zt, a, dtype=q_dt), x, (), code_checker(rounded, kind), f"quantize {dt} {cfg}")
    print(f"{x.numel()} elements, {x.shape[0]} scales x 3 ways")


@pytest.mark.parametrize("cfg", [("int", 8, None), ("fp8", 8, None), ("fp8", 8, "fp8")], ids=lambda c: f"{c[0]}{c[1]}-zp{c[2]}")
@pytest.mark.parametrize("dt", ["bf16", "fp16"])
def test_quantize_every_scale_pattern(dt, cfg):
    """QuantizeOp on all 2^32 (x, scale) pattern pairs of dt (every finite non-zero scale, CHANNEL scales, aligned): the quotient is
    the one rounding that depends on the scale's every bit, and the fast path forms it from a reciprocal (refined by one residual FMA
    step in fp16), so only the whole square shows that every quotient landing on a code's tie rounds like IEEE division.  int8 codes
    hold every half-integer tie of every integer width; e4m3 codes every e4m3 midpoint, and with e4m3 zero points their shifts"""
    kind, bits, zpk = cfg
    s_all = torch.arange(65536, dtype=torch.int32, device=DEV).to(torch.int16).view(TD[dt])
    s_all = s_all[s_all.isfinite() & (s_all != 0)]
    zp_all = zero_points(kind, bits, zpk, s_all.numel())
    zp_all = zp_all.to(DEV) if zp_all is not None else None
    rows = 1024
    x = torch.arange(65536, dtype=torch.int32, device=DEV).to(torch.int16).view(TD[dt])[None, :].expand(rows, -1).contiguous()
    q_dt = F8 if kind == "fp8" else torch.int8
    a = Args(kind, bits, zpk, "channel", None)
    for i in range(0, s_all.numel(), rows):
        s = s_all[i:i + rows]
        zp = None if zp_all is None else zp_all[i:i + rows]
        xs = x[: s.numel()]
        got = ops.quantize(xs, s[:, None].contiguous(), None if zp is None else zp[:, None].contiguous(), a, dtype=q_dt)
        code_checker(model_rounded(xs, s, zp, kind, bits), kind)(got, f"quantize {dt} {cfg} scales {i}..{i + s.numel()}")
    print(f"{65536 * s_all.numel()} pairs")


def pack_checker(rounded, bits):
    """expected int32 words of the codes, and a mask of the bits that hold a code made from a NaN quotient"""
    nan = rounded.isnan()
    u = (torch.nan_to_num(rounded, nan=0.0).long() + (1 << (bits - 1))) & ((1 << bits) - 1)
    per = 32 // bits
    R, C = u.shape
    shift = (torch.arange(per, device=DEV) * bits)[None, None, :]
    want = (u.reshape(R, C // per, per) << shift).sum(-1)
    mask = ((~nan).long().reshape(R, C // per, per) * (((1 << bits) - 1) << shift)).sum(-1)
    want, mask = want.to(torch.int64), mask.to(torch.int64)

    def check(got, what):
        g = got.reshape(R, -1).long() & 0xFFFFFFFF
        bad = int((((g ^ want) & mask) != 0).sum())
        assert bad == 0, f"{what}: {bad} words differ"
    return check


@pytest.mark.parametrize("group", GROUPS, ids=lambda g: f"g{g}" if g else "channel")
@pytest.mark.parametrize("bits,zpk", [(4, None), (4, "int8"), (8, None), (8, "int8")])
@pytest.mark.parametrize("dt", ["bf16", "fp16", "f32"])
def test_quantize_pack(dt, bits, zpk, group):
    """QuantPackOp (the W4A16 / W8A16 quantize + pack): every pattern under every scale, words against the model's codes packed"""
    x, s, zp = inputs(dt, "int", bits, zpk)
    rounded = model_rounded(x, s, zp, "int", bits)
    C = x.shape[1]
    rows = torch.arange(0, x.shape[0], 61, device=DEV)
    want_o = oracle.pack_to_int32(oracle.quantize(x[rows].cpu(), s[rows].cpu()[:, None], None if zp is None else zp[rows].cpu()[:, None],
                                                  strategy="channel", num_bits=bits, dtype=torch.int8), bits)
    pack_checker(rounded[rows], bits)(want_o.to(DEV), "oracle vs model")
    sc, zt = scale_tensor(s, C, group), zp_tensor(zp, C, group)
    a = args_for("int", bits, zpk, group)
    three_ways(lambda src: ops._quantize_pack_call(src, sc, zt, a), x, (), pack_checker(rounded, bits), f"quantize_pack {dt} {bits} {zpk}")
    print(f"{x.numel()} elements, {x.shape[0]} scales x 3 ways")


FAKE_CFGS = [("int", b, z) for b in range(2, 9) for z in (None, "int8")] + [("fp8", 8, None), ("fp8", 8, "int8"), ("fp8", 8, "fp8")]


@pytest.mark.parametrize("cfg", FAKE_CFGS, ids=lambda c: f"{c[0]}{c[1]}-zp{c[2]}")
@pytest.mark.parametrize("dt", ["bf16", "fp16", "f32"])
def test_fake_quantize(dt, cfg):
    """FakeQuantOp (QI_NARROW in T up to the magic's width, QI_WIDE above it and in float32, QF8): every pattern, every scale"""
    kind, bits, zpk = cfg
    x, s, zp = inputs(dt, kind, bits, zpk)
    rounded = model_rounded(x, s, zp, kind, bits)
    want = model_dequant(rounded, s, zp, x.dtype)
    check_model_sample(x, s, zp, kind, bits, rounded, want)
    rows, wo = oracle_rows(x, s, zp, kind, bits, "fake")
    same_nan(want[rows].cpu(), wo, "oracle vs model")
    group = 16 if dt != "f32" else None
    sc, zt = scale_tensor(s, x.shape[1], group), zp_tensor(zp, x.shape[1], group)
    a = args_for(kind, bits, zpk, group)
    three_ways(lambda src: ops._fake_quantize_call(src, sc, zt, a), x, (), lambda got, what: same_nan(got, want, what),
               f"fake_quantize {dt} {cfg}")
    print(f"{x.numel()} elements, {x.shape[0]} scales x 3 ways")


def test_fake_quantize_heads():
    """ct_fake_quantize_heads: one ATTN_HEAD scale per head from the bf16 ladder, NARROW int4 and QF8 with an fp8 zero point"""
    s = torch.tensor(ladder("bf16"), dtype=torch.float64).to(torch.bfloat16)
    H = s.numel()
    x = torch.arange(65536, dtype=torch.int32).to(torch.int16).view(torch.bfloat16).reshape(1, 1, 256, 256).expand(1, H, 256, 256)
    xd = x.to(DEV).transpose(1, 2).contiguous().transpose(1, 2)      # [B, H, S, D] as a transposed view, the way attention hands it over
    for kind, bits, zpk in (("int", 4, None), ("fp8", 8, "fp8")):
        zp = zero_points(kind, bits, zpk, H)
        a = Args(kind, bits, zpk, "attn_head", None)
        sd, zd = s.to(DEV).reshape(H, 1, 1), None if zp is None else zp.to(DEV).reshape(H, 1, 1)
        (got,) = ops.fake_quantize_heads([xd], [sd], [zd], a)
        flat = x.reshape(H, 65536).to(DEV)
        zr = None if zp is None else zp.to(DEV)
        want = model_dequant(model_rounded(flat, s.to(DEV), zr, kind, bits), s.to(DEV), zr, torch.bfloat16)
        same_nan(got.reshape(H, 65536), want, f"heads {kind}{bits}")


# ---------------------------------------------------------------------------------------------------------------------------------
# decode
# ---------------------------------------------------------------------------------------------------------------------------------
def code_rows(kind, bits, R):
    """R rows of every code of the width (int8 values or e4m3 bytes), 256 columns; and their values as float64"""
    if kind == "fp8":
        b = torch.arange(256, dtype=torch.int32, device=DEV).to(torch.uint8)[None, :].expand(R, -1).contiguous()
        return b.view(F8), torch.from_numpy(M.e4m3_decode(np.arange(256))).to(DEV)[None, :].expand(R, -1)
    lo = -(1 << (bits - 1))
    v = (torch.arange(256, device=DEV) % (1 << bits) + lo)[None, :].expand(R, -1)
    return v.to(torch.int8).contiguous(), v.double()


@pytest.mark.parametrize("cfg", [("int", None), ("int", "int8"), ("fp8", None), ("fp8", "int8"), ("fp8", "fp8")], ids=lambda c: f"{c[0]}-zp{c[1]}")
@pytest.mark.parametrize("dt", ["bf16", "fp16", "f32"])
def test_dequantize(dt, cfg):
    """DequantizeOp: every int8 code / every e4m3 byte under every scale of the ladder and every zero point"""
    kind, zpk = cfg
    s = torch.tensor(ladder(dt), dtype=torch.float64).to(TD[dt]).to(DEV)
    R = s.numel()
    q, qv = code_rows(kind, 8, R)
    zp = zero_points(kind, 8, zpk, R)
    zp = zp.to(DEV) if zp is not None else None
    want = model_dequant(qv, s, zp, TD[dt])
    rows = torch.arange(0, R, 61, device=DEV)
    same_nan(oracle.dequantize(q[rows].cpu(), s[rows].cpu()[:, None], None if zp is None else zp[rows].cpu()[:, None]), want[rows].cpu(),
             "oracle vs model")
    sc, zt = s[:, None].contiguous(), None if zp is None else zp[:, None].contiguous()
    three_ways(lambda src: ops._dequantize_call(src, sc, zt), q, (), lambda got, what: same_nan(got, want, what), f"dequantize {dt} {cfg}")


@pytest.mark.parametrize("odt", ["bf16", "fp16"])
def test_dequantize_fp8_with_f32_scales(odt):
    """DequantF32ScaleOp: (q.to(float32) * scale).to(T) for every e4m3 byte under every float32 binade at two mantissas"""
    s = torch.tensor(ladder("f32"), dtype=torch.float32).to(DEV)
    R = s.numel()
    q, qv = code_rows("fp8", 8, R)
    want = (qv * s.double()[:, None]).float().to(TD[odt])
    a = Args("fp8", 8, None, "group", 128)
    sc = s[:, None].expand(-1, 2).contiguous()
    three_ways(lambda src: ops._dequantize_call(src, sc, None, a, dtype=TD[odt]), q, (), lambda got, what: same_nan(got, want, what),
               f"dequantize fp8 f32 scales -> {odt}")


@pytest.mark.parametrize("bits,zpk", [(4, None), (4, "int8"), (8, None), (8, "int8")])
@pytest.mark.parametrize("dt", ["bf16", "fp16", "f32"])
def test_unpack_dequantize(dt, bits, zpk):
    """UnpackDequantOp: every code of the width, packed, under every scale of the ladder and every zero point"""
    s = torch.tensor(ladder(dt), dtype=torch.float64).to(TD[dt]).to(DEV)
    R = s.numel()
    q, qv = code_rows("int", bits, R)
    packed = torch.from_numpy(M.pack_int32(q.cpu().numpy(), bits)).to(DEV)
    zp = zero_points("int", bits, zpk, R)
    zp = zp.to(DEV) if zp is not None else None
    want = model_dequant(qv, s, zp, TD[dt])
    sc, zt = s[:, None].contiguous(), None if zp is None else zp[:, None].contiguous()
    three_ways(lambda src: ops._unpack_dequantize_call(src, sc, zt, bits, q.shape), packed, (), lambda got, what: same_nan(got, want, what),
               f"unpack_dequantize {dt} {bits} {zpk}")


def test_pack_and_unpack_every_code():
    """PackOp / UnpackOp: every code of 4 and 8 bits at every position of a word, against the model's bit stream"""
    for bits in (4, 8):
        v = torch.arange(4096, dtype=torch.int32) % (1 << bits) - (1 << (bits - 1))
        v = v.reshape(16, 256).to(torch.int8)
        want = torch.from_numpy(M.pack_int32(v.numpy(), bits))
        same(ops.pack_to_int32(v.to(DEV), bits).cpu(), want, f"pack {bits}")
        same(ops.unpack_from_int32(want.to(DEV), bits, v.shape).cpu(), v, f"unpack {bits}")


def test_host_resident_ops():
    """ct_host_run_many (ops.host_batched, CPU tensors) for quantize + pack and unpack + dequantize on every bf16 pattern"""
    x, s, zp = inputs("bf16", "int", 4, "int8")
    x, s, zp = x[::8].cpu(), s[::8].cpu(), zp[::8].cpu()
    rounded = model_rounded(x.to(DEV), s.to(DEV), zp.to(DEV), "int", 4)
    c = ops._quantize_pack_call(x, s[:, None].contiguous(), zp[:, None].contiguous(), args_for("int", 4, "int8", None))
    out = torch.empty(c.out_shape, dtype=c.out_dtype)
    ops.host_batched(c.op, [(c.desc, c.src, c.p.scale, c.p.zp, out)])
    pack_checker(rounded, 4)(out.to(DEV), "host quantize_pack")
    q, qv = code_rows("int", 4, s.numel())
    packed = torch.from_numpy(M.pack_int32(q.cpu().numpy(), 4))
    c = ops._unpack_dequantize_call(packed, s[:, None].contiguous(), zp[:, None].contiguous(), 4, q.shape)
    out = torch.empty(c.out_shape, dtype=c.out_dtype)
    ops.host_batched(c.op, [(c.desc, c.src, c.p.scale, c.p.zp, out)])
    same_nan(out.to(DEV), model_dequant(qv, s.to(DEV), zp.to(DEV), torch.bfloat16), "host unpack_dequantize")


# ---------------------------------------------------------------------------------------------------------------------------------
# the table above names every instantiation
# ---------------------------------------------------------------------------------------------------------------------------------
def test_every_instantiation_is_swept():
    doc = __doc__
    leaves = set()
    for f in ("fast_quant.cu", "fast_pack.cu", "fast_fake.cu"):
        with open(os.path.join(CSRC, f)) as fh:
            for m in re.finditer(r"stream_kernel<(\w+<[^<>]*>)>\(\)", fh.read()):
                leaves.add(re.sub(r"\s+", " ", m.group(1)))
    assert len(leaves) >= 20
    missing = sorted(l for l in leaves if l not in doc)
    assert not missing, f"streaming leaves missing from the docstring's table: {missing}"
