#!/usr/bin/env python
"""
Golden vectors of the reference on NaN and infinite inputs and scales, by importing the reference exactly like make_golden.py does.

    python tests/golden/make_golden_nonfinite.py   ->  tests/golden/nonfinite.pt.gz

  static   fake_quantize (int4 symmetric, int8 with zero point 3, fp8, NVFP4 with a global scale) on bf16 / fp16 inputs holding every
           NaN and +-inf bit pattern, +-0, +-max-finite and the smallest subnormal, each at every lane 0..7 of a 16-byte chunk between
           finite values (fp32: +-inf, the canonical NaN and a few payloads); per-tensor scales 2^-7, 1, 37.5 and +inf; one per-channel
           and one per-group case with a NaN and an inf scale among finite ones
  dynamic  compute_dynamic_scales_and_zp + forward_quantize for the schemes of make_golden_dynamic.py on seeded randn with planted
           canonical NaN (lane 0, lane 7, last of a row, a whole row, the last group of the last row), +inf, -inf, both in one group,
           and fp32 values above 65504 cast to fp16; planted rows alternate with clean ones.  `zp_defined` is False where the reference
           cast a NaN zero point to int8 (an undefined value)
  heads    fake_quantize with ATTN_HEAD and TENSOR scales on [B, H, S, D] states holding NaN and +-inf
  qparams  calculate_qparams on amin / amax of weights with one NaN or inf in the tensor, a channel or a group, and generate_gparam
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as mg  # noqa: E402  (imports the reference from a temp copy)
import make_golden_dynamic as mgd  # noqa: E402

from compressed_tensors.quantization import QuantizationArgs, QuantizationStatus  # noqa: E402
from compressed_tensors.quantization.lifecycle.forward import fake_quantize, forward_quantize  # noqa: E402
from compressed_tensors.quantization.utils import calculate_qparams, compute_dynamic_scales_and_zp, generate_gparam  # noqa: E402

SEED = 20261017
NAN = float("nan")
INF = float("inf")
STATIC_SCALES = [2.0 ** -7, 1.0, 37.5, INF]
STATIC = {
    "int4": dict(num_bits=4, type="int", symmetric=True),
    "int8_zp3": dict(num_bits=8, type="int", symmetric=False),
    "fp8": dict(num_bits=8, type="float", symmetric=True),
    "nvfp4": dict(num_bits=4, type="float", symmetric=True, strategy="tensor_group", group_size=16),
}
NVFP4_GS = 4.0


def special_bits(dtype):
    """every NaN and +-inf pattern, +-0, +-max-finite and the smallest subnormal (fp32: +-inf and a few NaNs)"""
    if dtype == torch.float32:
        return torch.tensor([0x7F800000, 0xFF800000, 0x7FC00000, 0xFFC00000, 0x7FC00001, 0x7F800001, 0xFFFFFFFF, 0x7FFFFFFF],
                            dtype=torch.int64).to(torch.int32)
    mant = 7 if dtype == torch.bfloat16 else 10
    exp_all = ((1 << (15 - mant)) - 1) << mant
    nan_inf = [exp_all | m for m in range(1 << mant)]
    pats = nan_inf + [0x8000 | p for p in nan_inf] + [0x0000, 0x8000, exp_all - 1, 0x8000 | (exp_all - 1), 0x0001]
    return torch.tensor(pats, dtype=torch.int32).to(torch.int16)


def finite_filler(n, dtype, gen):
    """finite values on a quarter grid in [-10, 10]: few distinct outputs keep the fixture small"""
    return (torch.randint(-40, 41, (n,), generator=gen) * 0.25).to(dtype)


def static_input(dtype, gen):
    """pattern i sits at element 2i + k of stretch k (k = 0..7), finite values everywhere else: each pattern meets every lane"""
    pats = special_bits(dtype).view(dtype)
    parts = []
    for k in range(8):
        s = finite_filler(-(-(k + 2 * len(pats)) // 8) * 8, dtype, gen)   # whole chunks: every stretch starts at lane 0
        s[k::2][: len(pats)] = pats
        parts.append(s)
    x = torch.cat(parts)
    pad = (-x.numel()) % 64
    x = torch.cat([x, finite_filler(pad, dtype, gen)])
    return x.reshape(-1, 64)


def static_case(name, xs, scale, zp, strategy, gs=None):
    x = xs[-1]
    kw = dict(STATIC[name])
    kw.setdefault("strategy", strategy)
    if kw["strategy"] == "group":
        kw["group_size"] = 16
    args = QuantizationArgs(**kw)
    out = fake_quantize(x, scale, zp, args, global_scale=gs)
    return dict(scheme=name, args=kw, x=len(xs) - 1, scale=scale, zero_point=zp, global_scale=gs, out=out)


def gen_static(gen):
    xs, cases = [], []
    for dtype in (torch.bfloat16, torch.float16, torch.float32):
        xs.append(static_input(dtype, gen))
        x = xs[-1]
        rows, cols = x.shape
        for name in STATIC:
            if dtype == torch.float32 and name == "int4":
                continue   # fp32 takes int8 / fp8 through the streaming kernel and NVFP4 through the generic one
            for sv in STATIC_SCALES:
                if name == "nvfp4":
                    scale = torch.full((rows, cols // 16), sv, dtype=dtype)
                    cases.append(static_case(name, xs, scale, None, "tensor_group", torch.tensor([NVFP4_GS])))
                    continue
                scale = torch.tensor([sv], dtype=dtype)
                zp = torch.tensor([3], dtype=torch.int8) if name == "int8_zp3" else None
                cases.append(static_case(name, xs, scale, zp, "tensor"))
        if dtype == torch.float32:
            continue
        # one NaN and one inf scale among finite ones, per channel and per group, on the first 16 rows
        xs.append(x[:16].clone())
        rows = 16
        for name in ("int4", "int8_zp3", "fp8"):
            ch = (torch.rand(rows, 1, generator=gen) * 0.5 + 0.01).to(dtype)
            ch[1, 0], ch[4, 0] = NAN, INF
            zc = torch.full((rows, 1), 3, dtype=torch.int8) if name == "int8_zp3" else None
            cases.append(static_case(name, xs, ch, zc, "channel"))
            gr = (torch.rand(rows, cols // 16, generator=gen) * 0.5 + 0.01).to(dtype)
            gr[0, 1], gr[2, 3] = NAN, INF
            zg = torch.full((rows, cols // 16), 3, dtype=torch.int8) if name == "int8_zp3" else None
            cases.append(static_case(name, xs, gr, zg, "group"))
    return xs, cases


# ---------------------------------------------------------------------------------------------------------------------------------
# dynamic activations
# ---------------------------------------------------------------------------------------------------------------------------------
TOKEN_SHAPES = [(2, 8, 256), (2, 12, 2, 64), (16, 512)]
GROUP_SHAPES = [(2, 3, 4, 128), (13, 384)]
WIDE = (1, 1, 32768)   # one row: the tail NaN lands in it


def plant(x2):
    """planted rows 1, 3, 5, ... of the reduction-row view x2 (fp32); the last row gets a NaN in its last group"""
    cols = x2.shape[1]
    plants = [
        lambda r: r.__setitem__(0, NAN),                                  # lane 0
        lambda r: r.__setitem__(31, NAN),                                 # lane 7
        lambda r: r.__setitem__(cols - 1, NAN),                           # last of the row
        lambda r: r.__setitem__(5, INF),
        lambda r: r.__setitem__(12, -INF),
        lambda r: (r.__setitem__(17, INF), r.__setitem__(20, -INF)),      # one group (16 wide and up)
        lambda r: r.fill_(NAN),
        lambda r: (r.mul_(4e4), r.__setitem__(2, 7e4), r.__setitem__(3, -1e5)),   # fp16 overflow
    ]
    for k, p in enumerate(plants):
        r = 2 * k + 1
        if r >= x2.shape[0]:
            break
        p(x2[r])
    x2[-1, cols - 3] = NAN                                                # the tail


def dynamic_input(shape, dtype, token, gen):
    x = (torch.randn(shape, generator=gen) * 32).round() / 16   # a 1/16 grid keeps the fixture small
    x2 = x.view(shape[0] * shape[1], -1) if token and len(shape) > 2 else x.view(-1, shape[-1])
    plant(x2)
    x = x.to(dtype)
    # canonical NaN bits (bf16 0x7fc0, fp16 0x7e00), which the reference's MX scale depends on; fp32 -> bf16 casts can give 0xffff
    canon = torch.tensor(0x7FC0 if dtype == torch.bfloat16 else 0x7E00, dtype=torch.int16).view(dtype)
    return torch.where(x.isnan(), canon, x)


def zp_defined(x, args, zp):
    """False where the reference's zero point was NaN before its cast to int8"""
    if args.symmetric:
        return torch.ones(zp.shape, dtype=torch.bool)
    if args.strategy == "token":
        dims = tuple(range(2, x.ndim))
        mn, mx = (torch.aminmax(x) if not dims else (torch.amin(x, dim=dims, keepdim=True), torch.amax(x, dim=dims, keepdim=True)))
    else:
        mn, mx = torch.aminmax(x)
    mn, mx = torch.min(mn, torch.zeros_like(mn)), torch.max(mx, torch.zeros_like(mx))
    s = (mx - mn) / 255.0
    z = -128 - (mn / s)
    return (~z.isnan()).reshape(zp.shape)


def gen_dynamic(gen):
    inputs, cases, index = [], [], {}
    for name in mgd.PRESETS + list(mgd.CUSTOM):
        args = mgd.scheme_args(name)
        grouped = args.strategy in ("group", "tensor_group")
        shapes = (GROUP_SHAPES if grouped else TOKEN_SHAPES) + ([WIDE] if name in mgd.WIDE_SCHEMES else [])
        for dtype in (torch.bfloat16, torch.float16):
            for shape in shapes:
                key = (shape, dtype, not grouped)
                if key not in index:
                    index[key] = len(inputs)
                    inputs.append(dynamic_input(shape, dtype, not grouped, gen))
                i = index[key]
                x = inputs[i]
                gscales = [None]
                if name == "NVFP4":
                    fin = x.float()[x.float().isfinite()]
                    gscales = [torch.ones(1), generate_gparam(fin.amin(), fin.amax())]
                for gs in gscales:
                    module = torch.nn.Module()
                    module.quantization_status = QuantizationStatus.FROZEN
                    if gs is not None:
                        module.input_global_scale = gs
                    scale, zp = compute_dynamic_scales_and_zp(value=x, args=args, module=module, global_scale=gs)
                    out = forward_quantize(module, x, "input", args)
                    cases.append(dict(scheme=name, args=dict(mgd.CUSTOM.get(name, {})), input=i, global_scale=gs, scale=scale,
                                      zero_point=zp, zp_defined=zp_defined(x, args, zp), out=out))
    return inputs, cases


# ---------------------------------------------------------------------------------------------------------------------------------
# KV heads
# ---------------------------------------------------------------------------------------------------------------------------------
def gen_heads(gen):
    cases = []
    for dtype in (torch.bfloat16, torch.float16):
        x = (torch.randn(2, 4, 8, 64, generator=gen) * 2)
        x[0, 1, 3, 5], x[1, 2, 0, 0], x[1, 3, 7, 63], x[0, 0, 2, 9], x[0, 0, 2, 10] = NAN, INF, -INF, INF, -INF
        x = x.to(dtype)
        head = dict(num_bits=8, type="int", symmetric=False, strategy="attn_head")
        s = (torch.rand(4, 1, 1, generator=gen) * 0.05 + 0.01).to(dtype)
        z = torch.randint(-8, 8, (4, 1, 1), generator=gen).to(torch.int8)
        cases.append(dict(args=head, x=x, scale=s, zero_point=z, out=fake_quantize(x, s, z, QuantizationArgs(**head))))
        s2 = s.clone()
        s2[2] = NAN
        cases.append(dict(args=head, x=x, scale=s2, zero_point=z, out=fake_quantize(x, s2, z, QuantizationArgs(**head))))
        tensor = dict(num_bits=8, type="float", symmetric=True, strategy="tensor")
        st = torch.tensor([0.03], dtype=dtype)
        cases.append(dict(args=tensor, x=x, scale=st, zero_point=None, out=fake_quantize(x, st, None, QuantizationArgs(**tensor))))
    return cases


# ---------------------------------------------------------------------------------------------------------------------------------
# observer qparams
# ---------------------------------------------------------------------------------------------------------------------------------
QP_SCHEMES = {
    "int4_sym": dict(num_bits=4, type="int", symmetric=True),
    "int4_asym": dict(num_bits=4, type="int", symmetric=False),
    "int8_sym": dict(num_bits=8, type="int", symmetric=True),
    "int8_asym": dict(num_bits=8, type="int", symmetric=False),
    "fp8": dict(num_bits=8, type="float", symmetric=True),
}
PLANTS = {"nan": [(2, 5, NAN)], "inf": [(5, 130, INF)], "-inf": [(9, 7, -INF)], "inf_and_-inf": [(12, 200, INF), (12, 250, -INF)]}


def observe(w, strategy, group):
    if strategy == "tensor":
        return w.amin().reshape(1), w.amax().reshape(1)
    if strategy == "channel":
        return w.amin(dim=1, keepdim=True), w.amax(dim=1, keepdim=True)
    g = w.unflatten(-1, (w.shape[1] // group, group))
    return g.amin(dim=-1), g.amax(dim=-1)


def gen_qparams(gen):
    cases = []
    for dtype in (torch.bfloat16, torch.float16, torch.float32):
        for plant_name, spots in PLANTS.items():
            w = (torch.randn(16, 256, generator=gen) * 16).round() / 256
            for r, c, v in spots:
                w[r, c] = v
            w = w.to(dtype)
            gparam = generate_gparam(w.amin(), w.amax())
            for strategy in ("tensor", "channel", "group"):
                if dtype == torch.float32 and strategy != "tensor":
                    continue   # the fused channel and group observers take bf16 / fp16
                for name, kw in QP_SCHEMES.items():
                    if strategy == "group" and kw["type"] == "float":
                        continue
                    full = dict(kw, strategy=strategy, **({"group_size": 128} if strategy == "group" else {}))
                    args = QuantizationArgs(**full)
                    mn, mx = observe(w, strategy, 128)
                    scale, zp = calculate_qparams(mn, mx, args)
                    defined = torch.ones(zp.shape, dtype=torch.bool)
                    if not args.symmetric:
                        lo, hi = torch.min(mn, torch.zeros_like(mn)), torch.max(mx, torch.zeros_like(mx))
                        s = (hi - lo) / float(2 ** args.num_bits - 1)
                        defined = ~(-(2 ** (args.num_bits - 1)) - lo / s).isnan().reshape(zp.shape)
                    cases.append(dict(scheme=name, args=full, plant=plant_name, x=w, scale=scale, zero_point=zp, zp_defined=defined,
                                      gparam=gparam))
    return cases


def main():
    gen = torch.Generator().manual_seed(SEED)
    static_inputs, static = gen_static(gen)
    inputs, dynamic = gen_dynamic(gen)
    heads = gen_heads(gen)
    qparams = gen_qparams(gen)
    mg.save("nonfinite.pt", dict(static_inputs=static_inputs, static=static, inputs=inputs, dynamic=dynamic, heads=heads, qparams=qparams))


if __name__ == "__main__":
    main()
