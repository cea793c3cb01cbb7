"""
ops.fake_quantize_heads (ct_fake_quantize_heads: K / V / Q fake quantization in their strided [B, H, S, D] layout, one launch) against
ops.fake_quantize on contiguous copies and the oracle, and the KV-cache / attention golden cases (tests/golden/kv.pt.gz) on CUDA.
"""
import types
import zlib

import pytest
import torch

import oracle
from compressed_tensors_b200 import _native as N
from compressed_tensors_b200 import ops
from tests import golden
from tests.util import same

pytestmark = pytest.mark.gpu
DEV = "cuda"


def qargs(strategy, type_, bits, symmetric, dynamic=False):
    from compressed_tensors_b200.quantization import QuantizationArgs

    return QuantizationArgs(num_bits=bits, type=type_, symmetric=symmetric, strategy=strategy, dynamic=dynamic)


def hf_states(b, h, s, d, dtype, gen, layout):
    """key / value states as transformers hands them over: `hf` = [B, S, H, D] projections viewed as [B, H, S, D]"""
    if layout == "hf":
        x = torch.randn(b, s, h, d, generator=gen).transpose(1, 2)
    else:
        x = torch.randn(b, h, s, d, generator=gen)
    x = x * (torch.rand(1, h, 1, 1, generator=gen) * 4 + 0.1)
    return x.to(dtype).to(DEV)


def qparams(x, args):
    from compressed_tensors_b200.quantization.utils import calculate_qparams

    if args.strategy == "attn_head":
        h = x.shape[1]
        lo, hi = x.amin((0, 2, 3)).reshape(h, 1, 1), x.amax((0, 2, 3)).reshape(h, 1, 1)
    else:
        lo, hi = x.amin().reshape(1), x.amax().reshape(1)
    scale, zp = calculate_qparams(lo, hi, args)
    return scale.to(x.dtype), (zp if not args.symmetric else None)


def check_pair(xs, args, what="", sz=None):
    """fake_quantize_heads of xs against fake_quantize and the oracle, with the qparams `sz` ([(scale, zero point)], default: the
    observer's); returns the number of launches"""
    sz = sz or [qparams(x, args) for x in xs]
    scales, zps = [s for s, _ in sz], [z for _, z in sz]
    n0 = N.launch_count()
    got = ops.fake_quantize_heads(xs, scales, zps, args)
    launches = N.launch_count() - n0
    for i, (x, g) in enumerate(zip(xs, got)):
        assert g.shape == x.shape and g.stride() == x.stride() and g.dtype == x.dtype
        if x.numel() == 0:
            continue
        want = ops.fake_quantize(x.contiguous(), scales[i], zps[i], args)
        same(g, want, f"{what} tensor {i} vs fake_quantize: ")
        ref = oracle.fake_quantize(x.cpu(), scales[i].cpu(), zps[i].cpu() if zps[i] is not None else None, strategy=str(getattr(args.strategy, "value", args.strategy)),
                                   num_bits=args.num_bits, qtype=str(getattr(args.type, "value", args.type)))
        same(g.cpu(), ref, f"{what} tensor {i} vs oracle: ")
    return launches


# int 2 .. 8 bits (bf16 at 7 bits is the last width of the narrow rounding, dispatch.cu), symmetric and asymmetric, and fp8
SCHEMES = [("int", 8, True), ("int", 8, False), ("int", 4, True), ("int", 4, False), ("float", 8, True), ("int", 2, False), ("int", 3, True),
           ("int", 5, False), ("int", 6, True), ("int", 7, True), ("int", 7, False)]
LAYOUTS = [("contiguous", 2, 4, 16, 64), ("hf", 2, 4, 16, 64), ("hf", 3, 8, 5, 128), ("hf", 64, 8, 1, 128)]   # GQA heads, decode (S = 1)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("strategy", ["tensor", "attn_head"])
@pytest.mark.parametrize("scheme", SCHEMES, ids=[f"{t}{b}{'s' if s else 'a'}" for t, b, s in SCHEMES])
@pytest.mark.parametrize("layout", LAYOUTS, ids=[f"{lay}-{b}x{h}x{s}x{d}" for lay, b, h, s, d in LAYOUTS])
def test_fake_quantize_heads_matches_fake_quantize_and_oracle(dtype, strategy, scheme, layout):
    lay, b, h, s, d = layout
    gen = torch.Generator().manual_seed(zlib.crc32(repr((str(dtype), strategy, scheme, layout)).encode()))
    args = qargs(strategy, scheme[0], scheme[1], scheme[2])
    k, v = hf_states(b, h, s, d, dtype, gen, lay), hf_states(b, h, s, d, dtype, gen, lay)
    assert check_pair([k, v], args) == 1        # one launch for the K / V pair
    q = hf_states(b, 2 * h, s, d, dtype, gen, lay)
    assert check_pair([q], args) == 1


def _per_head(values, dtype, strategy):
    """one value per head ([H, 1, 1], ATTN_HEAD) or the first one ([1], TENSOR)"""
    t = torch.tensor(values, dtype=torch.float64).to(dtype).to(DEV)
    return t.reshape(-1, 1, 1) if strategy == "attn_head" else t[:1]


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("strategy", ["tensor", "attn_head"])
def test_fp8_with_the_all_zero_float8_zero_point(dtype, strategy):
    """an FP8 KV scheme applied before compression registers an all-zero float8_e4m3fn zero point (initialize_qparams with
    force_zero_point): the kernel's third zero-point kind"""
    gen = torch.Generator().manual_seed(20)
    args = qargs(strategy, "float", 8, True)
    k, v = hf_states(2, 4, 16, 64, dtype, gen, "hf"), hf_states(2, 4, 16, 64, dtype, gen, "hf")
    sz = []
    for x in (k, v):
        scale, _ = qparams(x, args)
        sz.append((scale, torch.zeros(scale.shape, dtype=torch.float8_e4m3fn, device=DEV)))
    assert check_pair([k, v], args, sz=sz) == 1


@pytest.mark.parametrize("scheme", [("int", 8, False), ("float", 8, True)], ids=["int8a", "fp8"])
@pytest.mark.parametrize("strategy", ["tensor", "attn_head"])
def test_empty_key_and_unequal_pair(strategy, scheme):
    """an empty K beside a non-empty V (the whole grid is V's), and K / V of different shapes whose chunk counts (of 8 elements)
    are not multiples of the 1024 chunks of a block"""
    gen = torch.Generator().manual_seed(21)
    args = qargs(strategy, scheme[0], scheme[1], scheme[2])
    v = hf_states(2, 4, 5, 64, torch.bfloat16, gen, "hf")
    empty = hf_states(2, 4, 0, 64, torch.bfloat16, gen, "hf")
    vsz = qparams(v, args)
    assert check_pair([empty, v], args, sz=[vsz, vsz]) == 1
    k = hf_states(1, 8, 37, 128, torch.bfloat16, gen, "hf")
    assert (k.numel() // 8) % 1024 and (v.numel() // 8) % 1024
    assert check_pair([k, v], args) == 1
    assert check_pair([v, k], args) == 1


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("strategy", ["tensor", "attn_head"])
@pytest.mark.parametrize("scheme", [("int", 8, True), ("int", 4, False), ("float", 8, True)], ids=["int8s", "int4a", "fp8"])
def test_scales_outside_2_pow_100(dtype, strategy, scheme):
    """scales of 2^-101 and 2^101 (per head: both, and 1), where x / scale is an IEEE division rather than a reciprocal product"""
    gen = torch.Generator().manual_seed(22)
    args = qargs(strategy, scheme[0], scheme[1], scheme[2])
    qmax = 448.0 if scheme[0] == "float" else 2.0 ** (scheme[1] - 1)
    for values in ([2.0 ** -101, 2.0 ** 101, 1.0, 2.0 ** -101], [2.0 ** 101, 2.0 ** -101, 2.0 ** -101, 1.0]):
        scale = _per_head(values, dtype, strategy)
        heads = scale.reshape(-1).double().cpu() if strategy == "attn_head" else scale.double().cpu().expand(4)
        xs = [(torch.randn(2, 16, 4, 64, generator=gen, dtype=torch.float64) * heads.reshape(1, 1, 4, 1) * qmax / 3).to(dtype).to(DEV)
              .transpose(1, 2) for _ in range(2)]
        zp = None if scheme[2] else torch.randint(-3, 3, scale.shape, generator=gen, dtype=torch.int8).to(DEV)
        assert check_pair(xs, args, sz=[(scale, zp), (scale, zp)]) == 1


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32])
@pytest.mark.parametrize("scheme", [("int", 8, False), ("int", 4, True), ("float", 8, True)], ids=["int8a", "int4s", "fp8"])
def test_infinite_inputs(dtype, scheme):
    """+-inf states clamp to the ends of the grid as fake_quantize and the oracle clamp them"""
    gen = torch.Generator().manual_seed(23)
    for strategy in ("tensor", "attn_head"):
        args = qargs(strategy, scheme[0], scheme[1], scheme[2])
        k, v = hf_states(2, 4, 16, 64, dtype, gen, "hf"), hf_states(2, 4, 16, 64, dtype, gen, "hf")
        sz = [qparams(x, args) for x in (k, v)]
        k[0, 1, 3, 5], k[1, 3, 0, 63], v[0, 0, 0, 0], v[1, 2, 15, 8] = float("inf"), float("-inf"), float("-inf"), float("inf")
        assert check_pair([k, v], args, sz=sz) == 1


def test_llama3_8b_prefill_shape():
    gen = torch.Generator().manual_seed(8)
    args = qargs("tensor", "float", 8, True)
    k, v = hf_states(1, 8, 8192, 128, torch.bfloat16, gen, "hf"), hf_states(1, 8, 8192, 128, torch.bfloat16, gen, "hf")
    assert check_pair([k, v], args) == 1


def test_attn_golden_cases_through_the_strided_op():
    """tests/golden/attn.pt.gz (reference fake_quantize with ATTN_HEAD scales), fed to the new op in the transposed layout"""
    for i, c in enumerate(golden.load("attn")):
        args = types.SimpleNamespace(**c["args"])
        x = c["x"].transpose(1, 2).contiguous().transpose(1, 2).to(DEV)    # same values, HF-transposed strides
        assert not x.is_contiguous()
        zp = c["zp"].to(DEV) if c["zp"] is not None else None
        n0 = N.launch_count()
        got = ops.fake_quantize_heads([x], [c["scale"].to(DEV)], [zp], args)[0]
        assert N.launch_count() - n0 == 1
        same(got.cpu(), c["fq"], f"attn case {i}: ")


INELIGIBLE = ["d_not_multiple_of_8", "fp32_scale_bf16_x", "non_dense_v_from_fused_qkv", "scale_not_per_head_shape"]


@pytest.mark.parametrize("symmetric", [True, False], ids=["sym", "asym"])
@pytest.mark.parametrize("strategy", ["tensor", "attn_head"])
@pytest.mark.parametrize("what", INELIGIBLE)
def test_ineligible_inputs_fall_back_to_fake_quantize(what, strategy, symmetric):
    """inputs the strided kernel does not take run through fake_quantize with the scales and zero points as given: same results,
    and the fused kernel does not run (each tensor takes its own fake_quantize launch)"""
    if what == "scale_not_per_head_shape" and strategy == "tensor":
        pytest.skip("a one-element scale is per tensor in every shape")
    gen = torch.Generator().manual_seed(zlib.crc32(repr((what, strategy, symmetric)).encode()))
    args = qargs(strategy, "int", 8, symmetric)
    b, h, s, d = 2, 4, 16, 64
    if what == "d_not_multiple_of_8":
        d = 36
    if what == "scale_not_per_head_shape":
        h = d = 8          # a [H] scale broadcasts along D in fake_quantize, not per head
    k = hf_states(b, h, s, d, torch.bfloat16, gen, "hf")
    if what == "non_dense_v_from_fused_qkv":
        # fused-qkv attentions (e.g. Phi-3) slice K and V out of one [B, S, 3 * H * D] projection: V is a view with gaps
        qkv = torch.randn(b, s, 3 * h * d, generator=gen).to(torch.bfloat16).to(DEV)
        v = qkv[..., 2 * h * d:].view(b, s, h, d).transpose(1, 2)
        assert torch.empty_like(v).stride() != v.stride()
    else:
        v = hf_states(b, h, s, d, torch.bfloat16, gen, "hf")
    scales, zps = [], []
    for x in (k, v):
        scale, zp = qparams(x, args)
        if what == "fp32_scale_bf16_x":
            scale = scale.float()
        if what == "scale_not_per_head_shape":
            scale, zp = scale.reshape(-1), (zp.reshape(-1) if zp is not None else None)
        scales.append(scale)
        zps.append(zp)
    n0 = N.launch_count()
    got = ops.fake_quantize_heads([k, v], scales, zps, args)
    assert N.launch_count() - n0 >= 2
    for x, sc, zp, g in zip((k, v), scales, zps, got):
        same(g, ops.fake_quantize(x, sc, zp, args), f"{what}: ")


def test_dynamic_token_kv_scheme_runs_unfused():
    """a dynamic token kv scheme has no static qparams: the KV-cache path takes forward_quantize (no strided launch) and gives the
    oracle's fake_quantize with the per-(batch, head) scales of the reference's token observer (reduction over dims 2, 3)"""
    from compressed_tensors_b200.modeling.kvcache import quantize_attention_states
    from compressed_tensors_b200.quantization import QuantizationScheme
    from compressed_tensors_b200.quantization.utils import calculate_qparams

    args = qargs("token", "int", 8, True, dynamic=True)
    m = torch.nn.Module()
    m.quantization_scheme = QuantizationScheme(targets=["x"], input_activations=args)
    gen = torch.Generator().manual_seed(4)
    k, v = hf_states(2, 4, 16, 64, torch.bfloat16, gen, "hf"), hf_states(2, 4, 16, 64, torch.bfloat16, gen, "hf")
    n0 = N.launch_count()
    got = quantize_attention_states(m, ("k", "v"), (k, v))
    assert N.launch_count() - n0 >= 2
    for x, g in zip((k, v), got):
        scale, zp = calculate_qparams(x.amin((2, 3), keepdim=True), x.amax((2, 3), keepdim=True), args)
        want = oracle.fake_quantize(x.cpu(), scale.cpu(), zp.cpu(), strategy="token", num_bits=8, qtype="int")
        same(g.cpu(), want)


def test_static_attn_head_kv_pair_takes_one_launch_through_the_hook():
    from compressed_tensors_b200.modeling.kvcache import quantize_attention_states
    from compressed_tensors_b200.quantization import QuantizationScheme

    args = qargs("attn_head", "int", 8, False)
    gen = torch.Generator().manual_seed(5)
    k, v = hf_states(2, 4, 16, 64, torch.bfloat16, gen, "hf"), hf_states(2, 4, 16, 64, torch.bfloat16, gen, "hf")
    m = torch.nn.Module()
    m.quantization_scheme = QuantizationScheme(targets=["x"], input_activations=args)
    for base, x in (("k", k), ("v", v)):
        scale, zp = qparams(x, args)
        m.register_parameter(f"{base}_scale", torch.nn.Parameter(scale, requires_grad=False))
        m.register_parameter(f"{base}_zero_point", torch.nn.Parameter(zp, requires_grad=False))
    n0 = N.launch_count()
    got = quantize_attention_states(m, ("k", "v"), (k, v))
    assert N.launch_count() - n0 == 1
    for base, x, g in (("k", k, got[0]), ("v", v, got[1])):
        same(g, ops.fake_quantize(x, getattr(m, f"{base}_scale"), getattr(m, f"{base}_zero_point"), args), f"{base}: ")


def _model_cases():
    pytest.importorskip("transformers", reason="the model-level KV-cache cases need transformers")
    return golden.load("kv")


@pytest.mark.parametrize("idx", range(8))
def test_model_cases_on_cuda(idx):
    """post-quantization Q / K / V equal ops.fake_quantize of the pre-quantization states of the same run; logits within bf16 / fp32
    tolerance of the reference's CPU run"""
    from tests.test_kv_cache_host import DTYPES, replay

    case = _model_cases()[idx]
    from compressed_tensors_b200.quantization import QuantizationConfig

    cfg = QuantizationConfig(**case["config"])
    args = cfg.kv_cache_scheme or next(iter(cfg.config_groups.values())).input_activations
    model, pre, post, logits = replay(case, DEV)
    from tests.test_kv_cache_host import attention_modules

    for layer, (m, p, q) in enumerate(zip(attention_modules(model), pre, post)):
        for base, x in p.items():
            assert x.is_cuda
            if args.dynamic:
                from compressed_tensors_b200.quantization.lifecycle.forward import forward_quantize
                want = forward_quantize(m, x, base, args)
            else:
                want = ops.fake_quantize(x.contiguous(), getattr(m, f"{base}_scale"), getattr(m, f"{base}_zero_point", None), args)
            same(q[base], want, f"layer {layer} {base}: ")
    tol = dict(rtol=2e-2, atol=5e-2) if DTYPES[case["dtype"]] == torch.bfloat16 else dict(rtol=1e-3, atol=1e-3)
    torch.testing.assert_close(logits.cpu(), case["logits"], **tol)
