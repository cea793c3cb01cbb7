"""
Maximum sizes: one tensor of more than 2^31 elements (147456 x 16384 = 2.42 G elements, 4.8 GB of bf16) through each kernel
family.  No CPU oracle finishes at this size, so the check is a size-independent property: the tensor is a 64-row tile repeated
2304 times along the rows, every op on the path is row-local (scales travel with their rows), hence the output must be the tile's
output repeated -- and the tile's output is checked against the oracle.  A 32-bit element or byte index anywhere on the path
breaks the repetition in the upper half of the tensor.
"""
import pytest
import torch

import oracle
from compressed_tensors_b200 import ops
from compressed_tensors_b200.quantization import QuantizationArgs

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TILE_ROWS, COLS, REP = 64, 16384, 2304
assert TILE_ROWS * REP * COLS > 2 ** 31


def _need_memory():
    free, _ = torch.cuda.mem_get_info(0)
    if free < 40 * 2 ** 30:
        pytest.skip("needs 40 GB of free device memory")


def _tiled_equal(big: torch.Tensor, tile_out: torch.Tensor, what: str):
    """big == tile_out repeated REP times along dim 0, compared on the device slab by slab (no second multi-GB tensor)"""
    assert big.shape[0] == tile_out.shape[0] * REP and big.shape[1:] == tile_out.shape[1:], (what, big.shape, tile_out.shape)
    v = big.view(REP, *tile_out.shape)
    a, b = (v.view(torch.uint8), tile_out.view(torch.uint8)) if v.dtype == torch.float8_e4m3fn else (v, tile_out)
    bad = (a != b.unsqueeze(0)).flatten(1).any(1)
    if bool(bad.any()):
        first = int(bad.nonzero()[0])
        pytest.fail(f"{what}: repetition {first} of {REP} (element offset {first * tile_out.numel():,}) differs from the tile's output", pytrace=False)


@pytest.fixture(scope="module")
def weights():
    _need_memory()
    g = torch.Generator().manual_seed(11)
    tile = (torch.randn(TILE_ROWS, COLS, generator=g) * 0.02).to(torch.bfloat16)
    return tile, tile.to(DEV).repeat(REP, 1)


def test_w4a16_quantize_pack_and_back(weights):
    tile, big = weights
    a = QuantizationArgs(num_bits=4, type="int", symmetric=True, strategy="group", group_size=128)
    s = (tile.float().unflatten(-1, (-1, 128)).abs().amax(-1) / 7.5).to(torch.bfloat16)
    S = s.to(DEV).repeat(REP, 1)
    kw = dict(strategy="group", group_size=128, num_bits=4, qtype="int")
    want = oracle.pack_to_int32(oracle.quantize(tile, s, None, dtype=torch.int8, **kw), 4)
    packed = ops.quantize_pack(big, S, None, a)
    _tiled_equal(packed, want.to(DEV), "quantize_pack (streaming path)")
    back = ops.unpack_dequantize(packed, S, None, 4, tuple(big.shape))
    _tiled_equal(back, oracle.fake_quantize(tile, s, None, **kw).to(DEV), "unpack_dequantize")
    del back
    _tiled_equal(ops.fake_quantize(big, S, None, a), oracle.fake_quantize(tile, s, None, **kw).to(DEV), "fake_quantize")


def test_generic_kernels_with_g_idx(weights):
    """activation ordering sends the op to the generic (non-streaming) kernels"""
    tile, big = weights
    a = QuantizationArgs(num_bits=8, type="int", symmetric=True, strategy="group", group_size=128)
    g = torch.Generator().manual_seed(12)
    g_idx = (torch.arange(COLS) // 128)[torch.randperm(COLS, generator=g)].to(torch.int32)
    s = (torch.rand(TILE_ROWS, COLS // 128, generator=g) * 0.001 + 0.0005).to(torch.bfloat16)
    S = s.to(DEV).repeat(REP, 1)
    kw = dict(strategy="group", group_size=128, num_bits=8, qtype="int", g_idx=g_idx)
    want = oracle.quantize(tile, s, None, dtype=torch.int8, **kw)
    q = ops.quantize(big, S, None, a, dtype=torch.int8, g_idx=g_idx.to(DEV))
    _tiled_equal(q, want.to(DEV), "quantize with g_idx (generic kernel)")


def test_fp8_channel_and_int4_pack(weights):
    tile, big = weights
    a = QuantizationArgs(num_bits=8, type="float", symmetric=True, strategy="channel")
    s = (tile.float().abs().amax(-1, keepdim=True) / 448.0).to(torch.bfloat16)
    S = s.to(DEV).repeat(REP, 1)
    kw = dict(strategy="channel", num_bits=8, qtype="float")
    q = ops.quantize(big, S, None, a, dtype=torch.float8_e4m3fn)
    _tiled_equal(q, oracle.quantize(tile, s, None, dtype=torch.float8_e4m3fn, **kw).to(DEV), "fp8 quantize")
    _tiled_equal(ops.dequantize(q, S, None, args=a), oracle.dequantize(oracle.quantize(tile, s, None, dtype=torch.float8_e4m3fn, **kw), s, None, strategy="channel").to(DEV), "fp8 dequantize")
    del q
    g = torch.Generator().manual_seed(13)
    codes = torch.randint(-8, 8, (TILE_ROWS, COLS), dtype=torch.int8, generator=g)
    C = codes.to(DEV).repeat(REP, 1)
    p = ops.pack_to_int32(C, 4)
    _tiled_equal(p, oracle.pack_to_int32(codes, 4).to(DEV), "pack_to_int32")
    _tiled_equal(ops.unpack_from_int32(p, 4, tuple(C.shape)), codes.to(DEV), "unpack_from_int32")


def test_nvfp4_pack_and_back(weights):
    tile, big = weights
    a = QuantizationArgs(num_bits=4, type="float", symmetric=True, strategy="tensor_group", group_size=16, scale_dtype=torch.float8_e4m3fn)
    gs = torch.tensor([448.0 * 6.0 / float(tile.float().abs().max())])
    s = (tile.float().unflatten(-1, (-1, 16)).abs().amax(-1) / 6.0 * gs).clamp(2 ** -9, 448).to(torch.float8_e4m3fn).to(torch.bfloat16)
    S, GS = s.to(DEV).repeat(REP, 1), gs.to(DEV)
    kw = dict(strategy="tensor_group", group_size=16, num_bits=4, qtype="float", global_scale=gs)
    want = oracle.pack_fp4_to_uint8(oracle.quantize(tile, s, None, **kw))
    packed = ops.quantize_pack_fp4(big, S, None, a, global_scale=GS)
    _tiled_equal(packed, want.to(DEV), "quantize_pack_fp4")
    tile_back = ops.unpack_dequantize_fp4(want.to(DEV), s.to(DEV), GS, dtype=torch.bfloat16)
    _tiled_equal(ops.unpack_dequantize_fp4(packed, S, GS, dtype=torch.bfloat16), tile_back, "unpack_dequantize_fp4")


def test_hadamard_transform(weights):
    """rows of order 128 (signed, permuted) and 16384; the tile's output against the float64 reference"""
    from tests.test_transform_host import assert_online_bound, structured_reference

    tile, big = weights
    g = torch.Generator().manual_seed(14)
    for n, signed in ((128, True), (16384, False)):
        q = (torch.randint(0, 2, (n,), generator=g) * 2 - 1).to(torch.int8).to(DEV) if signed else None
        perm = torch.randperm(n, generator=g).to(DEV) if signed else None
        tile_out = ops.hadamard_transform(tile.to(DEV), n, q, perm)
        assert_online_bound(tile_out, structured_reference(tile.to(DEV), n, q, perm), tile.to(DEV), n)
        _tiled_equal(ops.hadamard_transform(big, n, q, perm), tile_out, f"hadamard_transform n={n}")


def test_attention_view_heads_and_hadamard(weights):
    """the tensor as strided [B, H, S, D] attention states (B = REP, H = 16, S = 64, D = 1024): fake_quantize_heads per tensor and per
    head against the oracle, and hadamard_transform along D"""
    from tests.test_transform_host import assert_online_bound, structured_reference

    tile, big = weights
    view = big.view(REP, TILE_ROWS, 16, COLS // 16).transpose(1, 2)
    tview = tile.to(DEV).view(1, TILE_ROWS, 16, COLS // 16).transpose(1, 2)
    amax = tview.float().abs().amax((0, 2, 3))
    for strategy, scale in (("tensor", (amax.max() / 127).reshape(1)), ("attn_head", (amax / 127).reshape(16, 1, 1))):
        a = QuantizationArgs(num_bits=8, type="int", symmetric=True, strategy=strategy)
        scale = scale.to(torch.bfloat16)
        want = oracle.fake_quantize(tview.cpu(), scale.cpu(), None, strategy=strategy, num_bits=8, qtype="int").to(DEV)
        (got,) = ops.fake_quantize_heads([view], [scale], [None], a)
        assert got.stride() == view.stride()
        _tiled_equal(got.transpose(1, 2).reshape(big.shape), want.transpose(1, 2).reshape(tile.shape), f"fake_quantize_heads {strategy}")
        del got
    tile_out = ops.hadamard_transform(tview, 1024)
    assert_online_bound(tile_out, structured_reference(tview, 1024), tview, 1024)
    out = ops.hadamard_transform(view, 1024)
    assert out.stride() == view.stride()
    _tiled_equal(out.transpose(1, 2).reshape(big.shape), tile_out.transpose(1, 2).reshape(tile.shape), "hadamard_transform [B, H, S, D]")


def test_sparse_formats(weights):
    tile, big = weights
    v, m = ops.sparse24_compress(big)
    tv, tm = ops.sparse24_compress(tile.to(DEV))
    _tiled_equal(v, tv, "sparse24 values")
    _tiled_equal(m, tm, "sparse24 bitmask")
    dense = ops.sparse24_decompress(v, m, tuple(big.shape))
    _tiled_equal(dense, ops.sparse24_decompress(tv, tm, tuple(tile.shape)), "sparse24 decompress")
    del v, m
    # unstructured: the 2:4-pruned tensor (exactly half non-zero) through the bitmask format; compact offsets exceed 2^30
    uv, um, uo = ops.bitmask_compress(dense)
    assert uv.numel() == int((dense != 0).sum())
    back = ops.bitmask_decompress(uv, um, uo, tuple(dense.shape))
    assert torch.equal(back, dense)
