"""
Maximum sizes for the kernel families `test_gpu_large.py` does not reach: the dynamic activation observers, the fused weight observers,
fused 2:4 + int4, the checkpoint converters, one-byte outputs past 2^32 bytes and a multi-tensor launch whose jobs add up to more than
2^32 elements.  The method is the one of `test_gpu_large.py`: a small tile repeated along the rows, ops that are row- or group-local,
so the big output must be the tile's output repeated, and the tile's output is checked against the CPU oracle (or, where the oracle
has no entry point, against the two-step GPU path that tests/golden/dynamic.pt.gz pins).  The comparison runs on the device slab by
slab.

The tile has 48 rows (3 * 2^4), so no power of two is a multiple of its size: an element or byte index that wraps at 2^31 or 2^32
lands on another phase of the tile, and the repetition breaks.  (A tile of 2^k elements would hide a wrapped read: x[i mod 2^32] is
the same value as x[i].)  `test_wrapped_stand_ins_are_rejected` shows on the CPU that the checks reject such wrapped outputs.

Tensor-wide reductions (per-tensor scales, the NVFP4 global scale) see every element, so repetition alone does not show that the upper
half was read: the tensor's unique extreme is planted in the last repetition, past element 2^32, and the scale must be the one of
(tile min, planted max).
"""
import contextlib
import math
import time
from fractions import Fraction

import pytest
import torch

import oracle
from compressed_tensors_b200 import _native as N
from compressed_tensors_b200 import ops
from compressed_tensors_b200.quantization import QuantizationArgs, preset_name_to_scheme
from oracle.qparams import calculate_qparams as orc_qparams
from tests.util import same

DEV = "cuda:0"
GIB = 2 ** 30
TILE_ROWS, COLS = 48, 16384
TILE = TILE_ROWS * COLS                       # 786432 = 3 * 2^18 elements
REP_BIG = 5472                                # 4.30 G elements, 8.6 GB of bf16: past 2^32 elements and one-byte outputs past 2^32 bytes
REP_S24 = 2736                                # 2.15 G elements (fused 2:4 + int4)
FP8_TILE_ROWS, REP_FP8 = 384, 683             # 128 x 128 blocks: a 3-block-row tile, 4.30 G fp8 bytes
AWQ_K, AWQ_TILE_WORDS, REP_AWQ = 4096, 96, 1366   # weight_packed [1049088, 512] int32: 2.15 GB
REP_JOB_A, REP_JOB_B = 2800, 2801             # 2.20 G elements per job, 4.40 G in the launch
BIG_ROWS = TILE_ROWS * REP_BIG
assert TILE_ROWS * REP_BIG * COLS > 2 ** 32 and TILE_ROWS * REP_S24 * COLS > 2 ** 31
assert FP8_TILE_ROWS * REP_FP8 * COLS > 2 ** 32 and AWQ_TILE_WORDS * 8 * REP_AWQ * (AWQ_K // 8) * 4 > 2 ** 31
assert 2 ** 31 < TILE * REP_JOB_A < TILE * REP_JOB_B < 2 ** 32 < TILE * (REP_JOB_A + REP_JOB_B)
assert (REP_BIG - 1) * TILE > 2 ** 32 - TILE and BIG_ROWS * COLS - 1 > 2 ** 32   # the planted element (the last one) lies past 2^32


# ---- checks (device independent: the CPU test below runs them on stand-ins) --------------------------------------------------------
def _bits(t: torch.Tensor) -> torch.Tensor:
    """an integer view of t: float equality would take -0.0 for +0.0 and never match a NaN"""
    if t.dtype.is_floating_point:
        return t.view({1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])
    return t.view(torch.uint8) if t.dtype == torch.bool else t


def _tiled_equal(big: torch.Tensor, tile_out: torch.Tensor, what: str):
    """big == tile_out repeated along the leading dimension, bit for bit; compared slab by slab, so no second multi-GB tensor is made"""
    n = tile_out.numel()
    assert big.dtype == tile_out.dtype and big.is_contiguous() and big.shape[-1] == tile_out.shape[-1], (what, big.dtype, big.shape, tile_out.shape)
    assert n > 0 and big.numel() % n == 0, (what, big.shape, tile_out.shape)
    rep = big.numel() // n
    v, t = _bits(big).reshape(rep, n), _bits(tile_out.contiguous()).reshape(1, n)
    slab = max(1, 2 ** 28 // n)
    for s in range(0, rep, slab):
        bad = (v[s:s + slab] != t).any(1)
        if bool(bad.any()):
            first = s + int(bad.nonzero()[0])
            pytest.fail(f"{what}: repetition {first} of {rep} (element offset {first * n:,}) differs from the tile's output", pytrace=False)


def _planted_qparams(tile: torch.Tensor, planted: torch.Tensor, **qkw):
    """the oracle's calculate_qparams of a tensor made of repetitions of `tile` and one planted element"""
    mn, mx = torch.minimum(tile.min(), planted), torch.maximum(tile.max(), planted)
    return orc_qparams(mn.reshape(1), mx.reshape(1), **qkw)


def _check_planted(got, want, what: str):
    """per-tensor qparams (scale, zero point or None) computed on the device against the ones of (tile min, planted max)"""
    for g, w, name in zip(got, want, ("scale", "zero point")):
        if w is None:
            continue
        g = g.cpu().reshape(w.shape)
        if g.dtype != w.dtype or not torch.equal(_bits(g), _bits(w)):
            pytest.fail(f"{what}: {name} {g.tolist()} is not the {w.tolist()} of the planted extreme: the reduction missed it", pytrace=False)


def _report(what: str, numel: int, largest_bytes: int, past: int):
    assert numel > past, (what, numel, past)
    print(f"\n  {what}: {numel:,} elements (> 2^{past.bit_length() - 1}), largest output {largest_bytes:,} bytes", end="")


# ---- GPU helpers -----------------------------------------------------------------------------------------------------------------
def _need_memory(gib: int = 40):
    free, _ = torch.cuda.mem_get_info(0)
    if free < gib * GIB:
        pytest.skip(f"needs {gib} GB of free device memory")


@pytest.fixture(autouse=True)
def _wall_time_and_peak_memory(request):
    if request.node.get_closest_marker("gpu") is None or not torch.cuda.is_available():
        yield
        return
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    print(f"\n  [{request.node.name}] {time.perf_counter() - t0:.1f} s, peak device memory {torch.cuda.max_memory_allocated() / GIB:.1f} GiB")


def _repeat(tile: torch.Tensor, rep: int) -> torch.Tensor:
    """tile repeated `rep` times along dim 0 on the device (float8 through its bytes: repeat has no float8 kernel)"""
    t = tile.to(DEV)
    if t.dtype == torch.float8_e4m3fn:
        return t.view(torch.uint8).repeat(rep, 1).view(torch.float8_e4m3fn)
    return t.repeat(rep, *([1] * (t.ndim - 1)))


def _tile(seed: int, rows: int = TILE_ROWS, cols: int = COLS) -> torch.Tensor:
    """bf16 rows whose magnitudes span 2^-6 .. 2^2 (every fp4 code and near-zero rows occur)"""
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(rows, cols, generator=g) * torch.exp2(torch.randint(-6, 3, (rows, 1), generator=g).float())).to(torch.bfloat16)


@contextlib.contextmanager
def _planted(big: torch.Tensor, value: torch.Tensor):
    """big's last element (in the last repetition, past element 2^32) set to `value` for the duration"""
    flat = big.view(-1)
    old = flat[-1].clone()
    flat[-1] = value.to(big.dtype).to(big.device)
    try:
        yield flat.numel() - 1
    finally:
        flat[-1] = old


def _tiled_equal_but_planted(big: torch.Tensor, tile_out: torch.Tensor, planted_out: torch.Tensor, what: str):
    """big == tile_out repeated, except its last element, which must be `planted_out` (the planted input's result)"""
    flat = big.view(-1)
    got = flat[-1:].clone()
    assert torch.equal(_bits(got.cpu()), _bits(planted_out.reshape(1).to(got.dtype))), (what, got.item(), planted_out.item())
    flat[-1] = tile_out.reshape(-1)[-1].to(big.device)
    _tiled_equal(big, tile_out.to(big.device), what)


def _two_step(x: torch.Tensor, args, gs=None):
    """compute_dynamic_scales_and_zp + fake_quantize on the device: the path tests/golden/dynamic.pt.gz pins"""
    from compressed_tensors_b200.quantization.utils import compute_dynamic_scales_and_zp

    scale, zp = compute_dynamic_scales_and_zp(value=x, args=args, module=None, global_scale=gs)
    return ops.fake_quantize(x, scale, zp, args, global_scale=gs), scale, zp


def _acts(**kw):
    return QuantizationArgs(**{"num_bits": 8, "type": "int", "strategy": "token", "symmetric": True, "dynamic": True, **kw})


# ---- the 4.30 G element tensor: dynamic activations, fused observers, one-byte outputs --------------------------------------------
@pytest.fixture(scope="class")
def big():
    """the tile and its 5472 repetitions on the device (262656 x 16384 bf16, 8.6 GB); freed after the class"""
    _need_memory()
    tile = _tile(21)
    yield tile, _repeat(tile, REP_BIG)


def _planted_value(tile: torch.Tensor) -> torch.Tensor:
    """a positive value four times larger than any |x| of the tile: the tensor's unique extreme"""
    return (tile.float().abs().max() * 4).to(tile.dtype)


@pytest.mark.gpu
class TestPast2To32Elements:
    # ---- 1. dynamic activations (ops.dynamic_fake_quantize, csrc/dynamic_fake.cu) ----
    @pytest.mark.parametrize("cols", [COLS, 2 * COLS])
    @pytest.mark.parametrize("scheme", ["fp8", "int8_asym"])
    def test_dynamic_token(self, big, cols, scheme):
        """TOKEN on [1, R, 16384] (the 256 x 8 CTA) and [1, R/2, 32768] (the 512-thread CTA), 4.30 G elements: guards the row offset
        row * cols and the 16-byte unit index of the fp8 / int8 per-token kernels, and the bf16 output past 2^33 bytes"""
        tile, x = big
        args = _acts(type="float") if scheme == "fp8" else _acts(symmetric=False)
        x3, t3 = x.view(1, -1, cols), tile.view(1, -1, cols)
        _report(f"dynamic token {scheme} [1, {x3.shape[1]}, {cols}]", x3.numel(), x3.numel() * 2, 2 ** 32)
        want = _two_step(t3.to(DEV), args)
        # the two-step result of the tile against the oracle: per-row min/max -> calculate_qparams -> fake_quantize
        qkw = dict(num_bits=8, qtype="float" if scheme == "fp8" else "int")
        s, z = orc_qparams(t3.amin(-1, keepdim=True), t3.amax(-1, keepdim=True), symmetric=args.symmetric, **qkw)
        z = None if args.symmetric else z
        same(want[1].cpu(), s, "tile scale vs oracle")
        if z is not None:
            same(want[2].cpu(), z, "tile zero point vs oracle")
        same(want[0].cpu(), oracle.fake_quantize(t3, s, z, strategy="token", **qkw), "tile output vs oracle")
        res = ops.dynamic_fake_quantize(x3, args)
        assert res is not None, N.last_error()
        for got, w, what in zip(res, want, ("output", "scale", "zero point")):
            _tiled_equal(got, w, f"dynamic token {scheme} {cols} {what}")

    @pytest.mark.parametrize("scheme", ["int8_group128", "fp8_group128", "nvfp4", "mxfp4"])
    def test_dynamic_group(self, big, scheme):
        """GROUP 128 (int8, and the fp8 activations of FP8_BLOCK), TENSOR_GROUP 16 (NVFP4, fp8 scales under a global scale) and MXFP4
        group 32 (E8M0 scales), 4.30 G elements: guards the 16-byte unit index n / 8 and the group index of the warp-shuffle kernel"""
        tile, x = big
        gs = None
        if scheme == "int8_group128":
            args = _acts(strategy="group", group_size=128)
        elif scheme == "fp8_group128":
            args = preset_name_to_scheme("FP8_BLOCK", ["Linear"]).input_activations
        elif scheme == "nvfp4":
            from compressed_tensors_b200.quantization.utils import generate_gparam

            args = preset_name_to_scheme("NVFP4", ["Linear"]).input_activations
            gs = generate_gparam(tile.min(), tile.max()).reshape(1).to(DEV)
        else:
            args = preset_name_to_scheme("MXFP4", ["Linear"]).input_activations
        x3, t3 = x.view(1, BIG_ROWS, COLS), tile.view(1, TILE_ROWS, COLS).to(DEV)
        _report(f"dynamic {scheme}", x3.numel(), x3.numel() * 2, 2 ** 32)
        want = _two_step(t3, args, gs)
        if scheme.endswith("group128"):
            # scales in x's dtype: the two-step tile result against the oracle as well
            qt = "float" if scheme.startswith("fp8") else "int"
            grp = tile.view(1, TILE_ROWS, -1, 128)
            s, _ = orc_qparams(grp.amin(-1), grp.amax(-1), num_bits=8, qtype=qt, symmetric=True)
            same(want[1].cpu(), s, "tile scale vs oracle")
            same(want[0].cpu(), oracle.fake_quantize(tile.view(1, TILE_ROWS, COLS), s, None, strategy="group", group_size=128, num_bits=8, qtype=qt),
                 "tile output vs oracle")
        res = ops.dynamic_fake_quantize(x3, args, global_scale=gs)
        assert res is not None, N.last_error()
        for got, w, what in zip(res, want, ("output", "scale", "zero point")):
            _tiled_equal(got, w, f"dynamic {scheme} {what}")

    def test_dynamic_tensor_planted_extreme(self, big):
        """TENSOR int8 asymmetric, the two-launch path (ct_observe_tensor's grid-stride min / max, then the streaming fake_quantize),
        4.30 G elements with the unique maximum planted at the last element: guards the reduction's element index and CTA stride"""
        tile, x = big
        args = _acts(strategy="tensor", symmetric=False)
        planted = _planted_value(tile)
        _report("dynamic tensor int8 asym", x.numel(), x.numel() * 2, 2 ** 32)
        s, z = _planted_qparams(tile, planted, num_bits=8, qtype="int", symmetric=False)
        kw = dict(strategy="tensor", num_bits=8, qtype="int")
        want = oracle.fake_quantize(tile, s, z, **kw)
        with _planted(x, planted):
            res = ops.dynamic_fake_quantize(x.view(1, BIG_ROWS, COLS), args)
            assert res is not None, N.last_error()
            out, scale, zp = res
            _check_planted((scale, zp), (s, z), "dynamic tensor")
        _tiled_equal_but_planted(out.view(BIG_ROWS, COLS), want, oracle.fake_quantize(planted.reshape(1, 1), s, z, **kw), "dynamic tensor output")

    # ---- 2. fused observers ----
    @pytest.mark.parametrize("group", [32, 128])
    @pytest.mark.parametrize("bits", [4, 8])
    @pytest.mark.parametrize("sym", [True, False])
    def test_observe_quantize_pack(self, big, group, bits, sym):
        """ct_observe_quantize_pack_int32, 4.30 G elements: guards the group index gi = fd_div(gc0, dc) (32-bit), the packed word
        offset and the scale / zero point offsets"""
        from tests.test_gpu_observe import _args, _want

        tile, x = big
        _report(f"observe_quantize_pack g{group} int{bits} {'sym' if sym else 'asym'}", x.numel(), x.numel() * bits // 8, 2 ** 32)
        want_p, want_s, want_z = _want(tile, bits, group, sym)
        n0 = N.launch_count()
        packed, scale, zp = ops.observe_quantize_pack(x, _args(bits, group, sym))
        assert N.launch_count() - n0 == 1, "the fused observer must take the tensor"
        _tiled_equal(scale, want_s.to(DEV), "observer scale")
        assert (zp is None) == sym
        if zp is not None:
            _tiled_equal(zp, want_z.to(DEV), "observer zero point")
        del scale, zp
        _tiled_equal(packed, want_p.to(DEV), "observer packed words")

    @pytest.mark.parametrize("kind", [("int", 4, False, True), ("float", 8, True, False)])
    def test_observe_quantize_channel(self, big, kind):
        """ct_observe_quantize_channel with 16384 columns (the 8-unit instantiation), packed int4 asymmetric and fp8 codes, 4.30 G
        elements: guards the row offset of the input and of the codes (fp8 codes past 2^32 bytes)"""
        from tests.test_gpu_observe import _chan_oracle

        tile, x = big
        qtype, bits, sym, pack = kind
        _report(f"observe_quantize channel {qtype}{bits}", x.numel(), x.numel() * bits // 8, 2 ** 32)
        wq, ws, wz = _chan_oracle(tile, qtype, bits, sym, pack)
        n0 = N.launch_count()
        q, s, z = ops.observe_quantize(x, QuantizationArgs(num_bits=bits, type=qtype, symmetric=sym, strategy="channel"), pack=pack)
        assert N.launch_count() - n0 == 1, "the fused channel observer must take the tensor"
        _tiled_equal(s, ws.to(DEV), "channel observer scale")
        assert (z is None) == sym
        if z is not None:
            _tiled_equal(z, wz.to(DEV), "channel observer zero point")
        _tiled_equal(q, wq.to(DEV), "channel observer codes")

    def test_observe_tensor_planted_extreme(self, big):
        """ct_observe_quantize_tensor (observe_quantize, TENSOR) and ops.observe_tensor_qparams, int8 asymmetric, and
        ops.observe_tensor_gparam (ct_observe_tensor kind 1, generate_gparam), 4.30 G elements with the unique extreme planted at the
        last element: guards the grid-stride reduction, its atomicMax / done-counter combine, and the int8 code offset past 2^32 bytes"""
        from compressed_tensors_b200.quantization.utils import generate_gparam

        tile, x = big
        a = QuantizationArgs(num_bits=8, type="int", symmetric=False, strategy="tensor")
        planted = _planted_value(tile)
        _report("observe tensor int8 asym", x.numel(), x.numel(), 2 ** 32)
        s, z = _planted_qparams(tile, planted, num_bits=8, qtype="int", symmetric=False)
        kw = dict(strategy="tensor", num_bits=8, qtype="int", dtype=torch.int8)
        want_q = oracle.quantize(tile, s, z, **kw)
        want_g = generate_gparam(torch.minimum(tile.min(), planted), torch.maximum(tile.max(), planted))
        with _planted(x, planted):
            _check_planted(ops.observe_tensor_qparams(x, a), (s, z), "observe_tensor_qparams")
            _check_planted((ops.observe_tensor_gparam(x),), (want_g.reshape(1),), "observe_tensor_gparam")
            n0 = N.launch_count()
            q, qs, qz = ops.observe_quantize(x, a)
            assert N.launch_count() - n0 == 2, "grid-wide min / max + qparams, then the streaming quantize"
            _check_planted((qs, qz), (s, z), "observe_quantize tensor")
        _tiled_equal_but_planted(q, want_q, oracle.quantize(planted.reshape(1, 1), s, z, **kw), "tensor observer codes")

    def test_observe_quantize_pack_nvfp4(self, big):
        """ops.observe_quantize_pack_nvfp4 without a given global scale (ct_observe_tensor kind 1, then
        ct_observe_quantize_pack_nvfp4), 4.30 G elements: guards the group index, the nibble byte offset and the fp8 scale offset"""
        from compressed_tensors_b200.quantization.utils import calculate_qparams, generate_gparam

        tile, x = big
        a = QuantizationArgs(num_bits=4, type="float", symmetric=True, strategy="tensor_group", group_size=16, scale_dtype=torch.float8_e4m3fn)
        _report("observe_quantize_pack_nvfp4", x.numel(), x.numel() // 2, 2 ** 32)
        gs = generate_gparam(tile.min(), tile.max()).reshape(1)
        grp = tile.unflatten(-1, (-1, 16))
        s, _ = calculate_qparams(grp.amin(-1), grp.amax(-1), a, global_scale=gs)
        want_p = oracle.pack_fp4_to_uint8(oracle.quantize(tile, s, None, strategy="tensor_group", group_size=16, num_bits=4, qtype="float", global_scale=gs))
        n0 = N.launch_count()
        packed, scale, got_gs = ops.observe_quantize_pack_nvfp4(x, a)
        assert N.launch_count() - n0 == 2
        assert torch.equal(got_gs.cpu(), gs), (got_gs, gs)
        _tiled_equal(scale, s.to(torch.float8_e4m3fn).to(DEV), "nvfp4 observer fp8 scales")
        _tiled_equal(packed, want_p.to(DEV), "nvfp4 observer nibbles")

    # ---- 5. one-byte outputs past 2^32 bytes ----
    def test_fp8_quantize_and_dequantize(self, big):
        """streaming fp8 quantize (QuantizeOp, per-channel scales) and its dequantize, 4.30 G elements: the fp8 codes cross 2^32
        bytes, the bf16 output 2^33 bytes: guards 32-bit byte and element offsets of one-byte outputs and inputs"""
        tile, x = big
        a = QuantizationArgs(num_bits=8, type="float", symmetric=True, strategy="channel")
        s = (tile.float().abs().amax(-1, keepdim=True) / 448.0).to(torch.bfloat16)
        S = _repeat(s, REP_BIG)
        kw = dict(strategy="channel", num_bits=8, qtype="float")
        want_q = oracle.quantize(tile, s, None, dtype=torch.float8_e4m3fn, **kw)
        _report("fp8 quantize / dequantize", x.numel(), x.numel() * 2, 2 ** 32)
        q = ops.quantize(x, S, None, a, dtype=torch.float8_e4m3fn)
        _tiled_equal(q, want_q.to(DEV), "fp8 quantize")
        back = ops.dequantize(q, S, None, args=a)
        _tiled_equal(back, oracle.dequantize(want_q, s, None, strategy="channel").to(DEV), "fp8 dequantize")

    def test_generic_int8_g_idx_and_8bit_pack(self, big):
        """int8 quantize with g_idx (the generic kernel) into 4.30 GB of codes, then the 8-bit pack_to_int32 / unpack_from_int32 of
        those codes: guards the generic kernel's element index and the word offsets of the 8-bit packers past 2^32 bytes"""
        tile, x = big
        a = QuantizationArgs(num_bits=8, type="int", symmetric=True, strategy="group", group_size=128)
        g = torch.Generator().manual_seed(22)
        g_idx = (torch.arange(COLS) // 128)[torch.randperm(COLS, generator=g)].to(torch.int32)
        s = (tile.float().unflatten(-1, (-1, 128)).abs().amax(-1) / 127.0 + 2.0 ** -12).to(torch.bfloat16)
        want_q = oracle.quantize(tile, s, None, dtype=torch.int8, strategy="group", group_size=128, num_bits=8, qtype="int", g_idx=g_idx)
        _report("int8 quantize with g_idx, 8-bit pack / unpack", x.numel(), x.numel(), 2 ** 32)
        q = ops.quantize(x, _repeat(s, REP_BIG), None, a, dtype=torch.int8, g_idx=g_idx.to(DEV))
        _tiled_equal(q, want_q.to(DEV), "quantize with g_idx (generic kernel)")
        p = ops.pack_to_int32(q, 8)
        want_p = oracle.pack_to_int32(want_q, 8)
        _tiled_equal(p, want_p.to(DEV), "8-bit pack_to_int32")
        del q
        _tiled_equal(ops.unpack_from_int32(p, 8, (BIG_ROWS, COLS)), want_q.to(DEV), "8-bit unpack_from_int32")

    def test_fake_quantize_bf16(self, big):
        """W4 group-128 fake_quantize, 4.30 G elements: the bf16 output crosses 2^33 bytes"""
        tile, x = big
        a = QuantizationArgs(num_bits=4, type="int", symmetric=True, strategy="group", group_size=128)
        s = (tile.float().unflatten(-1, (-1, 128)).abs().amax(-1) / 7.5 + 2.0 ** -12).to(torch.bfloat16)
        _report("fake_quantize bf16", x.numel(), x.numel() * 2, 2 ** 32)
        want = oracle.fake_quantize(tile, s, None, strategy="group", group_size=128, num_bits=4, qtype="int")
        _tiled_equal(ops.fake_quantize(x, _repeat(s, REP_BIG), None, a), want.to(DEV), "fake_quantize")

    def test_fp4_cast_pack_unpack(self, big):
        """standalone ops.cast_to_fp4 (bf16 out past 2^33 bytes), ops.pack_fp4_to_uint8 (input past 2^32 elements) and
        ops.unpack_fp4_from_uint8 (output past 2^33 bytes), 4.30 G elements"""
        tile, x = big
        _report("cast_to_fp4 / pack_fp4_to_uint8 / unpack_fp4_from_uint8", x.numel(), x.numel() * 2, 2 ** 32)
        want_c = oracle.cast_to_fp4(tile)
        want_p = oracle.pack_fp4_to_uint8(want_c)
        c = ops.cast_to_fp4(x)
        _tiled_equal(c, want_c.to(DEV), "cast_to_fp4")
        p = ops.pack_fp4_to_uint8(c)
        del c
        _tiled_equal(p, want_p.to(DEV), "pack_fp4_to_uint8")
        _tiled_equal(ops.unpack_fp4_from_uint8(p, BIG_ROWS, COLS, torch.bfloat16), oracle.unpack_fp4_from_uint8(want_p, TILE_ROWS, COLS).to(DEV),
                     "unpack_fp4_from_uint8")


# ---- 3. fused 2:4 + int4 ------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["group128", "channel"])
def test_sparse24_quantize_pack_and_back(mode):
    """ops.sparse24_quantize_pack / sparse24_unpack_dequantize (csrc/fast_sparse24q.cu, BASELINE config 4) on a 2:4-pruned tile
    repeated to 2.15 G elements: guards the input / dense-output element offsets past 2^31 and the packed-word and mask offsets"""
    _need_memory()
    tile = _tile(23)
    tile = oracle.sparse24_decompress(*oracle.sparse24_compress(tile), tile.shape)       # exactly 2 of every 4 kept
    if mode == "group128":
        s = (tile.float().unflatten(-1, (-1, 128)).abs().amax(-1) / 7.5 + 2.0 ** -12).to(torch.bfloat16)
        a = QuantizationArgs(num_bits=4, type="int", symmetric=True, strategy="group", group_size=128)
        okw = dict(strategy="group", group_size=128)
    else:
        s = (tile.float().abs().amax(-1, keepdim=True) / 7.5 + 2.0 ** -12).to(torch.bfloat16)
        a = QuantizationArgs(num_bits=4, type="int", symmetric=True, strategy="channel")
        okw = dict(strategy="channel")
    want_p, want_m = oracle.sparse24_quantize_pack(tile, s, None, **okw)
    want_d = oracle.sparse24_unpack_dequantize(want_p, want_m, s, None, 4, tile.shape)
    x, S = _repeat(tile, REP_S24), _repeat(s, REP_S24)
    _report(f"sparse24 int4 {mode}", x.numel(), x.numel() * 2, 2 ** 31)
    n0 = N.launch_count()
    packed, mask = ops.sparse24_quantize_pack(x, S, None, a)
    assert N.launch_count() - n0 == 1, "the fused 2:4 + int4 kernel must take the tensor"
    _tiled_equal(packed, want_p.to(DEV), "sparse24 packed words")
    _tiled_equal(mask, want_m.to(DEV), "sparse24 mask bytes")
    del x
    n0 = N.launch_count()
    dense = ops.sparse24_unpack_dequantize(packed, mask, S, None, 4, (TILE_ROWS * REP_S24, COLS))
    assert N.launch_count() - n0 == 1, "the fused decompress kernel must take the tensor"
    _tiled_equal(dense, want_d.to(DEV), "sparse24 dense result")


# ---- 4. converters --------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_dequantize_block_fp8():
    """ops.dequantize_block_fp8 (the streaming DequantF32ScaleOp) with 128 x 128 blocks on 4.30 GB of fp8: guards the fp8 byte offset
    past 2^32, the bf16 output offset past 2^33 bytes and the block-row index of the scale"""
    _need_memory()
    g = torch.Generator().manual_seed(24)
    tile = (torch.randn(FP8_TILE_ROWS, COLS, generator=g) * 20).to(torch.float8_e4m3fn)
    s = torch.rand(FP8_TILE_ROWS // 128, COLS // 128, generator=g) * 0.01 + 0.001
    want = oracle.dequantize_block_fp8(tile, s, (128, 128))
    w = _repeat(tile, REP_FP8)
    _report("dequantize_block_fp8", w.numel(), w.numel() * 2, 2 ** 32)
    _tiled_equal(ops.dequantize_block_fp8(w, _repeat(s, REP_FP8), (128, 128)), want.to(DEV), "dequantize_block_fp8")


@pytest.mark.gpu
def test_awq_repack():
    """ops.awq_repack (ct_awq_repack_int4) of a qweight [4096, 131136] whose weight_packed [1049088, 512] int32 is 2.15 GB: guards
    the output word offset past 2^31 bytes and the input word offset k * (N / 8) + n / 8.  The qweight repeats a [4096, 96] tile along
    its columns, so weight_packed repeats the tile's along its rows"""
    _need_memory()
    g = torch.Generator().manual_seed(25)
    tile = torch.randint(-2 ** 31, 2 ** 31, (AWQ_K, AWQ_TILE_WORDS), dtype=torch.int64, generator=g).to(torch.int32)
    want = oracle.awq_repack(tile)
    q = tile.to(DEV).repeat(1, REP_AWQ)
    out = ops.awq_repack(q)
    _report("awq_repack", q.numel() * 8, out.numel() * 4, 2 ** 32)
    assert out.numel() * 4 > 2 ** 31
    _tiled_equal(out, want.to(DEV), "awq_repack")


# ---- 6. one multi-tensor launch past 2^32 elements ------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_batched_jobs_past_2_to_32_elements():
    """ops.batched(OP_QUANTIZE_PACK) with two W4A16 jobs of 2.20 G elements each (each below 2^32, 4.40 G together) in one launch:
    guards the uint32 tile_begin / tile_end accumulation across jobs and the dynamic tile claim"""
    _need_memory()
    a = QuantizationArgs(num_bits=4, type="int", symmetric=True, strategy="group", group_size=128)
    jobs, wants = [], []
    for seed, rep in ((26, REP_JOB_A), (27, REP_JOB_B)):
        tile = _tile(seed)
        s = (tile.float().unflatten(-1, (-1, 128)).abs().amax(-1) / 7.5 + 2.0 ** -12).to(torch.bfloat16)
        wants.append(oracle.pack_to_int32(oracle.quantize(tile, s, None, strategy="group", group_size=128, num_bits=4, dtype=torch.int8), 4))
        x, S = _repeat(tile, rep), _repeat(s, rep)
        out = torch.empty(x.shape[0], COLS // 8, dtype=torch.int32, device=DEV)
        p = ops._resolve(x, S, None, a, None)
        jobs.append((ops._desc(p, x.dtype, S.dtype, None, x.dtype, torch.int8, None, N.Q_INT, 4), x, S, None, out))
    total = sum(j[1].numel() for j in jobs)
    _report("batched quantize_pack, two jobs", total, jobs[1][4].numel() * 4, 2 ** 32)
    n0 = N.launch_count()
    ops.batched(N.OP_QUANTIZE_PACK, jobs, 0)
    assert N.launch_count() - n0 == 1, "both jobs must run in one launch"
    for i, (j, want) in enumerate(zip(jobs, wants)):
        _tiled_equal(j[4], want.to(DEV), f"batched job {i}")


# ---- the host-resident pipeline past 4 GB ------------------------------------------------------------------------------------------------
def _host_bytes_available() -> int:
    import os

    try:
        return os.sysconf("SC_AVPHYS_PAGES") * os.sysconf("SC_PAGE_SIZE")
    except (ValueError, OSError):
        return 0


@pytest.mark.gpu
def test_host_resident_quantize_pack_past_4gb():
    """ops.quantize_pack of a 2.42 G element bf16 weight held in host memory (4.8 GB, the staged pipeline): guards the host-side
    chunk offsets past 2^32 bytes"""
    if _host_bytes_available() < 24 * GIB:
        pytest.skip("needs 24 GB of available host memory")
    _need_memory(8)
    tile = _tile(28)
    a = QuantizationArgs(num_bits=4, type="int", symmetric=True, strategy="group", group_size=128)
    s = (tile.float().unflatten(-1, (-1, 128)).abs().amax(-1) / 7.5 + 2.0 ** -12).to(torch.bfloat16)
    rep = 3078                                                        # 2.42 G elements, 4.84 GB
    x, S = tile.repeat(rep, 1), s.repeat(rep, 1)
    _report("host-resident quantize_pack", x.numel(), x.numel() // 2, 2 ** 31)
    packed = ops.quantize_pack(x, S, None, a)
    assert not packed.is_cuda
    _tiled_equal(packed, oracle.pack_to_int32(oracle.quantize(tile, s, None, strategy="group", group_size=128, num_bits=4, dtype=torch.int8), 4),
                 "host-resident quantize_pack")


# ---- the checks bite: wrapped stand-ins on scaled-down tensors (CPU) ---------------------------------------------------------------------
SHRINK = 128     # columns of the CPU stand-ins: cols / SHRINK, so every offset of the full-size case scales by the same factor

# case: (tile rows, cols, repetitions, outputs as (name, output elements per row as a function of cols, bytes per element))
_ROW = lambda c: c                  # noqa: E731  one output element per input element
_GEOMETRY = {
    "dynamic token 16384": (TILE_ROWS, COLS, REP_BIG, [("out", _ROW, 2), ("scale", lambda c: 1, 2)]),
    "dynamic token 32768": (TILE_ROWS // 2, 2 * COLS, REP_BIG, [("out", _ROW, 2), ("scale", lambda c: 1, 2)]),
    "dynamic group 128": (TILE_ROWS, COLS, REP_BIG, [("out", _ROW, 2), ("scale", lambda c: c // 128, 2)]),
    "dynamic nvfp4": (TILE_ROWS, COLS, REP_BIG, [("out", _ROW, 2), ("scale", lambda c: c // 16, 4)]),
    "dynamic mxfp4": (TILE_ROWS, COLS, REP_BIG, [("out", _ROW, 2), ("scale", lambda c: c // 32, 2)]),
    "observe_quantize_pack g32 int4": (TILE_ROWS, COLS, REP_BIG, [("packed", lambda c: c // 8, 4), ("scale", lambda c: c // 32, 2)]),
    "observe_quantize_pack g128 int8": (TILE_ROWS, COLS, REP_BIG, [("packed", lambda c: c // 4, 4), ("scale", lambda c: c // 128, 2)]),
    "observe channel int4 / fp8": (TILE_ROWS, COLS, REP_BIG, [("packed", lambda c: c // 8, 4), ("codes", _ROW, 1), ("scale", lambda c: 1, 2)]),
    "observe nvfp4": (TILE_ROWS, COLS, REP_BIG, [("nibbles", lambda c: c // 2, 1), ("scale", lambda c: c // 16, 1)]),
    "one-byte outputs": (TILE_ROWS, COLS, REP_BIG, [("codes", _ROW, 1), ("bf16", _ROW, 2), ("8-bit words", lambda c: c // 4, 4),
                                                    ("fp4 nibbles", lambda c: c // 2, 1)]),
    "sparse24 int4": (TILE_ROWS, COLS, REP_S24, [("packed", lambda c: c // 16, 4), ("mask", lambda c: c // 8, 1), ("dense", _ROW, 2)]),
    "dequantize_block_fp8": (FP8_TILE_ROWS, COLS, REP_FP8, [("out", _ROW, 2)]),
    "awq_repack (output rows)": (AWQ_TILE_WORDS * 8, AWQ_K, REP_AWQ, [("weight_packed", lambda c: c // 8, 4)]),
}


def _wrap_rows(rows: int, cols: int, per_row: int, size: int):
    """the positions, in rows of the full-size case (a Fraction), where a 32-bit index wraps: an input element index, an output
    element index or an output byte offset reaching 2^31 or 2^32 (2^33 for bytes)"""
    n_in, n_out = rows * cols, rows * per_row
    at = set()
    for p in (2 ** 31, 2 ** 32, 2 ** 33):
        if p < n_in:
            at.add(Fraction(p, cols))
        if p < n_out:
            at.add(Fraction(p, per_row))
        if p < n_out * size:
            at.add(Fraction(p, per_row * size))
    return sorted(at)


def _read_wrapped(flat: torch.Tensor, w: int) -> torch.Tensor:
    """what a kernel that reads element i from i mod w produces"""
    out = flat.clone()
    for s in range(w, flat.numel(), w):
        out[s:s + w] = flat[: min(w, flat.numel() - s)]
    return out


def _write_wrapped(flat: torch.Tensor, w: int) -> torch.Tensor:
    """what a kernel that writes element i to i mod w leaves, over a buffer that already held the right answer (the worst case)"""
    out = flat.clone()
    for s in range(w, flat.numel(), w):
        out[: min(w, flat.numel() - s)] = flat[s:s + w]
    return out


def _stand_ins(tile_out: torch.Tensor, rep: int, per_row_small: int, wrap_rows):
    big = tile_out.repeat(rep, 1)
    for r in wrap_rows:
        w = math.floor(r * per_row_small)
        for name, fn in (("read", _read_wrapped), ("write", _write_wrapped)):
            yield f"{name} wrap at row {float(r):.0f}", fn(big.view(-1), w).view(big.shape)


@pytest.mark.parametrize("case", list(_GEOMETRY))
def test_wrapped_stand_ins_are_rejected(case):
    """for each case, on a tensor whose columns are shrunk by SHRINK: outputs whose element index or byte offset wraps at the case's
    powers of two (read or write, scaled by the same factor) fail `_tiled_equal`; the right output passes"""
    rows, cols, rep, outputs = _GEOMETRY[case]
    g = torch.Generator().manual_seed(30)
    cs = cols // SHRINK
    seen = 0
    for name, per_row, size in outputs:
        wraps = _wrap_rows(rows * rep, cols, per_row(cols), size)
        dt = {1: torch.uint8, 2: torch.int16, 4: torch.int32}[size]
        tile_out = torch.randint(-100, 100, (rows, per_row(cs)), generator=g).to(dt)
        _tiled_equal(tile_out.repeat(rep, 1), tile_out, f"{case} {name}")
        for what, bad in _stand_ins(tile_out, rep, per_row(cs), wraps):
            with pytest.raises(pytest.fail.Exception):
                _tiled_equal(bad, tile_out, f"{case} {name} {what}")
            seen += 1
    assert seen > 0, f"{case}: no output crosses a 32-bit limit"


def test_wrapped_batched_launch_is_rejected():
    """two jobs of one launch whose combined element index wraps at 2^32: the job that receives the wrapped elements fails"""
    g = torch.Generator().manual_seed(31)
    cs = COLS // SHRINK
    tiles = [torch.randint(-2 ** 31, 2 ** 31, (TILE_ROWS, cs // 8), dtype=torch.int64, generator=g).to(torch.int32) for _ in range(2)]
    reps = (REP_JOB_A, REP_JOB_B)
    flat = torch.cat([t.repeat(r, 1).view(-1) for t, r in zip(tiles, reps)])
    w = 2 ** 32 // 8 // SHRINK                                  # the output word of input element 2^32
    for fn in (_read_wrapped, _write_wrapped):
        bad = fn(flat, w)
        a = bad[: TILE_ROWS * REP_JOB_A * cs // 8].view(-1, cs // 8)
        b = bad[TILE_ROWS * REP_JOB_A * cs // 8:].view(-1, cs // 8)
        failed = 0
        for got, t in ((a, tiles[0]), (b, tiles[1])):
            try:
                _tiled_equal(got, t, "job")
            except pytest.fail.Exception:
                failed += 1
        assert failed, fn.__name__


@pytest.mark.parametrize("kind", ["int8 asym qparams", "gparam"])
def test_missed_planted_extreme_is_rejected(kind):
    """a per-tensor reduction whose element index wraps at 2^31 or 2^32 (scaled) never reads the planted last element: the planted
    check rejects its qparams, and accepts those of the whole tensor"""
    from compressed_tensors_b200.quantization.utils import generate_gparam

    tile = _tile(32, TILE_ROWS, COLS // SHRINK)
    planted = _planted_value(tile)
    x = tile.repeat(REP_BIG, 1).view(-1)
    x[-1] = planted
    assert x.numel() - 1 > 2 ** 32 // SHRINK

    def qparams(v):
        if kind == "gparam":
            return (generate_gparam(v.min(), v.max()).reshape(1),)
        return orc_qparams(v.min().reshape(1), v.max().reshape(1), num_bits=8, qtype="int", symmetric=False)

    if kind == "gparam":
        want = (generate_gparam(torch.minimum(tile.min(), planted), torch.maximum(tile.max(), planted)).reshape(1),)
    else:
        want = _planted_qparams(tile, planted, num_bits=8, qtype="int", symmetric=False)
    _check_planted(qparams(x), want, kind)
    for p in (2 ** 31, 2 ** 32):
        with pytest.raises(pytest.fail.Exception):
            _check_planted(qparams(x[: p // SHRINK]), want, f"{kind} wrapped at 2^{p.bit_length() - 1}")
