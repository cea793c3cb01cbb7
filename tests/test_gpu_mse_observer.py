"""
The MSE weight observer on the H100: the MSE mode of ct_observe_quantize_pack_int32 (GROUP int, W4A16 / W4A16_ASYM / W8A16) against
the torch path and the float64 rule, its stop-step fix-up, the min-max outputs it must leave alone, the entry points that refuse an
MSE descriptor, and the torch path of the NVFP4 / MX observers (whose fake_quantize has no host twin).
"""
import ctypes

import numpy as np
import pytest
import torch

import compressed_tensors_b200.ops as ops
from compressed_tensors_b200 import _native as N
from compressed_tensors_b200.quantization import QuantizationArgs
from compressed_tensors_b200.quantization.utils.helpers import calculate_qparams
from tests import mse_model as MM
from tests.test_mse_observer_host import _args, _on_grid, _same, _weight


def _group_at(x, args, chosen, mse):
    g = x.unflatten(-1, (-1, args.group_size))
    mn, mx = g.amin(-1), g.amax(-1)
    p = torch.tensor(mse.shrink, dtype=torch.float32)[torch.as_tensor(chosen).cpu()].reshape(mn.shape).to(x.device)
    scale, zp = calculate_qparams((mn.float() * p).to(x.dtype), (mx.float() * p).to(x.dtype), args)
    zp = None if args.symmetric else zp
    return ops.quantize_pack(x, scale, zp, args), scale, zp


def _kernel(x, args):
    before = N.launch_count()
    with ops._mse_error_tables() as tables:
        out = ops.observe_quantize(x, args, pack=True)
    torch.cuda.synchronize()
    assert N.launch_count() - before == 2, "the MSE kernel and its fix-up, nothing else"
    return out, tables[0]


SHAPES = [(4096, 4096), (1024, 14336), (96, 768), (3, 1280)]


@pytest.mark.gpu
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("bits,sym,group", [(4, True, 128), (4, False, 128), (8, True, 128), (4, True, 32), (8, False, 256)],
                         ids=["w4g128", "w4asym", "w8g128", "w4g32", "w8asym256"])
def test_group_kernel(bits, sym, group, dtype, shape):
    args = _args(num_bits=bits, type="int", strategy="group", group_size=group, symmetric=sym)
    mse = ops._mse_params(args)
    x = _weight(*shape, dtype, heavy=True, seed=shape[0]).cuda()
    (q, scale, zp), table = _kernel(x, args)
    # (b) + (c): the rule on the kernel's own errors, and the outputs at its choice, bit for bit
    chosen, stop = MM.choose(table.double().numpy(), mse.patience)
    wq, ws, wz = _group_at(x, args, chosen, mse)
    assert _same(q, wq) and _same(scale, ws) and _same(zp, wz)
    # against the torch path: errors within 1e-4, the same choice wherever both tables decide alike
    with ops._mse_error_tables() as tables:
        tq, ts, tz = ops._observe_mse(x, args, mse, "pack")
    ref = tables[0].double().numpy()
    got = table.double().numpy()
    assert np.array_equal(got == 0, ref == 0)
    np.testing.assert_allclose(got, ref, rtol=1e-4, atol=0)
    tchosen, tstop = MM.choose(ref, mse.patience)
    flips = int((tchosen != chosen).sum())
    print(f"{flips} of {len(chosen)} groups chose another step on the torch path's errors (stop {stop} / {tstop})")
    assert flips <= max(2, len(chosen) // 100)
    same = torch.as_tensor(tchosen == chosen).to(x.device).reshape(scale.shape)
    assert torch.equal(scale[same].view(torch.int16), ts[same].view(torch.int16))
    # (d) no group worse than min-max on its own errors; the total strictly lower at 4 bits
    picked = got[np.arange(len(chosen)), chosen]
    assert np.all(picked <= got[:, 0]) and (bits == 8 or picked.sum() < got[:, 0].sum())


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_fixup_applies_the_stop_step(dtype):
    """(e) on the device: the last group's best step (4 or 5) is past the stop step 3, so the fix-up rewrites it with step 0"""
    args = _args(num_bits=4, type="int", strategy="group", group_size=32, symmetric=False, observer_kwargs={"patience": 3})
    mse = ops._mse_params(args)
    x = _on_grid(4, 256, 32, dtype)
    g = torch.Generator().manual_seed(21)
    x[-1, -32:] = (torch.randn(32, generator=g) * 0.02 * torch.exp(torch.randn(32, generator=g))).to(dtype)
    x = x.cuda()
    (q, scale, zp), table = _kernel(x, args)
    chosen, stop = MM.choose(table.double().numpy(), mse.patience)
    assert stop == 3 and chosen[-1] == 0 and table[-1, stop + 1:].lt(table[-1, 0]).any()
    assert all(_same(a, b) for a, b in zip((q, scale, zp), _group_at(x, args, np.zeros(len(chosen), np.int64), mse)))


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_nonfinite_groups_and_other_observers(dtype):
    """(f) NaN / inf / zero groups keep min-max; (h) every other observer, and a one-step search, give the min-max kernel's bytes"""
    base = dict(num_bits=4, type="int", strategy="group", group_size=128, symmetric=False)
    x = _weight(256, 1024, dtype, heavy=True).cuda()
    x[0, 3], x[1, 200], x[2, 256:384] = float("nan"), float("inf"), 0
    minmax = ops.observe_quantize(x, QuantizationArgs(**base), pack=True)
    for obs in ("minmax", "memoryless_minmax", "static_minmax", "imatrix_mse"):
        assert all(_same(a, b) for a, b in zip(ops.observe_quantize(x, QuantizationArgs(**base, observer=obs), pack=True), minmax))
    one = ops.observe_quantize(x, _args(**base, observer_kwargs={"maxshrink": 0.01}), pack=True)
    assert all(_same(a, b) for a, b in zip(one, minmax))
    (q, scale, zp), table = _kernel(x, _args(**base))
    for r, c in ((0, 0), (1, 1), (2, 2)):
        assert _same(scale[r, c:c + 1], minmax[1][r, c:c + 1]) and torch.equal(q[r, c * 16:(c + 1) * 16], minmax[0][r, c * 16:(c + 1) * 16])


@pytest.mark.gpu
def test_group_kernel_past_2_31_elements():
    args = _args(num_bits=4, type="int", strategy="group", group_size=128, symmetric=True, observer_kwargs={"norm": 2})
    mse = ops._mse_params(args)
    rows, cols = 2 ** 31 // 8192 + 64, 8192
    x = (torch.randn(rows, cols, device="cuda", dtype=torch.bfloat16) * 0.02)
    (q, scale, zp), table = _kernel(x, args)
    chosen, _ = MM.choose(table.double().numpy(), mse.patience)
    tail = slice(rows - 64, rows)
    wq, ws, _ = _group_at(x[tail], args, chosen.reshape(rows, -1)[tail].reshape(-1), mse)
    assert torch.equal(q[tail], wq) and _same(scale[tail], ws)


@pytest.mark.gpu
def test_entry_points_refuse_an_mse_descriptor():
    """nothing runs min-max on a descriptor that asks for MSE: the observers without a search (BLOCK, MX, TENSOR), and ct_batched's
    observer ops.  The block here is all zeros, which only an entry point that refuses it may be given."""
    lib = N.lib()
    x = torch.randn(64, 256, device="cuda", dtype=torch.bfloat16)
    blk = torch.zeros(512, dtype=torch.uint8, device="cuda")
    out = torch.empty(64 * 256, dtype=torch.int32, device="cuda")
    sc = torch.empty(64 * 256, dtype=torch.float32, device="cuda")
    s = N.stream_ptr(0)
    d = ops._qdesc(64, 256, 1, 16, 16, N.Q_FP4, 4, torch.ones(1, device="cuda").data_ptr(), x_dtype=x.dtype,
                   scale_dtype=torch.float8_e4m3fn, compute_dtype=torch.float32, q_dtype=x.dtype, seff_dtype=torch.float32)
    d.aux = blk.data_ptr()
    p = N.ptr
    calls = {
        "block": lambda: lib.ct_observe_quantize_block(ctypes.byref(d), p(x), p(sc), p(out), 0, s),
        "mx": lambda: lib.ct_observe_quantize_mx(ctypes.byref(d), p(x), p(sc), p(out), 0, s),
        "tensor": lambda: lib.ct_observe_tensor(ctypes.byref(d), p(x), 0, p(sc), None, 0, s),
        "quantize_tensor": lambda: lib.ct_observe_quantize_tensor(ctypes.byref(d), p(x), p(sc), None, p(out), 0, s),
    }
    for op in (7, 10, 13, 14):
        ins, scs, outs = (ctypes.c_void_p * 1)(x.data_ptr()), (ctypes.c_void_p * 1)(sc.data_ptr()), (ctypes.c_void_p * 1)(out.data_ptr())
        calls[f"batched {op}"] = lambda op=op, ins=ins, scs=scs, outs=outs: lib.ct_batched(op, 1, ctypes.byref(d), ins, scs, None, outs, 0, s)
    before = N.launch_count()
    for name, call in calls.items():
        assert call() == N.CT_E_UNSUPPORTED, name
    torch.cuda.synchronize()
    assert N.launch_count() == before


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32], ids=["bf16", "fp16", "f32"])
@pytest.mark.parametrize("scheme", ["nvfp4", "mxfp4", "mxfp8"])
def test_fp4_mx_search(scheme, dtype):
    """NVFP4 keeps the min-max global scale and searches its group-of-16 scales; MX searches its power-of-two scales.  The error table
    is checked against float64 errors of the library's own fake_quantize at each candidate."""
    if scheme.startswith("mx") and dtype == torch.float32:
        pytest.skip("MX scales are generated in bf16 / fp16")
    bits = 8 if scheme == "mxfp8" else 4
    if scheme == "nvfp4":
        args = _args(num_bits=4, type="float", strategy="tensor_group", group_size=16, scale_dtype=torch.float8_e4m3fn)
    else:
        args = _args(num_bits=bits, type="float", strategy="group", group_size=32, scale_dtype=torch.uint8)
    mse = ops._mse_params(args)
    x = _weight(32, 256, dtype, heavy=True).cuda()
    with ops._mse_error_tables() as tables:
        out = ops.observe_quantize_pack_nvfp4(x, args) if scheme == "nvfp4" else ops.observe_quantize_mx(x, args)
    (table,) = tables
    g = 16 if scheme == "nvfp4" else 32
    gs = out[2] if scheme == "nvfp4" else None
    xr = x.unflatten(-1, (-1, g))
    mn, mx = xr.amin(-1), xr.amax(-1)
    want = []
    for p in mse.shrink:
        scale, _ = calculate_qparams((mn.float() * p).to(dtype), (mx.float() * p).to(dtype), args, global_scale=gs)
        fq = ops.fake_quantize(x, scale, None, args, global_scale=gs)
        want.append(((fq.double() - x.double()).abs() ** mse.norm).unflatten(-1, (-1, g)).sum(-1).reshape(-1))
    want = torch.stack(want, 1).cpu().numpy()
    got = table.double().numpy()
    assert np.array_equal(got == 0, want == 0)
    np.testing.assert_allclose(got, want, rtol=1e-4, atol=0)
    chosen, _ = MM.choose(got, mse.patience)
    p = torch.tensor(mse.shrink)[torch.as_tensor(chosen)].reshape(mn.shape).cuda()
    scale, _ = calculate_qparams((mn.float() * p).to(dtype), (mx.float() * p).to(dtype), args, global_scale=gs)
    if scheme == "nvfp4":
        assert _same(out[0], ops.quantize_pack_fp4(x, scale, None, args, global_scale=gs)) and _same(out[1], scale.to(torch.float8_e4m3fn))
        assert _same(out[2], ops.observe_quantize_pack_nvfp4(x, args.model_copy(update={"observer": None}))[2])   # min-max global scale
    else:
        q = ops.quantize_pack_fp4(x, scale, None, args) if bits == 4 else ops.quantize(x, scale, None, args, dtype=torch.float8_e4m3fn)
        assert _same(out[0], q) and _same(out[1], ops.compress_mx_scale(scale, torch.uint8))
    picked = want[np.arange(want.shape[0]), chosen]
    assert np.all(picked <= want[:, 0] * (1 + 1e-4)) and (bits == 8 or picked.sum() < want[:, 0].sum())




# ---------------------------------------------------------------------------------------------------------------------------------
# the per-row CHANNEL kernel (FP8_DYNAMIC, W8A8, channel int) and the NVFP4 kernel (NVFP4A16 local scales)
# ---------------------------------------------------------------------------------------------------------------------------------
CHANNEL = {"fp8": dict(num_bits=8, type="float", strategy="channel", symmetric=True),
           "int8": dict(num_bits=8, type="int", strategy="channel", symmetric=True),
           "int4asym": dict(num_bits=4, type="int", strategy="channel", symmetric=False)}
NVFP4 = dict(num_bits=4, type="float", strategy="tensor_group", group_size=16, scale_dtype=torch.float8_e4m3fn)   # as NVFP4A16


def _run_mse(x, args, kind):
    """(outputs, error table) of the kernel path; exactly two launches: the search and its fix-up"""
    before = N.launch_count()
    with ops._mse_error_tables() as tables:
        if kind == "nvfp4":
            gs = ops.observe_tensor_gparam(x)
            torch.cuda.synchronize()
            before = N.launch_count()
            out = ops.observe_quantize_pack_nvfp4(x, args, global_scale=gs)
        else:
            out = ops.observe_quantize(x, args, pack=kind == "pack")
    torch.cuda.synchronize()
    assert N.launch_count() - before == 2, "the MSE kernel and its fix-up, nothing else"
    return out, tables[0]


def _outputs_at(x, args, chosen, mse, kind, gs=None):
    """calculate_qparams + the min-max path's output ops at each group's chosen step"""
    if kind == "nvfp4":
        g = x.unflatten(-1, (-1, 16))
        mn, mx = g.amin(-1), g.amax(-1)
    else:
        mn, mx = x.amin(-1, keepdim=True), x.amax(-1, keepdim=True)
    p = torch.tensor(mse.shrink, dtype=torch.float32)[torch.as_tensor(chosen).cpu()].reshape(mn.shape).to(x.device)
    scale, zp = calculate_qparams((mn.float() * p).to(x.dtype), (mx.float() * p).to(x.dtype), args, global_scale=gs)
    if kind == "nvfp4":
        return ops.quantize_pack_fp4(x, scale, None, args, global_scale=gs), scale.to(torch.float8_e4m3fn), gs
    zp = None if args.symmetric else zp
    if kind == "pack":
        return ops.quantize_pack(x, scale, zp, args), scale, zp
    return ops.quantize(x, scale, zp, args, dtype=args.pytorch_dtype()), scale, zp


def _check_kernel(x, args, kind):
    mse = ops._mse_params(args)
    out, table = _run_mse(x, args, kind)
    gs = out[2] if kind == "nvfp4" else None
    chosen, stop = MM.choose(table.double().numpy(), mse.patience)
    want = _outputs_at(x, args, chosen, mse, kind, gs)
    assert all(_same(a, b) for a, b in zip(out, want))
    with ops._mse_error_tables() as tables:
        ops._observe_mse(x, args, mse, "nvfp4" if kind == "nvfp4" else kind, args.pytorch_dtype() if kind == "codes" else None, global_scale=gs)
    ref, got = tables[0].double().numpy(), table.double().numpy()
    assert np.array_equal(got == 0, ref == 0)
    np.testing.assert_allclose(got, ref, rtol=1e-4, atol=0)
    tchosen, tstop = MM.choose(ref, mse.patience)
    flips = int((tchosen != chosen).sum())
    print(f"{kind}: {flips} of {len(chosen)} groups chose another step on the torch path's errors (stop {stop} / {tstop})")
    assert flips <= max(2, len(chosen) // 100)
    picked = got[np.arange(len(chosen)), chosen]
    assert np.all(picked <= got[:, 0])
    return out, table, chosen, stop


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(4096, 4096), (1024, 14336), (14336, 4096), (7, 776)], ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("scheme", list(CHANNEL))
def test_channel_kernel(scheme, dtype, shape):
    args = _args(**CHANNEL[scheme])
    x = _weight(*shape, dtype, heavy=True, seed=shape[1]).cuda()
    _check_kernel(x, args, "pack" if scheme == "int4asym" else "codes")


@pytest.mark.gpu
@pytest.mark.parametrize("shape", [(4096, 4096), (1024, 14336), (14336, 4096), (5, 96)], ids=lambda s: f"{s[0]}x{s[1]}")
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_nvfp4_kernel(dtype, shape):
    x = _weight(*shape, dtype, heavy=True, seed=shape[0]).cuda()
    out, table, chosen, _ = _check_kernel(x, _args(**NVFP4), "nvfp4")
    picked = table.double().numpy()[np.arange(len(chosen)), chosen]
    assert picked.sum() < table[:, 0].double().sum().item()


def _late_unit(kind, args, mse, dtype, width):
    """a group (NVFP4: 16 values with max |x| = 1) or row whose own errors improve at step 0, then not for `patience` steps, then
    again: found among seeded candidates with the torch path, which shares the kernel's decisions on them"""
    g = torch.Generator().manual_seed(7)
    pool = (torch.randn(512, width, generator=g) * torch.exp(torch.randn(512, width, generator=g))).to(dtype)
    if kind == "nvfp4":
        pool = (pool.float() / pool.float().abs().amax(-1, keepdim=True)).to(dtype).cuda()
        gs = ops.observe_tensor_gparam(pool)
    else:
        pool, gs = pool.cuda(), None
    with ops._mse_error_tables() as tables:
        ops._observe_mse(pool, args, mse, kind, args.pytorch_dtype() if kind == "codes" else None, global_scale=gs)
    e = tables[0].double().numpy()
    for r in range(e.shape[0]):
        imp, best = [], MM.FLT_MAX
        for v in e[r]:
            imp.append(v < best)
            best = v if v < best else best
        if imp[0] and not any(imp[1:mse.patience + 1]) and any(imp[mse.patience + 1:]):
            return pool[r]
    raise AssertionError("no candidate with a late improvement")


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("kind", ["nvfp4", "codes", "pack"])
def test_fixup_of_nvfp4_and_channel(kind, dtype):
    """zero groups / rows never improve after step 0, so the one late group alone decides `any`: the search stops at `patience` and
    the fix-up must rewrite that group, whose best step lies past the stop, with step 0"""
    scheme = {"nvfp4": NVFP4, "codes": CHANNEL["fp8"], "pack": CHANNEL["int4asym"]}[kind]
    args = _args(**scheme, observer_kwargs={"patience": 2})
    mse = ops._mse_params(args)
    width = 16 if kind == "nvfp4" else 64
    unit = _late_unit(kind, args, mse, dtype, width)
    x = torch.zeros((8, 64), dtype=dtype, device="cuda")
    x.view(-1)[-width:] = unit
    out, table = _run_mse(x, args, kind)
    chosen, stop = MM.choose(table.double().numpy(), mse.patience)
    last = table[-1].double().numpy()
    assert stop == mse.patience and chosen[-1] == 0 and (last[stop + 1:] < last[0]).any()
    gs = out[2] if kind == "nvfp4" else None
    assert all(_same(a, b) for a, b in zip(out, _outputs_at(x, args, chosen, mse, kind, gs)))


@pytest.mark.gpu
def test_wide_channel_rows_take_the_torch_path():
    """rows past 16384 columns (the cluster kernel) have no search on the device: the torch path runs, nothing runs min-max"""
    args = _args(**CHANNEL["fp8"])
    x = _weight(4, 16384 + 512, torch.bfloat16, heavy=True).cuda()
    mse = ops._mse_params(args)
    with ops._mse_error_tables() as tables:
        q, scale, _ = ops.observe_quantize(x, args)
    chosen, _ = MM.choose(tables[0].double().numpy(), mse.patience)
    assert all(_same(a, b) for a, b in zip((q, scale), _outputs_at(x, args, chosen, mse, "codes")[:2]))


# ---------------------------------------------------------------------------------------------------------------------------------
# write fences: every buffer an MSE call writes (outputs, the block's `any`, masks, errors) is cut from a poisoned, guard-banded one
# ---------------------------------------------------------------------------------------------------------------------------------
GUARD = 256
POISON = 0xA5


def _fenced(n_bytes):
    raw = torch.full((n_bytes + 2 * GUARD + 16,), POISON, dtype=torch.uint8, device="cuda")
    off = (-raw.data_ptr()) % 16 + GUARD
    return raw, raw[off:off + n_bytes]


def _guards_intact(raw, inner):
    lo = inner.data_ptr() - raw.data_ptr()
    hi = lo + inner.numel()
    return bool((raw[:lo] == POISON).all() and (raw[hi:] == POISON).all())


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["pack", "nvfp4", "codes"])
def test_mse_write_fences(kind):
    dtype = torch.bfloat16
    rows, cols = 96, 512
    x = _weight(rows, cols, dtype, heavy=True).cuda()
    if kind == "pack":
        args = _args(num_bits=4, type="int", strategy="group", group_size=128, symmetric=False)
        ng, shapes = rows * cols // 128, {"out": rows * cols // 2, "scale": rows * cols // 128 * 2, "zp": rows * cols // 128}
        d = ops._qdesc(rows, cols, 1, 128, cols // 128, N.Q_INT, 4, x_dtype=dtype, scale_dtype=dtype, compute_dtype=dtype,
                       zp_dtype=torch.int8, q_dtype=torch.int8)
    elif kind == "nvfp4":
        args = _args(**NVFP4)
        gs = ops.observe_tensor_gparam(x)
        ng, shapes = rows * cols // 16, {"out": rows * cols // 2, "scale": rows * cols // 16}
        d = ops._nvfp4_observe_desc(rows, cols, dtype, gs.data_ptr())
    else:
        args = _args(**CHANNEL["fp8"])
        ng, shapes = rows, {"out": rows * cols, "scale": rows * 2}
        d = ops._qdesc(rows, cols, 1, N.INF, 1, N.Q_FLOAT, 8, x_dtype=dtype, scale_dtype=dtype, compute_dtype=dtype, q_dtype=torch.float8_e4m3fn)
    mse = ops._mse_params(args)
    bufs = {k: _fenced(n) for k, n in shapes.items()}
    masks = _fenced(ng * 8)
    errors = _fenced(ng * mse.steps * 4)
    blk = N.MseBlock(steps=mse.steps, patience=mse.patience, norm=mse.norm, any=0xFFFF, masks=masks[1].data_ptr(), errors=errors[1].data_ptr())
    blk.shrink[:mse.steps] = list(mse.shrink)
    block = _fenced(ctypes.sizeof(N.MseBlock))
    block[1].copy_(torch.frombuffer(bytearray(bytes(blk)), dtype=torch.uint8))
    d.aux = block[1].data_ptr()
    lib, p, s = N.lib(), lambda k: ctypes.c_void_p(bufs[k][1].data_ptr()) if k in bufs else None, N.stream_ptr(0)
    if kind == "pack":
        rc = lib.ct_observe_quantize_pack_int32(ctypes.byref(d), N.ptr(x), p("scale"), p("zp"), p("out"), 0, s)
    elif kind == "nvfp4":
        rc = lib.ct_observe_quantize_pack_nvfp4(ctypes.byref(d), N.ptr(x), p("scale"), p("out"), 0, s)
    else:
        rc = lib.ct_observe_quantize_channel(ctypes.byref(d), N.ptr(x), p("scale"), None, p("out"), 0, s)
    assert rc == 0
    torch.cuda.synchronize()
    for name, (raw, inner) in {**bufs, "masks": masks, "errors": errors, "block": block}.items():
        assert _guards_intact(raw, inner), name
    # the block: only `any` changed, to the OR of the masks
    before, after = bytes(blk), bytes(block[1].cpu().numpy())
    at = N.MseBlock.any.offset
    assert after[:at] == before[:at] and after[at + 8:] == before[at + 8:]
    m = masks[1].view(torch.int64).cpu()
    anyv = int.from_bytes(after[at:at + 8], "little")
    ored = 0
    for v in m.tolist():
        ored |= v & 0xFFFFFFFFFFFFFFFF
    assert anyv == ored and not (errors[1] == POISON).all()
    # the outputs are those of the ops call, error table included
    with ops._mse_error_tables() as tables:
        ref = (ops.observe_quantize_pack_nvfp4(x, args, global_scale=gs) if kind == "nvfp4"
               else ops.observe_quantize(x, args, pack=kind == "pack"))
    assert torch.equal(errors[1].view(torch.float32).reshape(ng, mse.steps).cpu(), tables[0])
    assert torch.equal(bufs["out"][1].cpu(), ref[0].contiguous().view(torch.uint8).reshape(-1).cpu())
    assert torch.equal(bufs["scale"][1].cpu(), ref[1].contiguous().view(torch.uint8).reshape(-1).cpu())


# ---------------------------------------------------------------------------------------------------------------------------------
# convert_checkpoint with observer="mse"
# ---------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("preset", ["W4A16", "NVFP4A16", "FP8_DYNAMIC"])
def test_convert_checkpoint_with_mse(tmp_path, preset):
    import json

    from transformers import LlamaConfig, LlamaForCausalLM

    from compressed_tensors_b200.compressors import ModelCompressor
    from compressed_tensors_b200.entrypoints.convert import CompressedTensorsQuantizer, convert_checkpoint
    from compressed_tensors_b200.quantization import apply_quantization_config, preset_name_to_scheme
    from tests.golden import quantizer_checkpoint as qc
    from tests.test_quantizer_host import _read_all

    scheme = preset_name_to_scheme(preset, ["Linear"])
    scheme.weights.observer, scheme.weights.observer_kwargs = "mse", {"norm": 2.4, "patience": 4}
    tensors = qc.dense_tensors(torch.bfloat16)
    qc.write_checkpoint(str(tmp_path / "in"), tensors, torch.bfloat16)
    conv = CompressedTensorsQuantizer(scheme, ignore=list(qc.IGNORE))
    convert_checkpoint(str(tmp_path / "in"), str(tmp_path / "out"), conv, device="cuda")
    written = _read_all(str(tmp_path / "out"))
    with open(tmp_path / "out" / "config.json") as f:
        cfg = json.load(f)
    w = cfg["quantization_config"]["config_groups"]["group_0"]["weights"]
    assert w["observer"] == "mse" and w["observer_kwargs"] == {"norm": 2.4, "patience": 4}
    # the written tensors equal per-weight ops calls (NVFP4: with the fused group's shared global scale)
    args = scheme.weights
    names = [n[:-len(".weight")] for n in tensors if n.endswith(".weight") and f"{n[:-len('.weight')]}.weight_scale" in written]
    assert names
    expected = {}
    for name in names:
        wt = tensors[f"{name}.weight"].cuda()
        if preset == "NVFP4A16":
            gs = written[f"{name}.weight_global_scale"].cuda()
            packed, scale, _ = ops.observe_quantize_pack_nvfp4(wt, args, global_scale=gs)
            want = {"weight_packed": packed, "weight_scale": scale}
        elif preset == "W4A16":
            packed, scale, _ = ops.observe_quantize(wt, args, pack=True)
            want = {"weight_packed": packed, "weight_scale": scale}
        else:
            q, scale, _ = ops.observe_quantize(wt, args)
            want = {"weight_scale": scale}
            expected[name] = (scale, None)
        for k, v in want.items():
            assert _same(written[f"{name}.{k}"].cuda(), v), f"{name}.{k}"
        if preset != "FP8_DYNAMIC":
            expected[name] = (scale, written.get(f"{name}.weight_global_scale"))
    # decompress_model gives fake_quantize at the chosen qparams
    compressor = ModelCompressor.from_compression_config(cfg)
    kw = {k: v for k, v in cfg.items() if k not in ("architectures", "model_type", "torch_dtype", "quantization_config")}
    with torch.device("meta"):
        model = LlamaForCausalLM(LlamaConfig(**kw))
    apply_quantization_config(model, compressor.quantization_config)
    compressor.compress_model(model)
    model.load_state_dict({k: v.cuda() for k, v in written.items()}, assign=True, strict=True)
    compressor.decompress_model(model)
    for name, (scale, gs) in expected.items():
        wt = tensors[f"{name}.weight"].cuda()
        s = scale.to(wt.dtype) if preset != "NVFP4A16" else scale.float()
        want = ops.fake_quantize(wt, s.cuda(), None, args, global_scale=None if gs is None else gs.cuda())
        assert torch.equal(model.get_submodule(name).weight, want), name
