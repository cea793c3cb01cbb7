"""
The MSE weight observer's torch path on the CPU (the library's host twins): its error table against the float64 model of
tests/mse_model.py, the search rule, the outputs at the chosen step, the stop step, non-finite groups, observer_kwargs, and the
min-max outputs of every other observer.  The kernels are covered by tests/test_gpu_mse_observer.py.
"""
import numpy as np
import pytest
import torch

import compressed_tensors_b200.ops as ops
from compressed_tensors_b200.quantization import QuantizationArgs
from compressed_tensors_b200.quantization.utils.helpers import calculate_qparams
from tests import mse_model as MM

DT = {torch.bfloat16: "bf16", torch.float16: "fp16", torch.float32: "f32"}


@pytest.fixture(autouse=True)
def host_twins():
    prev = getattr(ops._mode, "cpu", False)
    ops._mode.cpu = True
    try:
        yield
    finally:
        ops._mode.cpu = prev


def _v(e):
    return getattr(e, "value", e)


def _weight(rows, cols, dtype, heavy, seed=0):
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(rows, cols, generator=g) * 0.02
    if heavy:   # a few large outliers per row: the min-max range is far too wide for the bulk
        w = w * torch.exp(torch.randn(rows, cols, generator=g) * 1.2)
    return w.to(dtype)


def _args(**kw):
    kw.setdefault("observer", "mse")
    return QuantizationArgs(**kw)


INT_CASES = [
    *[dict(num_bits=b, type="int", strategy="group", group_size=32, symmetric=s) for b in (2, 3, 4, 6, 8) for s in (True, False)],
    dict(num_bits=8, type="int", strategy="channel", symmetric=True),
    dict(num_bits=4, type="int", strategy="channel", symmetric=False),
    dict(num_bits=8, type="int", strategy="tensor", symmetric=False),
    dict(num_bits=8, type="float", strategy="channel", symmetric=True),
    dict(num_bits=8, type="float", strategy="tensor", symmetric=True),
    dict(num_bits=8, type="float", strategy="block", block_structure=[16, 32], symmetric=True),
]


def _ids(c):
    return "-".join(str(c[k]) for k in ("type", "num_bits", "strategy") if k in c) + ("-sym" if c.get("symmetric", True) else "-asym")


def _groups(args, shape):
    """group index of every element, number of groups"""
    rows, cols = shape
    r, c = np.meshgrid(np.arange(rows), np.arange(cols), indexing="ij")
    s = _v(args.strategy)
    if s in ("group", "tensor_group"):
        return r * (cols // args.group_size) + c // args.group_size, rows * (cols // args.group_size)
    if s == "channel":
        return r, rows
    if s == "tensor":
        return np.zeros_like(r), 1
    bh, bw = args.block_structure
    ncb = -(-cols // bw)
    return (r // bh) * ncb + c // bw, -(-rows // bh) * ncb


def _observe(x, args):
    with ops._mse_error_tables() as tables:
        out = ops.observe_quantize(x, args, pack=_v(args.strategy) == "group" and _v(args.type) == "int")
    assert len(tables) == 1
    return out, tables[0]


def _min_max(x, args):
    s = _v(args.strategy)
    if s == "group":
        g = x.unflatten(-1, (-1, args.group_size))
        return g.amin(-1), g.amax(-1)
    if s == "channel":
        return x.amin(-1, keepdim=True), x.amax(-1, keepdim=True)
    if s == "tensor":
        return x.amin().reshape(1), x.amax().reshape(1)
    bh, bw = args.block_structure
    r, c = x.shape
    p = torch.nn.functional.pad(x, (0, -(-c // bw) * bw - c, 0, -(-r // bh) * bh - r)).reshape(-(-r // bh), bh, -(-c // bw), bw)
    return p.amin(dim=(1, 3)), p.amax(dim=(1, 3))


def _at(x, args, chosen, mse):
    """calculate_qparams + quantize (+ pack) at each group's chosen step, with the library's public ops"""
    mn, mx = _min_max(x, args)
    p = torch.tensor(mse.shrink, dtype=torch.float32)[torch.as_tensor(chosen)].reshape(mn.shape)
    scale, zp = calculate_qparams((mn.float() * p).to(x.dtype), (mx.float() * p).to(x.dtype), args)
    zp = None if args.symmetric else zp
    if _v(args.strategy) == "group" and _v(args.type) == "int":
        return ops.quantize_pack(x, scale, zp, args), scale, zp
    return ops.quantize(x, scale, zp, args, dtype=args.pytorch_dtype()), scale, zp


def _same(a, b):
    if a is None or b is None:
        return a is None and b is None
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


@pytest.mark.parametrize("heavy", [False, True], ids=["gauss", "heavy"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16, torch.float32], ids=["bf16", "fp16", "f32"])
@pytest.mark.parametrize("case", INT_CASES, ids=_ids)
def test_int_fp8_search(case, dtype, heavy):
    args = _args(**case)
    mse = ops._mse_params(args)
    x = _weight(48, 256, dtype, heavy)
    (q, scale, zp), table = _observe(x, args)
    dt = DT[dtype]
    gid, ng = _groups(args, x.shape)
    kind = "fp8" if _v(args.type) == "float" else "int"
    want = MM.error_table(x.double().numpy(), gid, ng, dt, kind, args.num_bits, args.symmetric, np.array(mse.shrink), mse.norm)
    got = table.double().numpy()
    # (a) every entry within 1e-4 relative; zeros exactly
    assert got.shape == want.shape == (ng, mse.steps)
    assert np.array_equal(got == 0, want == 0)
    np.testing.assert_allclose(got, want, rtol=1e-4, atol=0)
    # (b) the rule on the returned table
    chosen, stop = MM.choose(got, mse.patience)
    lib_chosen, lib_stop = ops._mse_choose(table, mse)
    assert lib_stop == stop and np.array_equal(lib_chosen.numpy(), chosen)
    # (c) outputs at the chosen step
    wq, ws, wz = _at(x, args, chosen, mse)
    assert _same(q, wq) and _same(scale, ws) and _same(zp, wz)
    # (d) never worse than min-max per group; strictly better in total on heavy-tailed weights at 4 bits or fewer (at 8 bits the
    # min-max grid is already fine enough that shrinking rarely pays)
    picked = want[np.arange(ng), chosen]
    assert np.all(picked <= want[:, 0] * (1 + 1e-4))
    if heavy and kind == "int" and args.num_bits <= 4:
        assert picked.sum() < want[:, 0].sum()


def _on_grid(rows, cols, group, dtype, seed=1):
    """groups whose values all lie on their own min-max int4 grid: zero error at step 0, so they never improve afterwards"""
    g = torch.Generator().manual_seed(seed)
    codes = torch.randint(-8, 8, (rows, cols), generator=g).float()
    codes[:, ::group] = -8.0                      # every group spans the full range
    codes[:, 1::group] = 7.0
    return (codes * 2.0 ** -6).to(dtype)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_patience_stops_before_a_later_improvement(dtype):
    """(e) every group but one has error 0 at step 0 and never improves; the last one (picked with the model) improves at step 0 and
    next at step 4 (bf16) or 5 (fp16), after `patience` = 3 steps in which nothing improved: the search stops at step 3 first and
    that group keeps min-max"""
    args = _args(num_bits=4, type="int", strategy="group", group_size=32, symmetric=False, observer_kwargs={"patience": 3})
    mse = ops._mse_params(args)
    x = _on_grid(4, 256, 32, dtype)
    g = torch.Generator().manual_seed(21)
    x[-1, -32:] = (torch.randn(32, generator=g) * 0.02 * torch.exp(torch.randn(32, generator=g))).to(dtype)
    gid, ng = _groups(args, x.shape)
    e = MM.error_table(x.double().numpy(), gid, ng, DT[dtype], "int", 4, False, np.array(mse.shrink), mse.norm)
    assert np.all(e[:-1, 0] == 0)
    first = next(i for i in range(1, mse.steps) if e[-1, i] < e[-1, :i].min())
    assert first > mse.patience, "the constructed group must first improve after the stop step"
    chosen, stop = MM.choose(e, mse.patience)
    assert stop == mse.patience and chosen[-1] == 0
    (q, scale, zp), table = _observe(x, args)
    lib_chosen, lib_stop = ops._mse_choose(table, mse)
    assert lib_stop == mse.patience and int(lib_chosen[-1]) == 0
    assert all(_same(a, b) for a, b in zip((q, scale, zp), _at(x, args, np.zeros(ng, np.int64), mse)))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
def test_nonfinite_and_zero_groups_keep_min_max(dtype):
    """(f) a group holding a NaN or an inf, or only zeros, never improves: its outputs are the min-max ones"""
    args = _args(num_bits=4, type="int", strategy="group", group_size=32, symmetric=True)
    x = _weight(4, 128, dtype, heavy=True)
    x[0, 3] = float("nan")
    x[1, 40] = float("inf")
    x[2, 64:96] = 0
    (q, scale, zp), table = _observe(x, args)
    chosen, _ = ops._mse_choose(table, ops._mse_params(args))
    assert int(chosen[0]) == 0 and int(chosen[5]) == 0 and int(chosen[10]) == 0
    assert not torch.isfinite(table[0]).any() and not torch.isfinite(table[5]).any() and table[10].eq(0).all()
    mq, ms, _ = _at(x, args, np.zeros(16, np.int64), ops._mse_params(args))
    for g in (0, 5, 10):
        r, c = divmod(g, 4)
        assert _same(scale[r, c:c + 1], ms[r, c:c + 1]) and torch.equal(q[r, c * 4:(c + 1) * 4], mq[r, c * 4:(c + 1) * 4])


@pytest.mark.parametrize("kw,steps", [({"norm": 2}, 20), ({"grid": 50, "maxshrink": 0.3}, 15), ({"patience": 1}, 20), ({"maxshrink": 0.01}, 1)])
def test_observer_kwargs(kw, steps):
    """(g) the kwargs reach the search: steps, shrink factors, norm and patience"""
    args = _args(num_bits=4, type="int", strategy="group", group_size=32, symmetric=False, observer_kwargs=kw)
    mse = ops._mse_params(args)
    grid = float(kw.get("grid", 100.0))
    assert mse.steps == steps and mse.shrink == tuple(float(np.float32(1 - i / grid)) for i in range(steps))
    x = _weight(16, 128, torch.bfloat16, heavy=True)
    (q, scale, zp), table = _observe(x, args)
    gid, ng = _groups(args, x.shape)
    want = MM.error_table(x.double().numpy(), gid, ng, "bf16", "int", 4, False, np.array(mse.shrink), mse.norm)
    np.testing.assert_allclose(table.double().numpy(), want, rtol=1e-4, atol=0)
    chosen, stop = MM.choose(table.double().numpy(), mse.patience)
    assert _same(q, _at(x, args, chosen, mse)[0])
    if steps == 1:   # one candidate, p = 1: the min-max outputs
        assert all(_same(a, b) for a, b in zip((q, scale, zp), _at(x, args, np.zeros(ng, np.int64), mse)))


@pytest.mark.parametrize("kw", [{"shrink": 0.1}, {"maxshrink": 0.0}, {"maxshrink": 0.7}, {"grid": 1e9}, {"patience": 0},
                                {"patience": 2.5}, {"patience": "3"}, {"norm": 0}, {"norm": -1.0}, {"norm": float("inf")}, {"norm": float("nan")}])
def test_invalid_observer_kwargs(kw):
    args = _args(num_bits=4, type="int", strategy="group", group_size=32, observer_kwargs=kw)
    with pytest.raises(ValueError):
        ops.observe_quantize(_weight(2, 64, torch.bfloat16, False), args, pack=True)


@pytest.mark.parametrize("observer", [None, "minmax", "memoryless_minmax", "static_minmax", "imatrix_mse"])
def test_other_observers_are_min_max(observer):
    """(h) no observer other than mse / memoryless_mse reaches the search (their outputs are compared with the min-max kernels on
    the GPU)"""
    base = dict(num_bits=4, type="int", strategy="group", group_size=32, symmetric=False)
    assert ops._mse_params(QuantizationArgs(**base, observer=observer)) is None
    assert ops._mse_params(QuantizationArgs(**base, observer="memoryless_mse")).steps == 20
