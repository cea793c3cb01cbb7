"""
Random-hadamard transforms of orders n = K * 2^m on the H100: ct_hadamard_transform with a core against its CPU twin bit for bit
(every golden core and m, every form and inverse, both precisions, partial last tiles, more tiles than the grid, the fp64 scratch
tiles, strided [B, H, S, D] views and unaligned rows) and within the bound of DESIGN.md section 3 of the float64 product, the golden
factory cases and the n = 14336 case of tests/golden/transform_orders.pt.gz (make_golden_transform_orders.py) against the reference,
and the meta build -> load -> run flow of a Llama whose down_proj takes an order-448 rotation, on the kernel.
"""
import pytest
import torch

from compressed_tensors_b200 import _native as N
from compressed_tensors_b200 import ops
from compressed_tensors_b200.transform.factory.hadamard import HadamardTransform
from compressed_tensors_b200.transform.utils.hadamard import table_core_order
from tests.test_transform_orders_host import (
    DTYPES,
    GOLD,
    _eager,
    assert_core_bound,
    assert_near_reference,
    build_golden_model,
    core_cases,
    core_reference,
    forms,
    loaded_transform,
)

gpu = pytest.mark.gpu


def _no_dense(*a, **k):
    raise AssertionError("the dense formula ran")


@gpu
@pytest.mark.parametrize("k,m", core_cases(), ids=lambda v: str(v))
def test_kernel_with_core_equals_cpu_twin(k, m):
    """every form and inverse, both precisions and dtypes: the kernel equals the twin bit for bit and lies within the bound; rows of
    two blocks, and a partial last tile (one row more than a tile holds) for orders below 4096"""
    core = GOLD["cores"][k]
    n = k * m
    gen = torch.Generator().manual_seed(k * 31 + m)
    rows = max(3, 4096 // n + 1)
    for dtype in DTYPES:
        x = torch.randn(rows, 2 * n, generator=gen).to(dtype)
        xd = x.cuda()
        for sign, perm, inverse in forms(n, gen):
            ref = core_reference(x, core, n, sign, perm, inverse)
            for precision in (torch.float32, torch.float64):
                got = ops.hadamard_transform(xd, n, sign, perm, inverse, precision, core=core.cuda())
                assert torch.equal(got.cpu(), _eager(x, n, sign, perm, inverse, precision, core=core)), (k, m, dtype, precision)
                assert_core_bound(got.cpu(), ref, x, n, k, precision)


@gpu
@pytest.mark.parametrize("precision", (torch.float32, torch.float64))
def test_kernel_with_core_on_more_tiles_than_its_grid(precision):
    """K = 224 at n = 14336 and 28672: more rows than the grid's CTAs (persistent CTAs loop over tiles; fp64 at 28672 uses the global
    scratch tiles)"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    core = GOLD["cores"][224]
    gen = torch.Generator().manual_seed(5)
    for m, rows in ((64, 8 * sms + 5), (128, 2 * sms + 7)):
        n = 224 * m
        x = torch.randn(rows, n, generator=gen).to(torch.bfloat16)
        sign, perm, inverse = forms(n, gen)[-1]
        got = ops.hadamard_transform(x.cuda(), n, sign, perm, inverse, precision, core=core.cuda()).cpu()
        sel = torch.tensor([0, rows // 2, rows - 1])
        assert torch.equal(got[sel], _eager(x[sel], n, sign, perm, inverse, precision, core=core))


@gpu
@pytest.mark.parametrize("dtype", DTYPES)
def test_kernel_with_core_on_strided_views_and_unaligned_rows(dtype):
    """the transposed [B, H, S, D] view of a [B, S, H, D] tensor in place, and rows that start one element off 16 bytes"""
    core = GOLD["cores"][12]
    gen = torch.Generator().manual_seed(8)
    for n, d in ((12, 48), (96, 96), (12 * 64, 768)):
        base = torch.randn(2, 5, 3, d, generator=gen).to(dtype)
        view = base.cuda().transpose(1, 2)
        sign, perm, inverse = forms(n, gen)[5]
        got = ops.hadamard_transform(view, n, sign, perm, inverse, core=core.cuda())
        assert got.stride() == view.stride()
        assert torch.equal(got.cpu(), _eager(base.transpose(1, 2).contiguous(), n, sign, perm, inverse, core=core))
        flat = torch.randn(3 * d + 1, generator=gen).to(dtype)
        x = flat[1:].view(3, d)
        got = ops.hadamard_transform(x.cuda(), n, sign, perm, inverse, torch.float64, core=core.cuda())
        assert torch.equal(got.cpu(), _eager(x.contiguous(), n, sign, perm, inverse, torch.float64, core=core))


@gpu
@pytest.mark.parametrize("case", GOLD["factory"], ids=lambda c: f"{c['n']}-{c['randomize']}-{c['location']}-{c['dtype'][6:]}")
def test_factory_golden_on_the_kernel(case, monkeypatch):
    """loaded weights of orders 20 and 448 on CUDA run the kernel in one launch: fused weights equal the reference's bit for bit,
    online outputs lie within the bound"""
    tfm = loaded_transform(case, True, monkeypatch).cuda()
    n = case["n"]
    with torch.no_grad():
        if case["location"] in ("input", "output"):
            x = case["x"]
            tfm(x.cuda())
            launches = N.launch_count()
            y = tfm(x.cuda()).cpu()
            assert N.launch_count() - launches == 1
            w = tfm.weight.double().cpu()
            if tfm.perm is not None:
                w = w[tfm.perm.cpu()][:, tfm.perm.cpu()]
            ref = x.double() @ w / n ** 0.5
            assert_core_bound(y, ref, x, n, table_core_order(n))
            assert_near_reference(y, case["y"], ref, x, n, table_core_order(n))
        else:
            assert torch.equal(tfm(case["module_weight"].cuda()).cpu(), case["fused_weight"])
            if case["location"] == "weight_output":
                assert torch.equal(tfm(case["module_bias"].cuda().unsqueeze(-1)).squeeze(-1).cpu(), case["fused_bias"])


@gpu
def test_large_order_against_the_reference():
    large = GOLD["large"]
    n = large["n"]
    core = GOLD["cores"][224]
    q = large["first_column"] * core[0].repeat_interleave(n // 224)
    for row in large["rows"]:
        x = row["x"]
        y = ops.hadamard_transform(x.cuda(), n, q.cuda(), None, False, torch.float32, core=core.cuda()).cpu()
        assert torch.equal(y, _eager(x, n, q, None, False, torch.float32, core=core))
        ref = core_reference(x, core, n, q)
        assert_core_bound(y, ref, x, n, 224)
        assert_near_reference(y, row["y"], ref, x, n, 224)


@gpu
@pytest.mark.parametrize("case", GOLD["model"], ids=lambda c: f"{c['name']}{'-w4a16-kvfp8' if c['quant'] else ''}")
def test_model_load_flow_on_the_kernel(case, monkeypatch):
    """meta build -> apply_transform_config -> to_empty(cuda) -> load_state_dict(golden): the online R4 rotation of order 448 runs on
    the kernel (the dense formula raises) and the logits are the reference's within 2^-6"""
    pytest.importorskip("transformers")
    model = build_golden_model(case, "cuda")
    monkeypatch.setattr(HadamardTransform, "_dense", _no_dense)
    with torch.no_grad():
        logits = model(case["ids"].cuda(), use_cache=False).logits.cpu()
    assert torch.allclose(logits.float(), case["logits"].float(), atol=2.0 ** -6, rtol=0.0), \
        float((logits.float() - case["logits"].float()).abs().max())
