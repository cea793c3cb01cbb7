"""
Transforms (transform/) on the host: golden replay of tests/golden/transform.pt.gz (make_golden_transform.py, recorded from the
reference) through the CPU twin of ct_hadamard_transform (ImplBackend's eager body), the deliberate deviation and the reference's
errors, and apply_transform_config on small models.

Fused weights of the two Hadamard factories must equal the reference's bit for bit (float64 sums of bf16 / fp16 / fp32 weights are exact
here); online outputs must lie within (log2(n) + 1) * 2^-24 * |x_row| of the float64 product, plus half an ulp of the output dtype.
"""
import math

import pytest
import torch

from compressed_tensors_b200 import ops
from compressed_tensors_b200.transform import (
    TransformArgs,
    TransformConfig,
    TransformFactory,
    TransformScheme,
    apply_transform_config,
)
from compressed_tensors_b200.transform.utils.hadamard import deterministic_hadamard_matrix, is_pow2, random_hadamard_matrix
from tests import golden

GOLD = golden.load("transform")
HALF_ULP = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11, torch.float32: 0.0}


@pytest.fixture
def eager(monkeypatch):
    monkeypatch.setenv("CT_ENFORCE_EAGER", "1")


def dense_reference(weight, perm, x, inverse=False):
    """float64 x @ M / sqrt(n) row block by row block (block-diagonal over the last dimension)"""
    w = weight.double()
    if perm is not None:
        w = w[perm][:, perm]
    if inverse:
        w = w.T
    n = w.shape[0]
    return (x.double().unflatten(-1, (-1, n)) @ w).flatten(-2) / math.sqrt(n)


def assert_online_bound(y, ref, x, n):
    """each element within (log2 n + 1) 2^-24 |x_row| of the float64 product, plus half an ulp of y's dtype"""
    err = (y.double() - ref).abs().unflatten(-1, (-1, n))
    row_norm = x.double().unflatten(-1, (-1, n)).norm(dim=-1, keepdim=True)
    bound = (math.log2(n) + 1) * 2.0 ** -24 * row_norm + HALF_ULP[y.dtype] * ref.abs().unflatten(-1, (-1, n))
    assert bool((err <= bound).all()), float((err - bound).max())


def _case_id(c):
    return f"{c['type']}-{'rand' if c['randomize'] else 'fixed'}-{c['location']}-hd{c['head_dim']}-{c['dtype'].split('.')[-1]}"


@pytest.mark.parametrize("case", GOLD["factory"], ids=_case_id)
def test_factory_golden(case, eager):
    dtype = getattr(torch, case["dtype"].split(".")[-1])
    module = torch.nn.Linear(16, 64, bias=True).to(dtype)
    with torch.no_grad():
        module.weight.copy_(case["module_weight"])
        module.bias.copy_(case["module_bias"])
    scheme = TransformScheme(type=case["type"], randomize=case["randomize"], head_dim=case["head_dim"])
    factory = TransformFactory.from_scheme(scheme, name="", seed=42)
    args = TransformArgs(targets="Linear", location=case["location"])
    tfm = factory.create_transform(module, args)
    assert tfm.weight.dtype == case["weight"].dtype and torch.equal(tfm.weight, case["weight"])
    perm = getattr(tfm, "perm", None)
    assert (perm is None) == (case["perm"] is None)
    if perm is not None:
        assert torch.equal(perm, case["perm"])
    n = tfm.weight.shape[0]
    with torch.no_grad():
        if args.is_online():
            y = tfm(case["x"])
            assert y.dtype == case["y"].dtype and y.shape == case["y"].shape
            if case["type"] == "random-matrix":
                assert torch.equal(y, case["y"])
            else:
                assert_online_bound(y, dense_reference(tfm.weight, perm, case["x"]), case["x"], n)
        else:
            assert torch.equal(tfm(module.weight), case["fused_weight"])
            if case["location"] == "weight_output":
                assert torch.equal(tfm(module.bias.unsqueeze(-1)).squeeze(-1), case["fused_bias"])


def test_cpu_twin_matches_dense_product_for_every_form():
    """the four structured forms and their transposes, against the dense matrix the factories build"""
    gen = torch.Generator().manual_seed(0)
    for n in (2, 8, 64, 256):
        x = torch.randn(3, 2 * n, generator=gen)
        q = (torch.randint(0, 2, (n,), generator=gen) * 2 - 1).to(torch.int8)
        perm = torch.randperm(n, generator=gen)
        for sign in (None, q):
            for p in (None, perm):
                w = deterministic_hadamard_matrix(n, torch.float64)
                if sign is not None:
                    w = sign.double().unsqueeze(1) * w
                for inverse in (False, True):
                    ref = dense_reference(w, p, x, inverse)
                    y64 = _eager(x.bfloat16(), n, sign, p, inverse, torch.float64)
                    assert torch.equal(y64, dense_reference(w, p, x.bfloat16(), inverse).float().bfloat16())
                    assert_online_bound(_eager(x, n, sign, p, inverse, torch.float32), ref, x, n)


def _eager(*args):
    from compressed_tensors_b200.utils import ImplBackend

    return ImplBackend.call("hadamard_transform_eager", *args)


def test_errors_and_deviation():
    for size in (32, 48, 768):
        with pytest.raises(NotImplementedError, match=str(size)):
            random_hadamard_matrix(size)
    for size in (0, -4):
        with pytest.raises(ValueError):
            deterministic_hadamard_matrix(size)
    with pytest.raises(ValueError):
        deterministic_hadamard_matrix(48)
    assert is_pow2(64) and not is_pow2(48) and not is_pow2(0)
    with pytest.raises(ValueError):
        ops.hadamard_transform(torch.zeros(4, 48), 48)
    with pytest.raises(NotImplementedError):
        ops.hadamard_transform(torch.zeros(1, 1 << 16), 1 << 16)
    with pytest.raises(ValueError):
        ops.hadamard_transform(torch.zeros(4, 24), 16)
    x = torch.zeros(4, 16)
    for sign, perm in ((torch.ones(8, dtype=torch.int8), None), (None, torch.arange(8)), (None, torch.arange(16).flip(0) + 1),
                       (None, torch.zeros(16, dtype=torch.int64)), (None, torch.arange(16.0))):
        with pytest.raises(ValueError):
            ops.hadamard_transform(x, 16, sign, perm)
    module = torch.nn.Linear(48, 48)
    with pytest.raises(ValueError):
        TransformFactory.from_scheme(TransformScheme(type="hadamard"), name="").create_transform(
            module, TransformArgs(targets="Linear", location="input"))
    with pytest.raises(NotImplementedError, match="48"):
        TransformFactory.from_scheme(TransformScheme(type="random-hadamard"), name="").create_transform(
            module, TransformArgs(targets="Linear", location="input"))


def test_random_hadamard_is_signed_sylvester():
    """the deviation's premise: diag(Q) . H_n with Q drawn as the reference draws it (randint in the matrix dtype, then 2Q - 1)"""
    for n in (2, 64, 1024):
        m = random_hadamard_matrix(n, torch.float32, gen=torch.Generator().manual_seed(5))
        q = torch.randint(0, 2, (n,), generator=torch.Generator().manual_seed(5), dtype=torch.float32) * 2 - 1
        assert torch.equal(m, q.unsqueeze(1) * deterministic_hadamard_matrix(n, torch.float32))


@pytest.mark.parametrize("type_", ("hadamard", "random-hadamard", "random-matrix"))
@pytest.mark.parametrize("randomize", (True, False))
@pytest.mark.parametrize("embed_loc", ("weight_output", "output"))
@pytest.mark.parametrize("linear_loc", ("input", "weight_input"))
def test_embedding_and_linear(type_, randomize, embed_loc, linear_loc):
    torch.manual_seed(0)
    model = torch.nn.Sequential(torch.nn.Embedding(2, 4), torch.nn.Linear(4, 8, bias=False))
    ids = torch.randint(high=2, low=0, size=(17, 5, 2))
    expected = model(ids)
    config = TransformConfig(config_groups={"": TransformScheme(type=type_, randomize=randomize, apply=[
        TransformArgs(targets="Embedding", location=embed_loc),
        TransformArgs(targets="Linear", location=linear_loc, inverse=True)])})
    apply_transform_config(model, config)
    assert torch.allclose(expected, model(ids), atol=1e-5, rtol=0.0)
    assert model.transform_config is config


def test_non_hadamard_weight_takes_the_dense_formula(eager):
    """a loaded weight that is not diag(Q) . H must not reach the butterfly"""
    module = torch.nn.Linear(16, 16, bias=False)
    tfm = TransformFactory.from_scheme(TransformScheme(type="hadamard"), name="").create_transform(
        module, TransformArgs(targets="Linear", location="input"))
    x = torch.randn(4, 16)
    assert_online_bound(tfm(x), dense_reference(tfm.weight, None, x), x, 16)
    with torch.no_grad():
        tfm.weight.mul_(0.5)
        tfm.weight[3, 5] = 0.25
    assert torch.equal(tfm(x), tfm._dense(x))


def _model_id(c):
    return f"{c['name']}{'-w4a16-kvfp8' if c['quant'] else ''}"


@pytest.mark.parametrize("case", GOLD["model"], ids=_model_id)
def test_model_golden_structure(case, eager):
    """parameter names / shapes / dtypes, tied-weight keys, logits and the transform_config written by update_config"""
    pytest.importorskip("transformers")
    from tests.test_gpu_transform import _without_version, run_model_case

    got = run_model_case(case, "cpu")
    assert got["params"] == case["params"]
    assert got["tied"] == case["tied"]
    assert _without_version(got["written"]) == _without_version(case["written"])
    # online rotations may differ from the reference's by one bf16 ulp per element (DESIGN.md section 3), and that reaches the
    # logits (|logit| < 2 here): one ulp of the top of their range, twice the largest difference seen on the CPU (2^-8)
    assert torch.allclose(got["logits"].float(), case["logits"].float(), atol=2.0 ** -7, rtol=0.0), \
        float((got["logits"].float() - case["logits"].float()).abs().max())
