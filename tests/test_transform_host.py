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


def assert_fp64_result(y, ref, x, n):
    """fp64 compute: 16-bit inputs give the float64 value rounded through fp32 (their sums are exact in float64), fp32 inputs lie within
    half an fp32 ulp plus (log2 n + 1) 2^-53 |x_row| of it"""
    if x.dtype != torch.float32:
        assert torch.equal(y, ref.float().to(x.dtype)), int((y.double() != ref.float().to(x.dtype).double()).sum())
        return
    err = (y.double() - ref).abs().unflatten(-1, (-1, n))
    row_norm = x.double().unflatten(-1, (-1, n)).norm(dim=-1, keepdim=True)
    bound = (math.log2(n) + 1) * 2.0 ** -53 * row_norm + 2.0 ** -24 * ref.abs().unflatten(-1, (-1, n))
    assert bool((err <= bound).all()), float((err - bound).max())


def fwht64(z):
    """z . H_n along the last dimension in float64 (n its length, a power of two), by recursive halves:
    (a, b) . H_2m = ((a + b) . H_m, (a - b) . H_m), the halves taken first (the kernel pairs neighbours first)"""
    z = z.double()
    h = z.shape[-1] // 2
    while h >= 1:
        v = z.unflatten(-1, (-1, 2, h))
        z = torch.stack((v[..., 0, :] + v[..., 1, :], v[..., 0, :] - v[..., 1, :]), -2).flatten(-3)
        h //= 2
    return z


def structured_matrix(n, sign=None, perm=None, inverse=False):
    """the dense M of hadamard.cu's header, from its definition: (diag(Q) . H)[perm][:, perm], transposed for the inverse;
    H is scipy's Sylvester matrix"""
    import scipy.linalg

    m = torch.from_numpy(scipy.linalg.hadamard(n).astype("float64"))
    if sign is not None:
        m = torch.where(sign < 0, -1.0, 1.0).double().unsqueeze(1) * m
    if perm is not None:
        m = m[perm][:, perm]
    return m.T if inverse else m


def structured_reference(x, n, sign=None, perm=None, inverse=False):
    """float64 x . M / sqrt(n), block-diagonal over the last dimension, for every order through fwht64.  With p = perm and Q = sign,
    M[i][j] = Q[p[i]] H[p[i]][p[j]], so y[j] = (z . H)[p[j]] with z[p[i]] = Q[p[i]] x[i]; M^T[i][j] = Q[p[j]] H[p[j]][p[i]], so
    y[j] = Q[p[j]] (z . H)[p[j]] with z[p[i]] = x[i].  test_fwht_reference_equals_dense_product checks this against
    structured_matrix.  Runs on x's device (plain float64 additions, the same on every device)."""
    xb = x.double().unflatten(-1, (-1, n))
    q = torch.ones(n, dtype=torch.float64, device=x.device) if sign is None else torch.where(sign.to(x.device) < 0, -1.0, 1.0).double()
    p = torch.arange(n, device=x.device) if perm is None else perm.to(x.device)
    z = torch.empty_like(xb)
    z[..., p] = xb if inverse else xb * q[p]
    y = fwht64(z)[..., p]
    if inverse:
        y = y * q[p]
    return y.flatten(-2) / math.sqrt(n)


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


def transform_cases(n, gen):
    """(sign, perm, inverse) for the four structured forms and their transposes"""
    q = (torch.randint(0, 2, (n,), generator=gen) * 2 - 1).to(torch.int8)
    perm = torch.randperm(n, generator=gen)
    return [(s, p, inv) for s in (None, q) for p in (None, perm) for inv in (False, True)]


def test_fwht_reference_equals_dense_product():
    """structured_reference (recursive halves) against x . M with M built densely from scipy's Sylvester matrix, bit for bit on
    bf16-valued inputs (their float64 sums are exact, so the two summation orders agree)"""
    gen = torch.Generator().manual_seed(1)
    for log2_n in range(1, 13):
        n = 1 << log2_n
        x = torch.randn(3, 2 * n, generator=gen).bfloat16()
        for sign, p, inverse in transform_cases(n, gen):
            m = structured_matrix(n, sign, p, inverse)
            if sign is None and p is None:
                assert torch.equal(m, deterministic_hadamard_matrix(n, torch.float64))
            dense = (x.double().unflatten(-1, (-1, n)) @ m).flatten(-2) / math.sqrt(n)
            assert torch.equal(structured_reference(x, n, sign, p, inverse), dense), (n, sign is None, p is None, inverse)


def test_cpu_twin_matches_dense_product_for_every_form():
    """every order 2^1 .. 2^15, dtype, precision, the four structured forms and their transposes, against the float64 reference"""
    gen = torch.Generator().manual_seed(0)
    for log2_n in range(1, 16):
        n = 1 << log2_n
        for dtype in (torch.bfloat16, torch.float16, torch.float32):
            x = torch.randn(3 if n <= 4096 else 1, 2 * n, generator=gen).to(dtype)
            for sign, p, inverse in transform_cases(n, gen):
                ref = structured_reference(x, n, sign, p, inverse)
                assert_fp64_result(_eager(x, n, sign, p, inverse, torch.float64), ref, x, n)
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


def _random_hadamard_transform(device):
    module = torch.nn.Linear(64, 64).to(device)
    return TransformFactory.from_scheme(TransformScheme(type="random-hadamard", randomize=True), name="", seed=7).create_transform(
        module, TransformArgs(targets="Linear", location="input"))


def check_tracked_writes_are_followed(device):
    """a new signed Hadamard weight and permutation written by copy_, load_state_dict, update_offload_parameter or assignment to
    .data is what the next call computes with"""
    from compressed_tensors_b200.offload import update_offload_parameter

    gen = torch.Generator().manual_seed(8)
    x = torch.randn(4, 64, generator=gen).to(device)
    for write in ("copy_", "load_state_dict", "update_offload_parameter", "assign .data"):
        t = _random_hadamard_transform(device)
        before = t(x)
        q = (torch.randint(0, 2, (64,), generator=gen) * 2 - 1).to(torch.int8).to(device)
        perm = torch.randperm(64, generator=gen).to(device)
        weight = q.to(t.weight.dtype).unsqueeze(1) * deterministic_hadamard_matrix(64, t.weight.dtype, device)
        if write == "copy_":
            with torch.no_grad():
                t.weight.copy_(weight)
                t.perm.copy_(perm)
        elif write == "load_state_dict":
            t.load_state_dict({"weight": weight, "perm": perm})
        elif write == "update_offload_parameter":
            update_offload_parameter(t, "weight", weight)
            update_offload_parameter(t, "perm", perm)
        else:
            t.weight.data = weight
            t.perm.data = perm
        y = t(x)
        assert not torch.equal(y, before), write
        assert torch.equal(y, ops.hadamard_transform(x, 64, q, perm)), write
        assert_online_bound(y.cpu(), structured_reference(x.cpu(), 64, q, perm), x.cpu(), 64)


def check_data_writes_keep_the_verified_snapshot(device):
    """in-place writes through .data are not tracked: the transform keeps computing with the signs and permutation it verified, never
    with the stale signs and the live permutation; the next tracked write brings both up to date"""
    gen = torch.Generator().manual_seed(9)
    x = torch.randn(4, 64, generator=gen).to(device)
    t = _random_hadamard_transform(device)
    before = t(x)
    q = t.weight[:, 0].detach().clone()
    other = torch.randperm(64, generator=gen).to(device)
    t.weight.data.mul_(-1)                  # diag(-Q) . H: still a signed Hadamard matrix
    t.perm.data.copy_(other)                # still a permutation
    assert torch.equal(t(x), before)
    with torch.no_grad():
        t.weight.mul_(1)
        t.perm.add_(0)
    assert torch.equal(t(x), ops.hadamard_transform(x, 64, -q, other))
    # the op on its own: the permutation it checked, not one written through .data afterwards
    perm = torch.randperm(64, generator=gen).to(device)
    y = ops.hadamard_transform(x, 64, None, perm)
    perm.data.copy_(torch.randperm(64, generator=gen).to(device))
    assert torch.equal(ops.hadamard_transform(x, 64, None, perm), y)
    perm.add_(0)
    assert not torch.equal(ops.hadamard_transform(x, 64, None, perm), y)


def test_tracked_writes_are_followed(eager):
    check_tracked_writes_are_followed("cpu")


def test_data_writes_keep_the_verified_snapshot(eager):
    check_data_writes_keep_the_verified_snapshot("cpu")


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
