"""
Random-hadamard transforms of orders n = K * 2^m (K a core of the reference's table of known Hadamard matrices) on the host: the CPU
twin of ct_hadamard_transform with a core against a float64 restatement, replay of tests/golden/transform_orders.pt.gz
(make_golden_transform_orders.py, recorded from the reference), building on meta and loading a checkpoint's weights.

Online outputs must lie within (m + K + 1) * 2^-24 * |x_block| of the float64 product plus half an ulp of the output dtype
(DESIGN.md section 3); fp64 compute of 16-bit inputs gives the float64 value rounded through fp32 exactly.
"""
import math

import pytest
import torch

from compressed_tensors_b200 import ops
from compressed_tensors_b200.transform import TransformArgs, TransformConfig, TransformScheme, apply_transform_config
from compressed_tensors_b200.transform.factory.hadamard import HadamardTransform, _core_factors
from compressed_tensors_b200.transform.utils.hadamard import random_hadamard_matrix, table_core_order
from tests import golden
from tests.test_transform_host import fwht64

GOLD = golden.load("transform_orders")
HALF_ULP = {torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11, torch.float32: 0.0}
DTYPES = (torch.bfloat16, torch.float16, torch.float32)


@pytest.fixture
def eager(monkeypatch):
    monkeypatch.setenv("CT_ENFORCE_EAGER", "1")


def _eager(*args, **kwargs):
    from compressed_tensors_b200.utils import ImplBackend

    return ImplBackend.call("hadamard_transform_eager", *args, **kwargs)


def core_reference(x, core, n, sign=None, perm=None, inverse=False):
    """float64 x . M / sqrt(n) for M = (diag(Q) . (C ⊗ H_{2^m})^T)[perm][:, perm] (transposed for the inverse), block-diagonal over
    the last dimension: z scattered and signed as in structured_reference, Y[c] = sum_a C[c][a] FWHT(Z[a]) (C^T for the inverse)"""
    k = core.shape[0]
    xb = x.double().unflatten(-1, (-1, n))
    q = torch.ones(n, dtype=torch.float64, device=x.device) if sign is None else torch.where(sign.to(x.device) < 0, -1.0, 1.0).double()
    p = torch.arange(n, device=x.device) if perm is None else perm.to(x.device)
    z = torch.empty_like(xb)
    z[..., p] = xb if inverse else xb * q[p]
    u = fwht64(z.unflatten(-1, (k, n // k)))
    c = core.double().to(x.device)
    u = torch.einsum("ca,...ad->...cd", c.T if inverse else c, u).flatten(-2)
    y = u[..., p]
    if inverse:
        y = y * q[p]
    return y.flatten(-2) / math.sqrt(n)


def dense_matrix(core, m):
    """(C ⊗ H_m)^T in float64"""
    h = torch.ones(1, 1, dtype=torch.float64)
    while h.shape[0] < m:
        h = torch.cat((torch.cat((h, h), 1), torch.cat((h, -h), 1)), 0)
    return torch.kron(core.double(), h).T


def assert_core_bound(y, ref, x, n, k, precision=torch.float32):
    """fp32: each element within (m + K + 1) 2^-24 |x_block| of the float64 product plus half an ulp of y's dtype.  fp64: 16-bit inputs
    give the float64 value through fp32 exactly (their sums are exact in float64), fp32 inputs lie within half an fp32 ulp plus
    (m + K + 1) 2^-53 |x_block| of it"""
    if precision == torch.float64 and x.dtype != torch.float32:
        want = ref.float().to(x.dtype)
        assert torch.equal(y.cpu(), want.cpu()), int((y.cpu().double() != want.cpu().double()).sum())
        return
    m = int(math.log2(n // k))
    err = (y.double() - ref).abs().unflatten(-1, (-1, n))
    row_norm = x.double().unflatten(-1, (-1, n)).norm(dim=-1, keepdim=True)
    if precision == torch.float64:
        bound = (m + k + 1) * 2.0 ** -53 * row_norm + 2.0 ** -24 * ref.abs().unflatten(-1, (-1, n))
    else:
        bound = (m + k + 1) * 2.0 ** -24 * row_norm + HALF_ULP[y.dtype] * ref.abs().unflatten(-1, (-1, n))
    assert bool((err <= bound).all()), float((err - bound).max())


def assert_near_reference(y, y_ref, ref, x, n, k):
    """the reference's output (a dense product of its own rounding) within twice the bound of ours: one ulp of 16-bit dtypes"""
    m = int(math.log2(n // k))
    row_norm = x.double().unflatten(-1, (-1, n)).norm(dim=-1, keepdim=True)
    tol = 2 * ((m + k + 1) * 2.0 ** -24 * row_norm + HALF_ULP[y.dtype] * ref.abs().unflatten(-1, (-1, n)))
    err = (y.double() - y_ref.double()).abs().unflatten(-1, (-1, n))
    assert bool((err <= tol).all()), float((err - tol).max())


def core_cases():
    """(K, m) for every golden core and every m with K * 2^m <= 2^15"""
    out = []
    for k in sorted(GOLD["cores"]):
        m = 1
        while k * m <= ops.HADAMARD_MAX_ORDER:
            out.append((k, m))
            m *= 2
    return out


def forms(n, gen):
    q = (torch.randint(0, 2, (n,), generator=gen) * 2 - 1).to(torch.int8)
    perm = torch.randperm(n, generator=gen)
    return [(s, p, inv) for s in (None, q) for p in (None, perm) for inv in (False, True)]


@pytest.mark.parametrize("k,m", core_cases(), ids=lambda v: str(v))
def test_cpu_twin_with_core_within_the_bound(k, m):
    core = GOLD["cores"][k]
    n = k * m
    gen = torch.Generator().manual_seed(k * 7919 + m)
    rows = 2 if n <= 4096 else 1
    for dtype in DTYPES:
        x = torch.randn(rows, 2 * n if n <= 1024 else n, generator=gen).to(dtype)
        for sign, perm, inverse in forms(n, gen):
            ref = core_reference(x, core, n, sign, perm, inverse)
            for precision in (torch.float32, torch.float64):
                y = _eager(x, n, sign, perm, inverse, precision, core=core)
                assert y.dtype == dtype and y.shape == x.shape
                assert_core_bound(y, ref, x, n, k, precision)


def test_core_reference_equals_dense_product():
    """core_reference is the dense x . M / sqrt(n) of hadamard.cu's header"""
    gen = torch.Generator().manual_seed(3)
    for k, m in ((12, 4), (20, 1), (28, 8)):
        n = k * m
        g = dense_matrix(GOLD["cores"][k], m)
        x = torch.randn(3, n, generator=gen, dtype=torch.float64)
        for sign, perm, inverse in forms(n, gen):
            w = g if sign is None else sign.double().unsqueeze(1) * g
            if perm is not None:
                w = w[perm][:, perm]
            if inverse:
                w = w.T
            torch.testing.assert_close(core_reference(x, GOLD["cores"][k], n, sign, perm, inverse), x @ w / math.sqrt(n),
                                       rtol=0, atol=1e-12)


@pytest.mark.parametrize("n", sorted(GOLD["matrices"]))
def test_reference_matrices_factor(n):
    """the reference's random_hadamard_matrix is diag(s) . (C ⊗ H_{2^m})^T with the K of table_core_order, C its table core up to
    the sign of each column a, and the factors read off the weight reproduce it"""
    w = GOLD["matrices"][n].double()
    k = table_core_order(n)
    s, c = _core_factors(w)
    m = n // k
    assert torch.equal(s.double().unsqueeze(1) * dense_matrix(c, m), w)
    if k in GOLD["cores"]:
        table = GOLD["cores"][k]
        col_sign = (c * table)[0]            # C = table . diag(d), d = +-1 per column
        assert torch.equal(c, table * col_sign)


def _factory_id(c):
    return f"{c['n']}-{'rand' if c['randomize'] else 'fixed'}-{c['location']}-{c['dtype'].split('.')[-1]}"


def loaded_transform(case, dense_raises, monkeypatch):
    """a HadamardTransform holding the golden weight and perm, as loading a checkpoint leaves it"""
    weight_dtype = getattr(torch, case["weight_dtype"].split(".")[-1])
    weight = torch.nn.Parameter(GOLD["weights"][case["weight_id"]].to(weight_dtype), requires_grad=False)
    perm = None if case["perm"] is None else torch.nn.Parameter(case["perm"].clone(), requires_grad=False)
    args = TransformArgs(targets="Linear", location=case["location"])
    tfm = HadamardTransform(weight, perm, TransformScheme(type="random-hadamard", randomize=case["randomize"]), args, torch.nn.Linear)
    if dense_raises:
        def no_dense(*a, **k):
            raise AssertionError("the dense formula ran")

        monkeypatch.setattr(tfm, "_dense", no_dense)
    return tfm


@pytest.mark.parametrize("case", GOLD["factory"], ids=_factory_id)
def test_factory_golden_on_the_twin(case, eager, monkeypatch):
    """loaded weights of orders 20 and 448 run the core path: fused weights equal the reference's bit for bit, online outputs lie
    within the bound of the float64 product and within one ulp of the reference's"""
    tfm = loaded_transform(case, True, monkeypatch)
    n = case["n"]
    with torch.no_grad():
        if case["location"] in ("input", "output"):
            x = case["x"]
            y = tfm(x)
            w = tfm.weight.double()
            if tfm.perm is not None:
                w = w[tfm.perm][:, tfm.perm]
            ref = x.double() @ w / math.sqrt(n)
            assert_core_bound(y, ref, x, n, table_core_order(n))
            assert_near_reference(y, case["y"], ref, x, n, table_core_order(n))
        else:
            module_weight = case["module_weight"]
            assert torch.equal(tfm(module_weight), case["fused_weight"])
            if case["location"] == "weight_output":
                assert torch.equal(tfm(case["module_bias"].unsqueeze(-1)).squeeze(-1), case["fused_bias"])


def test_large_order_on_the_twin():
    """n = 14336 (K = 224, m = 6): the signs and core read off the reference's first column and table give its output"""
    large = GOLD["large"]
    n = large["n"]
    core = GOLD["cores"][224]
    m = n // 224
    # the reference's matrix is diag(Q) . (C ⊗ H)^T, whose first column is Q[i] C[0][a(i)]: Q follows from it and C's first row
    q = large["first_column"] * core[0].repeat_interleave(m)
    for row in large["rows"]:
        x = row["x"]
        y = _eager(x, n, q, None, False, torch.float32, core=core)
        ref = core_reference(x, core, n, q)
        assert_core_bound(y, ref, x, n, 224)
        assert_near_reference(y, row["y"], ref, x, n, 224)


def test_meta_construction_draws_the_reference_signs():
    for n in (12, 20, 28, 32, 48, 448, 768, 5120, 11008, 14336, 28672):
        gen, want = torch.Generator().manual_seed(9), torch.Generator().manual_seed(9)
        w = random_hadamard_matrix(n, torch.float32, torch.device("meta"), gen)
        assert w.device.type == "meta" and w.shape == (n, n) and w.dtype == torch.float32
        torch.randint(low=0, high=2, size=(n,), generator=want, dtype=torch.float32)
        assert torch.equal(gen.get_state(), want.get_state())
    for n in (6, 520, 3 * 2 ** 16 + 2):
        with pytest.raises(NotImplementedError):
            random_hadamard_matrix(n, torch.float32, torch.device("meta"))
    for n in (32, 48, 768):
        with pytest.raises(NotImplementedError):
            random_hadamard_matrix(n, torch.float32, torch.device("cpu"))


def test_core_errors():
    x = torch.zeros(2, 48)
    core = GOLD["cores"][12]
    for bad in (core[:, :6], core.float() * 0.5, GOLD["cores"][20], torch.ones(5, 5, dtype=torch.int8), torch.ones(1, 1, 1)):
        with pytest.raises(ValueError):
            ops.hadamard_transform(x, 48, core=bad)
    with pytest.raises(NotImplementedError):
        ops.hadamard_transform(torch.zeros(1, 12 << 12), 12 << 12, core=core)
    with pytest.raises(ValueError):
        ops.hadamard_transform(torch.zeros(4, 48), 48)
    y = ops.hadamard_transform(torch.ones(2, 48), 48, core=core.float(), precision=torch.float64)   # a float core is accepted too
    assert y.shape == (2, 48)


def build_golden_model(case, device):
    """build the Llama of the case on meta, apply its configs there, materialise it on `device` and load the golden state dict on top
    of the seeded model's (the golden holds what differs from it); rotary buffers are not in the state dict and are copied"""
    from transformers import LlamaConfig, LlamaForCausalLM

    from compressed_tensors_b200.quantization import QuantizationConfig, apply_quantization_config

    cfg = LlamaConfig(num_hidden_layers=2, hidden_size=256, num_attention_heads=4, num_key_value_heads=2, head_dim=64, vocab_size=256,
                      intermediate_size=case["intermediate_size"], max_position_embeddings=128)
    torch.manual_seed(1234)
    seeded = LlamaForCausalLM(cfg).to(torch.bfloat16).eval()
    with torch.device("meta"):
        model = LlamaForCausalLM(cfg).to(torch.bfloat16).eval()
    apply_transform_config(model, TransformConfig(**case["config"]))
    if case["quant"]:
        fp8 = dict(num_bits=8, type="float", symmetric=True, strategy="tensor", dynamic=False)
        apply_quantization_config(model, QuantizationConfig(
            config_groups={"w": dict(targets=["Linear"], weights=dict(num_bits=4, type="int", symmetric=True, strategy="group",
                                                                      group_size=64, dynamic=False))},
            ignore=["lm_head"], kv_cache_scheme=fp8))
    model.to_empty(device=device)
    state = {k: v for k, v in seeded.state_dict().items()}
    for c in GOLD["model"]:
        for k, v in c["state"].items():
            state[k] = v.to(getattr(torch, c["signs"][k].split(".")[-1])) if k in c["signs"] else v
        if c is case:
            break
    missing, unexpected = model.load_state_dict(state, strict=False)
    assert not unexpected and all(k.startswith("lm_head") for k in missing), (missing, unexpected)
    for (name, buf), (_, want) in zip(model.named_buffers(), seeded.named_buffers()):
        buf.copy_(want)
    if "lm_head.weight" in missing:
        model.lm_head.weight = model.model.embed_tokens.weight
    return model


def _model_id(c):
    return f"{c['name']}{'-w4a16-kvfp8' if c['quant'] else ''}"


@pytest.mark.parametrize("case", GOLD["model"], ids=_model_id)
def test_model_load_flow_on_the_twin(case, eager):
    """meta build -> apply_transform_config -> to_empty -> load_state_dict(golden) -> the reference's logits within 2^-7"""
    pytest.importorskip("transformers")
    model = build_golden_model(case, "cpu")
    with torch.no_grad():
        logits = model(case["ids"], use_cache=False).logits
    assert torch.allclose(logits.float(), case["logits"].float(), atol=2.0 ** -7, rtol=0.0), \
        float((logits.float() - case["logits"].float()).abs().max())
