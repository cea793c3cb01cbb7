#!/usr/bin/env python
"""
Golden vectors for random-hadamard transforms of orders that are not powers of two (and 32), recorded by importing the reference
exactly like make_golden.py does.  Needs transformers.

    python tests/golden/make_golden_transform_orders.py   ->  tests/golden/transform_orders.pt.gz

- "cores": the K x K matrices of the reference's table of known Hadamard matrices for a few K, as int8.  They are test fixtures only:
  the package never reads them (it reads the core off a loaded weight).
- "matrices": random_hadamard_matrix(n, float32, seeded generator) for orders up to 768, as int8 (+-1).
- "factory": random-hadamard x randomize x the four locations x bf16 / fp16 / fp32 on Linear(n, 4) (input, weight_input) and
  Linear(4, n) (weight_output, output) for n in {20, 448}: the transform weight (int8, deduplicated in "weights"), perm, the input and
  online output, or the fused weight and bias.
- "large": two bf16 rows at n = 14336 (K = 224, the Llama-3-8B MLP order) through the reference's random-hadamard matrix (seeded like
  "matrices"): its first column (the signs Q) and the output.
- "model": the seeded 2-layer Llama of make_golden_kv.py with intermediate_size = 448 under an R4-only random-hadamard config (the
  down_proj input and weight_input inverse), alone and followed by W4A16 + FP8 kv_cache_scheme: the ids, the logits and every entry of
  the state dict that the seeded model (and, for the quantized case, the unquantized case before it) does not already hold with the
  same value (transform weights as int8 with their dtype).
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as mg  # noqa: E402  (imports the reference from a temp copy)
import make_golden_kv as mgkv  # noqa: E402
import make_golden_transform as mgt  # noqa: E402

from compressed_tensors.transform import (  # noqa: E402
    TransformArgs,
    TransformConfig,
    TransformFactory,
    TransformScheme,
    apply_transform_config,
)
from compressed_tensors.transform.utils.hadamard import _fetch_hadamard_divisor, random_hadamard_matrix  # noqa: E402
from compressed_tensors.quantization import QuantizationConfig, apply_quantization_config  # noqa: E402
from transformers import LlamaConfig, LlamaForCausalLM  # noqa: E402

CORE_ORDERS = (12, 20, 28, 32, 140, 160, 172, 192, 224)
MATRIX_ORDERS = (12, 20, 28, 32, 48, 224, 448, 640, 768)
FACTORY_ORDERS = (20, 448)
MATRIX_SEED = 5
LARGE_N = 14336
INTERMEDIATE = 448
R4 = dict(config_groups={
    "R4": dict(type="random-hadamard", apply=[
        dict(targets=["re:.*down_proj$"], location="input"),
        dict(targets=["re:.*down_proj$"], location="weight_input", inverse=True)]),
})


def as_signs(t):
    assert bool(((t == 1) | (t == -1)).all())
    return t.to(torch.int8)


def factory_cases(weights):
    out = []
    for n in FACTORY_ORDERS:
        for randomize in (False, True):
            for location in mgt.LOCATIONS:
                for dtype in mgt.DTYPES:
                    torch.manual_seed(7)
                    shape = (n, 4) if location in ("input", "weight_input") else (4, n)
                    module = torch.nn.Linear(*shape, bias=True).to(dtype)
                    factory = TransformFactory.from_scheme(TransformScheme(type="random-hadamard", randomize=randomize), name="",
                                                           seed=mgt.FACTORY_SEED)
                    args = TransformArgs(targets="Linear", location=location)
                    tfm = factory.create_transform(module, args)
                    w = as_signs(tfm.weight.detach())
                    idx = next((i for i, u in enumerate(weights) if torch.equal(u, w)), None)
                    if idx is None:
                        weights.append(w)
                        idx = len(weights) - 1
                    case = dict(n=n, randomize=randomize, location=location, dtype=str(dtype), weight_id=idx,
                                weight_dtype=str(tfm.weight.dtype), perm=getattr(tfm, "perm", None),
                                module_weight=module.weight.detach().clone(), module_bias=module.bias.detach().clone())
                    if case["perm"] is not None:
                        case["perm"] = case["perm"].detach().clone()
                    with torch.no_grad():
                        if args.is_online():
                            x = torch.randn(2, n, generator=torch.Generator().manual_seed(11)).to(dtype)
                            case["x"], case["y"] = x, tfm(x)
                        else:
                            case["fused_weight"] = tfm(module.weight)
                            if location == "weight_output":
                                case["fused_bias"] = tfm(module.bias.unsqueeze(-1)).squeeze(-1)
                    out.append(case)
    return out


def large_case():
    gen = torch.Generator().manual_seed(MATRIX_SEED)
    w = random_hadamard_matrix(LARGE_N, torch.float32, gen=gen)
    q = w[:, 0].clone()
    out = dict(n=LARGE_N, first_column=as_signs(q), rows=[])
    for dtype in (torch.bfloat16,):
        x = torch.randn(2, LARGE_N, generator=torch.Generator().manual_seed(13)).to(dtype)
        y = ((x.to(torch.float32) @ w) / torch.tensor(LARGE_N, dtype=torch.float32).sqrt()).to(dtype)
        out["rows"].append(dict(dtype=str(dtype), x=x, y=y))
    return out


def build_model():
    torch.manual_seed(mgkv.SEED)
    return LlamaForCausalLM(LlamaConfig(**dict(mgkv.MODEL, intermediate_size=INTERMEDIATE))).to(torch.bfloat16).eval()


def model_case(quant, base):
    model = build_model()
    apply_transform_config(model, TransformConfig(**R4))
    if quant:
        apply_quantization_config(model, QuantizationConfig(**mgt.W4A16_KV))
        mgt.calibrate(model)
    ids = torch.randint(0, mgkv.MODEL["vocab_size"], (1, 8), generator=torch.Generator().manual_seed(mgkv.SEED + 1))
    with torch.no_grad():
        logits = model(ids, use_cache=False).logits
    state, signs = {}, {}
    for k, v in model.state_dict().items():
        if k in base and base[k].dtype == v.dtype and torch.equal(base[k], v):
            continue
        if k.endswith("R4_input.weight"):
            state[k], signs[k] = as_signs(v), str(v.dtype)
        else:
            state[k] = v.detach().clone()
    base.update(state)
    return dict(name="r4", quant=quant, config=R4, intermediate_size=INTERMEDIATE, ids=ids, logits=logits, state=state, signs=signs)


def main():
    cores = {k: as_signs(_fetch_hadamard_divisor(k, torch.float32)) for k in CORE_ORDERS}
    matrices = {n: as_signs(random_hadamard_matrix(n, torch.float32, gen=torch.Generator().manual_seed(MATRIX_SEED)))
                for n in MATRIX_ORDERS}
    weights = []
    factory = factory_cases(weights)
    out = dict(matrix_seed=MATRIX_SEED, cores=cores, matrices=matrices, weights=weights, factory=factory, large=large_case(),
               model=[])
    base = build_model().state_dict()
    out["model"] = [model_case(q, base) for q in (False, True)]
    mg.save("transform_orders.pt", out)


if __name__ == "__main__":
    main()
