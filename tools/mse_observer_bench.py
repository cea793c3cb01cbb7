"""
MSE weight observer timing on the Llama-3-8B weight set (32 layers of q / k / v / o / gate / up / down, bf16) for W4A16 g128,
NVFP4A16 and FP8_DYNAMIC: the fused MSE kernels (search + fix-up) against the fused min-max kernels, and the torch path
(`ops._observe_mse`) on one layer's weights; then `convert_checkpoint` wall time with `mse` against min-max on the 4-shard synthetic
checkpoint of tests/golden/quantizer_checkpoint.py.  Prints one JSON line with the card's name, power limit and clocks, read in the
same run.

    python tools/mse_observer_bench.py [--reps 3] [--layers 32]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from compressed_tensors_b200 import ops  # noqa: E402
from compressed_tensors_b200.quantization import preset_name_to_scheme  # noqa: E402

LAYER = [(4096, 4096), (1024, 4096), (1024, 4096), (4096, 4096), (14336, 4096), (14336, 4096), (4096, 14336)]
SCHEMES = ("W4A16", "NVFP4A16", "FP8_DYNAMIC")


def _card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def _time(fn, reps):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    best = float("inf")
    for _ in range(reps):
        a.record()
        fn()
        b.record()
        b.synchronize()
        best = min(best, a.elapsed_time(b))
    return best


def _weights_args(preset, observer):
    scheme = preset_name_to_scheme(preset, ["Linear"])
    scheme.weights.observer = observer
    return scheme


def _calls(preset, args, ws, gss):
    if preset == "NVFP4A16":
        return lambda: [ops.observe_quantize_pack_nvfp4(w, args, global_scale=g) for w, g in zip(ws, gss)]
    return lambda: [ops.observe_quantize(w, args, pack=preset == "W4A16") for w in ws]


def _convert_seconds(scheme, src, reps):
    from compressed_tensors_b200.entrypoints.convert import CompressedTensorsQuantizer, convert_checkpoint
    from tests.golden import quantizer_checkpoint as qc

    best = float("inf")
    for _ in range(reps + 1):   # the first run warms up every kernel and the import path
        with tempfile.TemporaryDirectory() as out:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            convert_checkpoint(src, out, CompressedTensorsQuantizer(scheme, ignore=list(qc.IGNORE)), device="cuda")
            torch.cuda.synchronize()
            best = min(best, time.perf_counter() - t0)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--layers", type=int, default=32)
    a = ap.parse_args()
    g = torch.Generator(device="cuda").manual_seed(0)
    ws = [torch.randn(s, device="cuda", dtype=torch.bfloat16, generator=g) * 0.02 for s in LAYER]
    gss = [ops.observe_tensor_gparam(w) for w in ws]
    res = {"card": _card(), "workload": f"Llama-3-8B weights, {a.layers} layers (one layer timed, x {a.layers})",
           "elements": sum(w.numel() for w in ws) * a.layers}
    for preset in SCHEMES:
        minmax, mse = _weights_args(preset, None).weights, _weights_args(preset, "mse").weights
        m = ops._mse_params(mse)
        kind = {"W4A16": "pack", "NVFP4A16": "nvfp4", "FP8_DYNAMIC": "codes"}[preset]
        qdt = torch.float8_e4m3fn if preset == "FP8_DYNAMIC" else None
        r = {"minmax_fused_ms": _time(_calls(preset, minmax, ws, gss), a.reps) * a.layers,
             "mse_fused_ms": _time(_calls(preset, mse, ws, gss), a.reps) * a.layers,
             "mse_torch_ms": _time(lambda: [ops._observe_mse(w, mse, m, kind, qdt, global_scale=gs if kind == "nvfp4" else None)
                                            for w, gs in zip(ws, gss)], 1) * a.layers}
        r["mse_over_minmax"] = r["mse_fused_ms"] / r["minmax_fused_ms"]
        r["torch_over_mse"] = r["mse_torch_ms"] / r["mse_fused_ms"]
        res[preset] = r
    from tests.golden import quantizer_checkpoint as qc

    with tempfile.TemporaryDirectory() as src:
        qc.write_checkpoint(src, qc.dense_tensors(torch.bfloat16), torch.bfloat16)
        for preset in SCHEMES:
            mm = _convert_seconds(_weights_args(preset, None), src, a.reps)
            ms = _convert_seconds(_weights_args(preset, "mse"), src, a.reps)
            res[f"convert_{preset}"] = {"minmax_s": mm, "mse_s": ms, "mse_over_minmax": ms / mm}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
