#!/usr/bin/env python
"""Launch each headline multi-tensor op a few times on `--layers` Llama-3-8B layers so that ncu can
capture one launch per kernel:  ncu --set full -k regex:stream_ ... python tools/profile_ops.py"""
import argparse
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from compressed_tensors_b200 import _native as N  # noqa: E402
from compressed_tensors_b200 import ops  # noqa: E402
from tools.headline_problems import build_problems  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--layers", type=int, default=4)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--ops", default="quantpack,unpackdeq,fp8_q,fp8_dq,fake_w4")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    P, OPS, n = build_problems(a.layers)
    for name in a.ops.split(","):
        for _ in range(a.reps):
            ops.batched(OPS[name][0], P[name], 0)
        torch.cuda.synchronize()
    print("launched", a.ops, "on", n, "elements")


if __name__ == "__main__":
    main()
