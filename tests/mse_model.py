"""
A float64 model of the MSE weight observer's grid search (observer "mse" / "memoryless_mse"), independent of ops.py and csrc/.

For each group and step i < steps = int(maxshrink * grid):
  p_i          float32(1 - i / grid)
  lo, hi       min / max of the group shrunk by p_i: x_dtype(float32(min) * p_i)  (torch's tensor * python float)
  qparams      calculate_qparams(lo, hi) (quantization/utils/helpers.py:74-131), each op rounded to the x dtype
  e(i)         sum over the group of |fake_quantize(x) - x| ** norm, exact in float64
Step i improves a group when e(i) < min(FLT_MAX, e(0 .. i-1)); S is the first step that ends `patience` steps in which no group
improved (steps - 1 if none); a group takes its last improving step <= S, or 0.

The integer and FP8 arithmetic is tests/int_fp8_model.py's; values are numpy float64 arrays holding values of "bf16", "fp16" or "f32".
"""
import numpy as np

from tests import int_fp8_model as M

FLT_MAX = float(np.finfo(np.float32).max)
EPS = {"bf16": 2.0 ** -7, "fp16": 2.0 ** -10, "f32": 2.0 ** -23}


def shrink(maxshrink=0.20, grid=100.0):
    steps = int(maxshrink * grid)
    return np.array([1 - i / grid for i in range(steps)], np.float64).astype(np.float32).astype(np.float64)


def qparams(mn, mx, dt, kind, bits, symmetric):
    """calculate_qparams of float64 min / max of dt for integer (kind "int") or float8 (kind "fp8") codes: (scale, zero point or None)"""
    qmin, qmax = M.q_range(kind, bits)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        lo, hi = np.minimum(mn, 0.0), np.maximum(mx, 0.0)
        if symmetric:
            s = M.op(np.maximum(np.abs(lo), np.abs(hi)) / ((qmax - qmin) / 2), dt)
            z = None
        else:
            s = M.op(M.op(hi - lo, dt) / (qmax - qmin), dt)
            z = np.clip(M.op(qmin - M.op(lo / s, dt), dt), qmin, qmax)
            z = np.round(np.clip(z, -128.0, 127.0))
            z = np.where(np.isnan(z), 0.0, z)
        s = np.where(s == 0, EPS[dt], s)
    return s, z


def candidate(mn, mx, p, dt):
    """the shrunk range of step p: float32 product, rounded to dt"""
    return M.rn(M.rn(mn * p, "f32"), dt), M.rn(M.rn(mx * p, "f32"), dt)


def error_table(x, group_of, n_groups, dt, kind, bits, symmetric, p, norm):
    """e[g, i] for x (float64 values of dt, any shape) whose element k belongs to group group_of[k]"""
    x = np.asarray(x, np.float64).reshape(-1)
    gid = np.asarray(group_of).reshape(-1)
    mn = np.full(n_groups, np.inf)
    mx = np.full(n_groups, -np.inf)
    np.minimum.at(mn, gid, x)
    np.maximum.at(mx, gid, x)
    nan = np.zeros(n_groups, bool)
    np.logical_or.at(nan, gid, np.isnan(x))
    mn, mx = np.where(nan, np.nan, mn), np.where(nan, np.nan, mx)
    e = np.zeros((n_groups, len(p)))
    for i, pi in enumerate(p):
        lo, hi = candidate(mn, mx, pi, dt)
        s, z = qparams(lo, hi, dt, kind, bits, symmetric)
        with np.errstate(invalid="ignore", over="ignore"):
            fq = M.fake_quantize(x, s[gid], dt, kind, bits, None if z is None else z[gid])
            d = np.abs(fq - x)
            np.add.at(e[:, i], gid, d ** norm)
    return e


def choose(e, patience):
    """(chosen step per group, stop step S) of the rule on an error table"""
    e = np.asarray(e, np.float64)
    n, steps = e.shape
    best = np.full(n, FLT_MAX)
    imp = np.zeros((n, steps), bool)
    with np.errstate(invalid="ignore"):
        for i in range(steps):
            imp[:, i] = e[:, i] < best
            best = np.where(imp[:, i], e[:, i], best)
    stop, run = steps - 1, 0
    for i in range(steps):
        run = 0 if imp[:, i].any() else run + 1
        if run >= patience:
            stop = i
            break
    idx = np.where(imp[:, :stop + 1], np.arange(stop + 1), -1).max(1) if n else np.zeros(0, np.int64)
    return np.maximum(idx, 0), stop
