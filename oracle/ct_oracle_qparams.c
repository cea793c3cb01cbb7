/*
 * oracle/ct_oracle_qparams.c -- TEST INFRASTRUCTURE ONLY (see ct_oracle.c header).
 * Included by ct_oracle_all.c after ct_oracle.c (uses its static conversion helpers).
 *
 * calculate_qparams: reference quantization/utils/helpers.py:50-137, restated with the same
 * per-op rounding to the min/max tensors' dtype T (each torch op on a T tensor rounds to T; python
 * scalars and 0-dim fp32 tensors do not promote).  Pinned by tests/golden/qparams.pt.gz.
 *
 *   min = min(min, 0); max = max(max, 0)                                   :74-75
 *   symmetric : scale = max(|min|, |max|) / (float(qmax - qmin) / 2) ; zp = 0   :84-91
 *   asymmetric: scale = (max - min) / float(qmax - qmin)                        :100
 *               zp = clamp(qmin - min / scale, qmin, qmax)                      :101-102
 *   scale == 0 -> eps(T)                                                         :113-126
 *   zp -> round(clamp(zp, iinfo(zp_dtype))).to(zp_dtype)   (int8)  /  .to(fp8)   :129-131
 */
static float dtype_eps(int dt) {
    switch (dt) {
    case DT_BF16: return 0.0078125f;
    case DT_F16: return 0.0009765625f;
    default: return 1.1920928955078125e-07f;
    }
}

int orc_calculate_qparams(const void* mn, const void* mx, int dt, void* scale_out, void* zp_out, int zp_dt, int64_t n,
                          int qtype, int bits, int symmetric) {
    if (!is_float_dt(dt)) return ORC_E_DTYPE;
    float qmin, qmax;
    q_range(qtype, bits, &qmin, &qmax);
    const float range = qmax - qmin;      /* 0-dim fp32 tensor arithmetic in the reference */
    for (int64_t i = 0; i < n; ++i) {
        float lo = load_as_f32(mn, i, dt), hi = load_as_f32(mx, i, dt);
        /* torch.min(x, 0) / torch.max(x, 0) keep a NaN; for -0.0 vs 0.0 either is fine downstream */
        lo = (lo != lo || lo < 0.0f) ? lo : 0.0f;
        hi = (hi != hi || hi > 0.0f) ? hi : 0.0f;
        float s, z;
        if (symmetric) {
            const float m = (lo != lo || fabsf(lo) > fabsf(hi)) ? fabsf(lo) : fabsf(hi);   /* torch.max propagates NaN */
            s = rnd(m / (range / 2.0f), dt);
            z = 0.0f;
        } else {
            s = rnd(rnd(hi - lo, dt) / range, dt);
            z = rnd(qmin - rnd(lo / s, dt), dt);
            z = clampf(z, qmin, qmax);
        }
        if (s == 0.0f) s = dtype_eps(dt);
        store_from_f32(scale_out, i, dt, s);
        if (zp_dt == DT_I8) {
            float zc = clampf(z, -128.0f, 127.0f);
            ((int8_t*)zp_out)[i] = f32_to_i8(nearbyintf(zc));
        } else if (zp_dt == DT_F8E4M3) {
            ((uint8_t*)zp_out)[i] = f32_to_f8e4m3(clampf(z, -448.0f, 448.0f));
        } else {
            return ORC_E_DTYPE;
        }
    }
    return ORC_OK;
}
