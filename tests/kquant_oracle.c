/* kquant_oracle.c -- TEST INFRASTRUCTURE: plain-C restatement of llama.cpp's K-quant reference quantisers at tag b3962 without an
 * importance matrix (quantize_row_q{2,3,4,5,6}_K_ref, make_qkx2_quants, make_q3_quants, make_qx_quants, nearest_int), written in
 * the serial shape of that code: one function per super-block type, loops in the reference's order.  It is the reference the
 * product's K-quant encoders (comfyui-gguf_b200/csrc/quantize.cuh) are compared against, on the host and on the GPU.
 *
 * Built with -ffp-contract=off -fno-fast-math on x86-64 (SSE scalar float): every operation below is one IEEE binary32
 * operation rounded to nearest, which is what makes the bytes a function of the input.  fp16 conversion rounds to nearest even.
 * Only the NaN case of nearest_int is written out: x86-64 gives every NaN an operation creates the payload 0x400000, which the
 * bit trick maps to 0, and the guard states that rather than relying on it. */
#include <math.h>
#include <stdint.h>
#include <string.h>

#define QK_K 256
#define GROUP_MAX_EPS 1e-15f
#define MAX(a, b) ((a) > (b) ? (a) : (b))
#define MIN(a, b) ((a) < (b) ? (a) : (b))

static inline int nearest_int(float fval) {
    if (fval != fval) return 0;
    float val = fval + 12582912.f;
    int i;
    memcpy(&i, &val, sizeof(int));
    return (i & 0x007fffff) - 0x00400000;
}

/* fp32 -> fp16, round to nearest even, overflow to inf (ggml's software conversion) */
static uint16_t fp32_to_fp16(float f) {
    const float scale_to_inf = 0x1.0p+112f;
    const float scale_to_zero = 0x1.0p-110f;
    float base = (fabsf(f) * scale_to_inf) * scale_to_zero;
    uint32_t w;
    memcpy(&w, &f, 4);
    const uint32_t shl1_w = w + w;
    const uint32_t sign = w & 0x80000000u;
    uint32_t bias = shl1_w & 0xFF000000u;
    if (bias < 0x71000000u) bias = 0x71000000u;
    uint32_t bb = (bias >> 1) + 0x07800000u;
    float fb;
    memcpy(&fb, &bb, 4);
    base = fb + base;
    uint32_t bits;
    memcpy(&bits, &base, 4);
    const uint32_t exp_bits = (bits >> 13) & 0x00007C00u;
    const uint32_t mantissa_bits = bits & 0x00000FFFu;
    const uint32_t nonsign = exp_bits + mantissa_bits;
    return (uint16_t)((sign >> 16) | (shl1_w > 0xFF000000u ? 0x7E00u : nonsign));
}

static float fp16_to_fp32(uint16_t h) {
    const uint32_t sign = (uint32_t)(h & 0x8000u) << 16;
    const uint32_t e = (h >> 10) & 0x1Fu, m = h & 0x3FFu;
    float v;
    if (e == 0) v = ldexpf((float)m, -24);
    else if (e == 31) v = m ? NAN : INFINITY;
    else v = ldexpf((float)(m | 0x400u), (int)e - 25);
    uint32_t b;
    memcpy(&b, &v, 4);
    b |= sign;
    memcpy(&v, &b, 4);
    return v;
}

static void put_fp16(uint8_t *p, float f) {
    const uint16_t h = fp32_to_fp16(f);
    p[0] = (uint8_t)h;
    p[1] = (uint8_t)(h >> 8);
}

static float get_fp16(const uint8_t *p) { return fp16_to_fp32((uint16_t)(p[0] | (p[1] << 8))); }

/* ---- counters of the branches the adversarial tests must reach (reset by kqor_reset_counters) ---- */
static long long g_cnt[4];   /* 0: D <= 0, 1: this_min > 0, 2: make_q3_quants early exit, 3: make_qkx2_quants max == min */

static float make_qkx2_quants(int n, int nmax, const float *x, const float *weights, uint8_t *L, float *the_min, uint8_t *Laux,
                              float rmin, float rdelta, int nstep, int use_mad) {
    float min = x[0];
    float max = x[0];
    float sum_w = weights[0];
    float sum_x = sum_w * x[0];
    for (int i = 1; i < n; ++i) {
        if (x[i] < min) min = x[i];
        if (x[i] > max) max = x[i];
        float w = weights[i];
        sum_w += w;
        sum_x += w * x[i];
    }
    if (min > 0) min = 0;
    if (max == min) {
        ++g_cnt[3];
        for (int i = 0; i < n; ++i) L[i] = 0;
        *the_min = -min;
        return 0.f;
    }
    float iscale = nmax / (max - min);
    float scale = 1 / iscale;
    float best_mad = 0;
    for (int i = 0; i < n; ++i) {
        int l = nearest_int(iscale * (x[i] - min));
        L[i] = MAX(0, MIN(nmax, l));
        float diff = scale * L[i] + min - x[i];
        diff = use_mad ? fabsf(diff) : diff * diff;
        float w = weights[i];
        best_mad += w * diff;
    }
    if (nstep < 1) {
        *the_min = -min;
        return scale;
    }
    for (int is = 0; is <= nstep; ++is) {
        iscale = (rmin + rdelta * is + nmax) / (max - min);
        float sum_l = 0, sum_l2 = 0, sum_xl = 0;
        for (int i = 0; i < n; ++i) {
            int l = nearest_int(iscale * (x[i] - min));
            l = MAX(0, MIN(nmax, l));
            Laux[i] = l;
            float w = weights[i];
            sum_l += w * l;
            sum_l2 += w * l * l;
            sum_xl += w * l * x[i];
        }
        float D = sum_w * sum_l2 - sum_l * sum_l;
        if (D > 0) {
            float this_scale = (sum_w * sum_xl - sum_x * sum_l) / D;
            float this_min = (sum_l2 * sum_x - sum_l * sum_xl) / D;
            if (this_min > 0) {
                ++g_cnt[1];
                this_min = 0;
                this_scale = sum_xl / sum_l2;
            }
            float mad = 0;
            for (int i = 0; i < n; ++i) {
                float diff = this_scale * Laux[i] + this_min - x[i];
                diff = use_mad ? fabsf(diff) : diff * diff;
                float w = weights[i];
                mad += w * diff;
            }
            if (mad < best_mad) {
                for (int i = 0; i < n; ++i) L[i] = Laux[i];
                best_mad = mad;
                scale = this_scale;
                min = this_min;
            }
        } else {
            ++g_cnt[0];
        }
    }
    *the_min = -min;
    return scale;
}

static float make_q3_quants(int n, int nmax, const float *x, int8_t *L, int do_rmse) {
    float max = 0;
    float amax = 0;
    for (int i = 0; i < n; ++i) {
        float ax = fabsf(x[i]);
        if (ax > amax) {
            amax = ax;
            max = x[i];
        }
    }
    if (amax < GROUP_MAX_EPS) {
        for (int i = 0; i < n; ++i) L[i] = 0;
        return 0.f;
    }
    float iscale = -nmax / max;
    if (do_rmse) {
        float sumlx = 0;
        float suml2 = 0;
        for (int i = 0; i < n; ++i) {
            int l = nearest_int(iscale * x[i]);
            l = MAX(-nmax, MIN(nmax - 1, l));
            L[i] = l;
            float w = x[i] * x[i];
            sumlx += w * x[i] * l;
            suml2 += w * l * l;
        }
        for (int itry = 0; itry < 5; ++itry) {
            int n_changed = 0;
            for (int i = 0; i < n; ++i) {
                float w = x[i] * x[i];
                float slx = sumlx - w * x[i] * L[i];
                if (slx > 0) {
                    float sl2 = suml2 - w * L[i] * L[i];
                    int new_l = nearest_int(x[i] * sl2 / slx);
                    new_l = MAX(-nmax, MIN(nmax - 1, new_l));
                    if (new_l != L[i]) {
                        slx += w * x[i] * new_l;
                        sl2 += w * new_l * new_l;
                        if (sl2 > 0 && slx * slx * suml2 > sumlx * sumlx * sl2) {
                            L[i] = new_l;
                            sumlx = slx;
                            suml2 = sl2;
                            ++n_changed;
                        }
                    }
                }
            }
            if (!n_changed) {
                if (itry < 4) ++g_cnt[2];
                break;
            }
        }
        for (int i = 0; i < n; ++i) L[i] += nmax;
        return sumlx / suml2;
    }
    for (int i = 0; i < n; ++i) {
        int l = nearest_int(iscale * x[i]);
        l = MAX(-nmax, MIN(nmax - 1, l));
        L[i] = l + nmax;
    }
    return 1 / iscale;
}

static float make_qx_quants(int n, int nmax, const float *x, int8_t *L, int rmse_type, const float *qw) {
    float max = 0;
    float amax = 0;
    for (int i = 0; i < n; ++i) {
        float ax = fabsf(x[i]);
        if (ax > amax) {
            amax = ax;
            max = x[i];
        }
    }
    if (amax < GROUP_MAX_EPS) {
        for (int i = 0; i < n; ++i) L[i] = 0;
        return 0.f;
    }
    float iscale = -nmax / max;
    float sumlx = 0;
    float suml2 = 0;
    for (int i = 0; i < n; ++i) {
        int l = nearest_int(iscale * x[i]);
        l = MAX(-nmax, MIN(nmax - 1, l));
        L[i] = l + nmax;
        float w = qw ? qw[i] : rmse_type == 1 ? x[i] * x[i] : rmse_type == 2 ? 1 : rmse_type == 3 ? fabsf(x[i]) : sqrtf(fabsf(x[i]));
        sumlx += w * x[i] * l;
        suml2 += w * l * l;
    }
    float scale = suml2 ? sumlx / suml2 : 0.0f;
    float best = scale * sumlx;
    for (int is = -9; is <= 9; ++is) {
        if (is == 0) continue;
        iscale = -(nmax + 0.1f * is) / max;
        sumlx = suml2 = 0;
        for (int i = 0; i < n; ++i) {
            int l = nearest_int(iscale * x[i]);
            l = MAX(-nmax, MIN(nmax - 1, l));
            float w = qw ? qw[i] : rmse_type == 1 ? x[i] * x[i] : rmse_type == 2 ? 1 : rmse_type == 3 ? fabsf(x[i]) : sqrtf(fabsf(x[i]));
            sumlx += w * x[i] * l;
            suml2 += w * l * l;
        }
        if (suml2 > 0 && sumlx * sumlx > best * suml2) {
            for (int i = 0; i < n; ++i) {
                int l = nearest_int(iscale * x[i]);
                L[i] = nmax + MAX(-nmax, MIN(nmax - 1, l));
            }
            scale = sumlx / suml2;
            best = scale * sumlx;
        }
    }
    return scale;
}

static inline void get_scale_min_k4(int j, const uint8_t *q, uint8_t *d, uint8_t *m) {
    if (j < 4) {
        *d = q[j] & 63;
        *m = q[j + 4] & 63;
    } else {
        *d = (q[j + 4] & 0xF) | ((q[j - 4] >> 6) << 4);
        *m = (q[j + 4] >> 4) | ((q[j - 0] >> 6) << 4);
    }
}

/* ---- block_q2_K: scales[16] qs[64] d dmin (84 bytes) ---- */
static void quantize_q2_K(const float *x, uint8_t *y) {
    uint8_t L[QK_K], Laux[16];
    float weights[16], mins[QK_K / 16], scales[QK_K / 16];
    uint8_t *ysc = y, *qs = y + 16;
    const float q4scale = 15.f;
    float max_scale = 0, max_min = 0;
    for (int j = 0; j < QK_K / 16; ++j) {
        for (int l = 0; l < 16; ++l) weights[l] = fabsf(x[16 * j + l]);
        scales[j] = make_qkx2_quants(16, 3, x + 16 * j, weights, L + 16 * j, &mins[j], Laux, -0.5f, 0.1f, 15, 1);
        float scale = scales[j];
        if (scale > max_scale) max_scale = scale;
        float min = mins[j];
        if (min > max_min) max_min = min;
    }
    if (max_scale > 0) {
        float iscale = q4scale / max_scale;
        for (int j = 0; j < QK_K / 16; ++j) {
            int l = nearest_int(iscale * scales[j]);
            ysc[j] = l;
        }
        put_fp16(y + 80, max_scale / q4scale);
    } else {
        for (int j = 0; j < QK_K / 16; ++j) ysc[j] = 0;
        put_fp16(y + 80, 0.f);
    }
    if (max_min > 0) {
        float iscale = q4scale / max_min;
        for (int j = 0; j < QK_K / 16; ++j) {
            int l = nearest_int(iscale * mins[j]);
            ysc[j] |= (uint8_t)((unsigned)l << 4);
        }
        put_fp16(y + 82, max_min / q4scale);
    } else {
        put_fp16(y + 82, 0.f);
    }
    for (int j = 0; j < QK_K / 16; ++j) {
        const float d = get_fp16(y + 80) * (ysc[j] & 0xF);
        if (!d) continue;
        const float dm = get_fp16(y + 82) * (ysc[j] >> 4);
        for (int ii = 0; ii < 16; ++ii) {
            int l = nearest_int((x[16 * j + ii] + dm) / d);
            l = MAX(0, MIN(3, l));
            L[16 * j + ii] = l;
        }
    }
    for (int j = 0; j < QK_K; j += 128)
        for (int l = 0; l < 32; ++l)
            qs[j / 4 + l] = L[j + l] | (L[j + l + 32] << 2) | (L[j + l + 64] << 4) | (L[j + l + 96] << 6);
}

/* ---- block_q3_K: hmask[32] qs[64] scales[12] d (110 bytes) ---- */
static void quantize_q3_K(const float *x, uint8_t *y) {
    int8_t L[QK_K];
    float scales[QK_K / 16];
    uint8_t *hmask = y, *qs = y + 32, *ysc = y + 96;
    float max_scale = 0, amax = 0;
    for (int j = 0; j < QK_K / 16; ++j) {
        scales[j] = make_q3_quants(16, 4, x + 16 * j, L + 16 * j, 1);
        float scale = fabsf(scales[j]);
        if (scale > amax) {
            amax = scale;
            max_scale = scales[j];
        }
    }
    memset(ysc, 0, 12);
    if (max_scale) {
        float iscale = -32.f / max_scale;
        for (int j = 0; j < QK_K / 16; ++j) {
            int8_t l = nearest_int(iscale * scales[j]);
            l = MAX(-32, MIN(31, l)) + 32;
            if (j < 8) ysc[j] = l & 0xF;
            else ysc[j - 8] |= ((l & 0xF) << 4);
            l >>= 4;
            ysc[j % 4 + 8] |= (l << (2 * (j / 4)));
        }
        put_fp16(y + 108, 1 / iscale);
    } else {
        put_fp16(y + 108, 0.f);
    }
    int8_t sc;
    for (int j = 0; j < QK_K / 16; ++j) {
        sc = j < 8 ? ysc[j] & 0xF : ysc[j - 8] >> 4;
        sc = (sc | (((ysc[8 + j % 4] >> (2 * (j / 4))) & 3) << 4)) - 32;
        float d = get_fp16(y + 108) * sc;
        if (!d) continue;
        for (int ii = 0; ii < 16; ++ii) {
            int l = nearest_int(x[16 * j + ii] / d);
            l = MAX(-4, MIN(3, l));
            L[16 * j + ii] = l + 4;
        }
    }
    memset(hmask, 0, QK_K / 8);
    int m = 0;
    uint8_t hm = 1;
    for (int j = 0; j < QK_K; ++j) {
        if (L[j] > 3) {
            hmask[m] |= hm;
            L[j] -= 4;
        }
        if (++m == QK_K / 8) {
            m = 0;
            hm <<= 1;
        }
    }
    for (int j = 0; j < QK_K; j += 128)
        for (int l = 0; l < 32; ++l)
            qs[j / 4 + l] = L[j + l] | (L[j + l + 32] << 2) | (L[j + l + 64] << 4) | (L[j + l + 96] << 6);
}

/* ---- block_q4_K / block_q5_K: d dmin scales[12] [qh[32]] qs[128] ---- */
static void quantize_q45_K(const float *x, uint8_t *y, int five) {
    uint8_t L[QK_K], Laux[32];
    float weights[32], mins[QK_K / 32], scales[QK_K / 32];
    uint8_t *ysc = y + 4;
    const int nmax = five ? 31 : 15;
    float max_scale = 0, max_min = 0;
    for (int j = 0; j < QK_K / 32; ++j) {
        float sum_x2 = 0;
        for (int l = 0; l < 32; ++l) sum_x2 += x[32 * j + l] * x[32 * j + l];
        float av_x = sqrtf(sum_x2 / 32);
        for (int l = 0; l < 32; ++l) weights[l] = av_x + fabsf(x[32 * j + l]);
        if (five) scales[j] = make_qkx2_quants(32, 31, x + 32 * j, weights, L + 32 * j, &mins[j], Laux, -0.5f, 0.1f, 15, 0);
        else scales[j] = make_qkx2_quants(32, 15, x + 32 * j, weights, L + 32 * j, &mins[j], Laux, -1.f, 0.1f, 20, 0);
        float scale = scales[j];
        if (scale > max_scale) max_scale = scale;
        float min = mins[j];
        if (min > max_min) max_min = min;
    }
    float inv_scale = max_scale > 0 ? 63.f / max_scale : 0.f;
    float inv_min = max_min > 0 ? 63.f / max_min : 0.f;
    for (int j = 0; j < QK_K / 32; ++j) {
        uint8_t ls = nearest_int(inv_scale * scales[j]);
        uint8_t lm = nearest_int(inv_min * mins[j]);
        ls = MIN(63, ls);
        lm = MIN(63, lm);
        if (j < 4) {
            ysc[j] = ls;
            ysc[j + 4] = lm;
        } else {
            ysc[j + 4] = (ls & 0xF) | ((lm & 0xF) << 4);
            ysc[j - 4] |= ((ls >> 4) << 6);
            ysc[j - 0] |= ((lm >> 4) << 6);
        }
    }
    put_fp16(y, max_scale / 63.f);
    put_fp16(y + 2, max_min / 63.f);
    uint8_t sc, m;
    for (int j = 0; j < QK_K / 32; ++j) {
        get_scale_min_k4(j, ysc, &sc, &m);
        const float d = get_fp16(y) * sc;
        if (!d) continue;
        const float dm = get_fp16(y + 2) * m;
        for (int ii = 0; ii < 32; ++ii) {
            int l = nearest_int((x[32 * j + ii] + dm) / d);
            l = MAX(0, MIN(nmax, l));
            L[32 * j + ii] = l;
        }
    }
    if (!five) {
        uint8_t *q = y + 16;
        for (int j = 0; j < QK_K; j += 64) {
            for (int l = 0; l < 32; ++l) q[l] = L[j + l] | (L[j + l + 32] << 4);
            q += 32;
        }
        return;
    }
    uint8_t *qh = y + 16, *ql = y + 48;
    memset(qh, 0, QK_K / 8);
    uint8_t m1 = 1, m2 = 2;
    for (int n = 0; n < QK_K; n += 64) {
        for (int j = 0; j < 32; ++j) {
            int l1 = L[n + j];
            if (l1 > 15) {
                l1 -= 16;
                qh[j] |= m1;
            }
            int l2 = L[n + j + 32];
            if (l2 > 15) {
                l2 -= 16;
                qh[j] |= m2;
            }
            ql[j] = l1 | (l2 << 4);
        }
        m1 <<= 2;
        m2 <<= 2;
        ql += 32;
    }
}

/* ---- block_q6_K: ql[128] qh[64] scales[16] (int8) d (210 bytes) ---- */
static void quantize_q6_K(const float *x, uint8_t *y) {
    int8_t L[QK_K];
    float scales[QK_K / 16];
    int8_t *ysc = (int8_t *)(y + 192);
    float max_scale = 0, max_abs_scale = 0;
    for (int ib = 0; ib < QK_K / 16; ++ib) {
        const float scale = make_qx_quants(16, 32, x + 16 * ib, L + 16 * ib, 1, NULL);
        scales[ib] = scale;
        const float abs_scale = fabsf(scale);
        if (abs_scale > max_abs_scale) {
            max_abs_scale = abs_scale;
            max_scale = scale;
        }
    }
    if (max_abs_scale < GROUP_MAX_EPS) {
        memset(y, 0, 210);
        put_fp16(y + 208, 0.f);
        return;
    }
    float iscale = -128.f / max_scale;
    put_fp16(y + 208, 1 / iscale);
    for (int ib = 0; ib < QK_K / 16; ++ib) ysc[ib] = MIN(127, nearest_int(iscale * scales[ib]));
    for (int j = 0; j < QK_K / 16; ++j) {
        float d = get_fp16(y + 208) * ysc[j];
        if (!d) continue;
        for (int ii = 0; ii < 16; ++ii) {
            int l = nearest_int(x[16 * j + ii] / d);
            l = MAX(-32, MIN(31, l));
            L[16 * j + ii] = l + 32;
        }
    }
    uint8_t *ql = y, *qh = y + 128;
    for (int j = 0; j < QK_K; j += 128) {
        for (int l = 0; l < 32; ++l) {
            const uint8_t q1 = L[j + l + 0] & 0xF;
            const uint8_t q2 = L[j + l + 32] & 0xF;
            const uint8_t q3 = L[j + l + 64] & 0xF;
            const uint8_t q4 = L[j + l + 96] & 0xF;
            ql[l + 0] = q1 | (q3 << 4);
            ql[l + 32] = q2 | (q4 << 4);
            qh[l] = (L[j + l] >> 4) | ((L[j + l + 32] >> 4) << 2) | ((L[j + l + 64] >> 4) << 4) | ((L[j + l + 96] >> 4) << 6);
        }
        ql += 64;
        qh += 32;
    }
}

/* x: n_blocks * 256 fp32 values; y: n_blocks * type_size bytes.  Returns -1 for a type that is not a K type. */
int kqor_quantize(int type, const float *x, long long n_blocks, uint8_t *y) {
    static const int ts[5] = {84, 110, 144, 176, 210};
    if (type < 10 || type > 14) return -1;
    for (long long b = 0; b < n_blocks; ++b) {
        const float *xb = x + b * QK_K;
        uint8_t *yb = y + b * ts[type - 10];
        switch (type) {
        case 10: quantize_q2_K(xb, yb); break;
        case 11: quantize_q3_K(xb, yb); break;
        case 12: quantize_q45_K(xb, yb, 0); break;
        case 13: quantize_q45_K(xb, yb, 1); break;
        case 14: quantize_q6_K(xb, yb); break;
        }
    }
    return 0;
}

void kqor_reset_counters(void) { memset(g_cnt, 0, sizeof g_cnt); }
long long kqor_counter(int i) { return (i >= 0 && i < 4) ? g_cnt[i] : -1; }
