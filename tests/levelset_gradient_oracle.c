/*
 * levelset_gradient_oracle.c -- the gradient of the level set at arbitrary points (DESIGN.md section 13.1) by a scan over all
 * particles in ascending index, TEST INFRASTRUCTURE ONLY.
 *
 * Built twice by tests/test_levelset_gradient.py into a temporary directory, with and without SO_FIELD_ANISO, on top of
 * tests/levelset_field_oracle.c (unchanged), which provides the value (so_field_scan), the records of the anisotropic mode and the
 * scalar kernel's constants.  The gradient folds are restated in the operation order of SsSphGradFold, SsAnisoGradFold,
 * SsAvgGradFold and SsAvgRadGradFold (splashsurf_b200/csrc/ss_field.cuh).  Compile it like the oracle: single precision,
 * un-contracted (-ffp-contract=off -fno-fast-math).
 */
#include "levelset_field_oracle.c"

/* W'(r) of the scalar cubic spline from the constants of k_scalar_cubic (ss_kernel_scalar_dr) */
static float so_kernel_dr(float h, float r) {
    const float sigma = 8.0f / ((h * h) * h), c_inner = 3.0f / (2.0f * SO_PI_F), c_outer = 1.0f / (4.0f * SO_PI_F);
    const float q = (r + r) / h;
    float f;
    if (q < 1.0f) f = c_inner * (q * (1.5f * q - 2.0f));
    else if (q < 2.0f) { const float x = 2.0f - q; f = ((-3.0f * c_outer) * x) * x; }
    else f = 0.0f;
    return (sigma * f) * (2.0f / h);
}

/* Values (so_field_scan) and gradients (m x 3) at m points; mode and arrays as so_field_scan (0 standard, 1 anisotropic, 2 averaged,
 * 4 averaged with radii; the corrected modes 3 and 5 have no gradient and leave grad untouched). */
void so_gradient_scan(int mode, const float *ctr, const float *w, const float *g6, const float *dlt, uint64_t n, float h, float rs,
                      const float *pts, uint64_t m, float *val, float *grad) {
    so_field_scan(mode, ctr, w, g6, dlt, n, h, rs, 0.4f, 3.5f, pts, m, val);
    if (mode == 3 || mode == 5) return;
    const float h2 = h * h, h2m = h2 * 1.01f;
    for (uint64_t q = 0; q < m; ++q) {
        const float *x = pts + 3 * q;
        float g[3] = { 0.0f, 0.0f, 0.0f }, sum[17];
        memset(sum, 0, sizeof(sum));                     /* S X Y Z, Tx Ty Tz, Mxx Mxy Mxz Myy Myz Mzz, Q, Ux Uy Uz */
        for (uint64_t j = 0; j < n; ++j) {
            const float *r = ctr + 3 * j;
            float d[3] = { r[0] - x[0], r[1] - x[1], r[2] - x[2] };
            if (mode == 1) {
                const float *G = g6 + 6 * j;
                float u0 = (G[0] * d[0] + G[1] * d[1]) + G[2] * d[2];
                float u1 = (G[1] * d[0] + G[3] * d[1]) + G[4] * d[2];
                float u2 = (G[2] * d[0] + G[4] * d[1]) + G[5] * d[2];
                float uu = (u0 * u0 + u1 * u1) + u2 * u2;
                if (!(uu < h2) || uu == 0.0f) continue;
                float rr = sqrtf(uu);
                float t = (w[j] * so_kernel_dr(h, rr)) / rr;
                float v[3] = { (G[0] * u0 + G[1] * u1) + G[2] * u2, (G[1] * u0 + G[3] * u1) + G[4] * u2, (G[2] * u0 + G[4] * u1) + G[5] * u2 };
                for (int b = 0; b < 3; ++b) g[b] = g[b] - t * v[b];
                continue;
            }
            float d2 = (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2];
            if (mode == 0) {
                if (!(d2 < h2m) || d2 == 0.0f) continue;
                float rr = sqrtf(d2);
                float t = (w[j] * so_kernel_dr(h, rr)) / rr;
                for (int b = 0; b < 3; ++b) g[b] = g[b] - t * d[b];
                continue;
            }
            if (!(d2 < h2)) continue;
            float u = 1.0f - d2 / h2;
            float uu = u * u;
            float wt = uu * u;
            sum[0] = sum[0] + wt;
            for (int b = 0; b < 3; ++b) sum[1 + b] = sum[1 + b] + wt * d[b];
            float e[3] = { uu * d[0], uu * d[1], uu * d[2] };
            for (int b = 0; b < 3; ++b) sum[4 + b] = sum[4 + b] + e[b];
            int slot = 7;
            for (int ia = 0; ia < 3; ++ia) for (int ib = ia; ib < 3; ++ib, ++slot) sum[slot] = sum[slot] + e[ia] * d[ib];
            if (mode == 4) {
                sum[13] = sum[13] + wt * dlt[j];
                float ed = uu * dlt[j];
                for (int b = 0; b < 3; ++b) sum[14 + b] = sum[14 + b] + ed * d[b];
            }
        }
        if (mode >= 2) {
            float s = sum[0];
            if (s > 0.0f) {
                float mm[3];
                for (int b = 0; b < 3; ++b) mm[b] = sum[1 + b] / s;
                float m2 = (mm[0] * mm[0] + mm[1] * mm[1]) + mm[2] * mm[2];
                float nm = sqrtf(m2);
                float k = 6.0f / h2;
                if (nm != 0.0f) {
                    const float M[3][3] = { { sum[7], sum[8], sum[9] }, { sum[8], sum[10], sum[11] }, { sum[9], sum[11], sum[12] } };
                    for (int i = 0; i < 3; ++i) {
                        float mv = (M[i][0] * mm[0] + M[i][1] * mm[1]) + M[i][2] * mm[2];
                        float jm = (k * (mv - m2 * sum[4 + i])) / s;
                        g[i] = (mm[i] - jm) / nm;
                    }
                }
                if (mode == 4) {
                    float b = sum[13] / s;
                    for (int i = 0; i < 3; ++i) g[i] = g[i] + (k * (sum[14 + i] - b * sum[4 + i])) / s;
                }
            }
        }
        for (int b = 0; b < 3; ++b) grad[3 * q + b] = g[b];
    }
}
