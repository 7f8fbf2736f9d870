/*
 * levelset_field_oracle.c -- the level set, its gradient, Hessian and curvature at arbitrary points (DESIGN.md sections 13, 13.1 and
 * 13.2) by a scan over all particles in ascending index, TEST INFRASTRUCTURE ONLY.
 *
 * Included unchanged by tests/levelset_sdf_oracle.c, whose library tests/levelset_field_harness.py builds once into a temporary
 * directory.  It includes tests/averaged_radii_oracle.c (unchanged; it includes the averaged, corrected and pinned oracles) for the
 * scalar kernel and the Jacobi rotation; the records of every mode are arrays (the anisotropic ones come from so_aniso_records in
 * tests/anisotropic_oracle.c).  The folds are restated in the operation order of SsSphFold, SsAnisoFold, SsAvgFold / SsAvgCorrFold /
 * SsAvgRadFold / SsAvgCorrRadFold (values), SsSphGradFold, SsAnisoGradFold, SsAvgGradFold, SsAvgRadGradFold (gradients),
 * SsSphHessFold, SsAnisoHessFold, SsAvgHessFold, SsAvgRadHessFold (Hessians) and ss_curvature (splashsurf_b200/csrc/ss_field.cuh,
 * ss_aniso.cuh, ss_averaged.cuh).  One pass over the records serves every output, but each accumulator keeps its own operation
 * sequence.  Compile it like the oracle: single precision, un-contracted (-ffp-contract=off -fno-fast-math).
 */
#include "averaged_radii_oracle.c"

static const int SO_HI[6] = { 0, 0, 0, 1, 1, 2 }, SO_HJ[6] = { 0, 1, 2, 1, 2, 2 };

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

/* W'(r) / r and W''(r) from the constants of k_scalar_cubic (ss_kernel_scalar_d2) */
static void so_kernel_d2(float h, float r, float *w1r, float *w2) {
    const float sigma = 8.0f / ((h * h) * h), c_inner = 3.0f / (2.0f * SO_PI_F), c_outer = 1.0f / (4.0f * SO_PI_F);
    const float q = (r + r) / h;
    const float t = 2.0f / h, s2 = t * t;
    float f1q, f2;
    if (q < 1.0f) { f1q = c_inner * (1.5f * q - 2.0f); f2 = c_inner * (3.0f * q - 2.0f); }
    else if (q < 2.0f) { const float x = 2.0f - q; f1q = (((-3.0f * c_outer) * x) * x) / q; f2 = (6.0f * c_outer) * x; }
    else { f1q = 0.0f; f2 = 0.0f; }
    *w1r = (sigma * f1q) * s2;
    *w2 = (sigma * f2) * s2;
}

/* H += a v v^T + b K (ss_hess_rank1) */
static void so_hess_rank1(float *H, float a, const float *v, float b, const float *K) {
    for (int e = 0; e < 6; ++e) H[e] = H[e] + ((a * v[SO_HI[e]]) * v[SO_HJ[e]] + b * K[e]);
}

/* (kappa_H, kappa_G) of ss_curvature */
static void so_curvature(const float *g, const float *H, float *kh, float *kg) {
    const float g2 = (g[0] * g[0] + g[1] * g[1]) + g[2] * g[2];
    if (g2 == 0.0f) { *kh = NAN; *kg = NAN; return; }
    const float ng = sqrtf(g2);
    const float n[3] = { g[0] / ng, g[1] / ng, g[2] / ng };
    const float M[3][3] = { { H[0], H[1], H[2] }, { H[1], H[3], H[4] }, { H[2], H[4], H[5] } };
    const float a00 = H[3] * H[5] - H[4] * H[4], a01 = H[2] * H[4] - H[1] * H[5], a02 = H[1] * H[4] - H[2] * H[3];
    const float a11 = H[0] * H[5] - H[2] * H[2], a12 = H[1] * H[2] - H[0] * H[4], a22 = H[0] * H[3] - H[1] * H[1];
    const float A[3][3] = { { a00, a01, a02 }, { a01, a11, a12 }, { a02, a12, a22 } };
    float hn[3], an[3];
    for (int i = 0; i < 3; ++i) {
        hn[i] = (M[i][0] * n[0] + M[i][1] * n[1]) + M[i][2] * n[2];
        an[i] = (A[i][0] * n[0] + A[i][1] * n[1]) + A[i][2] * n[2];
    }
    const float nHn = (n[0] * hn[0] + n[1] * hn[1]) + n[2] * hn[2];
    const float nAn = (n[0] * an[0] + n[1] * an[1]) + n[2] * an[2];
    const float tr = (H[0] + H[3]) + H[5];
    *kh = -((tr - nHn) / (2.0f * ng));
    *kg = nAn / g2;
}

/* The field at m points by one scan over the n records in ascending index per point (mode: 0 standard, 1 anisotropic, 2 averaged,
 * 3 corrected, 4 averaged with radii, 5 corrected with radii):
 *   ctr  kernel centres (n x 3): the particles, or x_bar in the anisotropic mode
 *   w    V_j = m / rho_j (standard) or V_j det G_j (anisotropic); unused otherwise
 *   g6   G_j (n x 6: g00 g01 g02 g11 g12 g22), anisotropic mode only
 *   dlt  delta_j = R_j - R_s, radii modes only
 * val (m) always; grad (m x 3), hess (m x 6: xx xy xz yy yz zz) and curv (m x 2: kappa_H, kappa_G) where not NULL, in the modes with
 * derivatives (0, 1, 2, 4): the corrected modes leave them untouched. */
void so_field_scan(int mode, const float *ctr, const float *w, const float *g6, const float *dlt, uint64_t n, float h, float rs, float t_low,
                   float t_high, const float *pts, uint64_t m, float *val, float *grad, float *hess, float *curv) {
    const float h2 = h * h, h2m = h2 * 1.01f;
    const k_scalar kern = k_scalar_new(h);
    const int corrected = mode == 3 || mode == 5;
    for (uint64_t q = 0; q < m; ++q) {
        const float *x = pts + 3 * q;
        float phi = 0.0f, g[3] = { 0.0f, 0.0f, 0.0f }, H[6] = { 0, 0, 0, 0, 0, 0 };
        /* S X Y Z, Tx Ty Tz, Mxx Mxy Mxz Myy Myz Mzz, Q, Ux Uy Uz | S2, N (6), O (10), S2d, Nd (6) */
        float sum[17], s2 = 0.0f, N[6], O[10], s2d = 0.0f, Nd[6];
        memset(sum, 0, sizeof(sum)); memset(N, 0, sizeof(N)); memset(O, 0, sizeof(O)); memset(Nd, 0, sizeof(Nd));
        for (uint64_t j = 0; j < n; ++j) {
            const float *r = ctr + 3 * j;
            float d[3] = { r[0] - x[0], r[1] - x[1], r[2] - x[2] };
            if (mode == 1) {
                const float *G = g6 + 6 * j;
                float u0 = (G[0] * d[0] + G[1] * d[1]) + G[2] * d[2];
                float u1 = (G[1] * d[0] + G[3] * d[1]) + G[4] * d[2];
                float u2 = (G[2] * d[0] + G[4] * d[1]) + G[5] * d[2];
                float uu = (u0 * u0 + u1 * u1) + u2 * u2;
                if (!(uu < h2)) continue;
                float rr = sqrtf(uu);
                phi = phi + w[j] * k_scalar_eval(&kern, rr);
                float v[3] = { (G[0] * u0 + G[1] * u1) + G[2] * u2, (G[1] * u0 + G[3] * u1) + G[4] * u2, (G[2] * u0 + G[4] * u1) + G[5] * u2 };
                if (uu != 0.0f) {
                    float t = (w[j] * so_kernel_dr(h, rr)) / rr;
                    for (int b = 0; b < 3; ++b) g[b] = g[b] - t * v[b];
                }
                float w1r, w2;
                so_kernel_d2(h, rr, &w1r, &w2);
                float ra = uu == 0.0f ? 0.0f : (w[j] * (w2 - w1r)) / uu;
                const float Gm[3][3] = { { G[0], G[1], G[2] }, { G[1], G[3], G[4] }, { G[2], G[4], G[5] } };
                float K[6];
                for (int e = 0; e < 6; ++e) {
                    const int a = SO_HI[e], b = SO_HJ[e];
                    K[e] = (Gm[a][0] * Gm[0][b] + Gm[a][1] * Gm[1][b]) + Gm[a][2] * Gm[2][b];
                }
                so_hess_rank1(H, ra, v, w[j] * w1r, K);
                continue;
            }
            float d2 = (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2];
            if (mode == 0) {
                if (!(d2 < h2m)) continue;
                float rr = sqrtf(d2);
                phi = phi + w[j] * k_scalar_eval(&kern, rr);
                if (d2 != 0.0f) {
                    float t = (w[j] * so_kernel_dr(h, rr)) / rr;
                    for (int b = 0; b < 3; ++b) g[b] = g[b] - t * d[b];
                }
                float w1r, w2;
                so_kernel_d2(h, rr, &w1r, &w2);
                float ra = d2 == 0.0f ? 0.0f : (w[j] * (w2 - w1r)) / d2;
                const float I6[6] = { 1.0f, 0.0f, 0.0f, 1.0f, 0.0f, 1.0f };
                so_hess_rank1(H, ra, d, w[j] * w1r, I6);
                continue;
            }
            if (!(d2 < h2)) continue;
            float u = 1.0f - d2 / h2;
            float uu = u * u;
            float wt = uu * u;
            sum[0] = sum[0] + wt;
            for (int b = 0; b < 3; ++b) sum[1 + b] = sum[1 + b] + wt * d[b];
            if (mode >= 4) sum[13] = sum[13] + wt * dlt[j];
            float e[3] = { uu * d[0], uu * d[1], uu * d[2] };
            for (int b = 0; b < 3; ++b) sum[4 + b] = sum[4 + b] + e[b];
            int slot = 7;
            for (int ia = 0; ia < 3; ++ia) for (int ib = ia; ib < 3; ++ib, ++slot) sum[slot] = sum[slot] + e[ia] * d[ib];
            if (corrected) continue;
            s2 = s2 + u * u;
            float ed[3] = { u * d[0], u * d[1], u * d[2] };
            float nn[6] = { ed[0] * d[0], ed[0] * d[1], ed[0] * d[2], ed[1] * d[1], ed[1] * d[2], ed[2] * d[2] };
            for (int i = 0; i < 6; ++i) N[i] = N[i] + nn[i];
            float oo[10] = { nn[0] * d[0], nn[0] * d[1], nn[0] * d[2], nn[1] * d[1], nn[1] * d[2],
                             nn[2] * d[2], nn[3] * d[1], nn[3] * d[2], nn[4] * d[2], nn[5] * d[2] };
            for (int i = 0; i < 10; ++i) O[i] = O[i] + oo[i];
            if (mode == 4) {
                float edl = uu * dlt[j];
                for (int b = 0; b < 3; ++b) sum[14 + b] = sum[14 + b] + edl * d[b];
                float ud = u * dlt[j];
                s2d = s2d + u * ud;
                float edd[3] = { ud * d[0], ud * d[1], ud * d[2] };
                for (int i = 0; i < 6; ++i) Nd[i] = Nd[i] + edd[SO_HI[i]] * d[SO_HJ[i]];
            }
        }
        if (mode <= 1) val[q] = phi;
        else if (!(sum[0] > 0.0f)) val[q] = 0.0f;
        else {
            const float s = sum[0];
            float mm[3];
            for (int b = 0; b < 3; ++b) mm[b] = sum[1 + b] / s;
            float m2 = (mm[0] * mm[0] + mm[1] * mm[1]) + mm[2] * mm[2];
            float nm = sqrtf(m2);
            float plain = h - nm;
            float bq = mode >= 4 ? sum[13] / s : 0.0f;
            if (mode == 2) val[q] = plain;
            else if (mode == 4) val[q] = plain + bq;
            else {
                float t[3], qq[3][3], A[3][3];
                for (int b = 0; b < 3; ++b) t[b] = sum[4 + b] / s;
                int slot = 7;
                for (int ia = 0; ia < 3; ++ia) for (int ib = ia; ib < 3; ++ib, ++slot) qq[ia][ib] = sum[slot] / s;
                for (int ia = 0; ia < 3; ++ia) for (int ib = ia; ib < 3; ++ib) {
                    A[ia][ib] = 0.5f * ((qq[ia][ib] - mm[ia] * t[ib]) + (qq[ia][ib] - mm[ib] * t[ia]));
                    A[ib][ia] = A[ia][ib];
                }
                for (int sweep = 0; sweep < 8; ++sweep) { ac_jacobi_rot(A, 0, 1); ac_jacobi_rot(A, 0, 2); ac_jacobi_rot(A, 1, 2); }
                float ev = A[0][0];
                if (A[1][1] > ev) ev = A[1][1];
                if (A[2][2] > ev) ev = A[2][2];
                ev = (6.0f / h2) * ev;
                float gc = (t_high - ev) / (t_high - t_low);
                gc = gc > 0.0f ? (gc < 1.0f ? gc : 1.0f) : 0.0f;
                float f = ((gc - 3.0f) * gc + 3.0f) * gc;
                f = f < 1.0f ? f : 1.0f;
                val[q] = mode == 3 ? plain - rs * (1.0f - f) : (plain + bq) - (rs + bq) * (1.0f - f);
            }
            if (!corrected) {
                const float k = 6.0f / h2, kh = 4.0f / h2;
                const float T[3] = { sum[4], sum[5], sum[6] };
                const float M[3][3] = { { sum[7], sum[8], sum[9] }, { sum[8], sum[10], sum[11] }, { sum[9], sum[11], sum[12] } };
                if (nm != 0.0f) {
                    for (int i = 0; i < 3; ++i) {               /* SsAvgGradFold::grad_f */
                        float mv = (M[i][0] * mm[0] + M[i][1] * mm[1]) + M[i][2] * mm[2];
                        float jm = (k * (mv - m2 * T[i])) / s;
                        g[i] = (mm[i] - jm) / nm;
                    }
                    const float mh[3] = { mm[0] / nm, mm[1] / nm, mm[2] / nm };
                    float J[3][3], B[3][3], cv[3];
                    for (int i = 0; i < 3; ++i)
                        for (int jj = 0; jj < 3; ++jj) {
                            J[i][jj] = (k * (M[i][jj] - mm[i] * T[jj])) / s;
                            B[i][jj] = (i == jj ? 1.0f : 0.0f) - J[i][jj];
                        }
                    for (int jj = 0; jj < 3; ++jj) cv[jj] = (J[0][jj] * mh[0] + J[1][jj] * mh[1]) + J[2][jj] * mh[2];
                    const float sig = nm * s2 - ((mh[0] * T[0] + mh[1] * T[1]) + mh[2] * T[2]);
                    const int OX[6] = { 0, 1, 2, 3, 4, 5 }, OY[6] = { 1, 3, 4, 6, 7, 8 }, OZ[6] = { 2, 4, 5, 7, 8, 9 };
                    for (int e = 0; e < 6; ++e) {
                        const int i = SO_HI[e], jj = SO_HJ[e];
                        float om = (O[OX[e]] * mh[0] + O[OY[e]] * mh[1]) + O[OZ[e]] * mh[2];
                        float p = kh * (om - nm * N[e]);
                        if (i == jj) p = p + sig;
                        p = (p - T[i] * cv[jj]) - cv[i] * T[jj];
                        float first = (k * p) / s;
                        float bb = (B[0][i] * B[0][jj] + B[1][i] * B[1][jj]) + B[2][i] * B[2][jj];
                        float second = (bb - g[i] * g[jj]) / nm;
                        H[e] = -(first + second);
                    }
                }
                if (mode == 4) {
                    float rg[3];
                    for (int i = 0; i < 3; ++i) rg[i] = (k * (sum[14 + i] - bq * T[i])) / s;
                    for (int i = 0; i < 3; ++i) g[i] = g[i] + rg[i];
                    float dg = bq * s2 - s2d;
                    for (int e = 0; e < 6; ++e) {
                        const int i = SO_HI[e], jj = SO_HJ[e];
                        float p = kh * (Nd[e] - bq * N[e]);
                        if (i == jj) p = p + dg;
                        p = (p - T[i] * rg[jj]) - rg[i] * T[jj];
                        H[e] = H[e] + (k * p) / s;
                    }
                }
            }
        }
        if (corrected) continue;
        if (grad) for (int b = 0; b < 3; ++b) grad[3 * q + b] = g[b];
        if (hess) for (int e = 0; e < 6; ++e) hess[6 * q + e] = H[e];
        if (curv) so_curvature(g, H, curv + 2 * q, curv + 2 * q + 1);
    }
}
