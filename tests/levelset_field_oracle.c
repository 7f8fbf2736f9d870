/*
 * levelset_field_oracle.c -- the level set at arbitrary points (DESIGN.md section 13) by a scan over all particles in ascending
 * index, TEST INFRASTRUCTURE ONLY.
 *
 * Built twice by tests/test_levelset_field.py into a temporary directory: with SO_FIELD_ANISO it includes
 * tests/anisotropic_oracle.c (unchanged) for the kernel centres x_bar, the matrices G and V det G; without, it includes
 * tests/averaged_radii_oracle.c (unchanged; it includes the averaged, corrected and pinned oracles) for the scalar kernel and the
 * Jacobi rotation.  The folds are restated in the operation order of SsSphFold (splashsurf_b200/csrc/ss_field.cuh), SsAnisoFold
 * (ss_aniso.cuh) and SsAvgFold / SsAvgCorrFold / SsAvgRadFold / SsAvgCorrRadFold (ss_averaged.cuh).  Compile it like the oracle:
 * single precision, un-contracted (-ffp-contract=off).
 */
#ifdef SO_FIELD_ANISO
#include "anisotropic_oracle.c"

/* x_bar (n x 3), G (n x 6) and V det G (n) of the n_filtered particles, as so_reconstruct_aniso computes them (the same filter,
 * grid, decompositions, densities and anisotropy); returns n_filtered, or -(error code). */
int64_t so_field_aniso_records(const float *xyz_in, uint64_t n_in, const so_params *p, float smoothing, float max_stretch, uint32_t min_neighbors,
                               float *xbar_out, float *g_out, float *vdet_out, float *rho_out) {
    const float *xyz = xyz_in; float *filtered = NULL; uint64_t n = n_in;
    if (p->has_particle_aabb) {
        filtered = (float *)malloc(sizeof(float) * 3 * (n_in ? n_in : 1));
        n = 0;
        for (uint64_t i = 0; i < n_in; ++i) {
            int in = 1;
            for (int d = 0; d < 3; ++d) { float v = xyz_in[3 * i + d]; if (!(v >= p->aabb_min[d] && v < p->aabb_max[d])) in = 0; }
            if (in) { memcpy(filtered + 3 * n, xyz_in + 3 * i, sizeof(float) * 3); ++n; }
        }
        xyz = filtered;
    }
    so_grid g0;
    int err = grid_for_reconstruction(&g0, xyz, n, p);
    if (err) { free(filtered); return -err; }
    int64_t S = (int64_t)p->subdomain_num_cubes_per_dim;
    float r2 = p->particle_radius + p->particle_radius;
    float rest_mass = (r2 * r2 * r2) * p->rest_density;
    float h = p->compact_support_radius, c = p->cube_size;
    float margin = f_ceil(h / c) * c * 1.01f;
    int64_t nsubd[3], ncg[3];
    for (int d = 0; d < 3; ++d) { nsubd[d] = (g0.nc[d] + S - 1) / S; ncg[d] = nsubd[d] * S; }
    so_grid gg; grid_new(&gg, g0.aabb_min, ncg, c);
    so_grid sg; grid_new(&sg, gg.aabb_min, nsubd, c * (float)S);
    so_decomp dstd; decompose(&dstd, xyz, n, &sg, margin);
    so_result res;
    memset(&res, 0, sizeof(res));
    res.densities = rho_out;
    memset(rho_out, 0, sizeof(float) * (n ? n : 1));
    g_an.on = 1; g_an.lambda = smoothing; g_an.kr = max_stretch; g_an.min_nb = min_neighbors;
    g_an.xbar = xbar_out; g_an.g = g_out; g_an.vdet = vdet_out;
    an_job job;
    memset(&job, 0, sizeof(job));
    job.xyz = xyz; job.sg = &sg; job.gg = &gg; job.dstd = &dstd; job.res = &res;
    job.h = h; job.c = c; job.margin = margin; job.rest_mass = rest_mass; job.S = S;
    parallel_for((int64_t)dstd.nsub, an_density_task, &job);
    for (uint64_t i = 0; i < n; ++i) {
        for (int d = 0; d < 3; ++d) g_an.xbar[3 * i + d] = xyz[3 * i + d];
        float id[6] = { 1, 0, 0, 1, 0, 1 };
        memcpy(g_an.g + 6 * i, id, sizeof(id));
        g_an.vdet[i] = 1.0f;
    }
    parallel_for((int64_t)dstd.nsub, an_aniso_task, &job);
    for (uint64_t i = 0; i < n; ++i) g_an.vdet[i] = (rest_mass / rho_out[i]) * g_an.vdet[i];
    memset(&g_an, 0, sizeof(g_an));
    free(dstd.flat); free(dstd.offset); free(dstd.members);
    free(filtered);
    return (int64_t)n;
}
#else
#include "averaged_radii_oracle.c"
#endif

/* The field at m points by a scan over the n records in ascending index (mode: 0 standard, 1 anisotropic, 2 averaged, 3 corrected,
 * 4 averaged with radii, 5 corrected with radii):
 *   ctr  kernel centres (n x 3): the particles, or x_bar in the anisotropic mode
 *   w    V_j = m / rho_j (standard) or V_j det G_j (anisotropic); unused otherwise
 *   g6   G_j (n x 6: g00 g01 g02 g11 g12 g22), anisotropic mode only
 *   dlt  delta_j = R_j - R_s, radii modes only */
void so_field_scan(int mode, const float *ctr, const float *w, const float *g6, const float *dlt, uint64_t n, float h, float rs, float t_low,
                   float t_high, const float *pts, uint64_t m, float *out) {
    const float h2 = h * h, h2m = h2 * 1.01f;
#ifndef SO_FIELD_ANISO
    const k_scalar kern = k_scalar_new(h);
#endif
    for (uint64_t q = 0; q < m; ++q) {
        const float *x = pts + 3 * q;
        float phi = 0.0f, sum[14];
        memset(sum, 0, sizeof(sum));                     /* S X Y Z, Tx Ty Tz, Mxx Mxy Mxz Myy Myz Mzz, Q */
        for (uint64_t j = 0; j < n; ++j) {
            const float *r = ctr + 3 * j;
            float d[3] = { r[0] - x[0], r[1] - x[1], r[2] - x[2] };
            if (mode == 1) {
                const float *g = g6 + 6 * j;
                float u0 = (g[0] * d[0] + g[1] * d[1]) + g[2] * d[2];
                float u1 = (g[1] * d[0] + g[3] * d[1]) + g[4] * d[2];
                float u2 = (g[2] * d[0] + g[4] * d[1]) + g[5] * d[2];
                float uu = (u0 * u0 + u1 * u1) + u2 * u2;
#ifdef SO_FIELD_ANISO
                if (uu < h2) { k_scalar kern = k_scalar_new(h); phi = phi + w[j] * k_scalar_eval(&kern, sqrtf(uu)); }
#endif
                continue;
            }
            float d2 = (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2];
            if (mode == 0) {
#ifndef SO_FIELD_ANISO
                if (d2 < h2m) phi = phi + w[j] * k_scalar_eval(&kern, sqrtf(d2));
#endif
                continue;
            }
            if (!(d2 < h2)) continue;
            float u = 1.0f - d2 / h2;
            float uu = u * u;
            float wt = uu * u;
            sum[0] = sum[0] + wt;
            for (int b = 0; b < 3; ++b) sum[1 + b] = sum[1 + b] + wt * d[b];
            if (mode >= 4) sum[13] = sum[13] + wt * dlt[j];
            if (mode != 3 && mode != 5) continue;
            float e[3] = { uu * d[0], uu * d[1], uu * d[2] };
            for (int b = 0; b < 3; ++b) sum[4 + b] = sum[4 + b] + e[b];
            int slot = 7;
            for (int ia = 0; ia < 3; ++ia) for (int ib = ia; ib < 3; ++ib, ++slot) sum[slot] = sum[slot] + e[ia] * d[ib];
        }
        if (mode <= 1) { out[q] = phi; continue; }
        float s = sum[0];
        if (!(s > 0.0f)) { out[q] = 0.0f; continue; }
        float mm[3];
        for (int b = 0; b < 3; ++b) mm[b] = sum[1 + b] / s;
        float m2 = (mm[0] * mm[0] + mm[1] * mm[1]) + mm[2] * mm[2];
        float plain = h - sqrtf(m2);
        float bq = mode >= 4 ? sum[13] / s : 0.0f;
        if (mode == 2) { out[q] = plain; continue; }
        if (mode == 4) { out[q] = plain + bq; continue; }
#ifndef SO_FIELD_ANISO
        float t[3], qq[3][3], A[3][3];
        for (int b = 0; b < 3; ++b) t[b] = sum[4 + b] / s;
        int slot = 7;
        for (int ia = 0; ia < 3; ++ia) for (int ib = ia; ib < 3; ++ib, ++slot) qq[ia][ib] = sum[slot] / s;
        for (int ia = 0; ia < 3; ++ia) for (int ib = ia; ib < 3; ++ib) {
            A[ia][ib] = 0.5f * ((qq[ia][ib] - mm[ia] * t[ib]) + (qq[ia][ib] - mm[ib] * t[ia]));
            A[ib][ia] = A[ia][ib];
        }
        for (int sweep = 0; sweep < 8; ++sweep) { ac_jacobi_rot(A, 0, 1); ac_jacobi_rot(A, 0, 2); ac_jacobi_rot(A, 1, 2); }
        float e = A[0][0];
        if (A[1][1] > e) e = A[1][1];
        if (A[2][2] > e) e = A[2][2];
        float ev = (6.0f / h2) * e;
        float g = (t_high - ev) / (t_high - t_low);
        g = g > 0.0f ? (g < 1.0f ? g : 1.0f) : 0.0f;
        float f = ((g - 3.0f) * g + 3.0f) * g;
        f = f < 1.0f ? f : 1.0f;
        out[q] = mode == 3 ? plain - rs * (1.0f - f) : (plain + bq) - (rs + bq) * (1.0f - f);
#endif
    }
}
