/*
 * averaged_radii_oracle.c -- plain-C restatement of the per-particle radii of the averaged-position surface (DESIGN.md section
 * 12.2), TEST INFRASTRUCTURE ONLY.
 *
 * Built by tests/test_averaged_radii.py into a temporary directory.  It includes tests/averaged_correction_oracle.c (unchanged; it
 * includes tests/averaged_oracle.c and the pinned oracle/splashsurf_oracle.c) for the grid, the particle-AABB filter, the
 * decomposition, the densities, the averaged sums, the Jacobi rotation, marching cubes and stitching, and adds the sum
 * Q = sum_j w_j delta_j in the operation order of SsAvgRadFold / SsAvgCorrRadFold (splashsurf_b200/csrc/ss_averaged.cuh).  Compile
 * it like the oracle: single precision, un-contracted (-ffp-contract=off).
 */
#include "averaged_correction_oracle.c"
/* ------------------------------------------------------------ per-particle radii (DESIGN.md section 12.2) ---- */
/* The sums of subdomain_levelset_averaged (S, X, Y, Z) and, when corrected, of subdomain_levelset_averaged_corrected (T, M), plus
 * Q = sum w delta_j with the same weight w; then b = Q / S and
 *     plain:      (h - |m|) + b
 *     corrected:  ((h - |m|) + b) - (R_s + b) (1 - f)      (f of section 12.1)
 * and 0 where !(S > 0).  delta: delta_j per (filtered) particle.  acc: 14 np^3 floats. */
static void subdomain_levelset_averaged_radii(float *phi, float *acc, const float *xyz, const float *delta, const uint64_t *mem, uint64_t nm,
                                              const so_grid *gg, const float smin[3], const int64_t sijk[3], int64_t S, float h, float rs,
                                              int corrected, float t_low, float t_high) {
    int64_t np = S + 1;
    size_t npts = (size_t)(np * np * np);
    float c = gg->cell_size;
    int64_t R = (int64_t)f_ceil(h / c);
    float *sum[14];
    for (int k = 0; k < 14; ++k) sum[k] = acc + (size_t)k * npts;      /* S X Y Z, Tx Ty Tz, Mxx Mxy Mxz Myy Myz Mzz, Q */
    memset(acc, 0, sizeof(float) * 14 * npts);
    float h2 = h * h;
    for (uint64_t a = 0; a < nm; ++a) {
        const float *p = xyz + 3 * mem[a];
        float dj = delta[mem[a]];
        int64_t lo[3], up[3];
        influence_box(p, smin, c, R, np, lo, up);
        for (int64_t i = lo[0]; i < up[0]; ++i) for (int64_t j = lo[1]; j < up[1]; ++j) for (int64_t k = lo[2]; k < up[2]; ++k) {
            float gx = grid_coord(gg, 0, sijk[0] * S + i), gy = grid_coord(gg, 1, sijk[1] * S + j), gz = grid_coord(gg, 2, sijk[2] * S + k);
            float d[3] = { p[0] - gx, p[1] - gy, p[2] - gz };
            float d2 = (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2];
            if (!(d2 < h2)) continue;
            float u = 1.0f - d2 / h2;
            float uu = u * u;
            float w = uu * u;
            size_t q = (size_t)((i * np + j) * np + k);
            sum[0][q] = sum[0][q] + w;
            for (int b = 0; b < 3; ++b) sum[1 + b][q] = sum[1 + b][q] + w * d[b];
            sum[13][q] = sum[13][q] + w * dj;
            if (!corrected) continue;
            float e[3] = { uu * d[0], uu * d[1], uu * d[2] };
            for (int b = 0; b < 3; ++b) sum[4 + b][q] = sum[4 + b][q] + e[b];
            int slot = 7;
            for (int ia = 0; ia < 3; ++ia) for (int ib = ia; ib < 3; ++ib, ++slot) sum[slot][q] = sum[slot][q] + e[ia] * d[ib];
        }
    }
    for (size_t q = 0; q < npts; ++q) {
        float s = sum[0][q];
        if (!(s > 0.0f)) { phi[q] = 0.0f; continue; }
        float m[3], t[3], qq[3][3];
        for (int b = 0; b < 3; ++b) m[b] = sum[1 + b][q] / s;
        float m2 = (m[0] * m[0] + m[1] * m[1]) + m[2] * m[2];
        float plain = h - sqrtf(m2);
        float bq = sum[13][q] / s;
        if (!corrected) { phi[q] = plain + bq; continue; }
        for (int b = 0; b < 3; ++b) t[b] = sum[4 + b][q] / s;
        int slot = 7;
        for (int ia = 0; ia < 3; ++ia) for (int ib = ia; ib < 3; ++ib, ++slot) qq[ia][ib] = sum[slot][q] / s;
        float A[3][3];
        for (int ia = 0; ia < 3; ++ia) for (int ib = ia; ib < 3; ++ib) {
            A[ia][ib] = 0.5f * ((qq[ia][ib] - m[ia] * t[ib]) + (qq[ia][ib] - m[ib] * t[ia]));
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
        phi[q] = (plain + bq) - (rs + bq) * (1.0f - f);
    }
}

typedef struct { av_job av; const float *delta; float rs, t_low, t_high; int corrected; } ar_job;

static void ar_recon_task(int64_t s, void *ctx, void **tls) {
    ar_job *rj = (ar_job *)ctx;
    av_job *jb = &rj->av;
    int64_t S = jb->S, np = S + 1;
    size_t npts = (size_t)(np * np * np);
    if (!*tls) *tls = malloc(sizeof(float) * 15 * npts + sizeof(int64_t) * 3 * npts);
    int64_t *ev = (int64_t *)*tls;
    float *phi = (float *)(ev + 3 * npts), *acc = phi + npts;
    int64_t sijk[3]; unflatten_sub(jb->sg, jb->dc->flat[s], sijk);
    float smin[3];
    for (int d = 0; d < 3; ++d) smin[d] = grid_coord(jb->sg, d, sijk[d]);
    uint64_t nm = jb->dc->offset[s + 1] - jb->dc->offset[s];
    jb->res->subdomain_sparse[s] = 0;
    subdomain_levelset_averaged_radii(phi, acc, jb->xyz, rj->delta, jb->dc->members + jb->dc->offset[s], nm, jb->gg, smin, sijk, S, jb->h,
                                      rj->rs, rj->corrected, rj->t_low, rj->t_high);
    if (jb->tile_out && jb->dc->flat[s] == jb->tile_sub_flat) memcpy(jb->tile_out, phi, sizeof(float) * npts);
    subdomain_mc(&jb->patches[s], phi, smin, sijk, S, jb->c, jb->thr, ev);
}

/* so_reconstruct_averaged (corrected = 0) or so_reconstruct_averaged_corrected (corrected = 1, thresholds t_low, t_high) with the
 * radii r_j of the n_in input particles: the same grid, decomposition, densities, threshold t = h - R_s and refusals, plus 6
 * (SS_ERR_INVALID_PARAMETER) unless every R_j = radius_factor * r_j (all n_in, before the particle-AABB filter) lies in (0, h).
 * delta_j = R_j - R_s is compacted with the positions by the filter. */
int so_reconstruct_averaged_radii(const float *xyz_in, uint64_t n_in, const so_params *p, float radius_factor, const float *radii,
                                  int corrected, float t_low, float t_high, so_result **out, int64_t tile_sub_flat, float *tile_out) {
    so_result *res = (so_result *)calloc(1, sizeof(so_result));
    *out = res;
    lut_init();
    if (corrected && (!isfinite(t_low) || !isfinite(t_high) || !(t_low >= 0.0f) || !(t_low < t_high))) return 6;
    if (p->decomposition != 1) return 7;
    float h = p->compact_support_radius, c = p->cube_size;
    float rs = radius_factor * p->particle_radius;
    if (!(rs > 0.0f && rs < h) || !isfinite(rs)) return 6;
    for (uint64_t i = 0; i < n_in; ++i) {
        float R = radius_factor * radii[i];
        if (!(R > 0.0f && R < h)) return 6;
    }
    float thr = h - rs;
    const float *xyz = xyz_in; float *filtered = NULL; uint64_t n = n_in;
    float *delta = (float *)malloc(sizeof(float) * (n_in ? n_in : 1));
    if (p->has_particle_aabb) {
        res->inside_aabb = (uint8_t *)malloc(n_in ? n_in : 1);
        filtered = (float *)malloc(sizeof(float) * 3 * (n_in ? n_in : 1));
        n = 0;
        for (uint64_t i = 0; i < n_in; ++i) {
            int in = 1;
            for (int d = 0; d < 3; ++d) { float v = xyz_in[3 * i + d]; if (!(v >= p->aabb_min[d] && v < p->aabb_max[d])) in = 0; }
            res->inside_aabb[i] = (uint8_t)in;
            if (in) { memcpy(filtered + 3 * n, xyz_in + 3 * i, sizeof(float) * 3); delta[n] = radius_factor * radii[i] - rs; ++n; }
        }
        xyz = filtered;
    } else {
        for (uint64_t i = 0; i < n_in; ++i) delta[i] = radius_factor * radii[i] - rs;
    }
    res->n_filtered = n;
    so_grid g0;
    int err = grid_for_reconstruction(&g0, xyz, n, p);
    if (err) { free(filtered); free(delta); return err; }
    res->used_decomposition = 1;
    int64_t S = (int64_t)p->subdomain_num_cubes_per_dim;
    float r2 = p->particle_radius + p->particle_radius;
    float rest_mass = (r2 * r2 * r2) * p->rest_density;
    float margin = f_ceil(h / c) * c * 1.01f;
    int64_t nsubd[3], ncg[3];
    for (int d = 0; d < 3; ++d) { nsubd[d] = (g0.nc[d] + S - 1) / S; ncg[d] = nsubd[d] * S; }
    so_grid gg; grid_new(&gg, g0.aabb_min, ncg, c);
    float sub_size = c * (float)S;
    so_grid sg; grid_new(&sg, gg.aabb_min, nsubd, sub_size);
    res->grid = gg; res->subdomain_grid = sg;
    so_decomp dc; decompose(&dc, xyz, n, &sg, margin);
    res->n_subdomains = dc.nsub;
    res->subdomain_flat = (int64_t *)malloc(sizeof(int64_t) * (dc.nsub ? dc.nsub : 1));
    res->subdomain_count = (uint64_t *)malloc(sizeof(uint64_t) * (dc.nsub ? dc.nsub : 1));
    res->subdomain_sparse = (uint8_t *)malloc(dc.nsub ? dc.nsub : 1);
    uint64_t maxp = 0;
    for (uint64_t s = 0; s < dc.nsub; ++s) {
        res->subdomain_flat[s] = dc.flat[s];
        res->subdomain_count[s] = dc.offset[s + 1] - dc.offset[s];
        if (res->subdomain_count[s] > maxp) maxp = res->subdomain_count[s];
    }
    res->max_particles = maxp; res->sparse_limit = maxp / 20 < 100 ? 100 : maxp / 20;
    res->densities = (float *)calloc(n ? n : 1, sizeof(float));

    ar_job job;
    memset(&job, 0, sizeof(job));
    job.av.xyz = xyz; job.av.sg = &sg; job.av.gg = &gg; job.av.dc = &dc; job.av.res = res;
    job.av.h = h; job.av.c = c; job.av.thr = thr; job.av.margin = margin; job.av.rest_mass = rest_mass; job.av.S = S;
    job.av.tile_sub_flat = tile_sub_flat; job.av.tile_out = tile_out;
    job.delta = delta; job.rs = rs; job.t_low = t_low; job.t_high = t_high; job.corrected = corrected;
    parallel_for((int64_t)dc.nsub, av_density_task, &job.av);
    so_patch *patches = (so_patch *)calloc(dc.nsub ? dc.nsub : 1, sizeof(so_patch));
    job.av.patches = patches;
    parallel_for((int64_t)dc.nsub, ar_recon_task, &job);
    stitch(res, patches, dc.nsub);
    for (uint64_t s = 0; s < dc.nsub; ++s) { free(patches[s].v); free(patches[s].vkey); free(patches[s].vinterior); free(patches[s].t); }
    free(patches);
    free(dc.flat); free(dc.offset); free(dc.members);
    free(filtered); free(delta);
    return 0;
}
