/*
 * averaged_oracle.c -- plain-C restatement of the averaged-position surface (DESIGN.md section 12), TEST INFRASTRUCTURE ONLY.
 *
 * Built by tests/test_averaged_surface.py into a temporary directory.  It includes the pinned oracle (oracle/splashsurf_oracle.c,
 * unchanged) for the grid, the decomposition, the densities, marching cubes and stitching, and adds the averaged level set in the
 * operation order of splashsurf_b200/csrc/ss_averaged.cuh.  Compile it like the oracle: single precision, un-contracted
 * (-ffp-contract=off).
 */
#include "../oracle/splashsurf_oracle.c"

/* f(g) = h - |sum_j w_j d_j / sum_j w_j| (the norm of the averaged offset), d_j = x_j - g, w_j = (1 - |d_j|^2 / h^2)^3 over the
 * members of one subdomain within h of g, ascending index; 0 where no member is within h (or the weights sum to 0).  acc: 4 np^3
 * floats of scratch. */
static void subdomain_levelset_averaged(float *phi, float *acc, const float *xyz, const uint64_t *mem, uint64_t nm, const so_grid *gg,
                                        const float smin[3], const int64_t sijk[3], int64_t S, float h) {
    int64_t np = S + 1;
    size_t npts = (size_t)(np * np * np);
    float c = gg->cell_size;
    int64_t R = (int64_t)f_ceil(h / c);
    float *sw = acc, *sx = acc + npts, *sy = acc + 2 * npts, *sz = acc + 3 * npts;
    memset(acc, 0, sizeof(float) * 4 * npts);
    float h2 = h * h;
    for (uint64_t a = 0; a < nm; ++a) {
        const float *p = xyz + 3 * mem[a];
        int64_t lo[3], up[3];
        influence_box(p, smin, c, R, np, lo, up);
        for (int64_t i = lo[0]; i < up[0]; ++i) for (int64_t j = lo[1]; j < up[1]; ++j) for (int64_t k = lo[2]; k < up[2]; ++k) {
            float gx = grid_coord(gg, 0, sijk[0] * S + i), gy = grid_coord(gg, 1, sijk[1] * S + j), gz = grid_coord(gg, 2, sijk[2] * S + k);
            float dx = p[0] - gx, dy = p[1] - gy, dz = p[2] - gz;
            float d2 = (dx * dx + dy * dy) + dz * dz;
            if (!(d2 < h2)) continue;
            float u = 1.0f - d2 / h2;
            float w = (u * u) * u;
            size_t q = (size_t)((i * np + j) * np + k);
            sw[q] = sw[q] + w;
            sx[q] = sx[q] + w * dx; sy[q] = sy[q] + w * dy; sz[q] = sz[q] + w * dz;
        }
    }
    for (size_t q = 0; q < npts; ++q) {
        if (!(sw[q] > 0.0f)) { phi[q] = 0.0f; continue; }
        float mx = sx[q] / sw[q], my = sy[q] / sw[q], mz = sz[q] / sw[q];
        float m2 = (mx * mx + my * my) + mz * mz;
        phi[q] = h - sqrtf(m2);
    }
}

/* ------------------------------------------------------------ top level ---- */
typedef struct {
    const float *xyz; const so_grid *sg, *gg; const so_decomp *dc; so_result *res;
    float h, c, thr, margin, rest_mass; int64_t S; int64_t tile_sub_flat; float *tile_out; so_patch *patches;
} av_job;

static void av_density_task(int64_t s, void *ctx, void **tls) {
    (void)tls;
    av_job *jb = (av_job *)ctx;
    const so_decomp *dd = jb->dc;
    int64_t sijk[3]; unflatten_sub(jb->sg, dd->flat[s], sijk);
    subdomain_densities(jb->xyz, jb->sg, sijk, dd->members + dd->offset[s], dd->offset[s + 1] - dd->offset[s], jb->h, jb->margin,
                        jb->rest_mass, jb->res->densities, NULL, NULL, NULL);
}

static void av_recon_task(int64_t s, void *ctx, void **tls) {
    av_job *jb = (av_job *)ctx;
    int64_t S = jb->S, np = S + 1;
    size_t npts = (size_t)(np * np * np);
    if (!*tls) *tls = malloc(sizeof(float) * 5 * npts + sizeof(int64_t) * 3 * npts);
    int64_t *ev = (int64_t *)*tls;
    float *phi = (float *)(ev + 3 * npts), *acc = phi + npts;
    int64_t sijk[3]; unflatten_sub(jb->sg, jb->dc->flat[s], sijk);
    float smin[3];
    for (int d = 0; d < 3; ++d) smin[d] = grid_coord(jb->sg, d, sijk[d]);
    uint64_t nm = jb->dc->offset[s + 1] - jb->dc->offset[s];
    jb->res->subdomain_sparse[s] = 0;
    subdomain_levelset_averaged(phi, acc, jb->xyz, jb->dc->members + jb->dc->offset[s], nm, jb->gg, smin, sijk, S, jb->h);
    if (jb->tile_out && jb->dc->flat[s] == jb->tile_sub_flat) memcpy(jb->tile_out, phi, sizeof(float) * npts);
    subdomain_mc(&jb->patches[s], phi, smin, sijk, S, jb->c, jb->thr, ev);
}

/* so_reconstruct with the averaged-position surface: always decomposed on the standard margin (decomposition == 0 -> 7,
 * SS_ERR_UNSUPPORTED), surface f = h - R_s with R_s = radius_factor * particle_radius (0 < R_s < h, finite, else 6,
 * SS_ERR_INVALID_PARAMETER).  iso_surface_threshold is not used.  tile_out receives the level-set tile of subdomain tile_sub_flat
 * (or -1). */
int so_reconstruct_averaged(const float *xyz_in, uint64_t n_in, const so_params *p, float radius_factor, so_result **out,
                            int64_t tile_sub_flat, float *tile_out) {
    so_result *res = (so_result *)calloc(1, sizeof(so_result));
    *out = res;
    lut_init();
    if (p->decomposition != 1) return 7;
    float h = p->compact_support_radius, c = p->cube_size;
    float rs = radius_factor * p->particle_radius;
    if (!(rs > 0.0f && rs < h) || !isfinite(rs)) return 6;
    float thr = h - rs;
    /* lib.rs:369-406 particle AABB filter (half-open contains_point) */
    const float *xyz = xyz_in; float *filtered = NULL; uint64_t n = n_in;
    if (p->has_particle_aabb) {
        res->inside_aabb = (uint8_t *)malloc(n_in ? n_in : 1);
        filtered = (float *)malloc(sizeof(float) * 3 * (n_in ? n_in : 1));
        n = 0;
        for (uint64_t i = 0; i < n_in; ++i) {
            int in = 1;
            for (int d = 0; d < 3; ++d) { float v = xyz_in[3 * i + d]; if (!(v >= p->aabb_min[d] && v < p->aabb_max[d])) in = 0; }
            res->inside_aabb[i] = (uint8_t)in;
            if (in) { memcpy(filtered + 3 * n, xyz_in + 3 * i, sizeof(float) * 3); ++n; }
        }
        xyz = filtered;
    }
    res->n_filtered = n;
    so_grid g0;
    int err = grid_for_reconstruction(&g0, xyz, n, p);
    if (err) { free(filtered); return err; }
    res->used_decomposition = 1;
    /* dense_subdomains.rs:89-244 initialize_parameters */
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

    av_job job;
    memset(&job, 0, sizeof(job));
    job.xyz = xyz; job.sg = &sg; job.gg = &gg; job.dc = &dc; job.res = res;
    job.h = h; job.c = c; job.thr = thr; job.margin = margin; job.rest_mass = rest_mass; job.S = S;
    job.tile_sub_flat = tile_sub_flat; job.tile_out = tile_out;
    parallel_for((int64_t)dc.nsub, av_density_task, &job);
    so_patch *patches = (so_patch *)calloc(dc.nsub ? dc.nsub : 1, sizeof(so_patch));
    job.patches = patches;
    parallel_for((int64_t)dc.nsub, av_recon_task, &job);
    stitch(res, patches, dc.nsub);
    for (uint64_t s = 0; s < dc.nsub; ++s) { free(patches[s].v); free(patches[s].vkey); free(patches[s].vinterior); free(patches[s].t); }
    free(patches);
    free(dc.flat); free(dc.offset); free(dc.members);
    free(filtered);
    return 0;
}
