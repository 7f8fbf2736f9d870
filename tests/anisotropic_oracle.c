/*
 * anisotropic_oracle.c -- plain-C restatement of the anisotropic-kernel mode (DESIGN.md section 11), TEST INFRASTRUCTURE ONLY.
 *
 * Built by tests/test_anisotropic.py into a temporary directory.  It includes the pinned oracle (oracle/splashsurf_oracle.c,
 * unchanged) for the grid, the decomposition, the densities, marching cubes and stitching, and adds the anisotropy of every
 * particle and the anisotropic level set in the operation order of splashsurf_b200/csrc/ss_aniso.cuh.  Compile it like the oracle:
 * single precision, un-contracted (-ffp-contract=off).
 */
#include "../oracle/splashsurf_oracle.c"

/* DESIGN.md section 11, restated in the operation order of splashsurf_b200/csrc/ss_aniso.cuh.  Not part of the reference. */
typedef struct { int on; float lambda, kr; uint32_t min_nb; float *xbar, *g, *vdet; } so_aniso_cfg;
static so_aniso_cfg g_an;

static void aniso_jacobi_rot(float a[3][3], float v[3][3], int p, int q) {
    int r = 3 - p - q;
    float apq = a[p][q];
    if (apq == 0.0f) return;
    float theta = (a[q][q] - a[p][p]) / (2.0f * apq);
    float t = 1.0f / (fabsf(theta) + sqrtf(theta * theta + 1.0f));
    if (theta < 0.0f) t = -t;
    float c = 1.0f / sqrtf(t * t + 1.0f);
    float s = t * c;
    float app = a[p][p] - t * apq, aqq = a[q][q] + t * apq;
    float arp = c * a[r][p] - s * a[r][q], arq = s * a[r][p] + c * a[r][q];
    a[p][p] = app; a[q][q] = aqq; a[p][q] = 0.0f; a[q][p] = 0.0f;
    a[r][p] = arp; a[p][r] = arp; a[r][q] = arq; a[q][r] = arq;
    for (int k = 0; k < 3; ++k) {
        float vkp = v[k][p], vkq = v[k][q];
        v[k][p] = c * vkp - s * vkq;
        v[k][q] = s * vkp + c * vkq;
    }
}

/* G (g00 g01 g02 g11 g12 g22) and det G of covariance a; nn = neighbours without the particle itself */
static void aniso_matrix(float a[3][3], uint64_t nn, float g[6], float *det) {
    float v[3][3] = { { 1, 0, 0 }, { 0, 1, 0 }, { 0, 0, 1 } };
    for (int sweep = 0; sweep < 8; ++sweep) { aniso_jacobi_rot(a, v, 0, 1); aniso_jacobi_rot(a, v, 0, 2); aniso_jacobi_rot(a, v, 1, 2); }
    float e[3] = { a[0][0], a[1][1], a[2][2] };
    int ord[3] = { 0, 1, 2 };
    const int cx[3][2] = { { 0, 1 }, { 1, 2 }, { 0, 1 } };
    for (int q = 0; q < 3; ++q) {
        int i = cx[q][0], j = cx[q][1];
        if (e[i] < e[j]) { float te = e[i]; e[i] = e[j]; e[j] = te; int to = ord[i]; ord[i] = ord[j]; ord[j] = to; }
    }
    for (int k = 0; k < 3; ++k) if (e[k] < 0.0f) e[k] = 0.0f;
    if (nn < g_an.min_nb || e[0] == 0.0f) {
        g[0] = 1; g[1] = 0; g[2] = 0; g[3] = 1; g[4] = 0; g[5] = 1; *det = 1.0f;
        return;
    }
    float floor_s = e[0] / g_an.kr, inv[3];
    for (int k = 0; k < 3; ++k) inv[k] = 1.0f / (fmaxf(e[k], floor_s) / e[0]);
    *det = (inv[0] * inv[1]) * inv[2];
    const int ia[6] = { 0, 0, 0, 1, 1, 2 }, ib[6] = { 0, 1, 2, 1, 2, 2 };
    for (int q = 0; q < 6; ++q) {
        float acc = (v[ia[q]][ord[0]] * inv[0]) * v[ib[q]][ord[0]];
        acc = acc + (v[ia[q]][ord[1]] * inv[1]) * v[ib[q]][ord[1]];
        acc = acc + (v[ia[q]][ord[2]] * inv[2]) * v[ib[q]][ord[2]];
        g[q] = acc;
    }
}

/* x_bar, G, det G of the particles inside one subdomain of the STANDARD decomposition: the density stage's neighbours
 * (d^2 < h^2, same NS grid and visiting order as subdomain_densities) */
static void subdomain_anisotropy(const float *xyz, const so_grid *sg, const int64_t sijk[3], const uint64_t *mem, uint64_t nm, float h, float margin) {
    float smin[3], smax[3], mmin[3], mmax[3];
    float grow = margin * 1.5f;
    for (int d = 0; d < 3; ++d) {
        smin[d] = grid_coord(sg, d, sijk[d]); smax[d] = grid_coord(sg, d, sijk[d] + 1);
        mmin[d] = smin[d] - grow; mmax[d] = smax[d] + grow;
    }
    so_grid ns;
    if (grid_from_aabb(&ns, mmin, mmax, h) != 0) { fprintf(stderr, "oracle: NS grid construction failed\n"); abort(); }
    int64_t ncell = ns.nc[0] * ns.nc[1] * ns.nc[2];
    uint64_t *cstart = (uint64_t *)calloc((size_t)ncell + 1, sizeof(uint64_t));
    int64_t *cell_of = (int64_t *)malloc(sizeof(int64_t) * (nm ? nm : 1));
    for (uint64_t a = 0; a < nm; ++a) {
        const float *p = xyz + 3 * mem[a];
        int64_t c[3];
        for (int d = 0; d < 3; ++d) c[d] = grid_cell_of(&ns, d, p[d]);
        cell_of[a] = c[0] * ns.nc[1] * ns.nc[2] + c[1] * ns.nc[2] + c[2];
        cstart[cell_of[a] + 1]++;
    }
    for (int64_t c = 0; c < ncell; ++c) cstart[c + 1] += cstart[c];
    uint64_t *order = (uint64_t *)malloc(sizeof(uint64_t) * (nm ? nm : 1));
    uint64_t *cur = (uint64_t *)malloc(sizeof(uint64_t) * (size_t)(ncell ? ncell : 1));
    memcpy(cur, cstart, sizeof(uint64_t) * (size_t)ncell);
    for (uint64_t a = 0; a < nm; ++a) order[cur[cell_of[a]]++] = a;
    free(cur);
    float h2 = h * h;
    for (uint64_t a = 0; a < nm; ++a) {
        const float *pi = xyz + 3 * mem[a];
        int inside = 1;
        for (int d = 0; d < 3; ++d) if (!(pi[d] >= smin[d] && pi[d] < smax[d])) inside = 0;
        if (!inside) continue;
        int64_t c[3];
        for (int d = 0; d < 3; ++d) c[d] = grid_cell_of(&ns, d, pi[d]);
        float sw = 1.0f, m[3] = { 0, 0, 0 }, cv[6];
        uint64_t nn = 0;
        for (int phase = 0; phase < 2; ++phase) {
            if (phase == 1) {
                for (int d = 0; d < 3; ++d) m[d] = m[d] / sw;
                float ex = 0.0f - m[0], ey = 0.0f - m[1], ez = 0.0f - m[2];
                cv[0] = ex * ex; cv[1] = ex * ey; cv[2] = ex * ez; cv[3] = ey * ey; cv[4] = ey * ez; cv[5] = ez * ez;
            }
            for (int pass = 0; pass < 2; ++pass)
            for (int sx = -1; sx <= 1; ++sx) for (int sy = -1; sy <= 1; ++sy) for (int sz = -1; sz <= 1; ++sz) {
                int self = (sx == 0 && sy == 0 && sz == 0);
                if ((pass == 0) == self) continue;
                int64_t q[3] = { c[0] + sx, c[1] + sy, c[2] + sz };
                if (q[0] < 0 || q[1] < 0 || q[2] < 0 || q[0] >= ns.nc[0] || q[1] >= ns.nc[1] || q[2] >= ns.nc[2]) continue;
                int64_t fc = q[0] * ns.nc[1] * ns.nc[2] + q[1] * ns.nc[2] + q[2];
                for (uint64_t t = cstart[fc]; t < cstart[fc + 1]; ++t) {
                    uint64_t b = order[t];
                    if (b == a) continue;
                    const float *pj = xyz + 3 * mem[b];
                    float dx = pj[0] - pi[0], dy = pj[1] - pi[1], dz = pj[2] - pi[2];
                    float d2 = dx * dx + dy * dy + dz * dz;
                    if (!(d2 < h2)) continue;
                    float qq = sqrtf(d2) / h;
                    float w = 1.0f - (qq * qq) * qq;
                    if (phase == 0) { sw = sw + w; m[0] = m[0] + w * dx; m[1] = m[1] + w * dy; m[2] = m[2] + w * dz; ++nn; }
                    else {
                        float ex = dx - m[0], ey = dy - m[1], ez = dz - m[2];
                        float wx = w * ex, wy = w * ey, wz = w * ez;
                        cv[0] = cv[0] + wx * ex; cv[1] = cv[1] + wx * ey; cv[2] = cv[2] + wx * ez;
                        cv[3] = cv[3] + wy * ey; cv[4] = cv[4] + wy * ez; cv[5] = cv[5] + wz * ez;
                    }
                }
            }
        }
        for (int k = 0; k < 6; ++k) cv[k] = cv[k] / sw;
        float A[3][3] = { { cv[0], cv[1], cv[2] }, { cv[1], cv[3], cv[4] }, { cv[2], cv[4], cv[5] } };
        uint64_t pid = mem[a];
        for (int d = 0; d < 3; ++d) g_an.xbar[3 * pid + d] = pi[d] + g_an.lambda * m[d];
        aniso_matrix(A, nn, g_an.g + 6 * pid, &g_an.vdet[pid]);
    }
    free(order); free(cell_of); free(cstart);
}

/* phi(x) = sum_j V_j det G_j W(|G_j (x - x_bar_j)|) over the members of one subdomain (WIDE decomposition), ascending index;
 * vdet = V det G per particle */
static void subdomain_levelset_aniso(float *phi, const uint64_t *mem, uint64_t nm, const so_grid *gg, const float smin[3],
                                     const int64_t sijk[3], int64_t S, float h) {
    int64_t np = S + 1;
    float c = gg->cell_size;
    int64_t R = (int64_t)f_ceil(h / c);
    memset(phi, 0, sizeof(float) * (size_t)(np * np * np));
    k_scalar kern = k_scalar_new(h);
    float h2 = h * h;
    for (uint64_t a = 0; a < nm; ++a) {
        uint64_t pid = mem[a];
        const float *p = g_an.xbar + 3 * pid, *g = g_an.g + 6 * pid;
        float vd = g_an.vdet[pid];
        int64_t lo[3], up[3];
        influence_box(p, smin, c, R, np, lo, up);
        for (int64_t i = lo[0]; i < up[0]; ++i) for (int64_t j = lo[1]; j < up[1]; ++j) for (int64_t k = lo[2]; k < up[2]; ++k) {
            float gx = grid_coord(gg, 0, sijk[0] * S + i), gy = grid_coord(gg, 1, sijk[1] * S + j), gz = grid_coord(gg, 2, sijk[2] * S + k);
            float dx = p[0] - gx, dy = p[1] - gy, dz = p[2] - gz;
            float u0 = (g[0] * dx + g[1] * dy) + g[2] * dz;
            float u1 = (g[1] * dx + g[3] * dy) + g[4] * dz;
            float u2 = (g[2] * dx + g[4] * dy) + g[5] * dz;
            float uu = (u0 * u0 + u1 * u1) + u2 * u2;
            if (uu < h2) phi[(i * np + j) * np + k] += vd * k_scalar_eval(&kern, sqrtf(uu));
        }
    }
}

/* ------------------------------------------------------------ top level ---- */
typedef struct {
    const float *xyz; const so_grid *sg, *gg; const so_decomp *dc, *dstd; so_result *res;
    float h, c, thr, margin, rest_mass; int64_t S; int64_t tile_sub_flat; float *tile_out; so_patch *patches;
} an_job;

static void an_density_task(int64_t s, void *ctx, void **tls) {
    (void)tls;
    an_job *jb = (an_job *)ctx;
    const so_decomp *dd = jb->dstd;
    int64_t sijk[3]; unflatten_sub(jb->sg, dd->flat[s], sijk);
    subdomain_densities(jb->xyz, jb->sg, sijk, dd->members + dd->offset[s], dd->offset[s + 1] - dd->offset[s], jb->h, jb->margin,
                        jb->rest_mass, jb->res->densities, NULL, NULL, NULL);
}

static void an_aniso_task(int64_t s, void *ctx, void **tls) {
    (void)tls;
    an_job *jb = (an_job *)ctx;
    const so_decomp *dd = jb->dstd;
    int64_t sijk[3]; unflatten_sub(jb->sg, dd->flat[s], sijk);
    subdomain_anisotropy(jb->xyz, jb->sg, sijk, dd->members + dd->offset[s], dd->offset[s + 1] - dd->offset[s], jb->h, jb->margin);
}

static void an_recon_task(int64_t s, void *ctx, void **tls) {
    an_job *jb = (an_job *)ctx;
    int64_t S = jb->S, np = S + 1;
    size_t npts = (size_t)(np * np * np);
    if (!*tls) *tls = malloc(sizeof(float) * npts + sizeof(int64_t) * 3 * npts);
    int64_t *ev = (int64_t *)*tls;
    float *phi = (float *)(ev + 3 * npts);
    int64_t sijk[3]; unflatten_sub(jb->sg, jb->dc->flat[s], sijk);
    float smin[3];
    for (int d = 0; d < 3; ++d) smin[d] = grid_coord(jb->sg, d, sijk[d]);
    uint64_t nm = jb->dc->offset[s + 1] - jb->dc->offset[s];
    jb->res->subdomain_sparse[s] = 0;
    subdomain_levelset_aniso(phi, jb->dc->members + jb->dc->offset[s], nm, jb->gg, smin, sijk, S, jb->h);
    if (jb->tile_out && jb->dc->flat[s] == jb->tile_sub_flat) memcpy(jb->tile_out, phi, sizeof(float) * npts);
    subdomain_mc(&jb->patches[s], phi, smin, sijk, S, jb->c, jb->thr, ev);
}

/* lib.rs:369-406 particle AABB filter (half-open contains_point; inside, when not NULL, receives the flags) and
 * dense_subdomains.rs:89-244 initialize_parameters: the filtered particles, the grid and the subdomain grid.  Returns the error of
 * grid_for_reconstruction; s->filtered is the caller's to free either way. */
typedef struct { const float *xyz; float *filtered; uint64_t n; so_grid gg, sg; float h, c, margin, rest_mass; int64_t S; } an_setup;

static int an_setup_new(an_setup *s, const float *xyz_in, uint64_t n_in, const so_params *p, uint8_t *inside) {
    s->xyz = xyz_in; s->filtered = NULL; s->n = n_in;
    if (p->has_particle_aabb) {
        s->filtered = (float *)malloc(sizeof(float) * 3 * (n_in ? n_in : 1));
        s->n = 0;
        for (uint64_t i = 0; i < n_in; ++i) {
            int in = 1;
            for (int d = 0; d < 3; ++d) { float v = xyz_in[3 * i + d]; if (!(v >= p->aabb_min[d] && v < p->aabb_max[d])) in = 0; }
            if (inside) inside[i] = (uint8_t)in;
            if (in) { memcpy(s->filtered + 3 * s->n, xyz_in + 3 * i, sizeof(float) * 3); ++s->n; }
        }
        s->xyz = s->filtered;
    }
    so_grid g0;
    int err = grid_for_reconstruction(&g0, s->xyz, s->n, p);
    if (err) return err;
    int64_t S = (int64_t)p->subdomain_num_cubes_per_dim;
    float r2 = p->particle_radius + p->particle_radius;
    s->S = S;
    s->rest_mass = (r2 * r2 * r2) * p->rest_density;
    s->h = p->compact_support_radius; s->c = p->cube_size;
    s->margin = f_ceil(s->h / s->c) * s->c * 1.01f;
    int64_t nsubd[3], ncg[3];
    for (int d = 0; d < 3; ++d) { nsubd[d] = (g0.nc[d] + S - 1) / S; ncg[d] = nsubd[d] * S; }
    grid_new(&s->gg, g0.aabb_min, ncg, s->c);
    float sub_size = s->c * (float)S;
    grid_new(&s->sg, s->gg.aabb_min, nsubd, sub_size);
    return 0;
}

/* The densities (rho), then x_bar (n x 3), G (n x 6) and V det G (n) of the set-up particles, on the standard decomposition; g_an
 * keeps pointing at them for the level set. */
static void an_records(const an_setup *s, float smoothing, float max_stretch, uint32_t min_neighbors, float *rho, float *xbar, float *g,
                       float *vdet) {
    so_decomp dstd; decompose(&dstd, s->xyz, s->n, &s->sg, s->margin);
    so_result res;
    memset(&res, 0, sizeof(res));
    res.densities = rho;
    memset(rho, 0, sizeof(float) * s->n);
    g_an.on = 1; g_an.lambda = smoothing; g_an.kr = max_stretch; g_an.min_nb = min_neighbors;
    g_an.xbar = xbar; g_an.g = g; g_an.vdet = vdet;
    an_job job;
    memset(&job, 0, sizeof(job));
    job.xyz = s->xyz; job.sg = &s->sg; job.gg = &s->gg; job.dstd = &dstd; job.res = &res;
    job.h = s->h; job.c = s->c; job.margin = s->margin; job.rest_mass = s->rest_mass; job.S = s->S;
    parallel_for((int64_t)dstd.nsub, an_density_task, &job);
    for (uint64_t i = 0; i < s->n; ++i) {
        for (int d = 0; d < 3; ++d) g_an.xbar[3 * i + d] = s->xyz[3 * i + d];
        float id[6] = { 1, 0, 0, 1, 0, 1 };
        memcpy(g_an.g + 6 * i, id, sizeof(id));
        g_an.vdet[i] = 1.0f;
    }
    parallel_for((int64_t)dstd.nsub, an_aniso_task, &job);
    for (uint64_t i = 0; i < s->n; ++i) g_an.vdet[i] = (s->rest_mass / rho[i]) * g_an.vdet[i];
    free(dstd.flat); free(dstd.offset); free(dstd.members);
}

/* The records of the anisotropic level set as so_reconstruct_aniso computes them: the densities (rho_out), x_bar (xbar_out, n x 3),
 * G (g_out, n x 6) and V det G (vdet_out) of the n filtered particles (buffers of n_in); returns n, or -(error code). */
int64_t so_aniso_records(const float *xyz_in, uint64_t n_in, const so_params *p, float smoothing, float max_stretch, uint32_t min_neighbors,
                         float *xbar_out, float *g_out, float *vdet_out, float *rho_out) {
    an_setup s;
    int err = an_setup_new(&s, xyz_in, n_in, p, NULL);
    if (!err) an_records(&s, smoothing, max_stretch, min_neighbors, rho_out, xbar_out, g_out, vdet_out);
    memset(&g_an, 0, sizeof(g_an));
    free(s.filtered);
    return err ? -(int64_t)err : (int64_t)s.n;
}

/* so_reconstruct with anisotropic kernels: always decomposed (decomposition == 0 -> 7, SS_ERR_UNSUPPORTED).  xbar_out (>= n_in x 3)
 * and g_out (>= n_in x 6: g00 g01 g02 g11 g12 g22) receive x_bar and G of the n_filtered particles; tile_out the level-set tile of
 * subdomain tile_sub_flat (or -1). */
int so_reconstruct_aniso(const float *xyz_in, uint64_t n_in, const so_params *p, float smoothing, float max_stretch, uint32_t min_neighbors,
                         so_result **out, int64_t tile_sub_flat, float *tile_out, float *xbar_out, float *g_out) {
    so_result *res = (so_result *)calloc(1, sizeof(so_result));
    *out = res;
    lut_init();
    if (p->decomposition != 1) return 7;
    if (p->has_particle_aabb) res->inside_aabb = (uint8_t *)malloc(n_in ? n_in : 1);
    an_setup s;
    int err = an_setup_new(&s, xyz_in, n_in, p, res->inside_aabb);
    res->n_filtered = s.n;
    if (err) { free(s.filtered); return err; }
    res->used_decomposition = 1;
    res->grid = s.gg; res->subdomain_grid = s.sg;
    uint64_t n = s.n;
    /* memberships within 2h (kernel centres move by up to smoothing * h); densities and anisotropy on the standard margin */
    so_decomp dc; decompose(&dc, s.xyz, n, &s.sg, f_ceil((2.0f * s.h) / s.c) * s.c * 1.01f);
    res->n_subdomains = dc.nsub;
    res->subdomain_flat = (int64_t *)malloc(sizeof(int64_t) * (dc.nsub ? dc.nsub : 1));
    res->subdomain_count = (uint64_t *)malloc(sizeof(uint64_t) * (dc.nsub ? dc.nsub : 1));
    res->subdomain_sparse = (uint8_t *)malloc(dc.nsub ? dc.nsub : 1);
    uint64_t maxp = 0;
    for (uint64_t k = 0; k < dc.nsub; ++k) {
        res->subdomain_flat[k] = dc.flat[k];
        res->subdomain_count[k] = dc.offset[k + 1] - dc.offset[k];
        if (res->subdomain_count[k] > maxp) maxp = res->subdomain_count[k];
    }
    res->max_particles = maxp; res->sparse_limit = maxp / 20 < 100 ? 100 : maxp / 20;
    res->densities = (float *)calloc(n ? n : 1, sizeof(float));
    float *vdet = (float *)malloc(sizeof(float) * (n ? n : 1));
    an_records(&s, smoothing, max_stretch, min_neighbors, res->densities, xbar_out, g_out, vdet);

    an_job job;
    memset(&job, 0, sizeof(job));
    job.xyz = s.xyz; job.sg = &s.sg; job.gg = &s.gg; job.dc = &dc; job.res = res;
    job.h = s.h; job.c = s.c; job.thr = p->iso_surface_threshold; job.margin = s.margin; job.rest_mass = s.rest_mass; job.S = s.S;
    job.tile_sub_flat = tile_sub_flat; job.tile_out = tile_out;
    so_patch *patches = (so_patch *)calloc(dc.nsub ? dc.nsub : 1, sizeof(so_patch));
    job.patches = patches;
    parallel_for((int64_t)dc.nsub, an_recon_task, &job);
    stitch(res, patches, dc.nsub);
    for (uint64_t k = 0; k < dc.nsub; ++k) { free(patches[k].v); free(patches[k].vkey); free(patches[k].vinterior); free(patches[k].t); }
    free(patches);
    free(dc.flat); free(dc.offset); free(dc.members);
    free(vdet);
    memset(&g_an, 0, sizeof(g_an));
    free(s.filtered);
    return 0;
}
