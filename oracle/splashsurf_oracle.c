/*
 * splashsurf_oracle.c -- CPU restatement of the splashsurf reconstruct hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under splashsurf_b200/ may import, link or
 * execute this file; only tests/, __graft_entry__.smoke() and bench.py's
 * cpu_baseline / --impl reference legs use it, and only as the checker.
 *
 * Parity status: PINNED.  tests/test_oracle_vs_reference.py checks this
 * restatement against the reference's own prebuilt binary (the pysplashsurf
 * 0.14.0 wheel shipped in /root/reference/splashsurf_studio/src/wheels, unpacked
 * by oracle/build_ref.sh into oracle/_ref/) -- particle densities bit-exact,
 * mesh connectivity identical after canonical ordering, vertex positions
 * bit-exact for interior vertices -- and against the golden fixtures generated
 * from that binary under tests/golden/.
 *
 * The file follows the f32 / i64 instantiation of the reference (the default
 * one in every front-end).  Each function cites the reference file:line whose
 * behaviour it restates (paths relative to splashsurf_lib/src/).  All float
 * arithmetic is single precision, un-contracted (-ffp-contract=off); fused
 * multiply-adds appear only where the reference's AVX2 path writes them
 * explicitly (fmaf below == _mm256_fmadd_ps lane).
 */
#include <math.h>
#include <float.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <stdio.h>
#include <pthread.h>
#include <stdatomic.h>
#include <unistd.h>

#define SO_PI_F 3.14159265358979323846f /* std::f32::consts::PI */

typedef struct {
    float particle_radius, rest_density, compact_support_radius, cube_size, iso_surface_threshold;
    int32_t has_particle_aabb;
    float aabb_min[3], aabb_max[3];
    int32_t enable_simd;      /* 1: AVX2-FMA grid loop semantics, 0: scalar grid loop */
    int32_t decomposition;    /* 1: UniformGrid, 0: None (global path, sequential semantics) */
    uint32_t subdomain_num_cubes_per_dim;
    int32_t auto_disable;
} so_params;

typedef struct {
    float aabb_min[3], aabb_max[3];
    float cell_size;
    int64_t np[3], nc[3];
} so_grid;

typedef struct {
    /* grids */
    so_grid grid;           /* SurfaceReconstruction.grid (subdomain-padded global MC grid) */
    so_grid subdomain_grid; /* grid of subdomains */
    int32_t used_decomposition;
    /* filtered particles */
    uint64_t n_filtered;
    uint8_t *inside_aabb;   /* n entries or NULL */
    float *densities;       /* n_filtered */
    /* mesh */
    uint64_t nv, nt;
    float *vertices;        /* nv*3 */
    uint64_t *triangles;    /* nt*3 */
    int64_t *vertex_keys;   /* nv*4: global point i,j,k + axis of the MC edge carrying the vertex */
    /* decomposition stats */
    uint64_t n_subdomains;
    int64_t *subdomain_flat;   /* n_subdomains, ascending flat index */
    uint64_t *subdomain_count; /* particles (owned+ghost) per subdomain */
    uint8_t *subdomain_sparse;
    uint64_t max_particles, sparse_limit;
} so_result;

/* ---------------------------------------------------------------- LUT ---- */
/* Classic 256x16 marching cubes triangle table; generated into mc_lut.inc by
 * tools/derive_mc_lut.py from black-box probing of the reference binary (see
 * tests/golden/mc_lut_cases.json).  Raw (un-reversed) edge triplets. */
#include "../splashsurf_b200/csrc/mc_lut.inc"
static signed char SS_MC_TRI_TABLE[256][16];
static int g_lut_ready = 0;
static void lut_init(void) { if (!g_lut_ready) { ss_mc_unpack(SS_MC_TRI_TABLE); g_lut_ready = 1; } }

/* ------------------------------------------------------------- helpers ---- */
static inline float f_floor(float x) { return floorf(x); }
static inline float f_ceil(float x) { return ceilf(x); }

/* uniform_grid.rs:175-232 (from_aabb / new / checked_aabb) */
static int grid_new(so_grid *g, const float min[3], const int64_t nc[3], float cell) {
    for (int d = 0; d < 3; ++d) {
        g->aabb_min[d] = min[d];
        g->nc[d] = nc[d];
        g->np[d] = nc[d] + 1;
        g->aabb_max[d] = min[d] + cell * (float)nc[d];
    }
    g->cell_size = cell;
    return 0;
}

static int grid_from_aabb(so_grid *g, const float mn[3], const float mx[3], float cell) {
    if (!(cell > 0.0f)) return 1;                       /* InvalidCellSize */
    if (mn[0] == mx[0] && mn[1] == mx[1] && mn[2] == mx[2]) return 2; /* DegenerateAabb: min == max (aabb.rs:159-161) */
    for (int d = 0; d < 3; ++d) if (!(mn[d] <= mx[d])) return 3; /* InconsistentAabb */
    float amin[3]; int64_t nc[3];
    for (int d = 0; d < 3; ++d) {
        amin[d] = f_floor(mn[d] / cell) * cell;         /* unscale, floor, scale */
        float ext = mx[d] - amin[d];
        float ncr = f_ceil(ext / cell);
        int64_t n = (int64_t)ncr;
        nc[d] = n > 1 ? n : 1;
    }
    return grid_new(g, amin, nc, cell);
}

/* uniform_grid.rs:418-437 point_coordinates: min + (i as R)*cell */
static inline float grid_coord(const so_grid *g, int d, int64_t i) {
    return g->aabb_min[d] + (float)i * g->cell_size;
}
/* uniform_grid.rs:444-451 enclosing_cell */
static inline int64_t grid_cell_of(const so_grid *g, int d, float x) {
    return (int64_t)f_floor((x - g->aabb_min[d]) / g->cell_size);
}

/* kernel.rs:51-107 scalar cubic spline */
typedef struct { float h, sigma; } k_scalar;
static k_scalar k_scalar_new(float h) { k_scalar k; k.h = h; k.sigma = 8.0f / (h * h * h); return k; }
static inline float k_scalar_cubic(float q) {
    if (q < 1.0f) {
        return (3.0f / (2.0f * SO_PI_F)) * ((2.0f / 3.0f) - q * q + 0.5f * q * q * q);
    } else if (q < 2.0f) {
        float x = 2.0f - q;
        return (1.0f / (4.0f * SO_PI_F)) * x * x * x;
    }
    return 0.0f;
}
static inline float k_scalar_eval(const k_scalar *k, float r) {
    float q = (r + r) / k->h;
    return k->sigma * k_scalar_cubic(q);
}

/* kernel.rs:321-379 AVX2+FMA cubic spline, one lane */
typedef struct { float hinv, sigma, s2, s6, s12; } k_avx;
static k_avx k_avx_new(float h) {
    k_avx k; k.hinv = 1.0f / h; float rrr = h * h * h;
    k.sigma = 8.0f / (SO_PI_F * rrr);
    k.s2 = 2.0f * k.sigma; k.s6 = 6.0f * k.sigma; k.s12 = 12.0f * k.sigma;
    return k;
}
static inline float k_avx_eval(const k_avx *k, float r) {
    float q = r * k->hinv;
    float v = 1.0f - q;
    v = v > 0.0f ? v : 0.0f;             /* _mm256_max_ps(v, 0) */
    float v2 = v * v, v3 = v2 * v;
    float outer = v3 * k->s2;
    float inner = k->sigma;
    inner = fmaf(-v, k->s6, inner);      /* fnmadd */
    inner = fmaf(v2, k->s12, inner);     /* fmadd  */
    inner = fmaf(-v3, k->s6, inner);     /* fnmadd */
    return (q <= 0.5f) ? inner : outer;  /* blendv on q <= 0.5 */
}

/* ------------------------------------------------------- grid for recon ---- */
/* lib.rs:476-516 + density_map.rs:551-580 */
static int grid_for_reconstruction(so_grid *g, const float *xyz, uint64_t n, const so_params *p) {
    float mn[3], mx[3];
    if (p->has_particle_aabb) {
        for (int d = 0; d < 3; ++d) { mn[d] = p->aabb_min[d]; mx[d] = p->aabb_max[d]; }
    } else {
        if (n == 0) { for (int d = 0; d < 3; ++d) mn[d] = mx[d] = 0.0f; }
        else {
            for (int d = 0; d < 3; ++d) mn[d] = mx[d] = xyz[d];
            for (uint64_t i = 1; i < n; ++i) for (int d = 0; d < 3; ++d) {
                float v = xyz[3 * i + d];
                if (v < mn[d]) mn[d] = v;
                if (v > mx[d]) mx[d] = v;
            }
        }
        for (int d = 0; d < 3; ++d) { mn[d] -= p->particle_radius; mx[d] += p->particle_radius; }
    }
    float half_cells = f_ceil(p->compact_support_radius / p->cube_size);
    float margin = p->cube_size * half_cells * (1.0f + sqrtf(FLT_EPSILON));
    for (int d = 0; d < 3; ++d) { mn[d] -= margin; mx[d] += margin; }
    return grid_from_aabb(g, mn, mx, p->cube_size);
}

/* ------------------------------------------------------ decomposition ---- */
typedef struct {
    uint64_t nsub;
    int64_t *flat;       /* ascending flat subdomain index */
    uint64_t *offset;    /* nsub+1 */
    uint64_t *members;   /* global particle indices, ascending within each subdomain */
} so_decomp;

/* dense_subdomains.rs:1810-1905: fills `out` with flat subdomain indices, returns count */
static int classify_particle(const float p[3], const so_grid *sg, float margin, int64_t *out, int cap) {
    int64_t ijk[3];
    for (int d = 0; d < 3; ++d) {
        ijk[d] = grid_cell_of(sg, d, p[d]);
        if (ijk[d] < 0 || ijk[d] >= sg->nc[d]) return 0; /* not part of computational domain */
    }
    float dx = sg->cell_size;
    int r = (int)f_ceil(margin / dx);
    float minc[3], maxc[3];
    for (int d = 0; d < 3; ++d) { minc[d] = grid_coord(sg, d, ijk[d]); maxc[d] = grid_coord(sg, d, ijk[d] + 1); }
    int cnt = 0;
    for (int i = -r; i <= r; ++i) for (int j = -r; j <= r; ++j) for (int k = -r; k <= r; ++k) {
        int st[3] = { i, j, k };
        int ok = 1;
        for (int d = 0; d < 3 && ok; ++d) {
            int s = st[d];
            float off = (float)((s < 0 ? -s : s) - 1);
            if (s > 0) ok = ((maxc[d] + off * dx) - p[d]) < margin;
            else if (s < 0) ok = (p[d] - (minc[d] - off * dx)) < margin;
        }
        if (!ok) continue;
        int64_t t[3]; int valid = 1;
        for (int d = 0; d < 3; ++d) { t[d] = ijk[d] + st[d]; if (t[d] < 0 || t[d] >= sg->nc[d]) valid = 0; }
        if (!valid) continue;
        if (cnt < cap) out[cnt] = t[0] * sg->nc[1] * sg->nc[2] + t[1] * sg->nc[2] + t[2];
        ++cnt;
    }
    return cnt;
}

static int cmp_i64(const void *a, const void *b) {
    int64_t x = *(const int64_t *)a, y = *(const int64_t *)b; return (x > y) - (x < y);
}

/* dense_subdomains.rs:349-494.  The reference's subdomain ORDER is hash-map iteration order
 * (machine dependent); we use ascending flat index, which the final mesh is canonicalised over. */
static void decompose(so_decomp *dc, const float *xyz, uint64_t n, const so_grid *sg, float margin) {
    int r = (int)f_ceil(margin / sg->cell_size);
    int cap = (2 * r + 1) * (2 * r + 1) * (2 * r + 1);
    int64_t *tmp = (int64_t *)malloc(sizeof(int64_t) * (size_t)cap);
    /* pass 1: collect all (flat) keys */
    uint64_t total = 0, capk = n * 2 + 16;
    int64_t *keys = (int64_t *)malloc(sizeof(int64_t) * capk);
    uint64_t *pidx = (uint64_t *)malloc(sizeof(uint64_t) * capk);
    for (uint64_t i = 0; i < n; ++i) {
        int c = classify_particle(xyz + 3 * i, sg, margin, tmp, cap);
        if (total + (uint64_t)c > capk) {
            capk = (total + (uint64_t)c) * 2;
            keys = (int64_t *)realloc(keys, sizeof(int64_t) * capk);
            pidx = (uint64_t *)realloc(pidx, sizeof(uint64_t) * capk);
        }
        for (int m = 0; m < c; ++m) { keys[total] = tmp[m]; pidx[total] = i; ++total; }
    }
    free(tmp);
    /* unique sorted subdomain ids */
    int64_t *sorted = (int64_t *)malloc(sizeof(int64_t) * (total ? total : 1));
    memcpy(sorted, keys, sizeof(int64_t) * total);
    qsort(sorted, total, sizeof(int64_t), cmp_i64);
    uint64_t nsub = 0;
    for (uint64_t i = 0; i < total; ++i) if (i == 0 || sorted[i] != sorted[i - 1]) sorted[nsub++] = sorted[i];
    dc->nsub = nsub;
    dc->flat = (int64_t *)malloc(sizeof(int64_t) * (nsub ? nsub : 1));
    memcpy(dc->flat, sorted, sizeof(int64_t) * nsub);
    free(sorted);
    dc->offset = (uint64_t *)calloc(nsub + 1, sizeof(uint64_t));
    /* count, then stable fill (particle order ascending => lists sorted, == sort_unstable result) */
    uint64_t *cid = (uint64_t *)malloc(sizeof(uint64_t) * (total ? total : 1));
    for (uint64_t i = 0; i < total; ++i) {
        uint64_t lo = 0, hi = nsub;
        while (lo + 1 < hi) { uint64_t mid = (lo + hi) / 2; if (dc->flat[mid] <= keys[i]) lo = mid; else hi = mid; }
        cid[i] = lo; dc->offset[lo + 1]++;
    }
    for (uint64_t s = 0; s < nsub; ++s) dc->offset[s + 1] += dc->offset[s];
    dc->members = (uint64_t *)malloc(sizeof(uint64_t) * (total ? total : 1));
    uint64_t *cur = (uint64_t *)malloc(sizeof(uint64_t) * (nsub ? nsub : 1));
    memcpy(cur, dc->offset, sizeof(uint64_t) * nsub);
    for (uint64_t i = 0; i < total; ++i) dc->members[cur[cid[i]]++] = pidx[i];
    free(cur); free(cid); free(keys); free(pidx);
}

static void unflatten_sub(const so_grid *sg, int64_t flat, int64_t ijk[3]) {
    ijk[0] = flat / (sg->nc[1] * sg->nc[2]);
    ijk[1] = (flat - ijk[0] * sg->nc[1] * sg->nc[2]) / sg->nc[2];
    ijk[2] = flat - ijk[0] * sg->nc[1] * sg->nc[2] - ijk[1] * sg->nc[2];
}

/* ------------------------------------------------ per-subdomain density ---- */
/* dense_subdomains.rs:496-646 + neighborhood_search.rs:345-438 + density_map.rs:150-186 */
static void subdomain_densities(const float *xyz, const so_grid *sg, const int64_t sijk[3],
                                const uint64_t *mem, uint64_t nm, float h, float margin, float rest_mass,
                                float *global_rho, int64_t *neighbor_counts, const int64_t *nbr_off, int64_t *nbr_out) {
    float smin[3], smax[3], mmin[3], mmax[3];
    float grow = margin * 1.5f;
    for (int d = 0; d < 3; ++d) {
        smin[d] = grid_coord(sg, d, sijk[d]); smax[d] = grid_coord(sg, d, sijk[d] + 1);
        mmin[d] = smin[d] - grow; mmax[d] = smax[d] + grow;
    }
    so_grid ns;
    if (grid_from_aabb(&ns, mmin, mmax, h) != 0) { fprintf(stderr, "oracle: NS grid construction failed\n"); abort(); }
    int64_t ncell = ns.nc[0] * ns.nc[1] * ns.nc[2];
    /* stable counting sort of members by NS cell (== per-cell Vec push order) */
    uint64_t *cstart = (uint64_t *)calloc((size_t)ncell + 1, sizeof(uint64_t));
    int64_t *cell_of = (int64_t *)malloc(sizeof(int64_t) * (nm ? nm : 1));
    for (uint64_t a = 0; a < nm; ++a) {
        const float *p = xyz + 3 * mem[a];
        int64_t c[3];
        for (int d = 0; d < 3; ++d) {
            c[d] = grid_cell_of(&ns, d, p[d]);
            if (c[d] < 0 || c[d] >= ns.nc[d]) { fprintf(stderr, "oracle: particle outside NS grid\n"); abort(); }
        }
        cell_of[a] = c[0] * ns.nc[1] * ns.nc[2] + c[1] * ns.nc[2] + c[2];
        cstart[cell_of[a] + 1]++;
    }
    for (int64_t c = 0; c < ncell; ++c) cstart[c + 1] += cstart[c];
    uint64_t *order = (uint64_t *)malloc(sizeof(uint64_t) * (nm ? nm : 1));
    uint64_t *cur = (uint64_t *)malloc(sizeof(uint64_t) * (size_t)(ncell ? ncell : 1));
    memcpy(cur, cstart, sizeof(uint64_t) * (size_t)ncell);
    for (uint64_t a = 0; a < nm; ++a) order[cur[cell_of[a]]++] = a;
    free(cur);

    k_scalar kern = k_scalar_new(h);
    float h2 = h * h;
    for (uint64_t a = 0; a < nm; ++a) {
        const float *pi = xyz + 3 * mem[a];
        /* is_inside = subdomain_aabb.contains_point (half-open), aabb.rs:220-222 */
        int inside = 1;
        for (int d = 0; d < 3; ++d) if (!(pi[d] >= smin[d] && pi[d] < smax[d])) inside = 0;
        if (!inside) continue;
        int64_t c[3];
        for (int d = 0; d < 3; ++d) c[d] = grid_cell_of(&ns, d, pi[d]);
        float rho = k_scalar_eval(&kern, 0.0f);
        int64_t nn = 0;
        /* 26 adjacent cells in x-major product order, then the own cell (neighborhood_search.rs:401-405) */
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
                if (d2 < h2) { rho += k_scalar_eval(&kern, sqrtf(d2)); if (nbr_out) nbr_out[nbr_off[mem[a]] + nn] = (int64_t)mem[b]; ++nn; }
            }
        }
        rho *= rest_mass;
        global_rho[mem[a]] = rho;
        if (neighbor_counts) neighbor_counts[mem[a]] = nn;
    }
    free(order); free(cell_of); free(cstart);
}

/* ----------------------------------------------- per-subdomain level set ---- */
/* dense_subdomains.rs:660-693 */
static inline void influence_box(const float p[3], const float smin[3], float c, int64_t R, int64_t np,
                                 int64_t lo[3], int64_t up[3]) {
    for (int d = 0; d < 3; ++d) {
        int64_t cell = (int64_t)f_floor((p[d] - smin[d]) / c);
        int64_t l = cell - R; if (l < 0) l = 0; if (l > np) l = np;
        int64_t u = cell + R + 2; if (u > np) u = np; if (u < 0) u = 0;
        lo[d] = l; up[d] = u;
    }
}

/* mode 0: AVX2-FMA loop (dense_subdomains.rs:991-1133); mode 1: scalar / sparse loop (:784-847, :1135-1213) */
static void subdomain_levelset(float *phi, const float *xyz, const float *rho, const uint64_t *mem, uint64_t nm,
                               const so_grid *gg, const float smin[3], const int64_t sijk[3], int64_t S,
                               float h, float rest_mass, int mode) {
    int64_t np = S + 1;
    float c = gg->cell_size;
    int64_t R = (int64_t)f_ceil(h / c);
    memset(phi, 0, sizeof(float) * (size_t)(np * np * np));
    if (mode == 0) {
        k_avx kern = k_avx_new(h);
        float h2 = h * h;
        for (uint64_t a = 0; a < nm; ++a) {
            const float *p = xyz + 3 * mem[a];
            float v = rest_mass / rho[mem[a]];
            int64_t lo[3], up[3];
            influence_box(p, smin, c, R, np, lo, up);
            int64_t rem = (up[2] > lo[2]) ? (up[2] - lo[2]) % 8 : 0;
            int64_t upk_al = up[2] - rem;
            for (int64_t i = lo[0]; i < up[0]; ++i) for (int64_t j = lo[1]; j < up[1]; ++j) {
                int32_t gi = (int32_t)sijk[0] * (int32_t)S + (int32_t)i;
                int32_t gj = (int32_t)sijk[1] * (int32_t)S + (int32_t)j;
                float gx = (float)gi * c + gg->aabb_min[0];
                float gy = (float)gj * c + gg->aabb_min[1];
                float dx = p[0] - gx, dy = p[1] - gy;
                for (int64_t k = lo[2]; k < up[2]; ++k) {
                    int32_t gk = (int32_t)sijk[2] * (int32_t)S + (int32_t)k;
                    float gz = fmaf((float)gk, c, gg->aabb_min[2]);
                    float dz = p[2] - gz;
                    float d2 = fmaf(dz, dz, fmaf(dx, dx, dy * dy));
                    float w = 0.0f;
                    if (d2 < h2) w = k_avx_eval(&kern, sqrtf(d2));
                    float *dst = phi + (i * np + j) * np + k;
                    if (k < upk_al) *dst = fmaf(w, v, *dst);
                    else *dst += w * v;              /* remainder lanes: mul then add */
                }
            }
        }
    } else {
        k_scalar kern = k_scalar_new(h);
        float h2m = (h * h) * 1.01f;
        for (uint64_t a = 0; a < nm; ++a) {
            const float *p = xyz + 3 * mem[a];
            float rho_i = rho[mem[a]];
            int64_t lo[3], up[3];
            influence_box(p, smin, c, R, np, lo, up);
            for (int64_t i = lo[0]; i < up[0]; ++i) for (int64_t j = lo[1]; j < up[1]; ++j)
            for (int64_t k = lo[2]; k < up[2]; ++k) {
                float gx = grid_coord(gg, 0, sijk[0] * S + i);
                float gy = grid_coord(gg, 1, sijk[1] * S + j);
                float gz = grid_coord(gg, 2, sijk[2] * S + k);
                float dx = p[0] - gx, dy = p[1] - gy, dz = p[2] - gz;
                float d2 = dx * dx + dy * dy + dz * dz;
                if (d2 < h2m) {
                    float v = rest_mass / rho_i;
                    float w = k_scalar_eval(&kern, sqrtf(d2));
                    phi[(i * np + j) * np + k] += v * w;
                }
            }
        }
    }
}

/* ----------------------------------------------------------- MC + stitch ---- */
static const int8_t CORNER[8][3] = { {0,0,0},{1,0,0},{1,1,0},{0,1,0},{0,0,1},{1,0,1},{1,1,1},{0,1,1} };
/* uniform_grid.rs:858-871: local edge -> (origin corner, axis) */
static const int8_t EDGE_CORNER[12] = { 0, 1, 3, 0, 4, 5, 7, 4, 0, 1, 2, 3 };
static const int8_t EDGE_AXIS[12]   = { 0, 1, 0, 1, 0, 1, 0, 1, 2, 2, 2, 2 };

typedef struct {
    uint64_t nv, nt, capv, capt;
    float *v;          /* nv*3 */
    int64_t *vkey;     /* nv*4 global point ijk + axis */
    uint8_t *vinterior;
    uint64_t *t;       /* nt*3, patch-local vertex ids */
} so_patch;

static void patch_push_v(so_patch *pt, const float x[3], const int64_t key[4], int interior) {
    if (pt->nv == pt->capv) {
        pt->capv = pt->capv ? pt->capv * 2 : 1024;
        pt->v = (float *)realloc(pt->v, sizeof(float) * 3 * pt->capv);
        pt->vkey = (int64_t *)realloc(pt->vkey, sizeof(int64_t) * 4 * pt->capv);
        pt->vinterior = (uint8_t *)realloc(pt->vinterior, pt->capv);
    }
    memcpy(pt->v + 3 * pt->nv, x, sizeof(float) * 3);
    memcpy(pt->vkey + 4 * pt->nv, key, sizeof(int64_t) * 4);
    pt->vinterior[pt->nv] = (uint8_t)interior;
    pt->nv++;
}
static void patch_push_t(so_patch *pt, const uint64_t tri[3]) {
    if (pt->nt == pt->capt) {
        pt->capt = pt->capt ? pt->capt * 2 : 2048;
        pt->t = (uint64_t *)realloc(pt->t, sizeof(uint64_t) * 3 * pt->capt);
    }
    memcpy(pt->t + 3 * pt->nt, tri, sizeof(uint64_t) * 3);
    pt->nt++;
}

/* dense_subdomains.rs:1470-1568 (per-cell triangulation of one subdomain tile) */
static void subdomain_mc(so_patch *pt, const float *phi, const float smin[3], const int64_t sijk[3],
                         int64_t S, float c, float thr, int64_t *edge_vertex /* 3*np^3 scratch */) {
    int64_t np = S + 1;
    size_t ne = (size_t)(3 * np * np * np);
    for (size_t e = 0; e < ne; ++e) edge_vertex[e] = -1;
    for (int64_t i = 0; i < S; ++i) for (int64_t j = 0; j < S; ++j) for (int64_t k = 0; k < S; ++k) {
        int idx = 0;
        for (int v = 0; v < 8; ++v) {
            float val = phi[((i + CORNER[v][0]) * np + (j + CORNER[v][1])) * np + (k + CORNER[v][2])];
            if (val > thr) idx |= (1 << v);
        }
        if (idx == 0) continue;
        const signed char *row = SS_MC_TRI_TABLE[idx];
        for (int t = 0; t < 5 && row[3 * t] >= 0; ++t) {
            uint64_t tri[3];
            for (int m = 0; m < 3; ++m) {
                int le = row[3 * t + (2 - m)];     /* reversed triplet, marching_cubes_lut.rs:338-342 */
                int oc = EDGE_CORNER[le], ax = EDGE_AXIS[le];
                int64_t o[3] = { i + CORNER[oc][0], j + CORNER[oc][1], k + CORNER[oc][2] };
                size_t eid = (size_t)(((o[0] * np + o[1]) * np + o[2]) * 3 + ax);
                if (edge_vertex[eid] < 0) {
                    int64_t tg[3] = { o[0], o[1], o[2] }; tg[ax] += 1;
                    float oc_[3], tc_[3];
                    for (int d = 0; d < 3; ++d) { oc_[d] = smin[d] + (float)o[d] * c; tc_[d] = smin[d] + (float)tg[d] * c; }
                    float a = phi[(o[0] * np + o[1]) * np + o[2]];
                    float b = phi[(tg[0] * np + tg[1]) * np + tg[2]];
                    float alpha = (thr - a) / (b - a);
                    float one_m = 1.0f - alpha;
                    float x[3];
                    for (int d = 0; d < 3; ++d) x[d] = oc_[d] * one_m + tc_[d] * alpha;
                    int boundary = 0;
                    for (int d = 0; d < 3; ++d) if (d != ax && (o[d] == 0 || o[d] + 1 == np)) boundary = 1;
                    int64_t key[4] = { sijk[0] * S + o[0], sijk[1] * S + o[1], sijk[2] * S + o[2], ax };
                    edge_vertex[eid] = (int64_t)pt->nv;
                    patch_push_v(pt, x, key, !boundary);
                }
                tri[m] = (uint64_t)edge_vertex[eid];
            }
            patch_push_t(pt, tri);
        }
    }
}

typedef struct { int64_t k[4]; uint64_t patch, local; } so_ext;
static int cmp_ext(const void *a, const void *b) {
    const so_ext *x = (const so_ext *)a, *y = (const so_ext *)b;
    for (int d = 0; d < 4; ++d) if (x->k[d] != y->k[d]) return (x->k[d] > y->k[d]) - (x->k[d] < y->k[d]);
    if (x->patch != y->patch) return (x->patch > y->patch) - (x->patch < y->patch);
    return (x->local > y->local) - (x->local < y->local);
}

/* dense_subdomains.rs:1603-1749.  Boundary vertices are de-duplicated by their globalised edge
 * (:1260-1329), which is equivalent to the global (point, axis) key used here; the first patch in
 * (ascending flat subdomain) order keeps its copy of the position, like the reference's or_insert. */
static void stitch(so_result *res, so_patch *patches, uint64_t npatch) {
    uint64_t nvi = 0, nti = 0, nve_raw = 0, nt_all = 0;
    for (uint64_t s = 0; s < npatch; ++s) {
        for (uint64_t v = 0; v < patches[s].nv; ++v) { if (patches[s].vinterior[v]) ++nvi; else ++nve_raw; }
        nt_all += patches[s].nt;
    }
    so_ext *ext = (so_ext *)malloc(sizeof(so_ext) * (nve_raw ? nve_raw : 1));
    uint64_t ne = 0;
    for (uint64_t s = 0; s < npatch; ++s) for (uint64_t v = 0; v < patches[s].nv; ++v) if (!patches[s].vinterior[v]) {
        memcpy(ext[ne].k, patches[s].vkey + 4 * v, sizeof(int64_t) * 4); ext[ne].patch = s; ext[ne].local = v; ++ne;
    }
    qsort(ext, ne, sizeof(so_ext), cmp_ext);
    uint64_t nve = 0;
    for (uint64_t e = 0; e < ne; ++e) if (e == 0 || memcmp(ext[e].k, ext[e - 1].k, sizeof(int64_t) * 4) != 0) ++nve;
    res->nv = nvi + nve; res->nt = nt_all;
    res->vertices = (float *)malloc(sizeof(float) * 3 * (res->nv ? res->nv : 1));
    res->vertex_keys = (int64_t *)malloc(sizeof(int64_t) * 4 * (res->nv ? res->nv : 1));
    res->triangles = (uint64_t *)malloc(sizeof(uint64_t) * 3 * (res->nt ? res->nt : 1));
    /* local -> global maps */
    uint64_t **l2g = (uint64_t **)malloc(sizeof(uint64_t *) * (npatch ? npatch : 1));
    uint64_t vo = 0;
    for (uint64_t s = 0; s < npatch; ++s) {
        l2g[s] = (uint64_t *)malloc(sizeof(uint64_t) * (patches[s].nv ? patches[s].nv : 1));
        for (uint64_t v = 0; v < patches[s].nv; ++v) if (patches[s].vinterior[v]) {
            memcpy(res->vertices + 3 * vo, patches[s].v + 3 * v, sizeof(float) * 3);
            memcpy(res->vertex_keys + 4 * vo, patches[s].vkey + 4 * v, sizeof(int64_t) * 4);
            l2g[s][v] = vo++;
        }
    }
    uint64_t cur = vo;
    for (uint64_t e = 0; e < ne; ++e) {
        if (e == 0 || memcmp(ext[e].k, ext[e - 1].k, sizeof(int64_t) * 4) != 0) {
            memcpy(res->vertices + 3 * cur, patches[ext[e].patch].v + 3 * ext[e].local, sizeof(float) * 3);
            memcpy(res->vertex_keys + 4 * cur, ext[e].k, sizeof(int64_t) * 4);
            ++cur;
        }
        l2g[ext[e].patch][ext[e].local] = cur - 1;
    }
    /* triangles: interior ones first, then exterior ones (ordering is canonicalised by the tests) */
    nti = 0;
    for (int pass = 0; pass < 2; ++pass)
    for (uint64_t s = 0; s < npatch; ++s) for (uint64_t t = 0; t < patches[s].nt; ++t) {
        const uint64_t *tr = patches[s].t + 3 * t;
        int interior = patches[s].vinterior[tr[0]] && patches[s].vinterior[tr[1]] && patches[s].vinterior[tr[2]];
        if ((pass == 0) != interior) continue;
        for (int m = 0; m < 3; ++m) res->triangles[3 * nti + m] = l2g[s][tr[m]];
        ++nti;
    }
    for (uint64_t s = 0; s < npatch; ++s) free(l2g[s]);
    free(l2g); free(ext);
}


/* ------------------------------------------------- global (non-decomposed) path ---- */
/* reconstruction.rs:65-194 with enable_multi_threading = false (the deterministic variant; the multi-threaded
 * variant sums thread-local maps in scheduling order and is not bit-reproducible):
 *   neighborhood_search_spatial_hashing (neighborhood_search.rs:148-230) over from_aabb(grid.aabb, h),
 *   sequential_compute_particle_densities (density_map.rs:130-186),
 *   sequential_generate_sparse_density_map (density_map.rs:370-412, support loop :677-736),
 *   construct_mc_input + triangulate (marching_cubes/narrow_band_extraction.rs:51-219, triangulation.rs:23-57). */
static int reconstruct_global(so_result *res, const float *xyz, uint64_t n, const so_params *p, const so_grid *g,
                              int64_t *neighbor_counts, const int64_t *nbr_off, int64_t *nbr_out, int64_t tile_sub_flat, float *tile_out) {
    const float h = p->compact_support_radius, c = p->cube_size, thr = p->iso_surface_threshold;
    float r2 = p->particle_radius + p->particle_radius;
    const float rest_mass = (r2 * r2 * r2) * p->rest_density;
    res->densities = (float *)calloc(n ? n : 1, sizeof(float));
    /* ---- densities on one neighbourhood-search grid over the whole domain */
    if (n) {
        so_grid ns;
        if (grid_from_aabb(&ns, g->aabb_min, g->aabb_max, h) != 0) return 6;
        int64_t ncell = ns.nc[0] * ns.nc[1] * ns.nc[2];
        uint64_t *cstart = (uint64_t *)calloc((size_t)ncell + 1, sizeof(uint64_t));
        int64_t *cell_of = (int64_t *)malloc(sizeof(int64_t) * n);
        for (uint64_t a = 0; a < n; ++a) {
            int64_t cc[3];
            for (int d = 0; d < 3; ++d) { cc[d] = grid_cell_of(&ns, d, xyz[3 * a + d]); if (cc[d] < 0 || cc[d] >= ns.nc[d]) { free(cstart); free(cell_of); return 6; } }
            cell_of[a] = cc[0] * ns.nc[1] * ns.nc[2] + cc[1] * ns.nc[2] + cc[2];
            cstart[cell_of[a] + 1]++;
        }
        for (int64_t q = 0; q < ncell; ++q) cstart[q + 1] += cstart[q];
        uint64_t *order = (uint64_t *)malloc(sizeof(uint64_t) * n);
        uint64_t *cur = (uint64_t *)malloc(sizeof(uint64_t) * (size_t)(ncell ? ncell : 1));
        memcpy(cur, cstart, sizeof(uint64_t) * (size_t)ncell);
        for (uint64_t a = 0; a < n; ++a) order[cur[cell_of[a]]++] = a;
        free(cur);
        k_scalar kern = k_scalar_new(h);
        float h2 = h * h;
        for (uint64_t a = 0; a < n; ++a) {
            const float *pi = xyz + 3 * a;
            int64_t cc[3];
            for (int d = 0; d < 3; ++d) cc[d] = grid_cell_of(&ns, d, pi[d]);
            float rho = k_scalar_eval(&kern, 0.0f);
            int64_t nn = 0;
            for (int pass = 0; pass < 2; ++pass)
            for (int sx = -1; sx <= 1; ++sx) for (int sy = -1; sy <= 1; ++sy) for (int sz = -1; sz <= 1; ++sz) {
                int self = (sx == 0 && sy == 0 && sz == 0);
                if ((pass == 0) == self) continue;
                int64_t q[3] = { cc[0] + sx, cc[1] + sy, cc[2] + sz };
                if (q[0] < 0 || q[1] < 0 || q[2] < 0 || q[0] >= ns.nc[0] || q[1] >= ns.nc[1] || q[2] >= ns.nc[2]) continue;
                int64_t fc = q[0] * ns.nc[1] * ns.nc[2] + q[1] * ns.nc[2] + q[2];
                for (uint64_t t = cstart[fc]; t < cstart[fc + 1]; ++t) {
                    uint64_t b = order[t];
                    if (b == a) continue;
                    const float *pj = xyz + 3 * b;
                    float dx = pj[0] - pi[0], dy = pj[1] - pi[1], dz = pj[2] - pi[2];
                    float d2 = dx * dx + dy * dy + dz * dz;
                    if (d2 < h2) { rho += k_scalar_eval(&kern, sqrtf(d2)); if (nbr_out) nbr_out[nbr_off[a] + nn] = (int64_t)b; ++nn; }
                }
            }
            res->densities[a] = rho * rest_mass;
            if (neighbor_counts) neighbor_counts[a] = nn;
        }
        free(order); free(cell_of); free(cstart);
    }
    /* ---- density map on the dense point array (missing == 0) */
    float half_real = f_ceil(h / c);
    int64_t half = (int64_t)half_real, supported = 2 * half + 2;
    float rev = c * half_real * (1.0f + sqrtf(FLT_EPSILON));
    float rev2 = rev * rev;
    float amin[3], amax[3];
    for (int d = 0; d < 3; ++d) { amin[d] = g->aabb_min[d] - (-rev); amax[d] = g->aabb_max[d] + (-rev); }
    if ((amin[0] == amax[0] && amin[1] == amax[1] && amin[2] == amax[2]) || !(amin[0] <= amax[0] && amin[1] <= amax[1] && amin[2] <= amax[2])) return 8;
    const int64_t np0 = g->np[0], np1 = g->np[1], np2 = g->np[2];
    size_t npts = (size_t)(np0 * np1 * np2);
    float *phi = (float *)calloc(npts, sizeof(float));
    k_scalar kern = k_scalar_new(h);
    for (uint64_t a = 0; a < n; ++a) {
        const float *pp = xyz + 3 * a;
        int in = 1;
        for (int d = 0; d < 3; ++d) if (!(pp[d] >= amin[d] && pp[d] < amax[d])) in = 0;
        if (!in) continue;
        float vol = rest_mass / res->densities[a];
        int64_t imin[3]; float mp[3];
        for (int d = 0; d < 3; ++d) { imin[d] = grid_cell_of(g, d, pp[d]) - half; mp[d] = grid_coord(g, d, imin[d]); }
        float dx = mp[0] - pp[0] - c;
        for (int64_t i = imin[0]; i != imin[0] + supported; ++i) {
            dx += c; float dxdx = dx * dx;
            float dy = mp[1] - pp[1] - c;
            for (int64_t j = imin[1]; j != imin[1] + supported; ++j) {
                dy += c; float dydy = dy * dy;
                float dz = mp[2] - pp[2] - c;
                for (int64_t k = imin[2]; k != imin[2] + supported; ++k) {
                    dz += c; float dzdz = dz * dz;
                    float rr = dxdx + dydy + dzdz;
                    if (rr < rev2) phi[(i * np1 + j) * np2 + k] += vol * k_scalar_eval(&kern, sqrtf(rr));
                }
            }
        }
    }
    /* debug tap: the 65^3 points of tile `tile_sub_flat` of the global grid cut into 64-cube tiles (the device's tiling of this
     * path); points past the grid stay 0 */
    if (tile_out && tile_sub_flat >= 0) {
        const int64_t T = 64, tn = T + 1, nsd1 = (g->nc[1] + T - 1) / T, nsd2 = (g->nc[2] + T - 1) / T;
        const int64_t ti = tile_sub_flat / (nsd1 * nsd2), tj = (tile_sub_flat / nsd2) % nsd1, tk = tile_sub_flat % nsd2;
        memset(tile_out, 0, sizeof(float) * (size_t)(tn * tn * tn));
        for (int64_t a = 0; a < tn; ++a) for (int64_t b = 0; b < tn; ++b) for (int64_t e = 0; e < tn; ++e) {
            const int64_t i = ti * T + a, j = tj * T + b, k = tk * T + e;
            if (i < np0 && j < np1 && k < np2) tile_out[(a * tn + b) * tn + e] = phi[(i * np1 + j) * np2 + k];
        }
    }
    /* ---- marching cubes input: vertices on edges from a point >= thr to a neighbour < thr */
    so_patch pt; memset(&pt, 0, sizeof(pt));
    int64_t *edge_vertex = (int64_t *)malloc(sizeof(int64_t) * 3 * npts);
    uint8_t *marked = (uint8_t *)calloc(npts, 1);      /* corner flagged Above by the edge loop */
    for (size_t e = 0; e < 3 * npts; ++e) edge_vertex[e] = -1;
    static const int NB[6][3] = { {1,0,0},{-1,0,0},{0,1,0},{0,-1,0},{0,0,1},{0,0,-1} };
    for (int64_t i = 0; i < np0; ++i) for (int64_t j = 0; j < np1; ++j) for (int64_t k = 0; k < np2; ++k) {
        float vp = phi[(i * np1 + j) * np2 + k];
        if (vp < thr) continue;
        for (int q = 0; q < 6; ++q) {
            int64_t ni = i + NB[q][0], nj = j + NB[q][1], nk = k + NB[q][2];
            if (ni < 0 || nj < 0 || nk < 0 || ni >= np0 || nj >= np1 || nk >= np2) continue;
            float vn = phi[(ni * np1 + nj) * np2 + nk];
            if (!(vn < thr)) continue;
            float alpha = (thr - vp) / (vn - vp);
            float one_m = 1.0f - alpha;
            float pc[3] = { grid_coord(g, 0, i), grid_coord(g, 1, j), grid_coord(g, 2, k) };
            float nc_[3] = { grid_coord(g, 0, ni), grid_coord(g, 1, nj), grid_coord(g, 2, nk) };
            float x[3];
            for (int d = 0; d < 3; ++d) x[d] = pc[d] * one_m + nc_[d] * alpha;
            int ax = q / 2;
            int64_t o[3] = { i < ni ? i : ni, j < nj ? j : nj, k < nk ? k : nk };
            int64_t key[4] = { o[0], o[1], o[2], ax };
            edge_vertex[((o[0] * np1 + o[1]) * np2 + o[2]) * 3 + ax] = (int64_t)pt.nv;
            patch_push_v(&pt, x, key, 1);
            marked[(i * np1 + j) * np2 + k] = 1;
        }
    }
    /* ---- triangulate every cell that touches a crossing edge */
    int rc = 0;
    for (int64_t i = 0; i + 1 < np0 && !rc; ++i) for (int64_t j = 0; j + 1 < np1 && !rc; ++j) for (int64_t k = 0; k + 1 < np2 && !rc; ++k) {
        int any_edge = 0;
        for (int le = 0; le < 12 && !any_edge; ++le) {
            int oc = EDGE_CORNER[le], ax = EDGE_AXIS[le];
            int64_t o[3] = { i + CORNER[oc][0], j + CORNER[oc][1], k + CORNER[oc][2] };
            if (edge_vertex[((o[0] * np1 + o[1]) * np2 + o[2]) * 3 + ax] >= 0) any_edge = 1;
        }
        if (!any_edge) continue;
        int idx = 0;
        for (int v = 0; v < 8; ++v) {
            size_t l = (size_t)(((i + CORNER[v][0]) * np1 + (j + CORNER[v][1])) * np2 + (k + CORNER[v][2]));
            /* narrow_band_extraction.rs:124-126 (Above set by the edge loop) and :179-184 (value > threshold) */
            if (marked[l] || phi[l] > thr) idx |= (1 << v);
        }
        const signed char *row = SS_MC_TRI_TABLE[idx];
        for (int t = 0; t < 5 && row[3 * t] >= 0; ++t) {
            uint64_t tri[3];
            for (int m = 0; m < 3; ++m) {
                int le = row[3 * t + (2 - m)];
                int oc = EDGE_CORNER[le], ax = EDGE_AXIS[le];
                int64_t o[3] = { i + CORNER[oc][0], j + CORNER[oc][1], k + CORNER[oc][2] };
                int64_t vid = edge_vertex[((o[0] * np1 + o[1]) * np2 + o[2]) * 3 + ax];
                if (vid < 0) { rc = 9; break; }       /* reference: "Missing iso surface vertex" error */
                tri[m] = (uint64_t)vid;
            }
            if (rc) break;
            patch_push_t(&pt, tri);
        }
    }
    res->nv = pt.nv; res->nt = pt.nt;
    res->vertices = pt.v ? pt.v : (float *)malloc(4);
    res->vertex_keys = pt.vkey ? pt.vkey : (int64_t *)malloc(8);
    res->triangles = pt.t ? pt.t : (uint64_t *)malloc(8);
    free(pt.vinterior); free(edge_vertex); free(marked); free(phi);
    return rc;
}

/* ------------------------------------------------------ thread helper ---- */
/* The reference parallelises over subdomains with rayon (dense_subdomains.rs:521-526, :1581-1598);
 * here: a pthread pool pulling subdomain indices from an atomic counter. */
static int g_num_threads = 0;
void so_set_num_threads(int n) { g_num_threads = n; }
int so_num_threads(void) {
    if (g_num_threads > 0) return g_num_threads;
    long n = sysconf(_SC_NPROCESSORS_ONLN);
    return n > 0 ? (int)n : 1;
}
typedef void (*so_task_fn)(int64_t idx, void *ctx, void **tls);
typedef struct { so_task_fn fn; void *ctx; int64_t n; atomic_llong next; } so_pool;
static void *pool_worker(void *arg) {
    so_pool *pl = (so_pool *)arg;
    void *tls = NULL;
    for (;;) {
        long long i = atomic_fetch_add(&pl->next, 1);
        if (i >= pl->n) break;
        pl->fn((int64_t)i, pl->ctx, &tls);
    }
    free(tls);
    return NULL;
}
static void parallel_for(int64_t n, so_task_fn fn, void *ctx) {
    so_pool pl; pl.fn = fn; pl.ctx = ctx; pl.n = n; atomic_init(&pl.next, 0);
    int nt = so_num_threads(); if ((int64_t)nt > n) nt = (int)(n > 0 ? n : 1);
    if (nt <= 1) { pool_worker(&pl); return; }
    pthread_t *th = (pthread_t *)malloc(sizeof(pthread_t) * (size_t)nt);
    for (int t = 0; t < nt; ++t) pthread_create(&th[t], NULL, pool_worker, &pl);
    for (int t = 0; t < nt; ++t) pthread_join(th[t], NULL);
    free(th);
}

typedef struct {
    const float *xyz; const so_grid *sg, *gg; const so_decomp *dc; so_result *res; const so_params *p;
    float h, c, thr, margin, rest_mass; int64_t S; uint64_t sparse_limit;
    int64_t *neighbor_counts; int64_t tile_sub_flat; float *tile_out; so_patch *patches;
    const int64_t *nbr_off; int64_t *nbr_out;
} so_job;

static void density_task(int64_t s, void *ctx, void **tls) {
    (void)tls;
    so_job *jb = (so_job *)ctx;
    int64_t sijk[3]; unflatten_sub(jb->sg, jb->dc->flat[s], sijk);
    subdomain_densities(jb->xyz, jb->sg, sijk, jb->dc->members + jb->dc->offset[s],
                        jb->dc->offset[s + 1] - jb->dc->offset[s], jb->h, jb->margin, jb->rest_mass,
                        jb->res->densities, jb->neighbor_counts, jb->nbr_off, jb->nbr_out);
}

static void recon_task(int64_t s, void *ctx, void **tls) {
    so_job *jb = (so_job *)ctx;
    int64_t S = jb->S, np = S + 1;
    size_t npts = (size_t)(np * np * np);
    if (!*tls) *tls = malloc(sizeof(float) * npts + sizeof(int64_t) * 3 * npts);
    int64_t *ev = (int64_t *)*tls;
    float *phi = (float *)(ev + 3 * npts);
    int64_t sijk[3]; unflatten_sub(jb->sg, jb->dc->flat[s], sijk);
    float smin[3];
    for (int d = 0; d < 3; ++d) smin[d] = grid_coord(jb->sg, d, sijk[d]);
    uint64_t nm = jb->dc->offset[s + 1] - jb->dc->offset[s];
    int sparse = nm <= jb->sparse_limit;
    jb->res->subdomain_sparse[s] = (uint8_t)sparse;
    int mode = (sparse || !jb->p->enable_simd) ? 1 : 0;
    subdomain_levelset(phi, jb->xyz, jb->res->densities, jb->dc->members + jb->dc->offset[s], nm, jb->gg,
                       smin, sijk, S, jb->h, jb->rest_mass, mode);
    if (jb->tile_out && jb->dc->flat[s] == jb->tile_sub_flat) memcpy(jb->tile_out, phi, sizeof(float) * npts);
    subdomain_mc(&jb->patches[s], phi, smin, sijk, S, jb->c, jb->thr, ev);
}

/* ------------------------------------------------------------ top level ---- */
void so_free(so_result *r) {
    if (!r) return;
    free(r->inside_aabb); free(r->densities); free(r->vertices); free(r->triangles); free(r->vertex_keys);
    free(r->subdomain_flat); free(r->subdomain_count); free(r->subdomain_sparse);
    free(r);
}

/* Optional debug taps: if tile_sub_flat >= 0, the level-set tile of that subdomain is copied to tile_out
 * ((S+1)^3 floats; on the global path the tile of that flat index in 64-cube tiles of the global grid, 65^3 floats whatever S
 * is, so tile_out must hold (max(S, 64) + 1)^3 floats). */
int so_reconstruct(const float *xyz_in, uint64_t n_in, const so_params *p, so_result **out,
                   int64_t tile_sub_flat, float *tile_out, int64_t *neighbor_counts, const int64_t *nbr_off, int64_t *nbr_out) {
    so_result *res = (so_result *)calloc(1, sizeof(so_result));
    *out = res;
    lut_init();
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
    res->grid = g0;
    /* lib.rs:421-464 decomposition decision */
    int use_dec = 0;
    if (p->decomposition == 1) {
        if (p->auto_disable) {
            int64_t mc = g0.nc[0]; if (g0.nc[1] > mc) mc = g0.nc[1]; if (g0.nc[2] > mc) mc = g0.nc[2];
            uint32_t with_margin = (uint32_t)(1.2 * (double)p->subdomain_num_cubes_per_dim);
            use_dec = (uint64_t)mc > (uint64_t)with_margin;
        } else use_dec = 1;
    }
    res->used_decomposition = use_dec;
    if (!use_dec) { int rcg = reconstruct_global(res, xyz, n, p, &g0, neighbor_counts, nbr_off, nbr_out, tile_sub_flat, tile_out); free(filtered); return rcg; }

    /* dense_subdomains.rs:89-244 initialize_parameters */
    int64_t S = (int64_t)p->subdomain_num_cubes_per_dim;
    float r2 = p->particle_radius + p->particle_radius;
    float rest_mass = (r2 * r2 * r2) * p->rest_density;
    float h = p->compact_support_radius, c = p->cube_size, thr = p->iso_surface_threshold;
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
    uint64_t sparse_limit = maxp / 20; if (sparse_limit < 100) sparse_limit = 100;
    res->max_particles = maxp; res->sparse_limit = sparse_limit;

    res->densities = (float *)calloc(n ? n : 1, sizeof(float));
    if (neighbor_counts) memset(neighbor_counts, 0, sizeof(int64_t) * n);
    so_job job;
    memset(&job, 0, sizeof(job));
    job.xyz = xyz; job.sg = &sg; job.gg = &gg; job.dc = &dc; job.res = res; job.p = p;
    job.h = h; job.c = c; job.thr = thr; job.margin = margin; job.rest_mass = rest_mass; job.S = S;
    job.sparse_limit = sparse_limit; job.neighbor_counts = neighbor_counts;
    job.tile_sub_flat = tile_sub_flat; job.tile_out = tile_out; job.nbr_off = nbr_off; job.nbr_out = nbr_out;
    parallel_for((int64_t)dc.nsub, density_task, &job);

    so_patch *patches = (so_patch *)calloc(dc.nsub ? dc.nsub : 1, sizeof(so_patch));
    job.patches = patches;
    parallel_for((int64_t)dc.nsub, recon_task, &job);
    stitch(res, patches, dc.nsub);
    for (uint64_t s = 0; s < dc.nsub; ++s) { free(patches[s].v); free(patches[s].vkey); free(patches[s].vinterior); free(patches[s].t); }
    free(patches);
    free(dc.flat); free(dc.offset); free(dc.members);
    free(filtered);
    return 0;
}

/* Stand-alone level-set tile evaluation for the reference's own hot-loop fixture
 * (data/density_grid_loop_subdomain_33.json; benches/bench_grid_loop.rs:203-262). */
void so_levelset_tile(float *phi, const float *xyz, const float *rho, uint64_t n,
                      const float gmin[3], float cube_size, const int64_t sijk[3], int64_t S,
                      const float smin[3], float h, float rest_mass, int mode) {
    so_grid gg; int64_t nc[3] = { 0, 0, 0 };
    grid_new(&gg, gmin, nc, cube_size);
    uint64_t *mem = (uint64_t *)malloc(sizeof(uint64_t) * (n ? n : 1));
    for (uint64_t i = 0; i < n; ++i) mem[i] = i;
    subdomain_levelset(phi, xyz, rho, mem, n, &gg, smin, sijk, S, h, rest_mass, mode);
    free(mem);
}

/* SPH normals at arbitrary points: sph_interpolation.rs:82-133 (+ kernel.rs:109-141 gradient norm).  The reference visits
 * neighbours in R-tree traversal order, which is not restated; the summation order here is cell order, so parity with the
 * reference binary is to rounding (tests use 2e-5 absolute on the unit vectors). */
static inline float k_scalar_dq(float q) {
    if (q < 1.0f) return (3.0f / (4.0f * SO_PI_F)) * (-4.0f * q + 3.0f * q * q);
    else if (q < 2.0f) { float x = 2.0f - q; return -(3.0f / (4.0f * SO_PI_F)) * x * x; }
    return 0.0f;
}
void so_sph_normals(const float *xyz, const float *rho, uint64_t n, float h, float rest_mass, const float *pts, uint64_t npts, float *out) {
    if (!npts) return;
    float mn[3] = { 1e30f, 1e30f, 1e30f }, mx[3] = { -1e30f, -1e30f, -1e30f };
    for (uint64_t a = 0; a < n; ++a) for (int d = 0; d < 3; ++d) { float v = xyz[3 * a + d]; if (v < mn[d]) mn[d] = v; if (v > mx[d]) mx[d] = v; }
    int64_t nc[3];
    for (int d = 0; d < 3; ++d) { nc[d] = n ? (int64_t)((mx[d] - mn[d]) / h) + 1 : 1; }
    int64_t ncell = nc[0] * nc[1] * nc[2];
    uint64_t *cstart = (uint64_t *)calloc((size_t)ncell + 1, sizeof(uint64_t));
    int64_t *cell_of = (int64_t *)malloc(sizeof(int64_t) * (n ? n : 1));
    for (uint64_t a = 0; a < n; ++a) {
        int64_t c[3];
        for (int d = 0; d < 3; ++d) { c[d] = (int64_t)((xyz[3 * a + d] - mn[d]) / h); if (c[d] >= nc[d]) c[d] = nc[d] - 1; if (c[d] < 0) c[d] = 0; }
        cell_of[a] = (c[0] * nc[1] + c[1]) * nc[2] + c[2]; cstart[cell_of[a] + 1]++;
    }
    for (int64_t q = 0; q < ncell; ++q) cstart[q + 1] += cstart[q];
    uint64_t *order = (uint64_t *)malloc(sizeof(uint64_t) * (n ? n : 1));
    uint64_t *cur = (uint64_t *)malloc(sizeof(uint64_t) * (size_t)ncell);
    memcpy(cur, cstart, sizeof(uint64_t) * (size_t)ncell);
    for (uint64_t a = 0; a < n; ++a) order[cur[cell_of[a]]++] = a;
    free(cur);
    k_scalar kern = k_scalar_new(h);
    float h2 = h * h, dqdr = (1.0f + 1.0f) / h;
    for (uint64_t v = 0; v < npts; ++v) {
        const float *x = pts + 3 * v;
        float g[3] = { 0.0f, 0.0f, 0.0f };
        int64_t c[3];
        for (int d = 0; d < 3; ++d) c[d] = (int64_t)floorf((x[d] - mn[d]) / h);
        for (int64_t i = c[0] - 1; i <= c[0] + 1; ++i) for (int64_t j = c[1] - 1; j <= c[1] + 1; ++j) for (int64_t k = c[2] - 1; k <= c[2] + 1; ++k) {
            if (i < 0 || j < 0 || k < 0 || i >= nc[0] || j >= nc[1] || k >= nc[2]) continue;
            int64_t fc = (i * nc[1] + j) * nc[2] + k;
            for (uint64_t t = cstart[fc]; t < cstart[fc + 1]; ++t) {
                uint64_t b = order[t];
                float dx = xyz[3 * b] - x[0], dy = xyz[3 * b + 1] - x[1], dz = xyz[3 * b + 2] - x[2];
                float d2 = dx * dx + dy * dy + dz * dz;
                if (!(d2 <= h2)) continue;
                float r = sqrtf(d2);
                float q = (r + r) / kern.h;
                float gn = kern.sigma * k_scalar_dq(q) * dqdr;
                float vol = rest_mass / rho[b];
                g[0] += (dx / r) * gn * vol; g[1] += (dy / r) * gn * vol; g[2] += (dz / r) * gn * vol;
            }
        }
        float nrm = sqrtf(g[0] * g[0] + g[1] * g[1] + g[2] * g[2]);
        out[3 * v] = g[0] / nrm; out[3 * v + 1] = g[1] / nrm; out[3 * v + 2] = g[2] / nrm;
    }
    free(order); free(cell_of); free(cstart);
}

/* scalar + AVX-lane kernels exposed for the kernel unit tests (kernel.rs:143-180, :381-481) */
float so_kernel_scalar(float h, float r) { k_scalar k = k_scalar_new(h); return k_scalar_eval(&k, r); }
float so_kernel_avx(float h, float r) { k_avx k = k_avx_new(h); return k_avx_eval(&k, r); }
