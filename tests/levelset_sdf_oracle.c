/* levelset_sdf_oracle.c -- the narrow-band signed distance grid of DESIGN.md section 14 restated as a brute-force scan: for every
 * point of every brick the f32 minimum over the triangles of the point-triangle distance, and the sign from the level-set field by
 * so_field_scan (tests/levelset_field_oracle.c, included unchanged).  Built with -ffp-contract=off -fno-fast-math, so every operation
 * below is one f32 rounding in the order written, the order of ss_sdf.cuh.
 *
 * A brick's scan may skip the triangles whose float64 AABB, grown by B plus one cell, misses the brick's points: such a triangle is
 * farther than B from every point of the brick and does not change min(d, B).  so_sdf_distance scans whatever it is given. */
#include "levelset_field_oracle.c"

static float sd_dot(const float *a, const float *b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }
static void sd_cross(const float *a, const float *b, float *x) {
    x[0] = a[1] * b[2] - a[2] * b[1];
    x[1] = a[2] * b[0] - a[0] * b[2];
    x[2] = a[0] * b[1] - a[1] * b[0];
}
static float sd_edge_d2(const float *p, const float *v0, const float *v1) {
    float e[3], w[3], r[3];
    for (int d = 0; d < 3; ++d) { e[d] = v1[d] - v0[d]; w[d] = p[d] - v0[d]; }
    float ee = sd_dot(e, e);
    float t = 0.0f;
    if (ee != 0.0f) t = fminf(fmaxf(sd_dot(w, e) / ee, 0.0f), 1.0f);
    for (int d = 0; d < 3; ++d) r[d] = p[d] - (v0[d] + t * e[d]);
    return sd_dot(r, r);
}
static float sd_side(const float *p, const float *v0, const float *v1, const float *n) {
    float e[3], w[3], x[3];
    for (int d = 0; d < 3; ++d) { e[d] = v1[d] - v0[d]; w[d] = p[d] - v0[d]; }
    sd_cross(e, w, x);
    return sd_dot(x, n);
}
/* squared distance from p to the triangle t = (a, b, c) */
float so_sdf_tri_d2(const float *p, const float *t) {
    const float *a = t, *b = t + 3, *c = t + 6;
    float d2 = fminf(fminf(sd_edge_d2(p, a, b), sd_edge_d2(p, b, c)), sd_edge_d2(p, c, a));
    float ab[3], ac[3], n[3];
    for (int d = 0; d < 3; ++d) { ab[d] = b[d] - a[d]; ac[d] = c[d] - a[d]; }
    sd_cross(ab, ac, n);
    float nn = sd_dot(n, n);
    if (nn > 0.0f && sd_side(p, a, b, n) >= 0.0f && sd_side(p, b, c, n) >= 0.0f && sd_side(p, c, a, n) >= 0.0f) {
        float w[3] = { p[0] - a[0], p[1] - a[1], p[2] - a[2] };
        float dn = sd_dot(w, n);
        d2 = fminf(d2, (dn * dn) / nn);
    }
    return d2;
}

static void sd_load(const float *verts, const uint32_t *tris, uint64_t k, float *t) {
    for (int v = 0; v < 3; ++v) for (int d = 0; d < 3; ++d) t[3 * v + d] = verts[3 * (uint64_t)tris[3 * k + v] + d];
}

/* d[q] = sqrt(min over the nt triangles of the squared distance) at m points (+inf without triangles) */
void so_sdf_distance(const float *verts, const uint32_t *tris, uint64_t nt, const float *pts, uint64_t m, float *d) {
    for (uint64_t q = 0; q < m; ++q) {
        float d2 = INFINITY, t[9];
        for (uint64_t k = 0; k < nt; ++k) { sd_load(verts, tris, k, t); d2 = fminf(d2, so_sdf_tri_d2(pts + 3 * q, t)); }
        d[q] = sqrtf(d2);
    }
}

static float sd_coord(const float *gmin, float c, int64_t i, int d) { return (float)i * c + gmin[d]; }

/* The grid of section 14: listed bricks in ascending (bx, by, bz) order (coords [B][3], values [B][512]; capacity: every brick of
 * the grid) and inside [nbx][nby][nbz].  The field arguments are those of so_field_scan; thr its threshold.  Returns B. */
int64_t so_sdf_grid(int mode, const float *ctr, const float *w, const float *g6, const float *dlt, uint64_t n, float h, float rs, float t_low,
                    float t_high, float thr, const float *verts, const uint32_t *tris, uint64_t nt, const float *gmin, float c, const int64_t *np,
                    uint32_t band, int32_t *coords, float *values, uint8_t *inside) {
    const float B = (float)band * c;
    const double reach = (double)B + (double)c;
    int64_t nb[3];
    for (int d = 0; d < 3; ++d) nb[d] = (np[d] + 7) / 8;
    double *box = (double *)malloc(sizeof(double) * 6 * (nt ? nt : 1));
    uint64_t *sel = (uint64_t *)malloc(sizeof(uint64_t) * (nt ? nt : 1));
    uint32_t *sub = (uint32_t *)malloc(sizeof(uint32_t) * 3 * (nt ? nt : 1));
    float *pts = (float *)malloc(sizeof(float) * 3 * 512), *dist = (float *)malloc(sizeof(float) * 512), *fv = (float *)malloc(sizeof(float) * 512);
    for (uint64_t k = 0; k < nt; ++k) {
        float t[9];
        sd_load(verts, tris, k, t);
        for (int d = 0; d < 3; ++d) {
            double lo = t[d], hi = t[d];
            for (int v = 1; v < 3; ++v) { lo = fmin(lo, (double)t[3 * v + d]); hi = fmax(hi, (double)t[3 * v + d]); }
            box[6 * k + d] = lo - reach; box[6 * k + 3 + d] = hi + reach;
        }
    }
    int64_t nl = 0;
    for (int64_t bx = 0; bx < nb[0]; ++bx) for (int64_t by = 0; by < nb[1]; ++by) for (int64_t bz = 0; bz < nb[2]; ++bz) {
        const int64_t b[3] = { bx, by, bz };
        uint64_t ns = 0;
        for (uint64_t k = 0; k < nt; ++k) {
            int meets = 1;
            for (int d = 0; d < 3; ++d)
                meets = meets && box[6 * k + 3 + d] >= (double)sd_coord(gmin, c, 8 * b[d], d) && box[6 * k + d] <= (double)sd_coord(gmin, c, 8 * b[d] + 7, d);
            if (meets) sel[ns++] = k;
        }
        for (uint64_t s = 0; s < ns; ++s) for (int v = 0; v < 3; ++v) sub[3 * s + v] = tris[3 * sel[s] + v];
        int listed = 0;
        for (int r = 0; r < 512; ++r) {
            const int64_t q[3] = { 8 * bx + (r >> 6), 8 * by + ((r >> 3) & 7), 8 * bz + (r & 7) };
            for (int d = 0; d < 3; ++d) pts[3 * r + d] = sd_coord(gmin, c, q[d], d);
        }
        so_sdf_distance(verts, sub, ns, pts, 512, dist);
        for (int r = 0; r < 512; ++r) {
            const int in = 8 * bx + (r >> 6) < np[0] && 8 * by + ((r >> 3) & 7) < np[1] && 8 * bz + (r & 7) < np[2];
            if (in && dist[r] < B) listed = 1;
        }
        if (!listed) continue;
        if (n) so_field_scan(mode, ctr, w, g6, dlt, n, h, rs, t_low, t_high, pts, 512, fv, NULL, NULL, NULL);
        else memset(fv, 0, sizeof(float) * 512);
        for (int d = 0; d < 3; ++d) coords[3 * nl + d] = (int32_t)b[d];
        for (int r = 0; r < 512; ++r) {
            const int in = 8 * bx + (r >> 6) < np[0] && 8 * by + ((r >> 3) & 7) < np[1] && 8 * bz + (r & 7) < np[2];
            const float dd = fminf(dist[r], B);
            values[512 * nl + r] = !in ? B : (fv[r] > thr ? -dd : dd);
        }
        ++nl;
    }
    for (int64_t bx = 0; bx < nb[0]; ++bx) for (int64_t by = 0; by < nb[1]; ++by) for (int64_t bz = 0; bz < nb[2]; ++bz) {
        const float p[3] = { sd_coord(gmin, c, 8 * bx, 0), sd_coord(gmin, c, 8 * by, 1), sd_coord(gmin, c, 8 * bz, 2) };
        float v = 0.0f;
        if (n) so_field_scan(mode, ctr, w, g6, dlt, n, h, rs, t_low, t_high, p, 1, &v, NULL, NULL, NULL);
        inside[(bx * nb[1] + by) * nb[2] + bz] = v > thr;
    }
    free(box); free(sel); free(sub); free(pts); free(dist); free(fv);
    return nl;
}
