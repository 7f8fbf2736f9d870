/*
 * levelset_raycast_oracle.c -- first crossings of the level-set field along rays (DESIGN.md section 15) by evaluating every sample,
 * TEST INFRASTRUCTURE ONLY.
 *
 * Includes tests/levelset_field_oracle.c unchanged and restates section 15 literally: every sample T_0 = 0, T_k = (float)k dt while
 * T_k < t_max and k < 2^24, then t_max if finite and > 0, is evaluated with so_field_scan, in order, with no skipping; the march
 * ends at the first crossing, at the first sample outside the grid on an axis the ray does not move back from, or after the last
 * sample; the bracket is halved up to `refine` times.  The device skips runs of value-0 samples by binary search; this file does not.
 * To keep the scan affordable each ray scans only the records within 2 h of its segment [0, T_last] (float64 distance), in
 * ascending index: every record farther than h from a point adds exactly nothing to any mode's fold there.  Compile it like the
 * oracle: single precision, un-contracted (-ffp-contract=off -fno-fast-math).
 */
#include "levelset_field_oracle.c"

#define SO_RAY_CAP 16777216u

typedef struct {
    int mode; uint64_t n; float h, rs, t_low, t_high, thr;
    const float *ctr, *w, *g6, *dlt;                         /* the ray's records (gathered) */
} so_ray_field;

static float so_ray_value(const so_ray_field *F, const float *p) {
    float v = 0.0f;
    if (F->n) so_field_scan(F->mode, F->ctr, F->w, F->g6, F->dlt, F->n, F->h, F->rs, F->t_low, F->t_high, p, 1, &v, NULL, NULL, NULL);
    return v;
}

static void so_ray_at(const float *o, const float *d, float t, float *p) {
    for (int a = 0; a < 3; ++a) p[a] = o[a] + t * d[a];
}

static int so_ray_gone(const float *p, const float *d, const float *gmin, const float *gmax) {
    for (int a = 0; a < 3; ++a)
        if ((p[a] > gmax[a] && d[a] >= 0.0f) || (p[a] < gmin[a] && d[a] <= 0.0f)) return 1;
    return 0;
}

/* m rays (o, d: m x 3; tmax: m, or NULL for +inf) against the n records of a mode (arrays as for so_field_scan).  Outputs as
 * ss_levelset_field_raycast_f32: t, pos (m x 3), val, status; grad (m x 3, or NULL) the gradient at the hit by so_field_scan (NaN
 * without a hit; modes with a gradient only).  Returns the total number of samples evaluated. */
int64_t so_raycast(int mode, const float *ctr, const float *w, const float *g6, const float *dlt, uint64_t n, float h, float rs, float t_low,
                   float t_high, float thr, const float *gmin, const float *gmax, const float *o, const float *d, const float *tmax, uint64_t m,
                   float step, uint32_t refine, float *t, float *pos, float *val, int8_t *status, float *grad) {
    float *c2 = malloc((n ? n : 1) * 3 * sizeof(float)), *w2 = malloc((n ? n : 1) * sizeof(float));
    float *g2 = malloc((n ? n : 1) * 6 * sizeof(float)), *d2 = malloc((n ? n : 1) * sizeof(float));
    int64_t evals = 0;
    for (uint64_t i = 0; i < m; ++i) {
        const float *oi = o + 3 * i, *di = d + 3 * i;
        const float tm = tmax ? tmax[i] : INFINITY;
        const float nd = sqrtf((di[0] * di[0] + di[1] * di[1]) + di[2] * di[2]);
        const float dt = step / nd;
        t[i] = INFINITY; val[i] = NAN; status[i] = 0;
        for (int a = 0; a < 3; ++a) pos[3 * i + a] = NAN;
        if (grad) for (int a = 0; a < 3; ++a) grad[3 * i + a] = NAN;
        /* the records within 2 h of the segment [0, T_last] (T_last <= 2^24 dt, or t_max) */
        double tend = (double)SO_RAY_CAP * (double)dt;
        if (isfinite(tm) && (double)tm < tend) tend = tm;
        const double dd = (double)di[0] * di[0] + (double)di[1] * di[1] + (double)di[2] * di[2];
        so_ray_field F = { mode, 0, h, rs, t_low, t_high, thr, c2, w2, g2, d2 };
        for (uint64_t j = 0; j < n; ++j) {
            double x[3], s = 0.0, q2 = 0.0;
            for (int a = 0; a < 3; ++a) { x[a] = (double)ctr[3 * j + a] - oi[a]; s += x[a] * di[a]; }
            s /= dd;
            if (s < 0.0) s = 0.0;
            if (s > tend) s = tend;
            for (int a = 0; a < 3; ++a) { const double e = x[a] - s * di[a]; q2 += e * e; }
            if (q2 > 4.0 * (double)h * h) continue;
            const uint64_t k = F.n++;
            memcpy(c2 + 3 * k, ctr + 3 * j, 12);
            if (w) w2[k] = w[j];
            if (g6) memcpy(g2 + 6 * k, g6 + 6 * j, 24);
            if (dlt) d2[k] = dlt[j];
        }
        if (!w) F.w = NULL;
        if (!g6) F.g6 = NULL;
        if (!dlt) F.dlt = NULL;
        /* T_0 */
        float p[3];
        so_ray_at(oi, di, 0.0f, p);
        const int in0 = so_ray_value(&F, p) > thr;
        ++evals;
        if (so_ray_gone(p, di, gmin, gmax)) continue;
        int found = 0, gone = 0, tail = 0;
        float prev = 0.0f, a = 0.0f, b = 0.0f, vb = 0.0f;
        for (uint32_t k = 1;; ++k) {
            float tk = (float)k * dt;
            if (!(k < SO_RAY_CAP && tk < tm)) {
                if (!(isfinite(tm) && tm > 0.0f)) break;
                tk = tm; tail = 1;
            }
            so_ray_at(oi, di, tk, p);
            const float v = so_ray_value(&F, p);
            ++evals;
            if ((v > thr) != in0) { found = 1; a = prev; b = tk; vb = v; break; }
            if (so_ray_gone(p, di, gmin, gmax)) { gone = 1; break; }
            if (tail) break;
            prev = tk;
        }
        if (!found) {
            status[i] = (!gone && (float)SO_RAY_CAP * dt < tm) ? 2 : 0;
            continue;
        }
        for (uint32_t r = 0; r < refine; ++r) {
            const float mid = a + ((b - a) * 0.5f);
            if (mid == a || mid == b) break;
            so_ray_at(oi, di, mid, p);
            const float v = so_ray_value(&F, p);
            ++evals;
            if ((v > thr) == in0) a = mid;
            else { b = mid; vb = v; }
        }
        so_ray_at(oi, di, b, p);
        t[i] = b; val[i] = vb; status[i] = in0 ? -1 : 1;
        for (int q = 0; q < 3; ++q) pos[3 * i + q] = p[q];
        if (grad && F.n) {
            float v, g[3] = { 0.0f, 0.0f, 0.0f };
            so_field_scan(mode, F.ctr, F.w, F.g6, F.dlt, F.n, h, rs, t_low, t_high, p, 1, &v, g, NULL, NULL);
            for (int q = 0; q < 3; ++q) grad[3 * i + q] = g[q];
        } else if (grad) {
            for (int q = 0; q < 3; ++q) grad[3 * i + q] = 0.0f;
        }
    }
    free(c2); free(w2); free(g2); free(d2);
    return evals;
}
