// ss_sdf.cuh -- narrow-band signed distance grid of a mesh on the lattice of a level-set field (ss_levelset_field_sdf_f32,
// DESIGN.md §14).
//
// The lattice is the field's grid, points gmin + index * cell (ss_grid_xy's formula), index in [0, n] per axis, in bricks of 8^3
// points.  d(p) is the f32 minimum over all triangles of ss_sdf_tri_d2 (every operation one rounding, no contraction), square-rooted
// once; B = band * cell.  A brick is listed iff one of its in-volume points has d < B; its values are -min(d, B) inside the field
// (value > threshold) and +min(d, B) outside, +B at points past the volume.
//
//   k_sdf_check_verts  lowest index of a vertex with a non-finite coordinate
//   k_sdf_count        per triangle: number of candidate bricks (its f32 AABB grown by B + cell, clamped to the grid) within a slab
//                      of brick columns, and once over the whole grid the candidate bricks per column and the lowest index of a
//                      triangle with a vertex index >= nv
//   k_sdf_emit         per triangle: (brick key, triangle) pairs of the slab at its scanned offset; the key sort (cub_sort) and
//                      k_field_starts give one run of triangles per candidate brick
//   k_sdf_brick        warp per candidate brick: its triangles staged in shared memory (9 floats each), then per 4x4x4 sub-box the
//                      triangles whose AABB lies within B + cell of the sub-box compacted by ballot; each lane keeps min d^2 of its two
//                      points.  Runs longer than the slice walk the triangles from global memory.  Writes d per point, the listed
//                      flag per brick and the tier counts
//   k_sdf_points       the grid points of the listed bricks, then the first point of every brick (the field's sign queries); the
//                      listed bricks' coordinates
//   k_sdf_sign         sign and clamp of the listed bricks' values; the inside flag of every brick
// A triangle farther than B from every point of a brick does not change min(d, B) there, so the binning and the sub-box cull (both
// conservative by one cell) change no output bit, and the minimum does not depend on the order the triangles are visited in.
// The host runs the slabs (whole brick columns bx, ascending) as passes whose pairs and bricks stay under a bound, so the working
// set of a call does not grow with the mesh.
#pragma once

#define SS_SDF_WARPS 2                  // candidate bricks per CTA
#define SS_SDF_CAP 320                  // triangles staged per warp (shared slice); longer runs take the global walk

struct SsSdfGrid {
    float gmin[3], c;                   // lattice: gmin + index * c
    int np[3], nb[3];                   // points and bricks per axis
    float B, reach;                     // background band * c; binning and culling margin B + c
};

__device__ __forceinline__ float ss_sdf_coord(const SsSdfGrid &G, int i, int d) { return __fadd_rn(__fmul_rn((float)i, G.c), G.gmin[d]); }

__device__ __forceinline__ float ss_sdf_dot(const float (&a)[3], const float (&b)[3]) {
    return __fadd_rn(__fadd_rn(__fmul_rn(a[0], b[0]), __fmul_rn(a[1], b[1])), __fmul_rn(a[2], b[2]));
}
__device__ __forceinline__ void ss_sdf_cross(const float (&a)[3], const float (&b)[3], float (&x)[3]) {
    x[0] = __fsub_rn(__fmul_rn(a[1], b[2]), __fmul_rn(a[2], b[1]));
    x[1] = __fsub_rn(__fmul_rn(a[2], b[0]), __fmul_rn(a[0], b[2]));
    x[2] = __fsub_rn(__fmul_rn(a[0], b[1]), __fmul_rn(a[1], b[0]));
}

// |p - (v0 + t e)|^2, e = v1 - v0, t = clamp(dot(p - v0, e) / dot(e, e), 0, 1) (t = 0 when dot(e, e) == 0)
__device__ __forceinline__ float ss_sdf_edge_d2(const float (&p)[3], const float *v0, const float *v1) {
    float e[3], w[3], r[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) { e[d] = __fsub_rn(v1[d], v0[d]); w[d] = __fsub_rn(p[d], v0[d]); }
    const float ee = ss_sdf_dot(e, e);
    const float t = ee == 0.0f ? 0.0f : fminf(fmaxf(__fdiv_rn(ss_sdf_dot(w, e), ee), 0.0f), 1.0f);
#pragma unroll
    for (int d = 0; d < 3; ++d) r[d] = __fsub_rn(p[d], __fadd_rn(v0[d], __fmul_rn(t, e[d])));
    return ss_sdf_dot(r, r);
}

// dot((v1 - v0) x (p - v0), n): >= 0 when p projects onto the inner side of edge v0 v1
__device__ __forceinline__ float ss_sdf_side(const float (&p)[3], const float *v0, const float *v1, const float (&n)[3]) {
    float e[3], w[3], x[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) { e[d] = __fsub_rn(v1[d], v0[d]); w[d] = __fsub_rn(p[d], v0[d]); }
    ss_sdf_cross(e, w, x);
    return ss_sdf_dot(x, n);
}

// Squared point-triangle distance, t = (a, b, c) as 9 floats: min of the edges (a, b), (b, c), (c, a), and of dot(p - a, n)^2 / |n|^2
// with n = (b - a) x (c - a) when |n|^2 > 0 and the three side tests are >= 0.  Defined for zero-area triangles.
__device__ __forceinline__ float ss_sdf_tri_d2(const float (&p)[3], const float *t) {
    const float *a = t, *b = t + 3, *c = t + 6;
    float d2 = fminf(fminf(ss_sdf_edge_d2(p, a, b), ss_sdf_edge_d2(p, b, c)), ss_sdf_edge_d2(p, c, a));
    float ab[3], ac[3], n[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) { ab[d] = __fsub_rn(b[d], a[d]); ac[d] = __fsub_rn(c[d], a[d]); }
    ss_sdf_cross(ab, ac, n);
    const float nn = ss_sdf_dot(n, n);
    if (nn > 0.0f && ss_sdf_side(p, a, b, n) >= 0.0f && ss_sdf_side(p, b, c, n) >= 0.0f && ss_sdf_side(p, c, a, n) >= 0.0f) {
        const float w[3] = { __fsub_rn(p[0], a[0]), __fsub_rn(p[1], a[1]), __fsub_rn(p[2], a[2]) };
        const float dn = ss_sdf_dot(w, n);
        d2 = fminf(d2, __fdiv_rn(__fmul_rn(dn, dn), nn));
    }
    return d2;
}

__device__ __forceinline__ void ss_sdf_load_tri(const float *__restrict__ verts, const uint32_t *__restrict__ tris, uint32_t t, float *dst) {
#pragma unroll
    for (int v = 0; v < 3; ++v) {
        const uint32_t i = tris[3 * (size_t)t + v];
        dst[3 * v] = verts[3 * (size_t)i]; dst[3 * v + 1] = verts[3 * (size_t)i + 1]; dst[3 * v + 2] = verts[3 * (size_t)i + 2];
    }
}

// Candidate bricks of a triangle: its AABB grown by B + cell, as point indices floor / ceil, clamped to the grid; false if empty
__device__ __forceinline__ bool ss_sdf_brick_range(const SsSdfGrid &G, const float *t, int (&lo)[3], int (&hi)[3]) {
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const float mn = fminf(fminf(t[d], t[3 + d]), t[6 + d]), mx = fmaxf(fmaxf(t[d], t[3 + d]), t[6 + d]);
        const float lim = (float)(G.np[d] + 8);
        const float fl = fminf(fmaxf(floorf(__fdiv_rn(__fsub_rn(__fsub_rn(mn, G.reach), G.gmin[d]), G.c)), -8.0f), lim);
        const float fh = fminf(fmaxf(ceilf(__fdiv_rn(__fsub_rn(__fadd_rn(mx, G.reach), G.gmin[d]), G.c)), -8.0f), lim);
        const int il = (int)fl, ih = (int)fh;
        if (ih < 0 || il > G.np[d] - 1) return false;
        lo[d] = max(il, 0) >> 3; hi[d] = min(ih, G.np[d] - 1) >> 3;
    }
    return true;
}

// chk[0]: lowest index of a vertex with a non-finite coordinate (preset ~0)
__global__ void k_sdf_check_verts(const float *__restrict__ verts, uint64_t nv, unsigned long long *__restrict__ chk) {
    const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nv) return;
    if (!isfinite(verts[3 * i]) || !isfinite(verts[3 * i + 1]) || !isfinite(verts[3 * i + 2])) atomicMin(&chk[0], (unsigned long long)i);
}

// The candidate bricks of a triangle within the slab of brick columns [bx0, bx1); false if none
__device__ __forceinline__ bool ss_sdf_slab_range(const SsSdfGrid &G, const float *t, int bx0, int bx1, int (&lo)[3], int (&hi)[3]) {
    if (!ss_sdf_brick_range(G, t, lo, hi)) return false;
    lo[0] = max(lo[0], bx0); hi[0] = min(hi[0], bx1 - 1);
    return lo[0] <= hi[0];
}

// cnt[t]: candidate bricks of triangle t in the slab [bx0, bx1); with hist, hist[bx] += its candidate bricks in column bx, and chk[1]:
// lowest index of a triangle with a vertex index >= nv (preset ~0), which counts 0
__global__ void k_sdf_count(SsSdfGrid G, const float *__restrict__ verts, uint64_t nv, const uint32_t *__restrict__ tris, uint32_t nt,
                            int bx0, int bx1, unsigned long long *__restrict__ cnt, unsigned long long *__restrict__ hist,
                            unsigned long long *__restrict__ chk) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nt) return;
    unsigned long long n = 0;
    if (tris[3 * (size_t)t] >= nv || tris[3 * (size_t)t + 1] >= nv || tris[3 * (size_t)t + 2] >= nv) {
        atomicMin(&chk[1], (unsigned long long)t);
    } else {
        float v[9];
        int lo[3], hi[3];
        ss_sdf_load_tri(verts, tris, t, v);
        if (ss_sdf_slab_range(G, v, bx0, bx1, lo, hi)) {
            const unsigned long long col = (unsigned long long)(hi[1] - lo[1] + 1) * (unsigned long long)(hi[2] - lo[2] + 1);
            n = (unsigned long long)(hi[0] - lo[0] + 1) * col;
            if (hist) for (int bx = lo[0]; bx <= hi[0]; ++bx) atomicAdd(&hist[bx], col);
        }
    }
    if (cnt) cnt[t] = n;
}

// (brick key, triangle) pairs of triangle t in the slab [bx0, bx1) at off[t]; key = (bx * nb1 + by) * nb2 + bz
__global__ void k_sdf_emit(SsSdfGrid G, const float *__restrict__ verts, const uint32_t *__restrict__ tris, uint32_t nt, int bx0, int bx1,
                           const unsigned long long *__restrict__ off, uint32_t *__restrict__ key, uint32_t *__restrict__ val) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nt) return;
    float v[9];
    int lo[3], hi[3];
    ss_sdf_load_tri(verts, tris, t, v);
    if (!ss_sdf_slab_range(G, v, bx0, bx1, lo, hi)) return;
    unsigned long long o = off[t];
    for (int bx = lo[0]; bx <= hi[0]; ++bx)
        for (int by = lo[1]; by <= hi[1]; ++by)
            for (int bz = lo[2]; bz <= hi[2]; ++bz, ++o) {
                key[o] = ((uint32_t)bx * (uint32_t)G.nb[1] + (uint32_t)by) * (uint32_t)G.nb[2] + (uint32_t)bz;
                val[o] = t;
            }
}

__device__ __forceinline__ void ss_sdf_brick_of(const SsSdfGrid &G, uint32_t k, int (&b)[3]) {
    b[2] = (int)(k % (uint32_t)G.nb[2]);
    b[1] = (int)(k / (uint32_t)G.nb[2] % (uint32_t)G.nb[1]);
    b[0] = (int)(k / ((uint32_t)G.nb[2] * (uint32_t)G.nb[1]));
}

// squared gap between the AABB of triangle t and the box [lo, hi].  Deliberately plain arithmetic (nvcc may contract it): it only
// culls, with a margin of one cell beyond B, so its rounding changes no output bit.
__device__ __forceinline__ float ss_sdf_box_gap2(const float *t, const float (&lo)[3], const float (&hi)[3]) {
    float s = 0.0f;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const float mn = fminf(fminf(t[d], t[3 + d]), t[6 + d]), mx = fmaxf(fmaxf(t[d], t[3 + d]), t[6 + d]);
        const float g = fmaxf(fmaxf(lo[d] - mx, mn - hi[d]), 0.0f);
        s += g * g;
    }
    return s;
}

struct SsSdfArgs {
    SsSdfGrid G;
    const float *verts;
    const uint32_t *tris;
    const uint32_t *key, *val;          // sorted pairs
    const uint32_t *starts;             // [ncand + 1] first pair of each candidate brick, then the number of pairs
    uint32_t ncand;
    float *dist;                        // [ncand][512] d per point (+inf where no triangle is within B + cell)
    uint32_t *listed;                   // [ncand] 1 if an in-volume point has d < B
    uint32_t *paths;                    // [2] candidate bricks through the shared slice, through the global walk
};

template <int WARPS, int CAP>
__global__ void __launch_bounds__(WARPS * 32)
k_sdf_brick(SsSdfArgs A) {
    __shared__ float s_tri[WARPS][CAP * 9];
    __shared__ uint16_t s_list[WARPS][CAP];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t cand = blockIdx.x * WARPS + wib;
    if (cand >= A.ncand) return;
    const SsSdfGrid &G = A.G;
    const uint32_t s0 = A.starts[cand], T = A.starts[cand + 1] - s0;
    int b[3];
    ss_sdf_brick_of(G, A.key[s0], b);
    const bool staged = T <= (uint32_t)CAP;
    if (staged)
        for (uint32_t j = lane; j < T; j += 32) ss_sdf_load_tri(A.verts, A.tris, A.val[s0 + j], &s_tri[wib][9 * j]);
    if (lane == 0) atomicAdd(&A.paths[staged ? 0 : 1], 1u);
    __syncwarp();
    const float reach2 = G.reach * G.reach;
    const int li = lane >> 3, lj = (lane >> 1) & 3, lk = (lane & 1) * 2;        // the lane's points (li, lj, lk) and (li, lj, lk + 1)
    bool listed = false;
    for (int sb = 0; sb < 8; ++sb) {
        const int o[3] = { 8 * b[0] + 4 * (sb >> 2), 8 * b[1] + 4 * ((sb >> 1) & 1), 8 * b[2] + 4 * (sb & 1) };
        float lo[3], hi[3];
#pragma unroll
        for (int d = 0; d < 3; ++d) { lo[d] = ss_sdf_coord(G, o[d], d); hi[d] = ss_sdf_coord(G, o[d] + 3, d); }
        const int gi = o[0] + li, gj = o[1] + lj, gk = o[2] + lk;
        const float pa[3] = { ss_sdf_coord(G, gi, 0), ss_sdf_coord(G, gj, 1), ss_sdf_coord(G, gk, 2) };
        const float pb[3] = { pa[0], pa[1], ss_sdf_coord(G, gk + 1, 2) };
        float da = INFINITY, db = INFINITY;
        if (staged) {
            int nlist = 0;
            for (uint32_t w = 0; w < (T + 31) >> 5; ++w) {
                const uint32_t j = w * 32 + lane;
                const bool keep = j < T && ss_sdf_box_gap2(&s_tri[wib][9 * j], lo, hi) < reach2;
                const unsigned m = __ballot_sync(0xffffffffu, keep);
                if (keep) s_list[wib][nlist + __popc(m & ((1u << lane) - 1u))] = (uint16_t)j;
                nlist += __popc(m);
            }
            __syncwarp();
            for (int n = 0; n < nlist; ++n) {
                const float *t = &s_tri[wib][9 * s_list[wib][n]];
                da = fminf(da, ss_sdf_tri_d2(pa, t)); db = fminf(db, ss_sdf_tri_d2(pb, t));
            }
            __syncwarp();                                        // the list is rebuilt for the next sub-box
        } else {
            for (uint32_t j = 0; j < T; ++j) {
                float t[9];
                ss_sdf_load_tri(A.verts, A.tris, A.val[s0 + j], t);
                if (!(ss_sdf_box_gap2(t, lo, hi) < reach2)) continue;
                da = fminf(da, ss_sdf_tri_d2(pa, t)); db = fminf(db, ss_sdf_tri_d2(pb, t));
            }
        }
        da = __fsqrt_rn(da); db = __fsqrt_rn(db);
        float *out = A.dist + (size_t)cand * 512;
        const int q = ((li + 4 * (sb >> 2)) * 8 + lj + 4 * ((sb >> 1) & 1)) * 8 + lk + 4 * (sb & 1);
        out[q] = da; out[q + 1] = db;
        const bool in_ij = gi < G.np[0] && gj < G.np[1];
        listed = listed || (in_ij && gk < G.np[2] && da < G.B) || (in_ij && gk + 1 < G.np[2] && db < G.B);
    }
    const bool any = __any_sync(0xffffffffu, listed);
    if (lane == 0) A.listed[cand] = any ? 1u : 0u;
}

// Query points: i < 512 nl: point i % 512 ([i][j][k], k fastest) of listed brick i / 512 (list: candidate indices); then the first point
// 8 b of brick b = i - 512 nl.  coords[3 l]: the brick coordinates of listed brick l.
__global__ void k_sdf_points(SsSdfGrid G, const uint32_t *__restrict__ key, const uint32_t *__restrict__ starts, const uint32_t *__restrict__ list,
                             uint32_t nl, uint32_t nbtot, float *__restrict__ pts, int32_t *__restrict__ coords) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t m = (uint64_t)nl * 512 + nbtot;
    if (i >= m) return;
    int b[3], q[3] = { 0, 0, 0 };
    if (i < nl * 512u) {
        ss_sdf_brick_of(G, key[starts[list[i >> 9]]], b);
        const int r = (int)(i & 511);
        q[0] = r >> 6; q[1] = (r >> 3) & 7; q[2] = r & 7;
        if (r == 0) { coords[3 * (size_t)(i >> 9)] = b[0]; coords[3 * (size_t)(i >> 9) + 1] = b[1]; coords[3 * (size_t)(i >> 9) + 2] = b[2]; }
    } else {
        ss_sdf_brick_of(G, i - nl * 512u, b);
    }
#pragma unroll
    for (int d = 0; d < 3; ++d) pts[3 * (size_t)i + d] = ss_sdf_coord(G, 8 * b[d] + q[d], d);
}

// values[l][r] = -min(d, B) inside (field value > thr), +min(d, B) outside, +B past the volume; inside[b] for every brick
__global__ void k_sdf_sign(SsSdfGrid G, float thr, const float *__restrict__ dist, const uint32_t *__restrict__ key, const uint32_t *__restrict__ starts,
                           const uint32_t *__restrict__ list, uint32_t nl, uint32_t nbtot, const float *__restrict__ fv, float *__restrict__ values,
                           uint8_t *__restrict__ inside) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    const uint64_t m = (uint64_t)nl * 512 + nbtot;
    if (i >= m) return;
    if (i < nl * 512u) {
        const uint32_t cand = list[i >> 9];
        const int r = (int)(i & 511);
        int b[3];
        ss_sdf_brick_of(G, key[starts[cand]], b);
        const bool in_volume = 8 * b[0] + (r >> 6) < G.np[0] && 8 * b[1] + ((r >> 3) & 7) < G.np[1] && 8 * b[2] + (r & 7) < G.np[2];
        const float d = fminf(dist[(size_t)cand * 512 + r], G.B);
        values[i] = !in_volume ? G.B : (fv[i] > thr ? -d : d);
    } else {
        inside[i - nl * 512u] = fv[i] > thr ? 1 : 0;
    }
}
