// ss_aniso.cuh -- anisotropic-kernel level set (J. Yu and G. Turk, "Reconstructing Surfaces of Particle-Based Fluids Using
// Anisotropic Kernels", ACM TOG 32(1), 2013), the opt-in mode of ss_context_set_anisotropy_f32.  DESIGN.md §11 is the
// specification; tests/anisotropic_oracle.c restates it in plain C in the same operation order, so results are bit-exact.
//
//   k_aniso_init        x_bar = x, G = I, det G = 1 for every particle (particles without an owning subdomain keep these)
//   k_aniso             per particle in its owning subdomain: weighted mean and covariance of its density neighbourhood (the
//                       density stage's walk, ss_nbr_walk), cyclic Jacobi, clamped stretch -> x_bar, G (6 entries), det G
//   k_records_aniso     splat records (x_bar, V det G) + the G entries of every binned membership
//   k_fold_levelset     warp per 8^3-point brick over the non-empty-brick work list: candidates of the brick's bins sorted by
//                       particle index, per 4x4x4 sub-box the candidates within h of the sub-box, two grid points per lane;
//                       bricks with more candidates than the slice go to a 4096-slot instantiation, beyond that to
//                       k_fold_select (O(C^2) selection in index order).  Templated on the fold: SsAnisoFold here, SsAvgFold
//                       and SsAvgCorrFold (averaged-position surface, plain and Jacobian-corrected, ss_averaged.cuh), and
//                       SsAvgRadFold / SsAvgCorrRadFold (the same with per-particle radii)
// Every value the level set writes is exact; there is no certification in this mode.
#pragma once

#define SS_AN_SWEEPS 8                  // cyclic Jacobi sweeps (pivots (0,1), (0,2), (1,2))
#define SS_AN_WARPS 4                   // bricks per CTA of the default slice
#define SS_AN_CAP 512                   // candidates staged per brick (default slice)
#define SS_AN_BIG_CAP 4096              // one warp per CTA: 40 KB of static shared memory

// ------------------------------------------------------------------ per-particle anisotropy ----
__global__ void k_aniso_init(const float *__restrict__ xyz, uint32_t n, float *__restrict__ xbar, float *__restrict__ gmat, float *__restrict__ gdet) {
    const uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    for (int d = 0; d < 3; ++d) xbar[3 * (uint64_t)p + d] = xyz[3 * (uint64_t)p + d];
    const float id[6] = { 1.0f, 0.0f, 0.0f, 1.0f, 0.0f, 1.0f };
    for (int q = 0; q < 6; ++q) gmat[6 * (uint64_t)p + q] = id[q];
    gdet[p] = 1.0f;
}

// One Jacobi rotation of the symmetric 3x3 matrix a (and the accumulated eigenvectors v, columns) that zeroes a[p][q];
// skipped when a[p][q] is exactly 0.  Classic formulas: theta = (a_qq - a_pp) / (2 a_pq), t = sgn(theta) / (|theta| +
// sqrt(theta^2 + 1)), c = 1 / sqrt(t^2 + 1), s = t c.
template <int p, int q>
__device__ __forceinline__ void ss_jacobi_rot(float (&a)[3][3], float (&v)[3][3]) {
    constexpr int r = 3 - p - q;
    const float apq = a[p][q];
    if (apq == 0.0f) return;
    const float theta = __fdiv_rn(__fsub_rn(a[q][q], a[p][p]), __fmul_rn(2.0f, apq));
    float t = __fdiv_rn(1.0f, __fadd_rn(fabsf(theta), __fsqrt_rn(__fadd_rn(__fmul_rn(theta, theta), 1.0f))));
    if (theta < 0.0f) t = -t;
    const float c = __fdiv_rn(1.0f, __fsqrt_rn(__fadd_rn(__fmul_rn(t, t), 1.0f)));
    const float s = __fmul_rn(t, c);
    const float app = __fsub_rn(a[p][p], __fmul_rn(t, apq)), aqq = __fadd_rn(a[q][q], __fmul_rn(t, apq));
    const float arp = __fsub_rn(__fmul_rn(c, a[r][p]), __fmul_rn(s, a[r][q]));
    const float arq = __fadd_rn(__fmul_rn(s, a[r][p]), __fmul_rn(c, a[r][q]));
    a[p][p] = app; a[q][q] = aqq; a[p][q] = 0.0f; a[q][p] = 0.0f;
    a[r][p] = arp; a[p][r] = arp; a[r][q] = arq; a[q][r] = arq;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        const float vkp = v[k][p], vkq = v[k][q];
        v[k][p] = __fsub_rn(__fmul_rn(c, vkp), __fmul_rn(s, vkq));
        v[k][q] = __fadd_rn(__fmul_rn(s, vkp), __fmul_rn(c, vkq));
    }
}

// G (g00, g01, g02, g11, g12, g22) and det G of a covariance matrix (DESIGN.md §11).
__device__ __forceinline__ void ss_aniso_matrix(const SsDev &P, float (&a)[3][3], uint32_t nn, float g[6], float &det) {
    float v[3][3] = { { 1.0f, 0.0f, 0.0f }, { 0.0f, 1.0f, 0.0f }, { 0.0f, 0.0f, 1.0f } };
#pragma unroll
    for (int sweep = 0; sweep < SS_AN_SWEEPS; ++sweep) {
        ss_jacobi_rot<0, 1>(a, v);
        ss_jacobi_rot<0, 2>(a, v);
        ss_jacobi_rot<1, 2>(a, v);
    }
    float e[3] = { a[0][0], a[1][1], a[2][2] };
    int ord[3] = { 0, 1, 2 };
    // descending, stable: compare-exchange (0,1), (1,2), (0,1)
#define SS_AN_CX(i, j) if (e[i] < e[j]) { const float te = e[i]; e[i] = e[j]; e[j] = te; const int to = ord[i]; ord[i] = ord[j]; ord[j] = to; }
    SS_AN_CX(0, 1) SS_AN_CX(1, 2) SS_AN_CX(0, 1)
#undef SS_AN_CX
#pragma unroll
    for (int k = 0; k < 3; ++k) e[k] = e[k] < 0.0f ? 0.0f : e[k];
    if (nn < P.an_min_nb || e[0] == 0.0f) {
        g[0] = 1.0f; g[1] = 0.0f; g[2] = 0.0f; g[3] = 1.0f; g[4] = 0.0f; g[5] = 1.0f; det = 1.0f;
        return;
    }
    const float floor_s = __fdiv_rn(e[0], P.an_kr);
    float inv[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) inv[k] = __fdiv_rn(1.0f, __fdiv_rn(fmaxf(e[k], floor_s), e[0]));
    det = __fmul_rn(__fmul_rn(inv[0], inv[1]), inv[2]);
    float R[3][3];                                  // R[row][k] = component `row` of the k-th eigenvector (descending)
#pragma unroll
    for (int row = 0; row < 3; ++row) {
#pragma unroll
        for (int k = 0; k < 3; ++k) R[row][k] = ord[k] == 0 ? v[row][0] : (ord[k] == 1 ? v[row][1] : v[row][2]);
    }
    const int ia[6] = { 0, 0, 0, 1, 1, 2 }, ib[6] = { 0, 1, 2, 1, 2, 2 };
#pragma unroll
    for (int q = 0; q < 6; ++q) {
        float acc = __fmul_rn(__fmul_rn(R[ia[q]][0], inv[0]), R[ib[q]][0]);
        acc = __fadd_rn(acc, __fmul_rn(__fmul_rn(R[ia[q]][1], inv[1]), R[ib[q]][1]));
        acc = __fadd_rn(acc, __fmul_rn(__fmul_rn(R[ia[q]][2], inv[2]), R[ib[q]][2]));
        g[q] = acc;
    }
}

// One thread per particle inside its subdomain (the density stage's compacted list).
__global__ void __launch_bounds__(128)
k_aniso(SsDev P, uint32_t m, const uint32_t *__restrict__ list, const uint32_t *__restrict__ list_off, const uint32_t *__restrict__ list_flag,
        const uint32_t *__restrict__ key, const float4 *__restrict__ spos, const uint32_t *__restrict__ sub_flat,
        const uint32_t *__restrict__ off, float *__restrict__ xbar, float *__restrict__ gmat,
        float *__restrict__ gdet) {
    const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
    if (tid >= list_off[m - 1] + list_flag[m - 1]) return;
    const SsWalk W = ss_walk_sub(P, list[tid], key, sub_flat, off);
    const float4 pi = spos[W.e];
    const uint32_t p = __float_as_uint(pi.w);
    // weighted mean of the offsets x_j - x_i (self: w = 1, offset 0)
    float sw = 1.0f, mx = 0.0f, my = 0.0f, mz = 0.0f;
    uint32_t nn = 0;
    ss_nbr_walk(P, W, pi, spos, [&](const float4 &, float dx, float dy, float dz, float d2) {
        const float q = __fdiv_rn(__fsqrt_rn(d2), P.h);
        const float w = __fsub_rn(1.0f, __fmul_rn(__fmul_rn(q, q), q));
        sw = __fadd_rn(sw, w);
        mx = __fadd_rn(mx, __fmul_rn(w, dx)); my = __fadd_rn(my, __fmul_rn(w, dy)); mz = __fadd_rn(mz, __fmul_rn(w, dz));
        ++nn;
    });
    const float ux = __fdiv_rn(mx, sw), uy = __fdiv_rn(my, sw), uz = __fdiv_rn(mz, sw);
    // weighted covariance about the mean, self term first
    float c00, c01, c02, c11, c12, c22;
    {
        const float ex = __fsub_rn(0.0f, ux), ey = __fsub_rn(0.0f, uy), ez = __fsub_rn(0.0f, uz);
        c00 = __fmul_rn(ex, ex); c01 = __fmul_rn(ex, ey); c02 = __fmul_rn(ex, ez);
        c11 = __fmul_rn(ey, ey); c12 = __fmul_rn(ey, ez); c22 = __fmul_rn(ez, ez);
    }
    ss_nbr_walk(P, W, pi, spos, [&](const float4 &, float dx, float dy, float dz, float d2) {
        const float q = __fdiv_rn(__fsqrt_rn(d2), P.h);
        const float w = __fsub_rn(1.0f, __fmul_rn(__fmul_rn(q, q), q));
        const float ex = __fsub_rn(dx, ux), ey = __fsub_rn(dy, uy), ez = __fsub_rn(dz, uz);
        const float wx = __fmul_rn(w, ex), wy = __fmul_rn(w, ey), wz = __fmul_rn(w, ez);
        c00 = __fadd_rn(c00, __fmul_rn(wx, ex)); c01 = __fadd_rn(c01, __fmul_rn(wx, ey)); c02 = __fadd_rn(c02, __fmul_rn(wx, ez));
        c11 = __fadd_rn(c11, __fmul_rn(wy, ey)); c12 = __fadd_rn(c12, __fmul_rn(wy, ez)); c22 = __fadd_rn(c22, __fmul_rn(wz, ez));
    });
    c00 = __fdiv_rn(c00, sw); c01 = __fdiv_rn(c01, sw); c02 = __fdiv_rn(c02, sw);
    c11 = __fdiv_rn(c11, sw); c12 = __fdiv_rn(c12, sw); c22 = __fdiv_rn(c22, sw);
    float a[3][3] = { { c00, c01, c02 }, { c01, c11, c12 }, { c02, c12, c22 } };
    float g[6], det;
    ss_aniso_matrix(P, a, nn, g, det);
    xbar[3 * (uint64_t)p] = __fadd_rn(pi.x, __fmul_rn(P.an_lambda, ux));
    xbar[3 * (uint64_t)p + 1] = __fadd_rn(pi.y, __fmul_rn(P.an_lambda, uy));
    xbar[3 * (uint64_t)p + 2] = __fadd_rn(pi.z, __fmul_rn(P.an_lambda, uz));
#pragma unroll
    for (int q = 0; q < 6; ++q) gmat[6 * (uint64_t)p + q] = g[q];
    gdet[p] = det;
}

// After k_records ran on the smoothed centres: rec.w = V det G, grec = (g00, g01, g02, g11), (g12, g22, 0, 0) per membership.
__global__ void k_records_aniso(uint32_t m, const uint32_t *__restrict__ key, const uint32_t *__restrict__ pidx, const float *__restrict__ gmat,
                                const float *__restrict__ gdet, float4 *__restrict__ rec, float4 *__restrict__ grec) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= m || key[e] == 0xffffffffu) return;
    const uint32_t p = pidx[e];
    const float *g = gmat + 6 * (uint64_t)p;
    rec[e].w = __fmul_rn(rec[e].w, gdet[p]);
    grec[2 * (uint64_t)e] = make_float4(g[0], g[1], g[2], g[3]);
    grec[2 * (uint64_t)e + 1] = make_float4(g[4], g[5], 0.0f, 0.0f);
}

// ------------------------------------------------------------------ level set ----
struct SsAnArgs {
    SsBins bins;                       // records: (x_bar, V det G), bin-sorted
    const float4 *grec;                // two per record: (g00, g01, g02, g11), (g12, g22, -, -)
    const float *rrec;                 // one per record: delta_j of the averaged surface's per-particle radii (ss_averaged.cuh)
    const uint32_t *bricks;            // listed bricks (linear index)
    uint32_t n_bricks;
    float *tiles;
    uint8_t *bstate;                   // set to 2 (exact values) by the first launch over the work list; NULL in fallback launches
    uint32_t *fallback;                // bricks left to the next stage: [0] = count, [1..] = linear brick indices
};

// One term of phi(x) = sum_j V_j det G_j W(|G_j (x - x_bar_j)|), counted when |G_j (x - x_bar_j)|^2 < h^2.
__device__ __forceinline__ float ss_aniso_term(const SsDev &P, const float4 r, const float4 g0, const float4 g1, float gx, float gy, float gz, float phi) {
    const float dx = __fsub_rn(r.x, gx), dy = __fsub_rn(r.y, gy), dz = __fsub_rn(r.z, gz);
    const float u0 = __fadd_rn(__fadd_rn(__fmul_rn(g0.x, dx), __fmul_rn(g0.y, dy)), __fmul_rn(g0.z, dz));
    const float u1 = __fadd_rn(__fadd_rn(__fmul_rn(g0.y, dx), __fmul_rn(g0.w, dy)), __fmul_rn(g1.x, dz));
    const float u2 = __fadd_rn(__fadd_rn(__fmul_rn(g0.z, dx), __fmul_rn(g1.x, dy)), __fmul_rn(g1.y, dz));
    const float uu = __fadd_rn(__fadd_rn(__fmul_rn(u0, u0), __fmul_rn(u1, u1)), __fmul_rn(u2, u2));
    return uu < P.h2 ? __fadd_rn(phi, __fmul_rn(r.w, ss_kernel_scalar(P, __fsqrt_rn(uu)))) : phi;
}

// a listed brick, its tile and its candidate bins (no extension planes: the single-point planes are bricks of their own)
struct SsAnBrick { SsBrick B; SsTile T; SsBrickBins K; };
__device__ __forceinline__ SsAnBrick ss_an_brick(const SsDev &P, const SsAnArgs &A, uint32_t brick_lin) {
    SsAnBrick N;
    N.B = ss_brick_from_lin(P, brick_lin);
    N.T = A.bins.tile_tab[N.B.tile];
    N.K = ss_brick_bins(P, A.bins.brick_rng, N.B.bx, N.B.by, N.B.bz, false);
    return N;
}

// The level sets of this file and of ss_averaged.cuh fold every candidate within h of a grid point, in ascending particle index,
// into per-point accumulators.  A fold F supplies
//   F::Cand  F::load(A, src)                      what the fold reads of record src
//   F::Acc   F::zero()                            the accumulators of one grid point
//   void     F::add(P, cand, gx, gy, gz, acc)     one candidate at the grid point (gx, gy, gz); tests its own support
//   float    F::value(P, acc)                     the tile value
//   int      F::SELECT_BOXES                      sub-boxes whose accumulators k_fold_select holds per walk (1, 2, 4 or 8)
// and the brick kernels below stage, order and cull the candidates once for every fold.  A fold's support must lie within the
// isotropic ball of radius h around the record's position (the sub-box cull).

// phi(x) = sum_j V_j det G_j W(|G_j (x - x_bar_j)|) (DESIGN.md §11)
struct SsAnisoFold {
    struct Cand { float4 r, g0, g1; };
    struct Acc { float phi; };
    static constexpr int SELECT_BOXES = 8;
    static __device__ __forceinline__ Cand load(const SsAnArgs &A, uint32_t src) {
        return Cand{ A.bins.rec[src], A.grec[2 * (size_t)src], A.grec[2 * (size_t)src + 1] };
    }
    static __device__ __forceinline__ Acc zero() { return Acc{ 0.0f }; }
    static __device__ __forceinline__ void add(const SsDev &P, const Cand &c, float gx, float gy, float gz, Acc &a) {
        a.phi = ss_aniso_term(P, c.r, c.g0, c.g1, gx, gy, gz, a.phi);
    }
    static __device__ __forceinline__ float value(const SsDev &, const Acc &a) { return a.phi; }
};

// The candidates of bins K of subdomain s, one warp: counts them, and when there are 1 to CAP of them stages their sort keys
// (particle index << 32 | record index) in s_key, run by run, and sorts them ascending.  Returns the count C (nothing is staged
// for C = 0 or C > CAP).  Shared by the brick kernels below and the point queries of ss_field.cuh.
template <int CAP>
__device__ __forceinline__ uint32_t ss_stage_candidates(const SsDev &P, const SsBins &B, uint32_t s, const SsBrickBins &K, unsigned long long *s_key,
                                                        int lane) {
    uint32_t C = 0;
    for (int r0 = 0; r0 < K.nruns; r0 += 32) {
        uint32_t a;
        uint32_t len = ss_brick_run(P, B, s, K, r0 + lane, a);
        for (int o = 16; o > 0; o >>= 1) len += __shfl_xor_sync(0xffffffffu, len, o);
        C += len;
    }
    if (C == 0 || C > (uint32_t)CAP) return C;
    uint32_t dst0 = 0;
    for (int r0 = 0; r0 < K.nruns; r0 += 32) {
        uint32_t a, tot;
        const uint32_t len = ss_brick_run(P, B, s, K, r0 + lane, a);
        const uint32_t dst = dst0 + ss_warp_excl_scan(len, lane, tot);
        const int nr = min(32, K.nruns - r0);
        for (int rr = 0; rr < nr; ++rr) {
            const uint32_t ra = __shfl_sync(0xffffffffu, a, rr), rl = __shfl_sync(0xffffffffu, len, rr), rd = __shfl_sync(0xffffffffu, dst, rr);
            for (uint32_t t = lane; t < rl; t += 32) s_key[rd + t] = ((unsigned long long)B.pidx[ra + t] << 32) | (unsigned long long)(ra + t);
        }
        dst0 += tot;
    }
    ss_sort_keys<true>(s_key, (int)C);
    return C;
}

// The selection walk over bins K of subdomain s, one warp: the smallest candidate key above `last` (any key when `first`), ~0 when
// none is left.  O(C / 32) per step; for bricks and point groups above the largest slice.
__device__ __forceinline__ unsigned long long ss_select_next(const SsDev &P, const SsBins &B, uint32_t s, const SsBrickBins &K, unsigned long long last,
                                                             bool first, int lane) {
    unsigned long long best = ~0ull;
    for (int r = 0; r < K.nruns; ++r) {
        uint32_t a;
        const uint32_t len = ss_brick_run(P, B, s, K, r, a);
        for (uint32_t t = a + lane; t < a + len; t += 32) {
            const unsigned long long kk = ((unsigned long long)B.pidx[t] << 32) | (unsigned long long)t;
            if ((first || kk > last) && kk < best) best = kk;
        }
    }
    for (int o = 16; o > 0; o >>= 1) { const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o); if (other < best) best = other; }
    return best;
}

template <class F, int CAP>
__device__ __forceinline__ void ss_fold_brick(const SsDev &P, const SsAnArgs &A, unsigned long long *s_key, uint16_t *s_list, uint32_t work, int lane) {
    const uint32_t brick_lin = A.bricks[work];
    const SsAnBrick N = ss_an_brick(P, A, brick_lin);
    if (A.bstate && lane == 0) A.bstate[brick_lin] = 2;
    const uint32_t C = ss_stage_candidates<CAP>(P, A.bins, N.T.s, N.K, s_key, lane);
    if (C == 0) return;                                      // pre-zeroed tile: the value of a point without candidates is 0
    if (C > (uint32_t)CAP) {
        if (lane == 0) A.fallback[1 + atomicAdd(&A.fallback[0], 1u)] = brick_lin;
        return;
    }

    float *const tile = A.tiles + (size_t)N.B.tile * P.np * P.np * P.np;
    const SsSubLane L = ss_sub_lane(P, lane);
    const float cull2 = P.h2 * 1.0001f;
    for (int b = 0; b < 8; ++b) {
        // grid point coordinates: point_coordinates (uniform_grid.rs:418-425), min + index * cell; culling box: every fold's support
        // lies within distance h of the record's position
        const SsSubBox X = ss_sub_box(P, N.T, N.B.bx, N.B.by, N.B.bz, b, L, true);
        if (!X.inside) continue;
        int nlist = 0;
        for (int w = 0; w < (int)((C + 31) >> 5); ++w) {
            const int rnk = w * 32 + lane;
            bool keep = false;
            if (rnk < (int)C) {
                const float4 r = A.bins.rec[(uint32_t)s_key[rnk]];
                keep = ss_axis_d2(r.x, X.bxl, X.bxh) + ss_axis_d2(r.y, X.byl, X.byh) + ss_axis_d2(r.z, X.bzl, X.bzh) < cull2;
            }
            const uint32_t mword = __ballot_sync(0xffffffffu, keep);
            if (keep) s_list[nlist + __popc(mword & ((1u << lane) - 1u))] = (uint16_t)rnk;
            nlist += __popc(mword);
        }
        __syncwarp();
        typename F::Acc accA = F::zero(), accB = F::zero();
        for (int n = 0; n < nlist; ++n) {
            const typename F::Cand cd = F::load(A, (uint32_t)s_key[s_list[n]]);
            F::add(P, cd, X.gx, X.gy, X.gzA, accA);
            F::add(P, cd, X.gx, X.gy, X.gzB, accB);
        }
        if (X.vA) tile[((size_t)X.i * P.np + X.j) * P.np + X.k] = F::value(P, accA);
        if (X.vB) tile[((size_t)X.i * P.np + X.j) * P.np + X.k + 1] = F::value(P, accB);
        __syncwarp();                                        // the list is rebuilt for the next sub-box
    }
}

template <class F, int CAP, int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
k_fold_levelset(SsDev P, SsAnArgs A) {
    __shared__ unsigned long long s_key[WARPS][CAP];
    __shared__ uint16_t s_list[WARPS][CAP];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t work = blockIdx.x * WARPS + wib;
    if (work >= A.n_bricks) return;
    ss_fold_brick<F, CAP>(P, A, s_key[wib], s_list[wib], work, lane);
}

// Bricks with more candidates than the largest slice (extreme clustering): one warp per brick walks the candidates in
// ascending particle index by repeated selection of the next key, O(C^2 / 32), and folds each into its grid points.  A lane holds
// the accumulators of two points per sub-box for F::SELECT_BOXES sub-boxes at a time; with fewer than 8 the walk is repeated per
// group of sub-boxes.
template <class F>
__global__ void __launch_bounds__(32)
k_fold_select(SsDev P, SsAnArgs A) {
    constexpr int NB = F::SELECT_BOXES;
    static_assert(8 % NB == 0, "the sub-boxes of a brick split into equal groups");
    if (blockIdx.x >= A.n_bricks) return;
    const int lane = threadIdx.x & 31;
    const SsAnBrick N = ss_an_brick(P, A, A.bricks[blockIdx.x]);
    const SsSubLane L = ss_sub_lane(P, lane);
#pragma unroll 1
    for (int b0 = 0; b0 < 8; b0 += NB) {
        typename F::Acc acc[2 * NB];
#pragma unroll
        for (int q = 0; q < 2 * NB; ++q) acc[q] = F::zero();
        unsigned long long last = 0;
        bool first = true;
        for (;;) {
            const unsigned long long best = ss_select_next(P, A.bins, N.T.s, N.K, last, first, lane);
            if (best == ~0ull) break;
            last = best; first = false;
            const typename F::Cand cd = F::load(A, (uint32_t)best);
#pragma unroll
            for (int b = 0; b < NB; ++b) {
                const SsSubBox X = ss_sub_box(P, N.T, N.B.bx, N.B.by, N.B.bz, b0 + b, L, true);
                F::add(P, cd, X.gx, X.gy, X.gzA, acc[2 * b]);
                F::add(P, cd, X.gx, X.gy, X.gzB, acc[2 * b + 1]);
            }
        }
        float *const tile = A.tiles + (size_t)N.B.tile * P.np * P.np * P.np;
#pragma unroll
        for (int b = 0; b < NB; ++b) {
            const SsSubBox X = ss_sub_box(P, N.T, N.B.bx, N.B.by, N.B.bz, b0 + b, L, true);
            if (X.vA) tile[((size_t)X.i * P.np + X.j) * P.np + X.k] = F::value(P, acc[2 * b]);
            if (X.vB) tile[((size_t)X.i * P.np + X.j) * P.np + X.k + 1] = F::value(P, acc[2 * b + 1]);
        }
    }
}
