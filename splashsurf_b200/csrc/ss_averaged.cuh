// ss_averaged.cuh -- averaged-position surface (Y. Zhu and R. Bridson, "Animating Sand as a Fluid", ACM TOG 24(3), 2005), the
// opt-in mode of ss_context_set_averaged_surface_f32.  DESIGN.md §12 is the specification; tests/averaged_oracle.c restates it in
// plain C in the same operation order, so results are bit-exact.
//
// At a grid point g, with d_j = x_j - g over the particles with |d_j|^2 < h^2 in ascending index and w_j = (1 - |d_j|^2 / h^2)^3:
//     f(g) = h - |sum_j w_j d_j / sum_j w_j|      (= h - |g - x_bar(g)|),   f = 0 without candidates or when the weights sum to 0
// and the surface is f = h - R_s.  Offsets are taken from the grid point, so the sums keep their precision far from the origin.  The
// norm is taken of the averaged offset, whose components are of the order of h: the raw sums carry the weights (down to 2^-72 for a
// candidate at the edge of the support) and their squares would underflow to 0, reading f = h (inside) at such a point.
// The level set runs through the warp-per-brick cascade of ss_aniso.cuh (k_fold_levelset, k_fold_select) on the standard splat
// records: the kernel centres are the particle positions, so the bins, candidate ranges and margins are the standard ones.
#pragma once

struct SsAvgFold {
    static constexpr int SELECT_BOXES = 8;
    struct Cand { float4 r; };
    struct Acc { float s, x, y, z; };
    static __device__ __forceinline__ Cand load(const SsAnArgs &A, uint32_t src) { return Cand{ A.bins.rec[src] }; }
    static __device__ __forceinline__ Acc zero() { return Acc{ 0.0f, 0.0f, 0.0f, 0.0f }; }
    static __device__ __forceinline__ void add(const SsDev &P, const Cand &c, float gx, float gy, float gz, Acc &a) {
        const float dx = __fsub_rn(c.r.x, gx), dy = __fsub_rn(c.r.y, gy), dz = __fsub_rn(c.r.z, gz);
        const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
        if (!(d2 < P.h2)) return;
        const float u = __fsub_rn(1.0f, __fdiv_rn(d2, P.h2));
        const float w = __fmul_rn(__fmul_rn(u, u), u);
        a.s = __fadd_rn(a.s, w);
        a.x = __fadd_rn(a.x, __fmul_rn(w, dx)); a.y = __fadd_rn(a.y, __fmul_rn(w, dy)); a.z = __fadd_rn(a.z, __fmul_rn(w, dz));
    }
    static __device__ __forceinline__ float value(const SsDev &P, const Acc &a) {
        if (!(a.s > 0.0f)) return 0.0f;
        const float mx = __fdiv_rn(a.x, a.s), my = __fdiv_rn(a.y, a.s), mz = __fdiv_rn(a.z, a.s);
        const float m2 = __fadd_rn(__fadd_rn(__fmul_rn(mx, mx), __fmul_rn(my, my)), __fmul_rn(mz, mz));
        return __fsub_rn(P.h, __fsqrt_rn(m2));
    }
};

// Jacobian correction of the averaged-position surface (B. Solenthaler, J. Schläfli and R. Pajarola, "A unified particle model for
// fluid-solid interactions", Computer Animation and Virtual Worlds 18(1), 2007), the opt-in of ss_context_set_averaged_correction_f32;
// DESIGN.md §12.1.  With u_j = 1 - d2_j / h2, besides SsAvgFold's sums S, X, Y, Z (same order, so x_bar is bit-identical):
//     T_b = sum_j u_j^2 d_jb,   M_ab = sum_j u_j^2 d_ja d_jb   (a <= b)
// J = grad_g x_bar = (6 / h^2) (M / S - m (T / S)^T) with m = (X, Y, Z) / S.  EV, the largest eigenvalue of the symmetric part of J
// (cyclic Jacobi, add / sub / mul / div / sqrt only), sets f in [0, 1] (1 for EV <= t_low, 0 for EV >= t_high), and the tile value
//     v = (h - |m|) - R_s (1 - f)
// puts the surface (v = h - R_s) where |m| = f R_s: the radius shrinks where the average is pulled between particle groups.
struct SsAvgCorrFold {
    static constexpr int SELECT_BOXES = 2;          // 13 accumulators per point: k_fold_select holds 4 points per lane, not 16
    using Cand = SsAvgFold::Cand;
    struct Acc { SsAvgFold::Acc a; float tx, ty, tz, mxx, mxy, mxz, myy, myz, mzz; };
    static __device__ __forceinline__ Cand load(const SsAnArgs &A, uint32_t src) { return SsAvgFold::load(A, src); }
    static __device__ __forceinline__ Acc zero() { return Acc{ SsAvgFold::zero(), 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f }; }
    static __device__ __forceinline__ void add(const SsDev &P, const Cand &c, float gx, float gy, float gz, Acc &a) {
        const float dx = __fsub_rn(c.r.x, gx), dy = __fsub_rn(c.r.y, gy), dz = __fsub_rn(c.r.z, gz);
        const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
        if (!(d2 < P.h2)) return;
        SsAvgFold::add(P, c, gx, gy, gz, a.a);
        const float u = __fsub_rn(1.0f, __fdiv_rn(d2, P.h2));
        const float uu = __fmul_rn(u, u);
        const float ex = __fmul_rn(uu, dx), ey = __fmul_rn(uu, dy), ez = __fmul_rn(uu, dz);
        a.tx = __fadd_rn(a.tx, ex); a.ty = __fadd_rn(a.ty, ey); a.tz = __fadd_rn(a.tz, ez);
        a.mxx = __fadd_rn(a.mxx, __fmul_rn(ex, dx)); a.mxy = __fadd_rn(a.mxy, __fmul_rn(ex, dy)); a.mxz = __fadd_rn(a.mxz, __fmul_rn(ex, dz));
        a.myy = __fadd_rn(a.myy, __fmul_rn(ey, dy)); a.myz = __fadd_rn(a.myz, __fmul_rn(ey, dz)); a.mzz = __fadd_rn(a.mzz, __fmul_rn(ez, dz));
    }
    static __device__ __forceinline__ float value(const SsDev &P, const Acc &a) {
        const float s = a.a.s;
        if (!(s > 0.0f)) return 0.0f;
        const float m[3] = { __fdiv_rn(a.a.x, s), __fdiv_rn(a.a.y, s), __fdiv_rn(a.a.z, s) };
        const float m2 = __fadd_rn(__fadd_rn(__fmul_rn(m[0], m[0]), __fmul_rn(m[1], m[1])), __fmul_rn(m[2], m[2]));
        const float plain = __fsub_rn(P.h, __fsqrt_rn(m2));           // SsAvgFold::value
        return __fsub_rn(plain, __fmul_rn(P.av_rs, __fsub_rn(1.0f, factor(P, a, m))));
    }
    // f of a point with S > 0 and averaged offset m = (X, Y, Z) / S (shared with SsAvgCorrRadFold)
    static __device__ __forceinline__ float factor(const SsDev &P, const Acc &a, const float (&m)[3]) {
        const float s = a.a.s;
        const float t[3] = { __fdiv_rn(a.tx, s), __fdiv_rn(a.ty, s), __fdiv_rn(a.tz, s) };
        const float q[3][3] = { { __fdiv_rn(a.mxx, s), __fdiv_rn(a.mxy, s), __fdiv_rn(a.mxz, s) },
                                { 0.0f, __fdiv_rn(a.myy, s), __fdiv_rn(a.myz, s) },
                                { 0.0f, 0.0f, __fdiv_rn(a.mzz, s) } };
        // symmetric part of J' = M / S - m t^T (J = (6 / h^2) J'): A_ab = 0.5 ((q_ab - m_a t_b) + (q_ab - m_b t_a))
        float A[3][3], v[3][3] = {};
#pragma unroll
        for (int i = 0; i < 3; ++i) {
#pragma unroll
            for (int j = i; j < 3; ++j) {
                A[i][j] = __fmul_rn(0.5f, __fadd_rn(__fsub_rn(q[i][j], __fmul_rn(m[i], t[j])), __fsub_rn(q[i][j], __fmul_rn(m[j], t[i]))));
                A[j][i] = A[i][j];
            }
        }
#pragma unroll
        for (int sweep = 0; sweep < SS_AN_SWEEPS; ++sweep) {           // eigenvalues only: v is never read
            ss_jacobi_rot<0, 1>(A, v);
            ss_jacobi_rot<0, 2>(A, v);
            ss_jacobi_rot<1, 2>(A, v);
        }
        float e = A[0][0];
        if (A[1][1] > e) e = A[1][1];
        if (A[2][2] > e) e = A[2][2];
        const float ev = __fmul_rn(__fdiv_rn(6.0f, P.h2), e);
        float g = __fdiv_rn(__fsub_rn(P.av_high, ev), __fsub_rn(P.av_high, P.av_low));
        g = g > 0.0f ? (g < 1.0f ? g : 1.0f) : 0.0f;                  // a NaN EV gives f = 0
        const float f = __fmul_rn(__fadd_rn(__fmul_rn(__fsub_rn(g, 3.0f), g), 3.0f), g);
        return f < 1.0f ? f : 1.0f;                                    // rounding gives 1 + 2^-23 for some gamma < 1
    }
};

// Per-particle radii of the averaged-position surface (Zhu & Bridson's r_bar), the opt-in of ss_context_set_averaged_radii_f32;
// DESIGN.md §12.2.  Each record carries delta_j = R_j - R_s (R_j = radius_factor * r_j) in the side array SsAnArgs::rrec, at the
// record's index; with the same weight w_j as S, X, Y, Z one more sum Q = sum_j w_j delta_j gives b = Q / S, r_bar = R_s + b and
//     plain:      v = (h - |m|) + b                      (inside where |m| < r_bar)
//     corrected:  v = ((h - |m|) + b) - (R_s + b) (1 - f)   (inside where |m| < f r_bar)
// against the unchanged threshold h - R_s.  Every delta_j = +0 gives Q = b = +0, and the values of SsAvgFold / SsAvgCorrFold bit
// for bit.  The folds compose those two: the candidates, their order and the other sums are theirs.
struct SsAvgRadFold {
    static constexpr int SELECT_BOXES = 4;          // 5 accumulators per point: k_fold_select holds 8 points per lane
    struct Cand { SsAvgFold::Cand c; float delta; };
    struct Acc { SsAvgFold::Acc a; float q; };
    static __device__ __forceinline__ Cand load(const SsAnArgs &A, uint32_t src) { return Cand{ SsAvgFold::load(A, src), A.rrec[src] }; }
    static __device__ __forceinline__ Acc zero() { return Acc{ SsAvgFold::zero(), 0.0f }; }
    // w_j delta_j added to q when the candidate is within the support (the weight of SsAvgFold::add)
    static __device__ __forceinline__ void add_q(const SsDev &P, const Cand &c, float gx, float gy, float gz, float &q) {
        const float dx = __fsub_rn(c.c.r.x, gx), dy = __fsub_rn(c.c.r.y, gy), dz = __fsub_rn(c.c.r.z, gz);
        const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
        if (!(d2 < P.h2)) return;
        const float u = __fsub_rn(1.0f, __fdiv_rn(d2, P.h2));
        const float w = __fmul_rn(__fmul_rn(u, u), u);
        q = __fadd_rn(q, __fmul_rn(w, c.delta));
    }
    static __device__ __forceinline__ void add(const SsDev &P, const Cand &c, float gx, float gy, float gz, Acc &a) {
        SsAvgFold::add(P, c.c, gx, gy, gz, a.a);
        add_q(P, c, gx, gy, gz, a.q);
    }
    static __device__ __forceinline__ float value(const SsDev &P, const Acc &a) {
        if (!(a.a.s > 0.0f)) return 0.0f;
        return __fadd_rn(SsAvgFold::value(P, a.a), __fdiv_rn(a.q, a.a.s));
    }
};

struct SsAvgCorrRadFold {
    static constexpr int SELECT_BOXES = 2;          // 14 accumulators per point: k_fold_select holds 4 points per lane
    using Cand = SsAvgRadFold::Cand;
    struct Acc { SsAvgCorrFold::Acc a; float q; };
    static __device__ __forceinline__ Cand load(const SsAnArgs &A, uint32_t src) { return SsAvgRadFold::load(A, src); }
    static __device__ __forceinline__ Acc zero() { return Acc{ SsAvgCorrFold::zero(), 0.0f }; }
    static __device__ __forceinline__ void add(const SsDev &P, const Cand &c, float gx, float gy, float gz, Acc &a) {
        SsAvgCorrFold::add(P, c.c, gx, gy, gz, a.a);
        SsAvgRadFold::add_q(P, c, gx, gy, gz, a.q);
    }
    static __device__ __forceinline__ float value(const SsDev &P, const Acc &a) {
        const float s = a.a.a.s;
        if (!(s > 0.0f)) return 0.0f;
        const float m[3] = { __fdiv_rn(a.a.a.x, s), __fdiv_rn(a.a.a.y, s), __fdiv_rn(a.a.a.z, s) };
        const float b = __fdiv_rn(a.q, s);
        const float f = SsAvgCorrFold::factor(P, a.a, m);
        return __fsub_rn(__fadd_rn(SsAvgFold::value(P, a.a.a), b), __fmul_rn(__fadd_rn(P.av_rs, b), __fsub_rn(1.0f, f)));
    }
};

// ------------------------------------------------------------------ per-particle radii (DESIGN.md §12.2) ----
// Validation of the n input radii (all of them, before the particle-AABB filter): R_j = radius_factor * r_j must be finite with
// 0 < R_j < h.  chk[0] counts the invalid radii, chk[1] receives the lowest invalid index (preset to 0 and 0xffffffff).
__global__ void k_radii_check(const float *__restrict__ radii, uint64_t n, float factor, float h, uint32_t *__restrict__ chk) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float R = __fmul_rn(factor, radii[i]);
    if (R > 0.0f && R < h) return;                      // NaN and +-inf fail both comparisons or the second
    atomicAdd(&chk[0], 1u);
    atomicMin(&chk[1], (uint32_t)i);
}

// delta_j = R_j - R_s of the particles the particle-AABB filter keeps, compacted with the filter's flags and offsets (those of
// k_filter_scatter, so that delta is indexed like the filtered positions); flag == NULL: no filter, delta_j for every particle.
__global__ void k_radii_delta(const float *__restrict__ radii, uint64_t n, const uint8_t *__restrict__ flag, const uint32_t *__restrict__ off,
                              float factor, float rs, float *__restrict__ delta) {
    const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= n || (flag && !flag[i])) return;
    delta[flag ? off[i] : i] = __fsub_rn(__fmul_rn(factor, radii[i]), rs);
}

// After k_records: the side array of SsAvgRadFold / SsAvgCorrRadFold, delta of every binned membership in bin order.
__global__ void k_records_radius(uint32_t m, const uint32_t *__restrict__ key, const uint32_t *__restrict__ pidx, const float *__restrict__ delta,
                                 float *__restrict__ out) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= m || key[e] == 0xffffffffu) return;
    out[e] = delta[pidx[e]];
}
