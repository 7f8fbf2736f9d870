// ss_field.cuh -- the level set of a reconstruction at arbitrary points (ss_levelset_field_*_f32, DESIGN.md §13).
//
// The value at a point p is the tile formula of the context's level set with p in place of the grid point: the same candidates
// (every record whose support reaches p), the same operations, ascending particle index.  The standard level set folds with
// SsSphFold below (the scalar formula of ss_accumulate<SPARSE = true>, the one of sparse subdomains and simd = off); the opt-in modes
// with their brick folds unchanged (SsAnisoFold, ss_aniso.cuh; SsAvgFold, SsAvgCorrFold, SsAvgRadFold, SsAvgCorrRadFold,
// ss_averaged.cuh).  Points no candidate reaches are 0.
//
//   k_field_keys      per point: group key (compressed subdomain, brick of its cell; ss_field_key, which the ray march of
//                     ss_raycast.cuh shares), or value 0 at once (outside the grid, subdomain without members); the first non-finite
//                     coordinate
//   k_field_starts    after the key sort: first point of every group
//   k_field_fold      warp per (subdomain, brick) group: the candidates of the group's bins staged and sorted as for a brick
//                     (ss_stage_candidates), then per batch of 32 points the candidates within h of the batch's bounding box
//                     (ballot compaction) folded by each lane for its point in index order, scattered to the caller's order; groups
//                     with more candidates than the slice go to a 4096-slot instantiation, beyond that to k_field_select
//   k_field_select    per batch of 32 points the selection walk of k_fold_select (ss_select_next)
// A group's candidate bins cover the cells [8b - R, 8b + 8 + R) along each axis (ss_pipeline.cu: upload_field_brick_ranges): a point lies
// anywhere in the closed cell box [8b, 8b + 8]^3 of its brick, one cell further than the brick's grid points reach.
// ss_levelset_field_gradient_at_f32 runs the same sequence with the gradient folds below (SsSphGradFold, SsAnisoGradFold,
// SsAvgGradFold, SsAvgRadGradFold), which k_field_fold and k_field_select recognise at compile time and also write the gradient for;
// ss_levelset_field_hessian_at_f32 likewise with the Hessian folds (SsSphHessFold, SsAnisoHessFold, SsAvgHessFold, SsAvgRadHessFold),
// and ss_levelset_field_curvature_at_f32 turns their gradients and Hessians into curvatures (k_field_curvature).
#pragma once
#include <type_traits>

#define SS_FLD_WARPS 4                  // groups per CTA of the default slice

// the fold of a field: the context's level set when the field was created
enum { SS_FLD_SPH = 0, SS_FLD_ANISO = 1, SS_FLD_AVG = 2, SS_FLD_AVG_CORR = 3, SS_FLD_AVG_RAD = 4, SS_FLD_AVG_CORR_RAD = 5 };

// phi(p) = sum_j V_j W(|x_j - p|) with the level set's scalar arithmetic (ss_accumulate<SPARSE = true>, dense_subdomains.rs:828-842):
// candidates with d2 < 1.01 h^2 are added, the kernel is 0 beyond h, so the support lies within h as the sub-box cull requires.
struct SsSphFold {
    static constexpr int SELECT_BOXES = 8;
    struct Cand { float4 r; };
    struct Acc { float phi; };
    static __device__ __forceinline__ Cand load(const SsAnArgs &A, uint32_t src) { return Cand{ A.bins.rec[src] }; }
    static __device__ __forceinline__ Acc zero() { return Acc{ 0.0f }; }
    static __device__ __forceinline__ void add(const SsDev &P, const Cand &c, float gx, float gy, float gz, Acc &a) {
        const float dx = __fsub_rn(c.r.x, gx), dy = __fsub_rn(c.r.y, gy), dz = __fsub_rn(c.r.z, gz);
        const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
        if (d2 < P.h2m) a.phi = __fadd_rn(a.phi, __fmul_rn(c.r.w, ss_kernel_scalar(P, __fsqrt_rn(d2))));
    }
    static __device__ __forceinline__ float value(const SsDev &, const Acc &a) { return a.phi; }
};

// ------------------------------------------------------------------ gradients (DESIGN.md §13.1) ----
// The gradient of the value at the query point p, d_j = x_j - p.  A gradient fold wraps its value fold: its Acc holds the value
// fold's Acc, its add calls the value fold's add first, and its value is the value fold's, so the value returned beside the gradient
// is bit-identical to the one of ss_levelset_field_at_f32.  It adds
//   void     F::gradient(P, acc, g)     the gradient (0 where no candidate reaches p)
// which k_field_fold / k_field_select write to SsFieldArgs::grad.  The corrected modes have no gradient fold (DESIGN.md §13.1).
template <class F, class = void> struct SsFoldHasGradient : std::false_type {};
template <class F> struct SsFoldHasGradient<F, std::void_t<decltype(&F::gradient)>> : std::true_type {};

// W'(r) of ss_kernel_scalar from the same constants: q = 2r / h, W' = sigma f'(q) (2 / h) with f' = c_inner q (1.5 q - 2) below 1,
// -3 c_outer (2 - q)^2 below 2, 0 beyond (continuous at q = 1 and 2, 0 at q = 0)
__device__ __forceinline__ float ss_kernel_scalar_dr(const SsDev &P, float r) {
    const float q = __fdiv_rn(__fadd_rn(r, r), P.h);
    float f;
    if (q < 1.0f) f = __fmul_rn(P.s_c_inner, __fmul_rn(q, __fsub_rn(__fmul_rn(1.5f, q), 2.0f)));
    else if (q < 2.0f) { const float x = __fsub_rn(2.0f, q); f = __fmul_rn(__fmul_rn(__fmul_rn(-3.0f, P.s_c_outer), x), x); }
    else f = 0.0f;
    return __fmul_rn(__fmul_rn(P.s_sigma, f), __fdiv_rn(2.0f, P.h));
}

// grad phi = -sum_j V_j W'(r) d_j / r over SsSphFold's candidates (d2 < 1.01 h^2); d2 == 0 is skipped (W'(0) = 0)
struct SsSphGradFold {
    using Cand = SsSphFold::Cand;
    struct Acc { SsSphFold::Acc v; float gx, gy, gz; };
    static __device__ __forceinline__ Cand load(const SsAnArgs &A, uint32_t src) { return SsSphFold::load(A, src); }
    static __device__ __forceinline__ Acc zero() { return Acc{ SsSphFold::zero(), 0.0f, 0.0f, 0.0f }; }
    static __device__ __forceinline__ void add(const SsDev &P, const Cand &c, float gx, float gy, float gz, Acc &a) {
        SsSphFold::add(P, c, gx, gy, gz, a.v);
        const float dx = __fsub_rn(c.r.x, gx), dy = __fsub_rn(c.r.y, gy), dz = __fsub_rn(c.r.z, gz);
        const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
        if (!(d2 < P.h2m) || d2 == 0.0f) return;
        const float r = __fsqrt_rn(d2);
        const float t = __fdiv_rn(__fmul_rn(c.r.w, ss_kernel_scalar_dr(P, r)), r);
        a.gx = __fsub_rn(a.gx, __fmul_rn(t, dx)); a.gy = __fsub_rn(a.gy, __fmul_rn(t, dy)); a.gz = __fsub_rn(a.gz, __fmul_rn(t, dz));
    }
    static __device__ __forceinline__ float value(const SsDev &P, const Acc &a) { return SsSphFold::value(P, a.v); }
    static __device__ __forceinline__ void gradient(const SsDev &, const Acc &a, float (&g)[3]) { g[0] = a.gx; g[1] = a.gy; g[2] = a.gz; }
};

// grad phi = -sum_j (V_j det G_j) W'(|u_j|) (G_j u_j) / |u_j|, u_j = G_j d_j as in ss_aniso_term (G symmetric); |u| == 0 is skipped
struct SsAnisoGradFold {
    using Cand = SsAnisoFold::Cand;
    struct Acc { SsAnisoFold::Acc v; float gx, gy, gz; };
    static __device__ __forceinline__ Cand load(const SsAnArgs &A, uint32_t src) { return SsAnisoFold::load(A, src); }
    static __device__ __forceinline__ Acc zero() { return Acc{ SsAnisoFold::zero(), 0.0f, 0.0f, 0.0f }; }
    static __device__ __forceinline__ void add(const SsDev &P, const Cand &c, float gx, float gy, float gz, Acc &a) {
        SsAnisoFold::add(P, c, gx, gy, gz, a.v);
        const float4 g0 = c.g0, g1 = c.g1;
        const float dx = __fsub_rn(c.r.x, gx), dy = __fsub_rn(c.r.y, gy), dz = __fsub_rn(c.r.z, gz);
        const float u0 = __fadd_rn(__fadd_rn(__fmul_rn(g0.x, dx), __fmul_rn(g0.y, dy)), __fmul_rn(g0.z, dz));
        const float u1 = __fadd_rn(__fadd_rn(__fmul_rn(g0.y, dx), __fmul_rn(g0.w, dy)), __fmul_rn(g1.x, dz));
        const float u2 = __fadd_rn(__fadd_rn(__fmul_rn(g0.z, dx), __fmul_rn(g1.x, dy)), __fmul_rn(g1.y, dz));
        const float uu = __fadd_rn(__fadd_rn(__fmul_rn(u0, u0), __fmul_rn(u1, u1)), __fmul_rn(u2, u2));
        if (!(uu < P.h2) || uu == 0.0f) return;
        const float r = __fsqrt_rn(uu);
        const float t = __fdiv_rn(__fmul_rn(c.r.w, ss_kernel_scalar_dr(P, r)), r);
        const float v0 = __fadd_rn(__fadd_rn(__fmul_rn(g0.x, u0), __fmul_rn(g0.y, u1)), __fmul_rn(g0.z, u2));
        const float v1 = __fadd_rn(__fadd_rn(__fmul_rn(g0.y, u0), __fmul_rn(g0.w, u1)), __fmul_rn(g1.x, u2));
        const float v2 = __fadd_rn(__fadd_rn(__fmul_rn(g0.z, u0), __fmul_rn(g1.x, u1)), __fmul_rn(g1.y, u2));
        a.gx = __fsub_rn(a.gx, __fmul_rn(t, v0)); a.gy = __fsub_rn(a.gy, __fmul_rn(t, v1)); a.gz = __fsub_rn(a.gz, __fmul_rn(t, v2));
    }
    static __device__ __forceinline__ float value(const SsDev &P, const Acc &a) { return SsAnisoFold::value(P, a.v); }
    static __device__ __forceinline__ void gradient(const SsDev &, const Acc &a, float (&g)[3]) { g[0] = a.gx; g[1] = a.gy; g[2] = a.gz; }
};

// f = h - |m|, m = X / S: grad f = (m - (6 / h^2) (M m - |m|^2 T) / S) / |m| = (I - J)^T m / |m| with §12.1's sums, which
// SsAvgCorrFold::add accumulates (S, X, Y, Z first, through SsAvgFold::add); 0 where !(S > 0) or |m| == 0.  g gets grad f; the
// return value is |m| (0 when g is the zero vector).
struct SsAvgGradFold {
    using Cand = SsAvgFold::Cand;
    using Acc = SsAvgCorrFold::Acc;                 // .a: SsAvgFold::Acc
    static __device__ __forceinline__ Cand load(const SsAnArgs &A, uint32_t src) { return SsAvgFold::load(A, src); }
    static __device__ __forceinline__ Acc zero() { return SsAvgCorrFold::zero(); }
    static __device__ __forceinline__ void add(const SsDev &P, const Cand &c, float gx, float gy, float gz, Acc &a) {
        SsAvgCorrFold::add(P, c, gx, gy, gz, a);
    }
    static __device__ __forceinline__ float value(const SsDev &P, const Acc &a) { return SsAvgFold::value(P, a.a); }
    static __device__ __forceinline__ float grad_f(const SsDev &P, const Acc &a, float (&g)[3]) {
        g[0] = 0.0f; g[1] = 0.0f; g[2] = 0.0f;
        const float s = a.a.s;
        if (!(s > 0.0f)) return 0.0f;
        const float m[3] = { __fdiv_rn(a.a.x, s), __fdiv_rn(a.a.y, s), __fdiv_rn(a.a.z, s) };
        const float m2 = __fadd_rn(__fadd_rn(__fmul_rn(m[0], m[0]), __fmul_rn(m[1], m[1])), __fmul_rn(m[2], m[2]));
        const float nm = __fsqrt_rn(m2);
        if (nm == 0.0f) return 0.0f;
        const float k = __fdiv_rn(6.0f, P.h2);
        const float M[3][3] = { { a.mxx, a.mxy, a.mxz }, { a.mxy, a.myy, a.myz }, { a.mxz, a.myz, a.mzz } };
        const float T[3] = { a.tx, a.ty, a.tz };
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            const float mm = __fadd_rn(__fadd_rn(__fmul_rn(M[i][0], m[0]), __fmul_rn(M[i][1], m[1])), __fmul_rn(M[i][2], m[2]));
            const float jm = __fdiv_rn(__fmul_rn(k, __fsub_rn(mm, __fmul_rn(m2, T[i]))), s);
            g[i] = __fdiv_rn(__fsub_rn(m[i], jm), nm);
        }
        return nm;
    }
    static __device__ __forceinline__ void gradient(const SsDev &P, const Acc &a, float (&g)[3]) { grad_f(P, a, g); }
};

// With radii: v = (h - |m|) + b, b = Q / S; grad v = grad f + (6 / h^2) (U - b T) / S with U_b = sum_j u_j^2 delta_j d_jb.  Q is
// SsAvgRadFold::add_q's sum; the value is SsAvgRadFold::value of (S, X, Y, Z, Q).
struct SsAvgRadGradFold {
    using Cand = SsAvgRadFold::Cand;
    struct Acc { SsAvgGradFold::Acc a; float q, ux, uy, uz; };
    static __device__ __forceinline__ Cand load(const SsAnArgs &A, uint32_t src) { return SsAvgRadFold::load(A, src); }
    static __device__ __forceinline__ Acc zero() { return Acc{ SsAvgGradFold::zero(), 0.0f, 0.0f, 0.0f, 0.0f }; }
    static __device__ __forceinline__ void add(const SsDev &P, const Cand &c, float gx, float gy, float gz, Acc &a) {
        SsAvgGradFold::add(P, c.c, gx, gy, gz, a.a);
        SsAvgRadFold::add_q(P, c, gx, gy, gz, a.q);
        const float dx = __fsub_rn(c.c.r.x, gx), dy = __fsub_rn(c.c.r.y, gy), dz = __fsub_rn(c.c.r.z, gz);
        const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
        if (!(d2 < P.h2)) return;
        const float u = __fsub_rn(1.0f, __fdiv_rn(d2, P.h2));
        const float e = __fmul_rn(__fmul_rn(u, u), c.delta);
        a.ux = __fadd_rn(a.ux, __fmul_rn(e, dx)); a.uy = __fadd_rn(a.uy, __fmul_rn(e, dy)); a.uz = __fadd_rn(a.uz, __fmul_rn(e, dz));
    }
    static __device__ __forceinline__ float value(const SsDev &P, const Acc &a) { return SsAvgRadFold::value(P, SsAvgRadFold::Acc{ a.a.a, a.q }); }
    static __device__ __forceinline__ void gradient(const SsDev &P, const Acc &a, float (&g)[3]) {
        SsAvgGradFold::grad_f(P, a.a, g);
        const float s = a.a.a.s;
        if (!(s > 0.0f)) return;
        const float k = __fdiv_rn(6.0f, P.h2), b = __fdiv_rn(a.q, s);
        const float U[3] = { a.ux, a.uy, a.uz }, T[3] = { a.a.tx, a.a.ty, a.a.tz };
#pragma unroll
        for (int i = 0; i < 3; ++i) g[i] = __fadd_rn(g[i], __fdiv_rn(__fmul_rn(k, __fsub_rn(U[i], __fmul_rn(b, T[i]))), s));
    }
};

// ------------------------------------------------------------------ Hessians (DESIGN.md §13.2) ----
// The second derivative of the value at the query point p, six entries xx, xy, xz, yy, yz, zz.  A Hessian fold wraps its gradient
// fold as that wraps the value fold: its Acc holds the gradient fold's Acc, its add calls the gradient fold's add first, and its
// value and gradient are the gradient fold's, bit for bit.  It adds
//   void     F::hessian(P, acc, H)      the Hessian (0 where no candidate reaches p)
// which k_field_fold / k_field_select write to SsFieldArgs::hess.
template <class F, class = void> struct SsFoldHasHessian : std::false_type {};
template <class F> struct SsFoldHasHessian<F, std::void_t<decltype(&F::hessian)>> : std::true_type {};

// W'(r) / r and W''(r) of ss_kernel_scalar from the same constants, with s2 = (2 / h)^2: W' / r = sigma s2 f'(q) / q, f' / q =
// c_inner (1.5 q - 2) below 1 (no division: finite at r = 0), -3 c_outer (2 - q)^2 / q below 2; W'' = sigma s2 f''(q), f'' =
// c_inner (3 q - 2) below 1, 6 c_outer (2 - q) below 2 (continuous at q = 1 and 2); both 0 beyond
__device__ __forceinline__ void ss_kernel_scalar_d2(const SsDev &P, float r, float &w1r, float &w2) {
    const float q = __fdiv_rn(__fadd_rn(r, r), P.h);
    const float t = __fdiv_rn(2.0f, P.h), s2 = __fmul_rn(t, t);
    float f1q, f2;
    if (q < 1.0f) {
        f1q = __fmul_rn(P.s_c_inner, __fsub_rn(__fmul_rn(1.5f, q), 2.0f));
        f2 = __fmul_rn(P.s_c_inner, __fsub_rn(__fmul_rn(3.0f, q), 2.0f));
    } else if (q < 2.0f) {
        const float x = __fsub_rn(2.0f, q);
        f1q = __fdiv_rn(__fmul_rn(__fmul_rn(__fmul_rn(-3.0f, P.s_c_outer), x), x), q);
        f2 = __fmul_rn(__fmul_rn(6.0f, P.s_c_outer), x);
    } else { f1q = 0.0f; f2 = 0.0f; }
    w1r = __fmul_rn(__fmul_rn(P.s_sigma, f1q), s2);
    w2 = __fmul_rn(__fmul_rn(P.s_sigma, f2), s2);
}

// H += a v v^T + b K (K symmetric, entries xx xy xz yy yz zz): per entry t = (a v_i) v_j + b K_ij, then H_ij + t
__device__ __forceinline__ void ss_hess_rank1(float (&H)[6], float a, const float (&v)[3], float b, const float (&K)[6]) {
    const int I[6] = { 0, 0, 0, 1, 1, 2 }, J[6] = { 0, 1, 2, 1, 2, 2 };
#pragma unroll
    for (int e = 0; e < 6; ++e) H[e] = __fadd_rn(H[e], __fadd_rn(__fmul_rn(__fmul_rn(a, v[I[e]]), v[J[e]]), __fmul_rn(b, K[e])));
}

// H phi = sum_j V_j [ (W'' - W'/r) / r^2 d d^T + (W'/r) I ] over SsSphFold's candidates (d2 < 1.01 h^2); at d2 == 0 only the I term
struct SsSphHessFold {
    using Cand = SsSphFold::Cand;
    struct Acc { SsSphGradFold::Acc g; float H[6]; };
    static __device__ __forceinline__ Cand load(const SsAnArgs &A, uint32_t src) { return SsSphFold::load(A, src); }
    static __device__ __forceinline__ Acc zero() { return Acc{ SsSphGradFold::zero(), { 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f } }; }
    static __device__ __forceinline__ void add(const SsDev &P, const Cand &c, float gx, float gy, float gz, Acc &a) {
        SsSphGradFold::add(P, c, gx, gy, gz, a.g);
        const float d[3] = { __fsub_rn(c.r.x, gx), __fsub_rn(c.r.y, gy), __fsub_rn(c.r.z, gz) };
        const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(d[0], d[0]), __fmul_rn(d[1], d[1])), __fmul_rn(d[2], d[2]));
        if (!(d2 < P.h2m)) return;
        float w1r, w2;
        ss_kernel_scalar_d2(P, __fsqrt_rn(d2), w1r, w2);
        const float ra = d2 == 0.0f ? 0.0f : __fdiv_rn(__fmul_rn(c.r.w, __fsub_rn(w2, w1r)), d2);
        const float I6[6] = { 1.0f, 0.0f, 0.0f, 1.0f, 0.0f, 1.0f };
        ss_hess_rank1(a.H, ra, d, __fmul_rn(c.r.w, w1r), I6);
    }
    static __device__ __forceinline__ float value(const SsDev &P, const Acc &a) { return SsSphGradFold::value(P, a.g); }
    static __device__ __forceinline__ void gradient(const SsDev &P, const Acc &a, float (&g)[3]) { SsSphGradFold::gradient(P, a.g, g); }
    static __device__ __forceinline__ void hessian(const SsDev &, const Acc &a, float (&H)[6]) {
#pragma unroll
        for (int e = 0; e < 6; ++e) H[e] = a.H[e];
    }
};

// H phi = sum_j (V_j det G_j) [ (W'' - W'/|u|) / |u|^2 (G u)(G u)^T + (W'/|u|) G^2 ], u = G d as in SsAnisoGradFold; candidates
// |u|^2 < h^2, at |u| == 0 only the G^2 term
struct SsAnisoHessFold {
    using Cand = SsAnisoFold::Cand;
    struct Acc { SsAnisoGradFold::Acc g; float H[6]; };
    static __device__ __forceinline__ Cand load(const SsAnArgs &A, uint32_t src) { return SsAnisoFold::load(A, src); }
    static __device__ __forceinline__ Acc zero() { return Acc{ SsAnisoGradFold::zero(), { 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f } }; }
    static __device__ __forceinline__ void add(const SsDev &P, const Cand &c, float gx, float gy, float gz, Acc &a) {
        SsAnisoGradFold::add(P, c, gx, gy, gz, a.g);
        const float4 g0 = c.g0, g1 = c.g1;
        const float dx = __fsub_rn(c.r.x, gx), dy = __fsub_rn(c.r.y, gy), dz = __fsub_rn(c.r.z, gz);
        const float u0 = __fadd_rn(__fadd_rn(__fmul_rn(g0.x, dx), __fmul_rn(g0.y, dy)), __fmul_rn(g0.z, dz));
        const float u1 = __fadd_rn(__fadd_rn(__fmul_rn(g0.y, dx), __fmul_rn(g0.w, dy)), __fmul_rn(g1.x, dz));
        const float u2 = __fadd_rn(__fadd_rn(__fmul_rn(g0.z, dx), __fmul_rn(g1.x, dy)), __fmul_rn(g1.y, dz));
        const float uu = __fadd_rn(__fadd_rn(__fmul_rn(u0, u0), __fmul_rn(u1, u1)), __fmul_rn(u2, u2));
        if (!(uu < P.h2)) return;
        float w1r, w2;
        ss_kernel_scalar_d2(P, __fsqrt_rn(uu), w1r, w2);
        const float ra = uu == 0.0f ? 0.0f : __fdiv_rn(__fmul_rn(c.r.w, __fsub_rn(w2, w1r)), uu);
        const float v[3] = { __fadd_rn(__fadd_rn(__fmul_rn(g0.x, u0), __fmul_rn(g0.y, u1)), __fmul_rn(g0.z, u2)),
                             __fadd_rn(__fadd_rn(__fmul_rn(g0.y, u0), __fmul_rn(g0.w, u1)), __fmul_rn(g1.x, u2)),
                             __fadd_rn(__fadd_rn(__fmul_rn(g0.z, u0), __fmul_rn(g1.x, u1)), __fmul_rn(g1.y, u2)) };
        // G^2 = G G: ((G_i0 G_0j + G_i1 G_1j) + G_i2 G_2j)
        const float G[3][3] = { { g0.x, g0.y, g0.z }, { g0.y, g0.w, g1.x }, { g0.z, g1.x, g1.y } };
        const int I[6] = { 0, 0, 0, 1, 1, 2 }, J[6] = { 0, 1, 2, 1, 2, 2 };
        float K[6];
#pragma unroll
        for (int e = 0; e < 6; ++e)
            K[e] = __fadd_rn(__fadd_rn(__fmul_rn(G[I[e]][0], G[0][J[e]]), __fmul_rn(G[I[e]][1], G[1][J[e]])), __fmul_rn(G[I[e]][2], G[2][J[e]]));
        ss_hess_rank1(a.H, ra, v, __fmul_rn(c.r.w, w1r), K);
    }
    static __device__ __forceinline__ float value(const SsDev &P, const Acc &a) { return SsAnisoGradFold::value(P, a.g); }
    static __device__ __forceinline__ void gradient(const SsDev &P, const Acc &a, float (&g)[3]) { SsAnisoGradFold::gradient(P, a.g, g); }
    static __device__ __forceinline__ void hessian(const SsDev &, const Acc &a, float (&H)[6]) {
#pragma unroll
        for (int e = 0; e < 6; ++e) H[e] = a.H[e];
    }
};

// The sums the averaged Hessian adds to §12.1's, with b = 1 - |d|^2 / h^2 over |d|^2 < h^2: S2 = sum b^2, N = sum b d d^T (xx xy xz
// yy yz zz), O = sum b d (x) d (x) d (xxx xxy xxz xyy xyz xzz yyy yyz yzz zzz); per candidate e = b d, n_ab = e_a d_b, o_abc = n_ab d_c.
struct SsAvgHessSums { float s2, n[6], o[10]; };
__device__ __forceinline__ void ss_avg_hess_sums(const float (&d)[3], float u, SsAvgHessSums &e) {
    e.s2 = __fadd_rn(e.s2, __fmul_rn(u, u));
    const float ed[3] = { __fmul_rn(u, d[0]), __fmul_rn(u, d[1]), __fmul_rn(u, d[2]) };
    const float n[6] = { __fmul_rn(ed[0], d[0]), __fmul_rn(ed[0], d[1]), __fmul_rn(ed[0], d[2]),
                         __fmul_rn(ed[1], d[1]), __fmul_rn(ed[1], d[2]), __fmul_rn(ed[2], d[2]) };
#pragma unroll
    for (int i = 0; i < 6; ++i) e.n[i] = __fadd_rn(e.n[i], n[i]);
    const float o[10] = { __fmul_rn(n[0], d[0]), __fmul_rn(n[0], d[1]), __fmul_rn(n[0], d[2]), __fmul_rn(n[1], d[1]), __fmul_rn(n[1], d[2]),
                          __fmul_rn(n[2], d[2]), __fmul_rn(n[3], d[1]), __fmul_rn(n[3], d[2]), __fmul_rn(n[4], d[2]), __fmul_rn(n[5], d[2]) };
#pragma unroll
    for (int i = 0; i < 10; ++i) e.o[i] = __fadd_rn(e.o[i], o[i]);
}

// d, |d|^2 and b of a candidate of the averaged folds; false outside the support
__device__ __forceinline__ bool ss_avg_offset(const SsDev &P, float4 r, float gx, float gy, float gz, float (&d)[3], float &u) {
    d[0] = __fsub_rn(r.x, gx); d[1] = __fsub_rn(r.y, gy); d[2] = __fsub_rn(r.z, gz);
    const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(d[0], d[0]), __fmul_rn(d[1], d[1])), __fmul_rn(d[2], d[2]));
    if (!(d2 < P.h2)) return false;
    u = __fsub_rn(1.0f, __fdiv_rn(d2, P.h2));
    return true;
}

// f = h - |m|: H f = -sum_a mh_a H m_a - (I - J)^T (I - mh mh^T) (I - J) / |m|, mh = m / |m|, J = (k / S)(M - m T^T), k = 6 / h^2,
// which DESIGN.md §13.2 reduces to
//   H f = -(k / S) [ A + sig I - T c^T - c T^T ] - (B^T B - g g^T) / |m|
// with B = I - J, g = B^T mh = grad f (SsAvgGradFold::grad_f, bit for bit), c = J^T mh, A = (4 / h^2)(sum_a mh_a O_a.. - |m| N),
// sig = |m| S2 - mh . T.  0 where !(S > 0) or |m| == 0.
struct SsAvgHessFold {
    using Cand = SsAvgFold::Cand;
    struct Acc { SsAvgGradFold::Acc g; SsAvgHessSums e; };
    static __device__ __forceinline__ Cand load(const SsAnArgs &A, uint32_t src) { return SsAvgFold::load(A, src); }
    static __device__ __forceinline__ Acc zero() { return Acc{ SsAvgGradFold::zero(), SsAvgHessSums{} }; }
    static __device__ __forceinline__ void add(const SsDev &P, const Cand &c, float gx, float gy, float gz, Acc &a) {
        SsAvgGradFold::add(P, c, gx, gy, gz, a.g);
        float d[3], u;
        if (ss_avg_offset(P, c.r, gx, gy, gz, d, u)) ss_avg_hess_sums(d, u, a.e);
    }
    static __device__ __forceinline__ float value(const SsDev &P, const Acc &a) { return SsAvgGradFold::value(P, a.g); }
    static __device__ __forceinline__ void gradient(const SsDev &P, const Acc &a, float (&g)[3]) { SsAvgGradFold::gradient(P, a.g, g); }
    static __device__ __forceinline__ void hess_f(const SsDev &P, const SsAvgGradFold::Acc &a, const SsAvgHessSums &e, float (&H)[6]) {
#pragma unroll
        for (int i = 0; i < 6; ++i) H[i] = 0.0f;
        float g[3];
        const float nm = SsAvgGradFold::grad_f(P, a, g);
        if (nm == 0.0f) return;                              // also !(S > 0)
        const float s = a.a.s;
        const float m[3] = { __fdiv_rn(a.a.x, s), __fdiv_rn(a.a.y, s), __fdiv_rn(a.a.z, s) };
        const float mh[3] = { __fdiv_rn(m[0], nm), __fdiv_rn(m[1], nm), __fdiv_rn(m[2], nm) };
        const float k = __fdiv_rn(6.0f, P.h2), kh = __fdiv_rn(4.0f, P.h2);
        const float M[3][3] = { { a.mxx, a.mxy, a.mxz }, { a.mxy, a.myy, a.myz }, { a.mxz, a.myz, a.mzz } };
        const float T[3] = { a.tx, a.ty, a.tz };
        float J[3][3], B[3][3];
#pragma unroll
        for (int i = 0; i < 3; ++i) {
#pragma unroll
            for (int j = 0; j < 3; ++j) {
                J[i][j] = __fdiv_rn(__fmul_rn(k, __fsub_rn(M[i][j], __fmul_rn(m[i], T[j]))), s);
                B[i][j] = __fsub_rn(i == j ? 1.0f : 0.0f, J[i][j]);
            }
        }
        float cv[3];                                         // c = J^T mh
#pragma unroll
        for (int j = 0; j < 3; ++j) cv[j] = __fadd_rn(__fadd_rn(__fmul_rn(J[0][j], mh[0]), __fmul_rn(J[1][j], mh[1])), __fmul_rn(J[2][j], mh[2]));
        const float sig = __fsub_rn(__fmul_rn(nm, e.s2), __fadd_rn(__fadd_rn(__fmul_rn(mh[0], T[0]), __fmul_rn(mh[1], T[1])), __fmul_rn(mh[2], T[2])));
        // O_aij of the six (i, j) entries for a = x, y, z (indices into SsAvgHessSums::o)
        const int OX[6] = { 0, 1, 2, 3, 4, 5 }, OY[6] = { 1, 3, 4, 6, 7, 8 }, OZ[6] = { 2, 4, 5, 7, 8, 9 };
        const int I[6] = { 0, 0, 0, 1, 1, 2 }, Jx[6] = { 0, 1, 2, 1, 2, 2 };
#pragma unroll
        for (int q = 0; q < 6; ++q) {
            const int i = I[q], j = Jx[q];
            const float om = __fadd_rn(__fadd_rn(__fmul_rn(e.o[OX[q]], mh[0]), __fmul_rn(e.o[OY[q]], mh[1])), __fmul_rn(e.o[OZ[q]], mh[2]));
            float p = __fmul_rn(kh, __fsub_rn(om, __fmul_rn(nm, e.n[q])));
            if (i == j) p = __fadd_rn(p, sig);
            p = __fsub_rn(__fsub_rn(p, __fmul_rn(T[i], cv[j])), __fmul_rn(cv[i], T[j]));
            const float first = __fdiv_rn(__fmul_rn(k, p), s);
            const float bb = __fadd_rn(__fadd_rn(__fmul_rn(B[0][i], B[0][j]), __fmul_rn(B[1][i], B[1][j])), __fmul_rn(B[2][i], B[2][j]));
            const float second = __fdiv_rn(__fsub_rn(bb, __fmul_rn(g[i], g[j])), nm);
            H[q] = -__fadd_rn(first, second);
        }
    }
    static __device__ __forceinline__ void hessian(const SsDev &P, const Acc &a, float (&H)[6]) { hess_f(P, a.g, a.e, H); }
};

// With radii: v = f + R, R = Q / S: H v = H f + (k / S) [ (4 / h^2)(Nd - R N) + (R S2 - S2d) I - T r^T - r T^T ] with r = grad R =
// k (U - R T) / S (SsAvgRadGradFold's term), Nd = sum b delta d d^T, S2d = sum b^2 delta; the R part wherever S > 0.
struct SsAvgRadHessFold {
    using Cand = SsAvgRadFold::Cand;
    struct Acc { SsAvgRadGradFold::Acc g; SsAvgHessSums e; float s2d, nd[6]; };
    static __device__ __forceinline__ Cand load(const SsAnArgs &A, uint32_t src) { return SsAvgRadFold::load(A, src); }
    static __device__ __forceinline__ Acc zero() { return Acc{ SsAvgRadGradFold::zero(), SsAvgHessSums{}, 0.0f, { 0.0f, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f } }; }
    static __device__ __forceinline__ void add(const SsDev &P, const Cand &c, float gx, float gy, float gz, Acc &a) {
        SsAvgRadGradFold::add(P, c, gx, gy, gz, a.g);
        float d[3], u;
        if (!ss_avg_offset(P, c.c.r, gx, gy, gz, d, u)) return;
        ss_avg_hess_sums(d, u, a.e);
        const float ud = __fmul_rn(u, c.delta);
        a.s2d = __fadd_rn(a.s2d, __fmul_rn(u, ud));
        const float ed[3] = { __fmul_rn(ud, d[0]), __fmul_rn(ud, d[1]), __fmul_rn(ud, d[2]) };
        const int I[6] = { 0, 0, 0, 1, 1, 2 }, J[6] = { 0, 1, 2, 1, 2, 2 };
#pragma unroll
        for (int q = 0; q < 6; ++q) a.nd[q] = __fadd_rn(a.nd[q], __fmul_rn(ed[I[q]], d[J[q]]));
    }
    static __device__ __forceinline__ float value(const SsDev &P, const Acc &a) { return SsAvgRadGradFold::value(P, a.g); }
    static __device__ __forceinline__ void gradient(const SsDev &P, const Acc &a, float (&g)[3]) { SsAvgRadGradFold::gradient(P, a.g, g); }
    static __device__ __forceinline__ void hessian(const SsDev &P, const Acc &a, float (&H)[6]) {
        SsAvgHessFold::hess_f(P, a.g.a, a.e, H);
        const float s = a.g.a.a.s;
        if (!(s > 0.0f)) return;
        const float k = __fdiv_rn(6.0f, P.h2), kh = __fdiv_rn(4.0f, P.h2), R = __fdiv_rn(a.g.q, s);
        const float U[3] = { a.g.ux, a.g.uy, a.g.uz }, T[3] = { a.g.a.tx, a.g.a.ty, a.g.a.tz };
        float r[3];
#pragma unroll
        for (int i = 0; i < 3; ++i) r[i] = __fdiv_rn(__fmul_rn(k, __fsub_rn(U[i], __fmul_rn(R, T[i]))), s);
        const float dg = __fsub_rn(__fmul_rn(R, a.e.s2), a.s2d);
        const int I[6] = { 0, 0, 0, 1, 1, 2 }, J[6] = { 0, 1, 2, 1, 2, 2 };
#pragma unroll
        for (int q = 0; q < 6; ++q) {
            const int i = I[q], j = J[q];
            float p = __fmul_rn(kh, __fsub_rn(a.nd[q], __fmul_rn(R, a.e.n[q])));
            if (i == j) p = __fadd_rn(p, dg);
            p = __fsub_rn(__fsub_rn(p, __fmul_rn(T[i], r[j])), __fmul_rn(r[i], T[j]));
            H[q] = __fadd_rn(H[q], __fdiv_rn(__fmul_rn(k, p), s));
        }
    }
};

// Curvature of the level set through p from g = grad phi and H (DESIGN.md §13.2): n = g / |g|, kappa_H = -(tr H - n^T H n) / (2 |g|)
// (half the divergence of the outward normal -g / |g|), kappa_G = n^T adj(H) n / |g|^2; both NaN where |g|^2 rounds to 0.
__device__ __forceinline__ void ss_curvature(const float (&g)[3], const float (&H)[6], float &kh, float &kg) {
    const float g2 = __fadd_rn(__fadd_rn(__fmul_rn(g[0], g[0]), __fmul_rn(g[1], g[1])), __fmul_rn(g[2], g[2]));
    if (g2 == 0.0f) { kh = __int_as_float(0x7fc00000); kg = kh; return; }
    const float ng = __fsqrt_rn(g2);
    const float n[3] = { __fdiv_rn(g[0], ng), __fdiv_rn(g[1], ng), __fdiv_rn(g[2], ng) };
    const float M[3][3] = { { H[0], H[1], H[2] }, { H[1], H[3], H[4] }, { H[2], H[4], H[5] } };
    // adj(H) of the symmetric H: cofactors, e.g. adj_xx = Hyy Hzz - Hyz Hyz, adj_xy = Hxz Hyz - Hxy Hzz
    const float A[3][3] = {
        { __fsub_rn(__fmul_rn(H[3], H[5]), __fmul_rn(H[4], H[4])), __fsub_rn(__fmul_rn(H[2], H[4]), __fmul_rn(H[1], H[5])),
          __fsub_rn(__fmul_rn(H[1], H[4]), __fmul_rn(H[2], H[3])) },
        { 0.0f, __fsub_rn(__fmul_rn(H[0], H[5]), __fmul_rn(H[2], H[2])), __fsub_rn(__fmul_rn(H[1], H[2]), __fmul_rn(H[0], H[4])) },
        { 0.0f, 0.0f, __fsub_rn(__fmul_rn(H[0], H[3]), __fmul_rn(H[1], H[1])) } };
    const float As[3][3] = { { A[0][0], A[0][1], A[0][2] }, { A[0][1], A[1][1], A[1][2] }, { A[0][2], A[1][2], A[2][2] } };
    float hn[3], an[3];
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        hn[i] = __fadd_rn(__fadd_rn(__fmul_rn(M[i][0], n[0]), __fmul_rn(M[i][1], n[1])), __fmul_rn(M[i][2], n[2]));
        an[i] = __fadd_rn(__fadd_rn(__fmul_rn(As[i][0], n[0]), __fmul_rn(As[i][1], n[1])), __fmul_rn(As[i][2], n[2]));
    }
    const float nHn = __fadd_rn(__fadd_rn(__fmul_rn(n[0], hn[0]), __fmul_rn(n[1], hn[1])), __fmul_rn(n[2], hn[2]));
    const float nAn = __fadd_rn(__fadd_rn(__fmul_rn(n[0], an[0]), __fmul_rn(n[1], an[1])), __fmul_rn(n[2], an[2]));
    const float tr = __fadd_rn(__fadd_rn(H[0], H[3]), H[5]);
    kh = -__fdiv_rn(__fsub_rn(tr, nHn), __fmul_rn(2.0f, ng));
    kg = __fdiv_rn(nAn, g2);
}

// (kappa_H, kappa_G) of m points from their gradients [m][3] and Hessians [m][6]
__global__ void k_field_curvature(const float *__restrict__ grad, const float *__restrict__ hess, uint32_t m, float *__restrict__ curv) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    const float g[3] = { grad[3 * (size_t)i], grad[3 * (size_t)i + 1], grad[3 * (size_t)i + 2] };
    float H[6];
#pragma unroll
    for (int e = 0; e < 6; ++e) H[e] = hess[6 * (size_t)i + e];
    float kh, kg;
    ss_curvature(g, H, kh, kg);
    curv[2 * (size_t)i] = kh; curv[2 * (size_t)i + 1] = kg;
}

struct SsFieldArgs {
    SsAnArgs A;                        // the mode's records (A.bins.brick_rng: the field's candidate ranges); bricks / tiles unused
    const float *pts;                  // [m][3] query points
    const uint32_t *key;               // sorted group keys: compressed subdomain * nb^3 + (bx * nb + by) * nb + bz
    const uint32_t *idx;               // caller's index of each sorted point
    const uint32_t *starts;            // [n_all + 1] first sorted point of each group, then the number of points inside a subdomain
    const uint32_t *groups;            // this launch's groups (NULL: 0 .. n_groups - 1)
    uint32_t n_groups;
    float *out;                        // [m] pre-zeroed
    uint32_t *fallback;                // groups left to the next tier: [0] = count, [1..] = group indices
    float *grad;                       // [m][3] pre-zeroed, written by gradient folds only
    float *hess;                       // [m][6] pre-zeroed, written by Hessian folds only
};

// the value of a point, and its gradient and Hessian when the fold has them
template <class F>
__device__ __forceinline__ void ss_field_store(const SsDev &P, const SsFieldArgs &Q, uint32_t dst, const typename F::Acc &acc) {
    Q.out[dst] = F::value(P, acc);
    if constexpr (SsFoldHasGradient<F>::value) {
        float g[3];
        F::gradient(P, acc, g);
        Q.grad[3 * (size_t)dst] = g[0]; Q.grad[3 * (size_t)dst + 1] = g[1]; Q.grad[3 * (size_t)dst + 2] = g[2];
    }
    if constexpr (SsFoldHasHessian<F>::value) {
        float H[6];
        F::hessian(P, acc, H);
#pragma unroll
        for (int e = 0; e < 6; ++e) Q.hess[6 * (size_t)dst + e] = H[e];
    }
}

// The cell of a point in the grid, clamped (a point on the grid's upper face belongs to the last cell); false outside [gmin, gmax]
// along an axis (gc then 0 from that axis on).  finite: whether every coordinate is finite.
__device__ __forceinline__ bool ss_field_cell(const SsDev &P, const float (&p)[3], float3 gmax, int (&gc)[3], bool &finite) {
    const float hi[3] = { gmax.x, gmax.y, gmax.z };
    bool inside = true;
    finite = true;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        finite = finite && isfinite(p[d]);
        inside = inside && p[d] >= P.gmin[d] && p[d] <= hi[d];
        gc[d] = inside ? min(max(ss_cell_of(p[d], P.gmin[d], P.c), 0), P.nsd[d] * P.S - 1) : 0;
    }
    return inside;
}

// The group key of a point (k_field_keys, ss_raycast.cuh): compressed subdomain * nb^3 + (bx * nb + by) * nb + bz of its cell, or
// 0xffffffff outside [gmin, gmax] along an axis, in a subdomain without members (sub_flat: the nsub subdomains with members,
// ascending) or at a non-finite coordinate.
__device__ __forceinline__ uint32_t ss_field_key(const SsDev &P, const float (&p)[3], float3 gmax, const uint32_t *__restrict__ sub_flat, uint32_t nsub,
                                                 bool &finite) {
    int gc[3];
    const bool inside = ss_field_cell(P, p, gmax, gc, finite);
    uint32_t k = 0xffffffffu;
    if (finite && inside) {
        int sd[3], lb[3];
#pragma unroll
        for (int d = 0; d < 3; ++d) { sd[d] = gc[d] / P.S; lb[d] = (gc[d] - sd[d] * P.S) >> 3; }
        const uint32_t flat = (uint32_t)(((int64_t)sd[0] * P.nsd[1] + sd[1]) * P.nsd[2] + sd[2]);
        uint32_t lo = 0, up = nsub;                             // sub_flat is ascending
        while (lo < up) { const uint32_t mid = (lo + up) >> 1; if (sub_flat[mid] < flat) lo = mid + 1; else up = mid; }
        if (lo < nsub && sub_flat[lo] == flat) k = lo * (uint32_t)(P.nb * P.nb * P.nb) + (uint32_t)((lb[0] * P.nb + lb[1]) * P.nb + lb[2]);
    }
    return k;
}

// Points outside [gmin, gmax] along an axis, or in a subdomain without members, get 0 and key 0xffffffff (sorted last); chk[0]:
// lowest index with a non-finite coordinate (preset 0xffffffff), chk[1]: points with a group (preset 0).
__global__ void k_field_keys(SsDev P, const float *__restrict__ pts, uint32_t m, float3 gmax, const uint32_t *__restrict__ sub_flat, uint32_t nsub,
                             uint32_t *__restrict__ key, uint32_t *__restrict__ idx, float *__restrict__ out, uint32_t *__restrict__ chk) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    bool grouped = false;
    if (i < m) {
        const float p[3] = { pts[3 * (size_t)i], pts[3 * (size_t)i + 1], pts[3 * (size_t)i + 2] };
        bool finite;
        const uint32_t k = ss_field_key(P, p, gmax, sub_flat, nsub, finite);
        if (!finite) atomicMin(&chk[0], i);
        grouped = k != 0xffffffffu;
        key[i] = k; idx[i] = i; out[i] = 0.0f;
    }
    const unsigned w = __ballot_sync(0xffffffffu, grouped);
    if ((threadIdx.x & 31) == 0 && w) atomicAdd(&chk[1], (uint32_t)__popc(w));
}

// flag[i] = 1 where sorted point i (< n) starts a group
__global__ void k_field_starts(const uint32_t *__restrict__ key, uint32_t n, uint32_t *__restrict__ flag) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) flag[i] = (i == 0 || key[i] != key[i - 1]) ? 1u : 0u;
}

// group g: compressed subdomain, candidate bins, sorted points [p0, p1)
struct SsFieldGroup { uint32_t s, p0, p1; SsBrickBins K; };
__device__ __forceinline__ SsFieldGroup ss_field_group(const SsDev &P, const SsFieldArgs &Q, uint32_t g) {
    SsFieldGroup G;
    G.p0 = Q.starts[g]; G.p1 = Q.starts[g + 1];
    const uint32_t nb3 = (uint32_t)(P.nb * P.nb * P.nb), k = Q.key[G.p0];
    G.s = k / nb3;
    const uint32_t b = k - G.s * nb3;
    G.K = ss_brick_bins(P, Q.A.bins.brick_rng, (int)(b / (uint32_t)(P.nb * P.nb)), (int)(b / (uint32_t)P.nb % (uint32_t)P.nb), (int)(b % (uint32_t)P.nb), false);
    return G;
}

// lane's point of the batch starting at sorted position q0: caller index and coordinates (on = false past the group's end)
struct SsFieldPoint { bool on; uint32_t dst; float x, y, z; };
__device__ __forceinline__ SsFieldPoint ss_field_point(const SsFieldArgs &Q, const SsFieldGroup &G, uint32_t q0, int lane) {
    SsFieldPoint p{ q0 + lane < G.p1, 0u, 0.0f, 0.0f, 0.0f };
    if (p.on) {
        p.dst = Q.idx[q0 + lane];
        p.x = Q.pts[3 * (size_t)p.dst]; p.y = Q.pts[3 * (size_t)p.dst + 1]; p.z = Q.pts[3 * (size_t)p.dst + 2];
    }
    return p;
}

template <class F, int CAP, int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
k_field_fold(SsDev P, SsFieldArgs Q) {
    __shared__ unsigned long long s_key[WARPS][CAP];
    __shared__ uint16_t s_list[WARPS][CAP];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t work = blockIdx.x * WARPS + wib;
    if (work >= Q.n_groups) return;
    const uint32_t g = Q.groups ? Q.groups[work] : work;
    const SsFieldGroup G = ss_field_group(P, Q, g);
    const uint32_t C = ss_stage_candidates<CAP>(P, Q.A.bins, G.s, G.K, s_key[wib], lane);
    if (C == 0) return;                                      // pre-zeroed: the value of a point without candidates is 0
    if (C > (uint32_t)CAP) {
        if (lane == 0) Q.fallback[1 + atomicAdd(&Q.fallback[0], 1u)] = g;
        return;
    }
    const float cull2 = P.h2 * 1.0001f;
    for (uint32_t q0 = G.p0; q0 < G.p1; q0 += 32) {
        const SsFieldPoint p = ss_field_point(Q, G, q0, lane);
        // the batch's bounding box (lanes past the end take lane 0's point, which is always on)
        const float x0 = __shfl_sync(0xffffffffu, p.x, 0), y0 = __shfl_sync(0xffffffffu, p.y, 0), z0 = __shfl_sync(0xffffffffu, p.z, 0);
        float xl = p.on ? p.x : x0, xh = xl, yl = p.on ? p.y : y0, yh = yl, zl = p.on ? p.z : z0, zh = zl;
        for (int o = 16; o > 0; o >>= 1) {
            xl = fminf(xl, __shfl_xor_sync(0xffffffffu, xl, o)); xh = fmaxf(xh, __shfl_xor_sync(0xffffffffu, xh, o));
            yl = fminf(yl, __shfl_xor_sync(0xffffffffu, yl, o)); yh = fmaxf(yh, __shfl_xor_sync(0xffffffffu, yh, o));
            zl = fminf(zl, __shfl_xor_sync(0xffffffffu, zl, o)); zh = fmaxf(zh, __shfl_xor_sync(0xffffffffu, zh, o));
        }
        int nlist = 0;
        for (int w = 0; w < (int)((C + 31) >> 5); ++w) {
            const int rnk = w * 32 + lane;
            bool keep = false;
            if (rnk < (int)C) {
                const float4 r = Q.A.bins.rec[(uint32_t)s_key[wib][rnk]];
                keep = ss_axis_d2(r.x, xl, xh) + ss_axis_d2(r.y, yl, yh) + ss_axis_d2(r.z, zl, zh) < cull2;
            }
            const uint32_t mword = __ballot_sync(0xffffffffu, keep);
            if (keep) s_list[wib][nlist + __popc(mword & ((1u << lane) - 1u))] = (uint16_t)rnk;
            nlist += __popc(mword);
        }
        __syncwarp();
        typename F::Acc acc = F::zero();
        for (int n = 0; n < nlist; ++n) F::add(P, F::load(Q.A, (uint32_t)s_key[wib][s_list[wib][n]]), p.x, p.y, p.z, acc);
        if (p.on) ss_field_store<F>(P, Q, p.dst, acc);
        __syncwarp();                                        // the list is rebuilt for the next batch
    }
}

// Groups with more candidates than the largest slice (extreme clustering): per batch of 32 points the candidates in ascending
// particle index by repeated selection, O(C^2 / 32) per batch.
template <class F>
__global__ void __launch_bounds__(32)
k_field_select(SsDev P, SsFieldArgs Q) {
    if (blockIdx.x >= Q.n_groups) return;
    const int lane = threadIdx.x & 31;
    const SsFieldGroup G = ss_field_group(P, Q, Q.groups ? Q.groups[blockIdx.x] : blockIdx.x);
    for (uint32_t q0 = G.p0; q0 < G.p1; q0 += 32) {
        const SsFieldPoint p = ss_field_point(Q, G, q0, lane);
        typename F::Acc acc = F::zero();
        unsigned long long last = 0;
        bool first = true;
        for (;;) {
            const unsigned long long best = ss_select_next(P, Q.A.bins, G.s, G.K, last, first, lane);
            if (best == ~0ull) break;
            last = best; first = false;
            F::add(P, F::load(Q.A, (uint32_t)best), p.x, p.y, p.z, acc);
        }
        if (p.on) ss_field_store<F>(P, Q, p.dst, acc);
    }
}
