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
