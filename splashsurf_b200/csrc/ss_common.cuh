// ss_common.cuh -- shared types and the exact-arithmetic helpers of the H100 reconstruct path.
//
// Parity rule: every float operation that decides a result of the reference is written with an explicit
// round-to-nearest intrinsic (__fadd_rn/__fmul_rn/__fmaf_rn/...), so that it is neither contracted into
// an FMA nor reassociated, and a fused multiply-add appears exactly where the reference's AVX2 grid loop
// has one (splashsurf_lib/src/dense_subdomains.rs:991-1133, kernel.rs:321-379).  The translation unit is
// additionally compiled with -fmad=false.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

#define SS_PI_F 3.14159265358979323846f

// ------------------------------------------------------------------ parameters on device ----
struct SsDev {
    float gmin[3];        // global MC grid aabb.min
    float c;              // cube size
    float h, h2, h2m;     // compact support, h*h, (h*h)*1.01f
    float thr;            // iso-surface threshold
    float rest_mass;      // (2r)^3 * rho0
    float sub_size;       // c * (float)S
    float margin;         // ghost particle margin
    float grow;           // margin * 1.5f (neighbourhood-search domain growth)
    int S, np;            // cubes per subdomain, points per subdomain (S+1)
    uint32_t np_magic;    // floor(2^32 / np) + 1: l / np == umulhi(l, np_magic) for l < np^2
    int nsd[3];           // subdomains per dimension
    int R;                // cube_radius = ceil(h/c)
    int srad;             // subdomain radius for ghost classification
    // kernels
    float a_hinv, a_sigma, a_s2, a_s6, a_s12;   // AVX-path cubic spline constants
    float s_sigma;                                // scalar-path normalisation 8/h^3
    float s_c_inner, s_c_outer, s_two_thirds;     // 3/(2pi), 1/(4pi), 2/3 in f32
    // neighbourhood-search grid bound and level-set binning
    int nsD, ns_stride;   // max NS cells per dim per subdomain, nsD^3
    int nb;               // bricks per dim = ceil(np / 8)
    int ext_bricks;       // 1: np == 8 (nb - 1) + 1 -> the np-1 planes are evaluated by the last full brick's CTA
    int be;               // bin edge in cells (multiple of 8; 8 unless h/c is large)
    int nlo;              // bin index offset = ceil(R / be): local coordinate u lands in bin floor(u/be)+nlo
    int nbin, nbin_sub;   // bins per dim, nbin^3
    float inv_c;          // 1/c (binning only; not parity relevant)
    float rr_cells;       // R + slack: particles farther than this from the tile are dropped (binning only)
    int simd;             // 1: AVX-path arithmetic for dense subdomains
    // global (non-decomposed) path, reconstruction.rs:65-194: one neighbourhood-search grid over the whole domain,
    // incremental stencil distances, narrow-band marching cubes; tiles are only an implementation detail there
    int gmode;
    float g_ns_amin[3]; int g_ns_nc[3];        // from_aabb(grid.aabb, h)
    float g_allow_min[3], g_allow_max[3];      // grid.aabb shrunk by the kernel evaluation radius (density_map.rs:606-610)
    float rev2;                                // kernel_evaluation_radius^2
    int sup;                                   // supported points per axis = 2R + 2
    // multi-GPU partition: memberships are kept only for subdomains with keep_lo <= ijk[part_axis] < keep_hi
    int part_axis, keep_lo, keep_hi;
    // anisotropic kernels (ss_aniso.cuh): margin is the wider membership margin, grow / nsD stay on the standard one
    int aniso;                                 // 1: memberships outside the neighbourhood-search grid are dropped, not an error
    float an_lambda, an_kr;                    // smoothing of the kernel centres, maximum stretch k_r
    uint32_t an_min_nb;                        // fewer neighbours than this: isotropic kernel
    // Jacobian correction of the averaged-position surface (ss_averaged.cuh, SsAvgCorrFold)
    float av_rs, av_low, av_high;              // R_s, t_low, t_high
};

// ------------------------------------------------------------------ exact helpers ----
__host__ __device__ inline float ss_coord(float mn, int64_t i, float cell) {
#ifdef __CUDA_ARCH__
    return __fadd_rn(mn, __fmul_rn((float)i, cell));           // uniform_grid.rs:418-425
#else
    volatile float t = (float)i * cell; return mn + t;
#endif
}

__host__ __device__ inline int ss_floor_div(int a, int b) { int q = a / b; return (a % b != 0 && ((a < 0) != (b < 0))) ? q - 1 : q; }

__device__ __forceinline__ int ss_cell_of(float x, float mn, float cell) {
    return (int)floorf(__fdiv_rn(__fsub_rn(x, mn), cell));      // uniform_grid.rs:444-451
}

// scalar cubic spline, kernel.rs:61-107
__device__ __forceinline__ float ss_kernel_scalar(const SsDev &P, float r) {
    float q = __fdiv_rn(__fadd_rn(r, r), P.h);
    float f;
    if (q < 1.0f) {
        float qq = __fmul_rn(q, q);
        float t = __fsub_rn(P.s_two_thirds, qq);
        float q3 = __fmul_rn(__fmul_rn(__fmul_rn(0.5f, q), q), q);
        f = __fmul_rn(P.s_c_inner, __fadd_rn(t, q3));
    } else if (q < 2.0f) {
        float x = __fsub_rn(2.0f, q);
        f = __fmul_rn(__fmul_rn(__fmul_rn(P.s_c_outer, x), x), x);
    } else {
        f = 0.0f;
    }
    return __fmul_rn(P.s_sigma, f);
}

// one lane of CubicSplineKernelAvxF32::evaluate, kernel.rs:343-378
__device__ __forceinline__ float ss_kernel_avx(const SsDev &P, float r) {
    float q = __fmul_rn(r, P.a_hinv);
    float v = fmaxf(__fsub_rn(1.0f, q), 0.0f);
    float v2 = __fmul_rn(v, v);
    float v3 = __fmul_rn(v2, v);
    float outer = __fmul_rn(v3, P.a_s2);
    float inner = __fmaf_rn(-v, P.a_s6, P.a_sigma);
    inner = __fmaf_rn(v2, P.a_s12, inner);
    inner = __fmaf_rn(-v3, P.a_s6, inner);
    return (q <= 0.5f) ? inner : outer;
}

// 64-bit key of a global MC edge: (point i, j, k) 20 bits each + axis
__host__ __device__ inline uint64_t ss_edge_key(int gi, int gj, int gk, int axis) {
    return ((uint64_t)(uint32_t)gi << 42) | ((uint64_t)(uint32_t)gj << 22) | ((uint64_t)(uint32_t)gk << 2) | (uint64_t)axis;
}
