// ss_field.cuh -- the level set of a reconstruction at arbitrary points (ss_levelset_field_*_f32, DESIGN.md §13).
//
// The value at a point p is the tile formula of the context's level set with p in place of the grid point: the same candidates
// (every record whose support reaches p), the same operations, ascending particle index.  The standard level set folds with
// SsSphFold below (the scalar formula of ss_accumulate<SPARSE = true>, the one of sparse subdomains and simd = off); the opt-in modes
// with their brick folds unchanged (SsAnisoFold, ss_aniso.cuh; SsAvgFold, SsAvgCorrFold, SsAvgRadFold, SsAvgCorrRadFold,
// ss_averaged.cuh).  Points no candidate reaches are 0.
//
//   k_field_keys      per point: group key (compressed subdomain, brick of its cell), or value 0 at once (outside the grid, subdomain
//                     without members); the first non-finite coordinate
//   k_field_starts    after the key sort: first point of every group
//   k_field_fold      warp per (subdomain, brick) group: the candidates of the group's bins staged and sorted as for a brick
//                     (ss_stage_candidates), then per batch of 32 points the candidates within h of the batch's bounding box
//                     (ballot compaction) folded by each lane for its point in index order, scattered to the caller's order; groups
//                     with more candidates than the slice go to a 4096-slot instantiation, beyond that to k_field_select
//   k_field_select    per batch of 32 points the selection walk of k_fold_select (ss_select_next)
// A group's candidate bins cover the cells [8b - R, 8b + 8 + R) along each axis (ss_pipeline.cu: upload_field_brick_ranges): a point lies
// anywhere in the closed cell box [8b, 8b + 8]^3 of its brick, one cell further than the brick's grid points reach.
#pragma once

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
};

// Points outside [gmin, gmax] along an axis, or in a subdomain without members, get 0 and key 0xffffffff (sorted last); chk[0]:
// lowest index with a non-finite coordinate (preset 0xffffffff), chk[1]: points with a group (preset 0).
__global__ void k_field_keys(SsDev P, const float *__restrict__ pts, uint32_t m, float3 gmax, const uint32_t *__restrict__ sub_flat, uint32_t nsub,
                             uint32_t *__restrict__ key, uint32_t *__restrict__ idx, float *__restrict__ out, uint32_t *__restrict__ chk) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    bool grouped = false;
    if (i < m) {
        const float p[3] = { pts[3 * (size_t)i], pts[3 * (size_t)i + 1], pts[3 * (size_t)i + 2] };
        const float hi[3] = { gmax.x, gmax.y, gmax.z };
        bool finite = true, inside = true;
        int gc[3];
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            finite = finite && isfinite(p[d]);
            inside = inside && p[d] >= P.gmin[d] && p[d] <= hi[d];
            // the cell of the point, clamped: a point on the grid's upper face belongs to the last cell
            gc[d] = inside ? min(max(ss_cell_of(p[d], P.gmin[d], P.c), 0), P.nsd[d] * P.S - 1) : 0;
        }
        if (!finite) atomicMin(&chk[0], i);
        uint32_t k = 0xffffffffu;
        if (finite && inside) {
            int sd[3], lb[3];
#pragma unroll
            for (int d = 0; d < 3; ++d) { sd[d] = gc[d] / P.S; lb[d] = (gc[d] - sd[d] * P.S) >> 3; }
            const uint32_t flat = (uint32_t)(((int64_t)sd[0] * P.nsd[1] + sd[1]) * P.nsd[2] + sd[2]);
            uint32_t lo = 0, up = nsub;                             // sub_flat is ascending
            while (lo < up) { const uint32_t mid = (lo + up) >> 1; if (sub_flat[mid] < flat) lo = mid + 1; else up = mid; }
            if (lo < nsub && sub_flat[lo] == flat) {
                k = lo * (uint32_t)(P.nb * P.nb * P.nb) + (uint32_t)((lb[0] * P.nb + lb[1]) * P.nb + lb[2]);
                grouped = true;
            }
        }
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
        if (p.on) Q.out[p.dst] = F::value(P, acc);
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
        if (p.on) Q.out[p.dst] = F::value(P, acc);
    }
}
