// ss_raycast.cuh -- first crossings of the level-set field along rays and segments (ss_levelset_field_raycast_f32, DESIGN.md §15).
//
// A wavefront march in rounds over per-ray state in global memory (SsRay).  Each round:
//   k_ray_keys        per active ray: its next point (sample T_j, or the bisection midpoint), keyed by the rule of k_field_keys
//                     (ss_field_key).  A point without a key has value 0: the rule is applied at once and the rest of the run of
//                     samples that shares the point's empty box (outside the grid on the approach, or a subdomain without members)
//                     is skipped by binary search, until the ray has a key or is done.  Writes (key, ray) of the keyed rays.
//   (sort, k_field_starts, scan_compact as for a field query)
//   k_ray_fold        warp per (subdomain, brick) group: the group's candidates staged as in k_field_fold; per batch of 32 rays,
//                     while a lane still has a point in the group, the lanes fold their points over the candidates within h of the
//                     active points' bounding box, apply the crossing / bisection rule and compute their next points; a lane whose
//                     next point has another key stores its state and stops.  A group without candidates skips each ray's run in
//                     its brick by binary search.  Groups beyond the slice go to the 4096-slot instantiation, then to k_ray_select.
//   k_ray_select      the same per batch with the candidates walked in ascending index by ss_select_next.
// The samples of a ray inside any axis-aligned box form one contiguous run of sample indices (DESIGN.md §15's lemma), so a skipped
// run is exactly a run of value-0 samples after its first one, which was evaluated.
#pragma once

#define SS_RAY_CAP (1u << 24)           // regular samples per ray: k < 2^24, where (float)k is exact

enum { SS_RAY_MARCH = 0, SS_RAY_REFINE = 1, SS_RAY_DONE = 2 };

// Per-ray state.  st: phase (bits 0-1), in(T_0) (bit 2), bisection steps taken (bits 3-9).
struct SsRay {
    float o[3], d[3];
    float dt, tmax;
    float a, b, vb;                    // bracket while refining, and the value at p(b)
    uint32_t j;                        // index of the sample to evaluate while marching
    uint32_t last;                     // index of the ray's last sample
    uint32_t st;
};

// The results of a call: t, position, value and status per ray (preset to +inf, NaN, NaN, 0 by k_ray_init)
struct SsRayOut { float *t, *pos, *val; int8_t *status; };

__device__ __forceinline__ uint32_t ss_ray_phase(const SsRay &r) { return r.st & 3u; }
__device__ __forceinline__ bool ss_ray_in0(const SsRay &r) { return (r.st >> 2) & 1u; }
__device__ __forceinline__ uint32_t ss_ray_nref(const SsRay &r) { return r.st >> 3; }

// whether k >= 1 is a regular sample, (float)k * dt < t_max and k < 2^24
__device__ __forceinline__ bool ss_ray_regular(const SsRay &r, uint32_t k) {
    return k >= 1 && k < SS_RAY_CAP && __fmul_rn((float)k, r.dt) < r.tmax;
}
// t of sample j <= last: 0, (float)j * dt, or t_max (the sample after the regular ones)
__device__ __forceinline__ float ss_ray_sample_t(const SsRay &r, uint32_t j) {
    return j == 0 ? 0.0f : (ss_ray_regular(r, j) ? __fmul_rn((float)j, r.dt) : r.tmax);
}
__device__ __forceinline__ float ss_ray_mid(float a, float b) { return __fadd_rn(a, __fmul_rn(__fsub_rn(b, a), 0.5f)); }
__device__ __forceinline__ void ss_ray_at(const SsRay &r, float t, float (&p)[3]) {
#pragma unroll
    for (int d = 0; d < 3; ++d) p[d] = __fadd_rn(r.o[d], __fmul_rn(t, r.d[d]));
}
// the point the ray evaluates next: p(T_j) while marching, p(mid) while refining
__device__ __forceinline__ void ss_ray_point(const SsRay &r, float (&p)[3]) {
    ss_ray_at(r, ss_ray_phase(r) == SS_RAY_REFINE ? ss_ray_mid(r.a, r.b) : ss_ray_sample_t(r, r.j), p);
}
// p lies outside [gmin, gmax] on an axis the direction does not move back from: every later sample has value 0
__device__ __forceinline__ bool ss_ray_gone(const SsDev &P, const SsRay &r, const float (&p)[3], float3 gmax) {
    const float hi[3] = { gmax.x, gmax.y, gmax.z };
    bool gone = false;
#pragma unroll
    for (int d = 0; d < 3; ++d) gone = gone || (p[d] > hi[d] && r.d[d] >= 0.0f) || (p[d] < P.gmin[d] && r.d[d] <= 0.0f);
    return gone;
}

// The march ends without a crossing: status 2 where the cap cut the regular samples short ((float)2^24 * dt < t_max), else 0
__device__ __forceinline__ void ss_ray_miss(SsRay &r, const SsRayOut &O, uint32_t i, bool gone) {
    O.status[i] = (!gone && __fmul_rn((float)SS_RAY_CAP, r.dt) < r.tmax) ? 2 : 0;
    r.st = (r.st & ~3u) | SS_RAY_DONE;
}
// The bracket [a, b] is final: t = b, position p(b), value at p(b), status +1 (enters) or -1 (leaves)
__device__ __forceinline__ void ss_ray_hit(SsRay &r, const SsRayOut &O, uint32_t i) {
    float p[3];
    ss_ray_at(r, r.b, p);
    O.t[i] = r.b; O.val[i] = r.vb;
    O.pos[3 * (size_t)i] = p[0]; O.pos[3 * (size_t)i + 1] = p[1]; O.pos[3 * (size_t)i + 2] = p[2];
    O.status[i] = ss_ray_in0(r) ? -1 : 1;
    r.st = (r.st & ~3u) | SS_RAY_DONE;
}
// after a bisection step (or at the crossing): the next midpoint, or the end of the refinement
__device__ __forceinline__ void ss_ray_refine_next(SsRay &r, const SsRayOut &O, uint32_t i, uint32_t refine) {
    const float mid = ss_ray_mid(r.a, r.b);
    if (ss_ray_nref(r) >= refine || mid == r.a || mid == r.b) ss_ray_hit(r, O, i);
    else r.st = (r.st & ~3u) | SS_RAY_REFINE;
}

// One evaluated point of ray i with value v (the point of ss_ray_point): §15's rule.  In(T_0) at sample 0; a crossing opens the
// bracket [T_{j-1}, T_j]; otherwise the march ends where the ray is gone from the grid, at its last sample, or moves on: to the
// next sample, or with `skip` (v is 0 along the run of samples for which in_run(point) holds, monotone in the index) to the first
// sample after the run.  A bisection step halves the bracket.  Returns whether the ray has a next point.
template <class Run>
__device__ __forceinline__ bool ss_ray_step(const SsDev &P, const SsRayOut &O, uint32_t i, SsRay &r, float v, const float (&p)[3], float3 gmax,
                                            uint32_t refine, bool skip, Run in_run) {
    const bool in = v > P.thr;
    if (ss_ray_phase(r) == SS_RAY_REFINE) {
        const float mid = ss_ray_mid(r.a, r.b);
        if (in == ss_ray_in0(r)) r.a = mid;
        else { r.b = mid; r.vb = v; }
        r.st += 8u;
        ss_ray_refine_next(r, O, i, refine);
        return ss_ray_phase(r) != SS_RAY_DONE;
    }
    if (r.j == 0) r.st = (r.st & ~4u) | (in ? 4u : 0u);
    else if (in != ss_ray_in0(r)) {
        r.a = ss_ray_sample_t(r, r.j - 1); r.b = ss_ray_sample_t(r, r.j); r.vb = v;
        ss_ray_refine_next(r, O, i, refine);
        return ss_ray_phase(r) != SS_RAY_DONE;
    }
    if (ss_ray_gone(P, r, p, gmax)) { ss_ray_miss(r, O, i, true); return false; }
    if (r.j == r.last) { ss_ray_miss(r, O, i, false); return false; }
    if (!skip) { ++r.j; return true; }
    // first sample in (j, last] outside the run
    uint32_t lo = r.j + 1, up = r.last + 1;
    while (lo < up) {
        const uint32_t mid = lo + ((up - lo) >> 1);
        float q[3];
        ss_ray_at(r, ss_ray_sample_t(r, mid), q);
        if (in_run(q)) lo = mid + 1; else up = mid;
    }
    if (lo > r.last) {                                       // the run reaches the last sample: no crossing after its first one
        float q[3];
        ss_ray_at(r, ss_ray_sample_t(r, r.last), q);
        ss_ray_miss(r, O, i, ss_ray_gone(P, r, q, gmax));
        return false;
    }
    r.j = lo;
    return true;
}

// Per ray: |d| = sqrt((dx dx + dy dy) + dz dz), dt = step / |d|, the index of its last sample, and the preset outputs.  chk[0]: first
// ray with a non-finite origin or direction, chk[1]: first with a zero direction or a zero or non-finite dt, chk[2]: first with a NaN
// or negative t_max (each preset 0xffffffff).  tmax == nullptr: +inf for every ray.
__global__ void k_ray_init(const float *__restrict__ o, const float *__restrict__ d, const float *__restrict__ tmax, uint32_t m, float step,
                           SsRay *__restrict__ rays, SsRayOut O, uint32_t *__restrict__ chk) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    SsRay r;
    bool finite = true;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        r.o[a] = o[3 * (size_t)i + a]; r.d[a] = d[3 * (size_t)i + a];
        finite = finite && isfinite(r.o[a]) && isfinite(r.d[a]);
    }
    const float nd = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(r.d[0], r.d[0]), __fmul_rn(r.d[1], r.d[1])), __fmul_rn(r.d[2], r.d[2])));
    r.dt = __fdiv_rn(step, nd);
    r.tmax = tmax ? tmax[i] : __int_as_float(0x7f800000);
    if (!finite) atomicMin(&chk[0], i);
    if ((r.d[0] == 0.0f && r.d[1] == 0.0f && r.d[2] == 0.0f) || !(r.dt > 0.0f) || !isfinite(r.dt)) atomicMin(&chk[1], i);
    if (!(r.tmax >= 0.0f)) atomicMin(&chk[2], i);
    // last regular sample: the largest k < 2^24 with (float)k * dt < t_max (0 if none), then t_max if it is finite and > 0
    uint32_t lo = 1, up = SS_RAY_CAP;
    while (lo < up) { const uint32_t mid = lo + ((up - lo) >> 1); if (ss_ray_regular(r, mid)) lo = mid + 1; else up = mid; }
    r.last = lo - 1 + ((isfinite(r.tmax) && r.tmax > 0.0f) ? 1u : 0u);
    r.a = 0.0f; r.b = 0.0f; r.vb = 0.0f; r.j = 0; r.st = SS_RAY_MARCH;
    rays[i] = r;
    const float nan = __int_as_float(0x7fc00000);
    O.t[i] = __int_as_float(0x7f800000); O.val[i] = nan; O.status[i] = 0;
    O.pos[3 * (size_t)i] = nan; O.pos[3 * (size_t)i + 1] = nan; O.pos[3 * (size_t)i + 2] = nan;
}

struct SsRayArgs {
    SsFieldArgs F;                     // A (records, the field's candidate ranges), key, idx (ray indices), starts, groups, n_groups, fallback
    SsRay *rays;
    SsRayOut O;
    float3 gmax;
    const uint32_t *sub_flat;
    uint32_t nsub, refine;
};

// Rays not yet done: advance through points without a key (value 0) until the ray has a key or is done; the keyed rays' (key, ray)
// at count[0]++ (count preset 0).
__global__ void k_ray_keys(SsDev P, SsRayArgs Q, uint32_t m, uint32_t *__restrict__ key, uint32_t *__restrict__ idx, uint32_t *__restrict__ count) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    uint32_t k = 0xffffffffu;
    if (i < m && ss_ray_phase(Q.rays[i]) != SS_RAY_DONE) {
        SsRay r = Q.rays[i];
        for (;;) {
            float p[3];
            ss_ray_point(r, p);
            bool finite;
            int gc[3];
            k = ss_field_key(P, p, Q.gmax, Q.sub_flat, Q.nsub, finite);
            if (k != 0xffffffffu) break;
            // the run: inside the grid, the samples in the same subdomain; outside, those not yet inside the grid on every
            // axis the ray approaches it along
            const bool inbox = ss_field_cell(P, p, Q.gmax, gc, finite);
            int sd[3];
#pragma unroll
            for (int d = 0; d < 3; ++d) sd[d] = gc[d] / P.S;
            const float hi[3] = { Q.gmax.x, Q.gmax.y, Q.gmax.z };
            const auto in_run = [&](const float (&q)[3]) {
                bool f;
                int qc[3];
                if (inbox) return ss_field_cell(P, q, Q.gmax, qc, f) && qc[0] / P.S == sd[0] && qc[1] / P.S == sd[1] && qc[2] / P.S == sd[2];
                bool out = false;
#pragma unroll
                for (int d = 0; d < 3; ++d) out = out || (r.d[d] > 0.0f && q[d] < P.gmin[d]) || (r.d[d] < 0.0f && q[d] > hi[d]);
                return out;
            };
            if (!ss_ray_step(P, Q.O, i, r, 0.0f, p, Q.gmax, Q.refine, true, in_run)) break;
        }
        Q.rays[i] = r;
    }
    const bool keyed = k != 0xffffffffu;
    const unsigned w = __ballot_sync(0xffffffffu, keyed);
    uint32_t base = 0;
    if ((threadIdx.x & 31) == 0 && w) base = atomicAdd(count, (uint32_t)__popc(w));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (keyed) {
        const uint32_t slot = base + __popc(w & ((1u << (threadIdx.x & 31)) - 1u));
        key[slot] = k; idx[slot] = i;
    }
}

// The rays of group G in batches of 32: while a lane still has a point in the group, value(active, x, y, z) folds the active lanes' points
// (warp-collective; every lane calls it) and each active lane applies the rule and moves on.  A group without candidates (empty)
// skips each ray's run in its brick.
template <class Value>
__device__ __forceinline__ void ss_ray_batches(const SsDev &P, const SsRayArgs &Q, const SsFieldGroup &G, bool empty, int lane, Value value) {
    const uint32_t gkey = Q.F.key[G.p0];
    const auto in_group = [&](const float (&q)[3]) { bool f; return ss_field_key(P, q, Q.gmax, Q.sub_flat, Q.nsub, f) == gkey; };
    for (uint32_t q0 = G.p0; q0 < G.p1; q0 += 32) {
        const bool on = q0 + lane < G.p1;
        const uint32_t i = on ? Q.F.idx[q0 + lane] : 0u;
        SsRay r;
        float p[3] = { 0.0f, 0.0f, 0.0f };
        if (on) { r = Q.rays[i]; ss_ray_point(r, p); }
        bool act = on;
        while (__any_sync(0xffffffffu, act)) {
            const float v = empty ? 0.0f : value(act, p[0], p[1], p[2]);
            if (act) {
                act = ss_ray_step(P, Q.O, i, r, v, p, Q.gmax, Q.refine, empty, in_group);
                if (act) { ss_ray_point(r, p); act = in_group(p); }
            }
        }
        if (on) Q.rays[i] = r;
    }
}

template <class F, int CAP, int WARPS>
__global__ void __launch_bounds__(WARPS * 32, 1)
k_ray_fold(SsDev P, SsRayArgs Q) {
    __shared__ unsigned long long s_key[WARPS][CAP];
    __shared__ uint16_t s_list[WARPS][CAP];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t work = blockIdx.x * WARPS + wib;
    if (work >= Q.F.n_groups) return;
    const uint32_t g = Q.F.groups ? Q.F.groups[work] : work;
    const SsFieldGroup G = ss_field_group(P, Q.F, g);
    const uint32_t C = ss_stage_candidates<CAP>(P, Q.F.A.bins, G.s, G.K, s_key[wib], lane);
    if (C > (uint32_t)CAP) {
        if (lane == 0) Q.F.fallback[1 + atomicAdd(&Q.F.fallback[0], 1u)] = g;
        return;
    }
    const float cull2 = P.h2 * 1.0001f;
    ss_ray_batches(P, Q, G, C == 0, lane, [&](bool act, float px, float py, float pz) {
        // the candidates within h of the active points' bounding box (inactive lanes take the first active lane's point)
        const int src = __ffs(__ballot_sync(0xffffffffu, act)) - 1;
        const float x0 = __shfl_sync(0xffffffffu, px, src), y0 = __shfl_sync(0xffffffffu, py, src), z0 = __shfl_sync(0xffffffffu, pz, src);
        float xl = act ? px : x0, xh = xl, yl = act ? py : y0, yh = yl, zl = act ? pz : z0, zh = zl;
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
                const float4 r = Q.F.A.bins.rec[(uint32_t)s_key[wib][rnk]];
                keep = ss_axis_d2(r.x, xl, xh) + ss_axis_d2(r.y, yl, yh) + ss_axis_d2(r.z, zl, zh) < cull2;
            }
            const uint32_t mword = __ballot_sync(0xffffffffu, keep);
            if (keep) s_list[wib][nlist + __popc(mword & ((1u << lane) - 1u))] = (uint16_t)rnk;
            nlist += __popc(mword);
        }
        __syncwarp();
        typename F::Acc acc = F::zero();
        if (act)
            for (int n = 0; n < nlist; ++n) F::add(P, F::load(Q.F.A, (uint32_t)s_key[wib][s_list[wib][n]]), px, py, pz, acc);
        __syncwarp();                                        // the list is rebuilt for the next points
        return F::value(P, acc);
    });
}

// Groups with more candidates than the largest slice: the candidates of every step in ascending particle index by repeated selection
template <class F>
__global__ void __launch_bounds__(32)
k_ray_select(SsDev P, SsRayArgs Q) {
    if (blockIdx.x >= Q.F.n_groups) return;
    const int lane = threadIdx.x & 31;
    const SsFieldGroup G = ss_field_group(P, Q.F, Q.F.groups ? Q.F.groups[blockIdx.x] : blockIdx.x);
    ss_ray_batches(P, Q, G, false, lane, [&](bool act, float px, float py, float pz) {
        typename F::Acc acc = F::zero();
        unsigned long long last = 0;
        bool first = true;
        for (;;) {
            const unsigned long long best = ss_select_next(P, Q.F.A.bins, G.s, G.K, last, first, lane);
            if (best == ~0ull) break;
            last = best; first = false;
            if (act) F::add(P, F::load(Q.F.A, (uint32_t)best), px, py, pz, acc);
        }
        return F::value(P, acc);
    });
}

// hit rays (status +-1): flag[i] = 1
__global__ void k_ray_hit_flags(const int8_t *__restrict__ status, uint32_t m, uint32_t *__restrict__ flag) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < m) flag[i] = (status[i] == 1 || status[i] == -1) ? 1u : 0u;
}
// positions of the n listed rays, packed
__global__ void k_ray_gather(const uint32_t *__restrict__ list, uint32_t n, const float *__restrict__ pos, float *__restrict__ out) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n) return;
    const uint32_t i = list[q];
#pragma unroll
    for (int a = 0; a < 3; ++a) out[3 * (size_t)q + a] = pos[3 * (size_t)i + a];
}
// n floats of NaN
__global__ void k_ray_fill_nan(float *__restrict__ out, uint64_t n) {
    const uint64_t q = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (q < n) out[q] = __int_as_float(0x7fc00000);
}
// the packed gradients of the n listed rays at their rays' places
__global__ void k_ray_scatter_hits(const uint32_t *__restrict__ list, uint32_t n, const float *__restrict__ g, float *__restrict__ out) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= n) return;
    const uint32_t i = list[q];
#pragma unroll
    for (int a = 0; a < 3; ++a) out[3 * (size_t)i + a] = g[3 * (size_t)q + a];
}
