// ss_certify.cuh -- level-set variant 1: certification in its own, barrier-light kernel (candidate for round 2; selected with
// ss_context_set_levelset_variant(ctx, 1), the default stays k_levelset's fused certify + exact pass).
//
// Why: in k_levelset a large share of the warp-time goes to CTA barriers: every warp
// waits for warp 0's run scan and, after certifying its own 32 points, for the slowest warp of the brick before it may
// store its markers -- although 94 % of the bricks of a bulk fluid never enter the exact path.  Here a brick's warps
//   * compute the candidate-run table redundantly in registers (shuffles, no shared table, no scan barrier),
//   * stage only the particle records (x, y, z, V) -- no sort keys, no k-split -- behind ONE barrier,
//   * certify their box, store markers or raise a per-box flag, and retire independently.
// Boxes whose certification fails are then evaluated by k_levelset in SS_LS_FIX mode (an extra, small launch over the flagged
// bricks), exactly like the boxes the fix-up sweep flags.  Results are identical to the fused pass by construction: the same
// ss_certify_box decides, the same SS_LS_FIX code evaluates.
//
// Per-box state wstate[brick * 16 + box] : 0 untouched (all zero), 1 every valid point carries SS_MARKER, 2 needs exact values,
// 3 exact values already in place (no candidate within the support of any point of the box: the pre-zeroed tile IS the result).
#pragma once

struct SsCertArgs {
    SsBins bins;
    const uint4 *work_desc;      // per listed brick: (linear brick index, tile, bx | by << 10 | bz << 20, 0)
    float *tiles;
    uint8_t *wstate;             // [batch][nb^3][16]
};

// work list with decoded brick coordinates (no runtime divisions in the kernel)
__global__ void k_compact_desc(SsDev P, const uint32_t *__restrict__ flag, const uint32_t *__restrict__ off, uint32_t n, uint4 *__restrict__ desc) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n || !flag[b]) return;
    const SsBrick B = ss_brick_from_lin(P, b);
    desc[off[b]] = make_uint4(b, (uint32_t)B.tile, (uint32_t)B.bx | ((uint32_t)B.by << 10) | ((uint32_t)B.bz << 20), 0u);
}

// marks the standard 2x4x4 boxes of brick (vbx, vby, vbz) that the point box W overlaps
__device__ __forceinline__ void ss_mark_boxes(const SsDev &P, uint8_t *__restrict__ wstate, int tile, int vbx, int vby, int vbz, const SsWarpBox &W, uint8_t value) {
    const size_t base = ((((size_t)tile * P.nb + vbx) * P.nb + vby) * P.nb + vbz) * SS_LS_WARPS;
    const int i0 = W.i0 - 8 * vbx, j0 = W.j0 - 8 * vby, k0 = W.k0 - 8 * vbz;
    for (int a = i0 >> 1; a <= min((i0 + W.dx - 1) >> 1, 3); ++a)
        for (int b = j0 >> 2; b <= min((j0 + W.dy - 1) >> 2, 1); ++b)
            for (int c = k0 >> 2; c <= min((k0 + W.dz - 1) >> 2, 1); ++c) wstate[base + (size_t)(a * 4 + b * 2 + c)] = value;
}

// true when some staged candidate lies within the kernel support of the warp's point box (the cull of ss_exact_box)
template <bool GLOBAL>
__device__ __forceinline__ bool ss_box_has_candidate(const SsDev &P, const SsLanePoint &L, bool sparse, const float4 *s_rec, int C, int lane) {
    const float cull2 = (GLOBAL ? P.rev2 : (sparse ? P.h2m : P.h2)) * 1.0001f;
    for (int w = 0; w < ((C + 31) >> 5); ++w) {
        const int c = w * 32 + lane;
        if (__any_sync(0xffffffffu, c < C && ss_box_dist2(L, s_rec[c < C ? c : 0]) < cull2)) return true;
    }
    return false;
}

template <bool GLOBAL>
__global__ void __launch_bounds__(SS_LS_THREADS, 3)
k_certify(SsDev P, SsCertArgs A) {
    __shared__ float4 s_rec[SS_LS_CAP];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint4 desc = A.work_desc[blockIdx.x];
    const int tile_idx = (int)desc.y;
    const int bx = (int)(desc.z & 1023u), by = (int)((desc.z >> 10) & 1023u), bz = (int)(desc.z >> 20);
    const SsTile T = A.bins.tile_tab[tile_idx];

    // ---- candidate runs (one per lane, host guarantees <= 32 for this variant) and their exclusive prefix, per warp
    const SsBrickBins K = ss_brick_bins(P, A.bins.brick_rng, bx, by, bz, P.ext_bricks != 0);
    const bool ex = K.ex, ey = K.ey, ez = K.ez;
    const int nyr = K.nyr, nruns = K.nruns;
    uint32_t run_a, total;
    const uint32_t run_len = ss_brick_run(P, A.bins, T.s, K, lane, run_a);
    const uint32_t run_dst = ss_warp_excl_scan(run_len, lane, total);
    const int C = (int)total;
    if (C == 0) return;                                         // tile is pre-zeroed: phi = 0 exactly (wstate stays 0)

    const SsWarpBox Wm = { bx * 8 + (warp >> 2) * 2, by * 8 + ((warp >> 1) & 1) * 4, bz * 8 + (warp & 1) * 4, 2, 4, 4 };
    SsWarpBox We = Wm;
    int vbx = bx, vby = by, vbz = bz;
    const bool has_ext = (ex || ey || ez) && warp < 10 && ss_ext_task(warp, bx, by, bz, ex, ey, ez, We, vbx, vby, vbz);
    const bool sparse = GLOBAL || T.sparse != 0;

    if (C > SS_LS_CAP) {
        // oversized brick: everything goes to the exact pass (k_levelset's oversized path honours the per-box flags)
        const SsLanePoint L = ss_lane_point(P, T, Wm, tile_idx, lane, sparse);
        if (L.warp_valid && lane == 0) A.wstate[(size_t)desc.x * SS_LS_WARPS + warp] = 2;
        if (has_ext) { const SsLanePoint Le = ss_lane_point(P, T, We, tile_idx, lane, sparse); if (Le.warp_valid && lane == 0) ss_mark_boxes(P, A.wstate, tile_idx, vbx, vby, vbz, We, 2); }
        return;
    }

    // ---- stage the records (bin order): warp w takes runs w, w + 16
    for (int r = warp; r < nruns; r += SS_LS_WARPS) {
        const uint32_t a = __shfl_sync(0xffffffffu, run_a, r), len = __shfl_sync(0xffffffffu, run_len, r), dst = __shfl_sync(0xffffffffu, run_dst, r);
        for (uint32_t t = lane; t < len; t += 32) {
            float4 rc = A.bins.rec[a + t];
            if (GLOBAL) { int im[3]; float d0[3]; if (!ss_global_candidate(P, rc, im, d0)) rc.w = 0.0f; }   // skipped particle: no volume
            s_rec[dst + t] = rc;
        }
    }
    // the candidate sweep starts at the run that holds the brick's own bin
    int w0;
    {
        const int ox = min(max(ss_floor_div(8 * bx, P.be) + P.nlo - K.rx.x, 0), K.rx.y - K.rx.x), oy = min(max(ss_floor_div(8 * by, P.be) + P.nlo - K.ry.x, 0), nyr - 1);
        w0 = (int)(__shfl_sync(0xffffffffu, run_dst, ox * nyr + oy) >> 5);
        if (w0 >= ((C + 31) >> 5)) w0 = 0;
    }
    __syncthreads();

    {
        const SsLanePoint L = ss_lane_point(P, T, Wm, tile_idx, lane, sparse);
        if (L.warp_valid) {
            const bool ok = ss_certify_box(P, L, s_rec, C, lane, w0);
            if (ok && L.valid) A.tiles[L.out_idx] = SS_MARKER;
            const uint8_t st = ok ? 1 : (ss_box_has_candidate<GLOBAL>(P, L, sparse, s_rec, C, lane) ? 2 : 3);
            if (lane == 0) A.wstate[(size_t)desc.x * SS_LS_WARPS + warp] = st;
        }
    }
    if (has_ext) {
        const SsLanePoint L = ss_lane_point(P, T, We, tile_idx, lane, sparse);
        if (L.warp_valid) {
            const bool ok = ss_certify_box(P, L, s_rec, C, lane, w0);
            if (ok && L.valid) A.tiles[L.out_idx] = SS_MARKER;
            const uint8_t st = ok ? 1 : (ss_box_has_candidate<GLOBAL>(P, L, sparse, s_rec, C, lane) ? 2 : 3);
            if (lane == 0) ss_mark_boxes(P, A.wstate, tile_idx, vbx, vby, vbz, We, st);
        }
    }
}

// per brick: state = max over its boxes (0 untouched, 1 certified, 2 has exact values -- box states 2 and 3), and the flags of
// the exact launch: need[b] = some box of b is in state 2, wflag = per-box "evaluate exactly"
__global__ void k_wstate_reduce(const uint8_t *__restrict__ wstate, uint32_t nbricks, uint8_t *__restrict__ bstate, uint32_t *__restrict__ need,
                                uint8_t *__restrict__ wflag) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nbricks) return;
    const uint4 w = *reinterpret_cast<const uint4 *>(wstate + (size_t)b * SS_LS_WARPS);
    const uint32_t q[4] = { w.x, w.y, w.z, w.w };
    uint32_t mx = 0, any_need = 0, f[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        f[k] = 0;
#pragma unroll
        for (int s = 0; s < 32; s += 8) { const uint32_t v = (q[k] >> s) & 0xffu; mx = max(mx, min(v, 2u)); if (v == 2u) { f[k] |= 1u << s; any_need = 1u; } }
    }
    bstate[b] = (uint8_t)mx;
    need[b] = any_need;
    *reinterpret_cast<uint4 *>(wflag + (size_t)b * SS_LS_WARPS) = make_uint4(f[0], f[1], f[2], f[3]);
}

// ====================================================================================================================
// Level-set variant 2: warp-per-brick certification, TMA-staged, paired FP32 (sm_90a).
//
// One WARP owns one 8x8x8-point brick from start to finish, so the kernel has no CTA barrier at all:
//   1. lanes 0..nruns-1 each look up one candidate run ((X, Y) bin column, Z contiguous) and a shuffle scan lays the runs out
//      back to back in the warp's private slice of shared memory;
//   2. every lane that owns a non-empty run issues ONE bulk asynchronous copy (cp.async.bulk, TMA engine) for it; the copies
//      complete on the warp's mbarrier -- no per-record loads, no register staging;
//   3. level 1 (once per brick): lane = candidate; squared distances to the eight 4x4x4-point sub-boxes of the brick are built
//      from per-axis half-brick distances, giving one byte per candidate: bit b = "within ring 0 (0.55 h) of sub-box b";
//   4. level 2 (per sub-box): lane = TWO grid points (k, k+1) of the 4x4x4 box.  The ring-0 candidates (ballot over the mask
//      bytes) are folded into both running lower bounds with paired arithmetic (ss_sm90.cuh): d^2 = (dz, dz')^2 + (dx^2 + dy^2)
//      as one FMA pair, the cubic bound g(d^2) as three FMA pairs, clamp, and one FMA pair for the volume-weighted sum.  The sub-box is certified when all 64 sums exceed threshold * (1 + 1e-4); a ring-1 sweep
//      (0.55 h .. 0.76 h, where g vanishes) follows only for the few boxes that are still short;
//   5. certified sub-boxes store SS_MARKER, the others raise their per-box flag for the exact pass (k_levelset, SS_LS_FIX).
// The +1 planes of tiles with 8 k + 1 points per axis (extension tasks) reuse the scalar one-point-per-lane sweep.
// Warps are persistent and claim bricks in work-list order; step 1 of the next brick runs while step 2's copies are in flight.
// Soundness is that of variant 0/1: every term of the reference's sum is >= 0 and g <= W / sigma, so a certified point is
// inside for the reference too; failing to certify only costs time.  Results are therefore identical by construction.
#include "ss_sm90.cuh"

// two instantiations: up to 3 candidate bins per axis (h <= 8 cells; bulk fluid at h = 4 r, c = 0.5 r: 216 candidates) and wider
// reaches (c = 0.45 r: 343 .. 512 candidates, depending on how the 4.44-cell lattice falls into the 32-cell reach)
#define SS_CW_CAP_S 384                // candidates staged per brick, small variant: 4 bricks in flight per CTA (4 x 9.8 KB)
#define SS_CW_WARPS_S 4
#define SS_CW_CAP_L 576                // large variant: 3 bricks in flight per CTA (3 x 13.1 KB)
#define SS_CW_WARPS_L 3
#define SS_CW_MAXRUNS 32               // candidate runs per brick: one per lane

struct SsCwArgs {
    SsBins bins;
    const uint4 *work_desc;            // per listed brick: (linear brick index, tile, bx | by << 10 | bz << 20, 0)
    uint32_t n_work;
    float *tiles;
    uint8_t *wstate;                   // [batch][nb^3][16]
    unsigned long long *evals;         // optional work counter: candidate evaluations of the certification (lane-level)
    uint32_t *taken;                   // work-list entries handed out beyond the first wave (zero at launch)
    float cs;                          // coordinate scale of the bound: 2^-e with h cs in [1, 2) (exact in f32)
    float g1, g2, g3;                  // cubic bound in scaled d^2: g = G0 + g1 d2 + g2 d2^2 + g3 d2^3 (G_k / (h cs)^(2k), host-computed)
    float r0sq, r1sq;                  // ring radii squared, unscaled: (0.55 h)^2, (0.76 h)^2
};

#define SS_CW_PAIRS 24                 // capacity of one sub-box's ring-0 list in candidate PAIRS (bulk fluid: ~13); extra candidates are dropped (sound)
// one list entry = two candidates, component-interleaved so that both halves of a pair load as one aligned 64-bit value
struct __align__(16) SsCwPair { float x[2], y[2], z[2], v[2]; };
template <int CAP>
struct __align__(16) SsCwSlice {
    float4 rec[CAP];                   // staged candidate records (bulk-copy destination)
    SsCwPair list[4][SS_CW_PAIRS];     // ring-0 lists of the four sub-boxes of one x-half of the brick
    uint16_t cidx[CAP];                // candidates within ring 0 of the whole brick (pre-filter)
    unsigned long long mbar;
    unsigned long long pad_;
};

// squared distance of coordinate u to the interval [lo, hi]
__device__ __forceinline__ float ss_axis_d2(float u, float lo, float hi) { const float d = fmaxf(fmaxf(lo - u, u - hi), 0.0f); return d * d; }


// Folds the candidates flagged in `mword` (bit = index into wrec) into the two running lower bounds of a lane (points k, k + 1):
//   d^2 = (dz, dz')^2 + (dx^2 + dy^2),  sum += max(g(d^2), 0) * V   with g = G0 + g1 d2 + g2 d2^2 + g3 d2^3 <= W / sigma.
// Distances are in coordinates scaled by cs (SsCwArgs): the point is stored scaled, a staged record is scaled by the fused
// multiply-add that takes the difference (r cs is exact, so this rounds like (r - g) cs).
// Two candidates per iteration (independent accumulators); an odd tail re-reads the last record with zero volume.
struct SsCwPoint { float gx, gy; ss_f2 ngz; float cs, g1, g2, g3; };
__device__ __forceinline__ void ss_cw_eval(const SsCwPoint &Q, const float4 r, const float vol, ss_f2 &sum) {
    const float dx = fmaf(r.x, Q.cs, -Q.gx), dy = fmaf(r.y, Q.cs, -Q.gy);
    const float t = fmaf(dx, dx, dy * dy);
    const ss_f2 dz = ss_fma2(ss_pack(r.z, r.z), ss_pack(Q.cs, Q.cs), Q.ngz);
    const ss_f2 d2 = ss_fma2(dz, dz, ss_pack(t, t));
    ss_f2 g = ss_fma2(d2, ss_pack(Q.g3, Q.g3), ss_pack(Q.g2, Q.g2));
    g = ss_fma2(d2, g, ss_pack(Q.g1, Q.g1));
    g = ss_fma2(d2, g, ss_pack(SS_G0, SS_G0));
    float ga, gb;
    ss_unpack(g, ga, gb);
    sum = ss_fma2(ss_pack(fmaxf(ga, 0.0f), fmaxf(gb, 0.0f)), ss_pack(vol, vol), sum);
}
__device__ __forceinline__ void ss_cw_accumulate(const SsCwPoint &Q, const float4 *wrec, uint32_t mword, ss_f2 &sum0, ss_f2 &sum1) {
    while (mword) {
        const int b0 = __ffs(mword) - 1;
        mword &= mword - 1;
        const bool two = mword != 0u;
        const int b1 = two ? __ffs(mword) - 1 : b0;
        mword &= mword - 1;                                     // no-op when mword is already 0
        const float4 ra = wrec[b0], rb = wrec[b1];
        ss_cw_eval(Q, ra, ra.w, sum0);
        ss_cw_eval(Q, rb, two ? rb.w : 0.0f, sum1);
    }
}

// Ring-0 fold over a pair list: lane = grid points (k, k + 1); each iteration folds TWO candidates into both points, every
// operand a natural register pair (x, y, z, V of the two candidates):
//   (dx, dx') = (x, x') - gx;  (dy, dy') likewise;  t = dx^2 + dy^2 (paired);  per point: d2 = dz^2 + t,  g(d2) by Horner,
//   sum += max(g, 0) * (V, V')
// sumA / sumB hold the two candidates' partial sums side by side.
__device__ __forceinline__ void ss_cw_fold_pairs(const SsCwPoint &Q, float ngzA, float ngzB, const SsCwPair *list, int first, int last, ss_f2 &sumA, ss_f2 &sumB) {
    const ss_f2 G0 = ss_pack(SS_G0, SS_G0), G1 = ss_pack(Q.g1, Q.g1), G2 = ss_pack(Q.g2, Q.g2), G3 = ss_pack(Q.g3, Q.g3);
    const ss_f2 ngx = ss_pack(-Q.gx, -Q.gx), ngy = ss_pack(-Q.gy, -Q.gy), nza = ss_pack(ngzA, ngzA), nzb = ss_pack(ngzB, ngzB);
#pragma unroll 2
    for (int n = first; n < last; ++n) {
        const SsCwPair &E = list[n];
        const ss_f2 dx = ss_add2(ss_pack(E.x[0], E.x[1]), ngx), dy = ss_add2(ss_pack(E.y[0], E.y[1]), ngy);
        const ss_f2 t = ss_fma2(dx, dx, ss_mul2(dy, dy));
        const ss_f2 z = ss_pack(E.z[0], E.z[1]), v = ss_pack(E.v[0], E.v[1]);
        const ss_f2 dza = ss_add2(z, nza), dzb = ss_add2(z, nzb);
        const ss_f2 d2a = ss_fma2(dza, dza, t), d2b = ss_fma2(dzb, dzb, t);
        ss_f2 ga = ss_fma2(d2a, G3, G2), gb = ss_fma2(d2b, G3, G2);
        ga = ss_fma2(d2a, ga, G1); gb = ss_fma2(d2b, gb, G1);
        ga = ss_fma2(d2a, ga, G0); gb = ss_fma2(d2b, gb, G0);
        float a0, a1, b0, b1;
        ss_unpack(ga, a0, a1); ss_unpack(gb, b0, b1);
        sumA = ss_fma2(ss_pack(fmaxf(a0, 0.0f), fmaxf(a1, 0.0f)), v, sumA);
        sumB = ss_fma2(ss_pack(fmaxf(b0, 0.0f), fmaxf(b1, 0.0f)), v, sumB);
    }
}

// A listed brick's candidate runs, one per lane (ss_cw_lookup), ready to be copied into the warp's slice (ss_cw_issue).
struct SsCwRuns {
    uint4 desc;                        // work descriptor
    uint32_t run_a, run_len, run_dst;  // this lane's run: source record, length, destination slot
    int C;                             // candidates to certify; 0: the brick needs no sweep
};

// Looks up the candidate runs of the brick `desc` (global loads and shuffles only, the slice is not touched).  C = 0 when the
// brick needs no sweep: no candidate (its boxes stay in state 0, exact zeros) or more than CAP (every box goes to the exact pass,
// recorded here).
template <int CAP>
__device__ __forceinline__ SsCwRuns ss_cw_lookup(const SsDev &P, const SsCwArgs &A, const uint4 desc, int lane) {
    SsCwRuns R;
    R.desc = desc; R.run_a = 0; R.run_len = 0; R.run_dst = 0; R.C = 0;
    const int tile_idx = (int)desc.y;
    const int bx = (int)(desc.z & 1023u), by = (int)((desc.z >> 10) & 1023u), bz = (int)(desc.z >> 20);
    const uint32_t tile_s = A.bins.tile_tab[tile_idx].s;
    uint8_t *const wst = A.wstate + (size_t)desc.x * SS_LS_WARPS;

    // ---- candidate runs: one per lane (host guarantees <= SS_CW_MAXRUNS for this variant), exclusive prefix by shuffles
    const SsBrickBins K = ss_brick_bins(P, A.bins.brick_rng, bx, by, bz, P.ext_bricks != 0);
    const bool ex = K.ex, ey = K.ey, ez = K.ez;
    uint32_t run_a, total;
    const uint32_t run_len = ss_brick_run(P, A.bins, tile_s, K, lane, run_a);
    const uint32_t run_dst = ss_warp_excl_scan(run_len, lane, total);
    const int C = (int)total;
    if (C == 0) return R;                                       // phi = 0 exactly (wstate stays 0)

    if (C > CAP) {
        // oversized brick: everything goes to the exact pass (k_levelset's oversized path honours the per-box flags)
        if (lane < SS_LS_WARPS) {
            const int i0 = bx * 8 + (lane >> 2) * 2, j0 = by * 8 + ((lane >> 1) & 1) * 4, k0 = bz * 8 + (lane & 1) * 4;
            if (i0 < P.np && j0 < P.np && k0 < P.np) wst[lane] = 2;
        }
        if (ex || ey || ez) {
            for (int t = 0; t < 10; ++t) {
                SsWarpBox We; int vbx, vby, vbz;
                if (!ss_ext_task(t, bx, by, bz, ex, ey, ez, We, vbx, vby, vbz)) continue;
                if (lane == 0 && We.i0 < P.np && We.j0 < P.np && We.k0 < P.np) ss_mark_boxes(P, A.wstate, tile_idx, vbx, vby, vbz, We, 2);
            }
        }
        return R;
    }
    R.run_a = run_a; R.run_len = run_len; R.run_dst = run_dst; R.C = C;
    return R;
}

// Starts the bulk asynchronous copies (TMA engine) of the runs R into the warp's slice; they complete on its mbarrier.
// The slice was last read (and, on the global path, written) by this warp's ordinary accesses: order those before the async
// proxy's writes.
template <int CAP>
__device__ __forceinline__ void ss_cw_issue(SsCwSlice<CAP> &S, const SsCwArgs &A, const SsCwRuns &R, int lane) {
    __syncwarp();
    ss_fence_proxy_async();
    if (lane == 0) ss_mbar_arrive_expect_tx(&S.mbar, (uint32_t)R.C * 16u);
    __syncwarp();
    if (R.run_len) ss_bulk_g2s(&S.rec[R.run_dst], A.bins.rec + R.run_a, R.run_len * 16u, &S.mbar);
    __syncwarp();
}

// Certifies one brick whose C candidate records are in place in the slice; returns the lane-level bound evaluations (COUNT).
template <bool GLOBAL, bool COUNT, int CAP>
__device__ __forceinline__ unsigned long long ss_cw_brick(const SsDev &P, const SsCwArgs &A, SsCwSlice<CAP> &S, const uint4 desc, int C, int lane) {
    const int nb = P.nb;
    const int tile_idx = (int)desc.y;
    const int bx = (int)(desc.z & 1023u), by = (int)((desc.z >> 10) & 1023u), bz = (int)(desc.z >> 20);
    const bool ext = P.ext_bricks != 0;
    const bool ex = ext && bx == nb - 2, ey = ext && by == nb - 2, ez = ext && bz == nb - 2;
    const SsTile T = A.bins.tile_tab[tile_idx];
    const bool sparse = GLOBAL || T.sparse != 0;
    uint8_t *const wst = A.wstate + (size_t)desc.x * SS_LS_WARPS;

    // ---- level 1: per candidate, ring-0 membership for the eight sub-boxes (bit b = a * 4 + bb * 2 + cc: upper half in x, y, z)
    const int nwords = (C + 31) >> 5;
    const int pmax = P.np - 1;
    // world coordinates of the half-brick point intervals [lo, hi] per axis (culling only; the grid points' own expressions, so
    // that the intervals contain the points: ss_grid_xy / ss_grid_z)
    float xl0, xl1, xh0, xh1, yl0, yl1, yh0, yh1, zl0, zl1, zh0, zh1;
    {
        const int ox = bx * 8, oy = by * 8, oz = bz * 8;
        xl0 = ss_grid_xy(P, T.gbase[0] + min(ox, pmax), 0);     xh0 = ss_grid_xy(P, T.gbase[0] + min(ox + 3, pmax), 0);
        xl1 = ss_grid_xy(P, T.gbase[0] + min(ox + 4, pmax), 0); xh1 = ss_grid_xy(P, T.gbase[0] + min(ox + 7, pmax), 0);
        yl0 = ss_grid_xy(P, T.gbase[1] + min(oy, pmax), 1);     yh0 = ss_grid_xy(P, T.gbase[1] + min(oy + 3, pmax), 1);
        yl1 = ss_grid_xy(P, T.gbase[1] + min(oy + 4, pmax), 1); yh1 = ss_grid_xy(P, T.gbase[1] + min(oy + 7, pmax), 1);
        zl0 = ss_grid_z(P, T.gbase[2] + min(oz, pmax), sparse);     zh0 = ss_grid_z(P, T.gbase[2] + min(oz + 3, pmax), sparse);
        zl1 = ss_grid_z(P, T.gbase[2] + min(oz + 4, pmax), sparse); zh1 = ss_grid_z(P, T.gbase[2] + min(oz + 7, pmax), sparse);
    }
    // ---- pre-filter: candidates within ring 0 of the whole brick, compacted (sub-box distances are never smaller)
    int n0 = 0;
    for (int w = 0; w < nwords; ++w) {
        const int c = w * 32 + lane;
        bool keep = false;
        if (c < C) {
            const float4 r = S.rec[c];
            if (GLOBAL) { int im[3]; float d0[3]; if (!ss_global_candidate(P, r, im, d0)) S.rec[c].w = 0.0f; }   // skipped particle: no volume
            keep = ss_axis_d2(r.x, xl0, xh1) + ss_axis_d2(r.y, yl0, yh1) + ss_axis_d2(r.z, zl0, zh1) < A.r0sq;
        }
        const uint32_t mword = __ballot_sync(0xffffffffu, keep);
        if (keep) S.cidx[n0 + __popc(mword & ((1u << lane) - 1u))] = (uint16_t)c;
        n0 += __popc(mword);
    }
    __syncwarp();

    // ---- level 2: the eight 4x4x4 sub-boxes, one x-half of the brick at a time; lane = points (i, j, k) and (i, j, k + 1)
    const float cert = (P.thr + fabsf(P.thr) * 1.0e-4f + 1.0e-30f) / P.a_sigma;     // compare the un-normalised sum
    const float cull2 = (GLOBAL ? P.rev2 : (sparse ? P.h2m : P.h2)) * 1.0001f;
    const int li = lane >> 3, lj = (lane >> 1) & 3, lk = (lane & 1) * 2;
    // this lane's first point of sub-box (0, 0, 0); the other sub-boxes are constant strides away
    float *const lane_out = A.tiles + (size_t)tile_idx * P.np * P.np * P.np + ((size_t)(bx * 8 + li) * P.np + (by * 8 + lj)) * P.np + (bz * 8 + lk);
    const int np1 = P.np, np2 = P.np * P.np;
    unsigned long long n_eval = 0;
    for (int ha = 0; ha < 2; ++ha) {
        if (bx * 8 + 4 * ha > pmax) break;
        // ---- ring-0 lists of the four sub-boxes (hb, hc) of this half: pair-interleaved records, closest-first is not needed
        int cnt0 = 0, cnt1 = 0, cnt2 = 0, cnt3 = 0;
        const float axl = ha ? xl1 : xl0, axh = ha ? xh1 : xh0;
        for (int w0 = 0; w0 < n0; w0 += 32) {
            const int q = w0 + lane;
            float4 r = make_float4(0.f, 0.f, 0.f, 0.f);
            uint32_t m = 0;
            if (q < n0) {
                r = S.rec[S.cidx[q]];
                const float ax = ss_axis_d2(r.x, axl, axh);
                const float xy0 = ax + ss_axis_d2(r.y, yl0, yh0), xy1 = ax + ss_axis_d2(r.y, yl1, yh1);
                const float az0 = ss_axis_d2(r.z, zl0, zh0), az1 = ss_axis_d2(r.z, zl1, zh1);
                m = ((xy0 + az0 < A.r0sq) ? 1u : 0u) | ((xy0 + az1 < A.r0sq) ? 2u : 0u) | ((xy1 + az0 < A.r0sq) ? 4u : 0u) | ((xy1 + az1 < A.r0sq) ? 8u : 0u);
            }
#define SS_CW_APPEND(s4, cnt_)                                                                                   \
            {                                                                                                            \
                const uint32_t bal = __ballot_sync(0xffffffffu, (m >> (s4)) & 1u);                                       \
                const int pos = cnt_ + __popc(bal & ((1u << lane) - 1u));                                                \
                if (((m >> (s4)) & 1u) && pos < 2 * SS_CW_PAIRS) {                                                       \
                    SsCwPair &E = S.list[s4][pos >> 1];                                                                  \
                    E.x[pos & 1] = r.x * A.cs; E.y[pos & 1] = r.y * A.cs; E.z[pos & 1] = r.z * A.cs; E.v[pos & 1] = r.w; \
                }                                                                                                        \
                cnt_ = min(cnt_ + __popc(bal), 2 * SS_CW_PAIRS);                                                         \
            }
            SS_CW_APPEND(0, cnt0) SS_CW_APPEND(1, cnt1) SS_CW_APPEND(2, cnt2) SS_CW_APPEND(3, cnt3)
#undef SS_CW_APPEND
        }
        __syncwarp();
        // odd lists: the free half of the last pair repeats its partner with zero volume
        const int cnt_l = lane == 0 ? cnt0 : (lane == 1 ? cnt1 : (lane == 2 ? cnt2 : cnt3));
        if (lane < 4 && (cnt_l & 1)) {
            SsCwPair &E = S.list[lane][cnt_l >> 1];
            E.x[1] = E.x[0]; E.y[1] = E.y[0]; E.z[1] = E.z[0]; E.v[1] = 0.0f;
        }
        __syncwarp();
        for (int s4 = 0; s4 < 4; ++s4) {
            const int hb = s4 >> 1, hc = s4 & 1;
            const int i0 = bx * 8 + 4 * ha, j0 = by * 8 + 4 * hb, k0 = bz * 8 + 4 * hc;
            if (j0 > pmax || k0 > pmax) continue;                                        // sub-box outside the tile (warp-uniform)
            const int i = i0 + li, j = j0 + lj, k = k0 + lk;
            const bool row_ok = i <= pmax && j <= pmax;
            const bool vA = row_ok && k <= pmax, vB = row_ok && k + 1 <= pmax;
            // grid point coordinates from GLOBAL indices, the reference's expressions, scaled like the list entries
            const float gx = ss_grid_xy(P, T.gbase[0] + i, 0) * A.cs;
            const float gy = ss_grid_xy(P, T.gbase[1] + j, 1) * A.cs;
            const float gzA = ss_grid_z(P, T.gbase[2] + k, sparse) * A.cs;
            const float gzB = ss_grid_z(P, T.gbase[2] + k + 1, sparse) * A.cs;
            SsCwPoint Q;
            Q.gx = gx; Q.gy = gy; Q.ngz = ss_pack(-gzA, -gzB); Q.cs = A.cs; Q.g1 = A.g1; Q.g2 = A.g2; Q.g3 = A.g3;
            const int ns4 = s4 == 0 ? cnt0 : (s4 == 1 ? cnt1 : (s4 == 2 ? cnt2 : cnt3));
            const int npairs = (ns4 + 1) >> 1;
            ss_f2 sumA = ss_pack(0.0f, 0.0f), sumB = ss_pack(0.0f, 0.0f);
            bool done = false;
            float sa = 0.0f, sb = 0.0f;
            // ring 0 in chunks of four pairs, checking after each chunk
            for (int first = 0; first < npairs && !done; first += 4) {
                const int last = min(first + 4, npairs);
                ss_cw_fold_pairs(Q, -gzA, -gzB, S.list[s4], first, last, sumA, sumB);
                if (COUNT) n_eval += 4ull * (unsigned)(last - first);
                float a0, a1, b0, b1;
                ss_unpack(sumA, a0, a1); ss_unpack(sumB, b0, b1);
                sa = a0 + a1; sb = b0 + b1;
                done = __all_sync(0xffffffffu, (!vA || sa > cert) && (!vB || sb > cert));
            }
            uint32_t any_sup = ns4 ? 1u : 0u;
            if (!done) {
                // ring 1: the remaining candidates the bound can see (g vanishes at 0.755 h), tested against this sub-box directly;
                // "not in ring 0" is the complement of the very comparison that built the list, so nobody is counted twice
                ss_f2 sum0 = ss_pack(sa, sb), sum1 = ss_pack(0.0f, 0.0f);
                const float bxl = axl, bxh = axh, byl = hb ? yl1 : yl0, byh = hb ? yh1 : yh0, bzl = hc ? zl1 : zl0, bzh = hc ? zh1 : zh0;
                for (int w = 0; w < nwords && !done; ++w) {
                    const int c = w * 32 + lane;
                    bool keep = false, sup = false;
                    if (c < C) {
                        const float4 r = S.rec[c];
                        const float db2 = (ss_axis_d2(r.x, bxl, bxh) + ss_axis_d2(r.y, byl, byh)) + ss_axis_d2(r.z, bzl, bzh);
                        sup = db2 < cull2;
                        keep = (db2 < A.r1sq) && !(db2 < A.r0sq);
                    }
                    any_sup |= __ballot_sync(0xffffffffu, sup);
                    const uint32_t mword = __ballot_sync(0xffffffffu, keep);
                    if (!mword) continue;
                    if (COUNT) n_eval += 2ull * (unsigned)__popc(mword);
                    ss_cw_accumulate(Q, S.rec + w * 32, mword, sum0, sum1);
                    float ta, tb;
                    ss_unpack(ss_add2(sum0, sum1), ta, tb);
                    done = __all_sync(0xffffffffu, (!vA || ta > cert) && (!vB || tb > cert));
                }
            }
            if (done || !any_sup) {
                // certified: markers; no candidate within the support of the sub-box: the value is exactly 0 (stored, so that the
                // tiles need no zero-fill beforehand)
                float *out = lane_out + (4 * ha * np2 + 4 * hb * np1 + 4 * hc);
                const float val = done ? SS_MARKER : 0.0f;
                if (vA) out[0] = val;
                if (vB) out[1] = val;
            }
            // per-box state of the two standard 2x4x4 boxes this sub-box covers: 1 markers, 2 needs exact values, 3 exact zeros in place
            if (lane < 2) {
                const int is = i0 + 2 * lane;                      // first plane of the standard box
                if (is <= pmax) wst[(2 * ha + lane) * 4 + hb * 2 + hc] = done ? 1 : (any_sup ? 2 : 3);
            }
        }
        __syncwarp();                                              // the lists are rebuilt for the other half
    }

    // ---- extension tasks (planes at index np - 1): scalar one-point-per-lane sweep over the staged candidates
    if (ex || ey || ez) {
        for (int t = 0; t < 10; ++t) {
            SsWarpBox We; int vbx, vby, vbz;
            if (!ss_ext_task(t, bx, by, bz, ex, ey, ez, We, vbx, vby, vbz)) continue;
            const SsLanePoint L = ss_lane_point(P, T, We, tile_idx, lane, sparse);
            if (!L.warp_valid) continue;
            const bool ok = ss_certify_box(P, L, S.rec, C, lane, 0);
            if (ok && L.valid) A.tiles[L.out_idx] = SS_MARKER;
            const uint8_t st = ok ? 1 : (ss_box_has_candidate<GLOBAL>(P, L, sparse, S.rec, C, lane) ? 2 : 3);
            if (st == 3 && L.valid) A.tiles[L.out_idx] = 0.0f;        // exact zero, stored (no zero-fill of the tiles beforehand)
            if (lane == 0) ss_mark_boxes(P, A.wstate, tile_idx, vbx, vby, vbz, We, st);
        }
    }
    __syncwarp();                                                  // the slice is refilled for the next brick
    return n_eval;
}

// Persistent warps: warp g of G starts with listed brick g and then takes the next unclaimed entry of the work list (a counter), so
// the bricks in flight stay a window of neighbouring bricks, whose candidates share the L2; each brick's result depends on that
// brick only, whichever warp takes it.  The run lookup of the next brick -- a chain of dependent global loads: work descriptor, tile table, brick
// ranges, bin table -- is done while the current brick's bulk copies are in flight, so the two latencies overlap instead of adding
// up.  One slice per warp, so the occupancy stays that of one brick per warp (20 warps per SM).
template <bool GLOBAL, bool COUNT, int CAP, int WARPS>
__global__ void __launch_bounds__(WARPS * 32, 20 / WARPS)
k_certify_warp(SsDev P, SsCwArgs A) {
    __shared__ SsCwSlice<CAP> s_slice[WARPS];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    SsCwSlice<CAP> &S = s_slice[wib];
    const uint32_t stride = gridDim.x * WARPS;
    uint32_t work = blockIdx.x * WARPS + wib;
    if (work >= A.n_work) return;
    if (lane == 0) { ss_mbar_init(&S.mbar, 1); ss_mbar_fence_init(); }
    __syncwarp();                                                  // barrier initialised before anyone arrives / copies
    SsCwRuns R = ss_cw_lookup<CAP>(P, A, A.work_desc[work], lane);
    uint32_t phase = 0;
    unsigned long long n_eval = 0;
    while (work < A.n_work) {
        if (R.C) ss_cw_issue(S, A, R, lane);
        uint32_t next = 0;
        if (lane == 0) next = stride + atomicAdd(A.taken, 1u);
        next = __shfl_sync(0xffffffffu, next, 0);
        SsCwRuns Rn = R;
        Rn.C = 0;
        if (next < A.n_work) Rn = ss_cw_lookup<CAP>(P, A, A.work_desc[next], lane);
        if (R.C) {
            ss_mbar_wait(&S.mbar, phase);
            phase ^= 1u;
            n_eval += ss_cw_brick<GLOBAL, COUNT, CAP>(P, A, S, R.desc, R.C, lane);
        }
        R = Rn;
        work = next;
    }
    if (COUNT && A.evals) {
        for (int o = 16; o > 0; o >>= 1) n_eval += __shfl_xor_sync(0xffffffffu, n_eval, o);
        if (lane == 0 && n_eval) atomicAdd(A.evals, n_eval);
    }
}


// Level-set variant 2 leaves the tiles un-zeroed (16 GB of memset at 50 M particles): every value a later pass can read is written by
// the certification / exact kernels -- except in bricks nobody evaluated (no candidate particle: state 0), whose exact value is 0.
// Readers (fix-up sweep, marching cubes) touch the listed bricks and at most one brick around them, so only untouched bricks with a
// listed brick in their 3x3x3 neighbourhood (themselves included) are filled.  One warp per brick of the batch.
__global__ void __launch_bounds__(256)
k_zero_untouched(SsDev P, const uint8_t *__restrict__ bstate, const uint32_t *__restrict__ flag_mc, const uint32_t *__restrict__ flag_fix,
                 uint32_t nbricks_total, float *__restrict__ tiles) {
    const uint32_t b = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (b >= nbricks_total || bstate[b] != 0) return;
    const int nb = P.nb;
    const SsBrick B = ss_brick_from_lin(P, b);
    const int bx = B.bx, by = B.by, bz = B.bz;
    const uint32_t tile = (uint32_t)B.tile;
    bool listed = false;
    if (lane < 27) {
        const int x = bx + lane / 9 - 1, y = by + (lane / 3) % 3 - 1, z = bz + lane % 3 - 1;
        if (x >= 0 && y >= 0 && z >= 0 && x < nb && y < nb && z < nb) {
            const uint32_t o = ((tile * (uint32_t)nb + (uint32_t)x) * (uint32_t)nb + (uint32_t)y) * (uint32_t)nb + (uint32_t)z;
            listed = (flag_mc[o] | flag_fix[o]) != 0u;
        }
    }
    if (!__any_sync(0xffffffffu, listed)) return;
    const int np = P.np;
    float *t = tiles + (size_t)tile * np * np * np;
    for (int p = lane; p < 512; p += 32) {
        const int i = bx * 8 + (p >> 6), j = by * 8 + ((p >> 3) & 7), k = bz * 8 + (p & 7);
        if (i < np && j < np && k < np) t[((size_t)i * np + j) * np + k] = 0.0f;
    }
}
