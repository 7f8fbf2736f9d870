// ss_exact.cuh -- exact pass of level-set variant 2: the ordered cubic-spline fold for the boxes certification could not
// settle (surface band, outside points near the fluid, fix-up points), one WARP per flagged brick, no CTA barrier.
//
// The values must equal the reference's bit for bit (dense_subdomains.rs:1044-1128): per grid point an ordered fold over the
// subdomain's particles in ascending global index with fixed roundings.  Per brick the warp
//   1. stages the candidate records with bulk asynchronous copies (TMA engine) like the certification kernel, plus the
//      particle index (sort key) and the AVX-remainder split of every candidate with ordinary loads, all in flight at once
//      (4-byte runs start anywhere, so they cannot be bulk-copied into the slice without staging windows it has no room for);
//   2. sorts the (index, slot) keys once -- a bitonic network in its private shared-memory slice, warp-synchronous;
//   3. for every 4x4x4-point sub-box with a flagged 2x4x4 box: compacts, in sorted order, the candidates within the kernel
//      support of the sub-box, then folds them into TWO grid points per lane (k, k + 1) as FP32 pairs (ss_sm90.cuh: two scalar
//      IEEE operations per pair), and the operation sequence per element is the reference's:
//          d^2 = fma(dz, dz, fma(dx, dx, dy * dy));  r = sqrt(d^2);  W = the AVX kernel's fnmadd / fmadd chain;
//          phi = fma(W, V, phi)      (phi + W * V in the 8-lane remainder of the particle's stencil)
//      A candidate outside the support of one of the two points contributes an exact zero there (W := 0).
// Scalar-arithmetic tiles (sparse subdomains, simd off) and the global path use the one-point formulas twice.
// Bricks this kernel cannot take (more candidates than its slice holds) are appended to a fallback list for the next tier.
#pragma once

#define SS_XW_WARPS 3                  // bricks in flight per CTA (3 x 13.5 KB of static shared memory)
#define SS_XW_THREADS (SS_XW_WARPS * 32)
#define SS_XW_CAP 512                  // candidates staged per brick
#define SS_XW_LIST 224                 // candidates within the support of one 4x4x4 sub-box

struct SsXwArgs {
    SsBins bins;
    const uint32_t *bricks;            // flagged bricks (linear index)
    uint32_t n_bricks;
    const uint8_t *wflag;              // [batch][nb^3][16] boxes that need exact values
    float *tiles;
    uint32_t *fallback;                // bricks left to k_levelset (SS_LS_FIX): [0] = count, [1..] = linear brick indices
    unsigned long long *pairs;         // work counter (in-support evaluations), only with COUNT
    uint32_t *taken;                   // list entries handed out beyond the first wave of the persistent tier (zero at launch)
    unsigned long long *phases;        // [SS_XP_N + 1]: clock64() cycles per phase summed over the warps, then bricks; only with PHASES
};

// Phases of the exact pass, timed per warp by the PHASES instantiation of k_exact_warp (ss_context_set_exact_phases,
// tools/profile_exact_phases.py).  The default instantiation reads no clock.
enum { SS_XP_LOOKUP, SS_XP_COPY_WAIT, SS_XP_STAGE, SS_XP_SORT, SS_XP_LIST, SS_XP_FOLD, SS_XP_STORE, SS_XP_N };
template <bool ON>
struct SsXpClock {
    long long t = 0;
    unsigned long long acc[SS_XP_N] = {};
    __device__ __forceinline__ void start() { if (ON) t = clock64(); }
    // the cycles since the last lap (or start) go to phase p
    __device__ __forceinline__ void lap(int p) { if (ON) { const long long n = clock64(); acc[p] += (unsigned long long)(n - t); t = n; } }
    __device__ __forceinline__ void flush(unsigned long long *out, unsigned long long bricks, int lane) {
        if (ON && lane == 0 && out) {
            for (int p = 0; p < SS_XP_N; ++p) atomicAdd(&out[p], acc[p]);
            atomicAdd(&out[SS_XP_N], bricks);
        }
    }
};

template <int CAP, int LIST, int KEYS>
struct __align__(16) SsXwSliceT {
    float4 rec[CAP];
    unsigned long long key[KEYS];      // (particle index << 32) | slot, sorted ascending
    uint16_t ks[CAP];                  // AVX-remainder split per slot
    uint16_t list[LIST];               // slots within the support of the current sub-box, ascending particle index
    unsigned long long mbar;
    unsigned long long pad_;
};
typedef SsXwSliceT<SS_XW_CAP, SS_XW_LIST, 512> SsXwSlice;
// Dense clusters (overlapping droplets, cfg-5): the same kernel with one warp per CTA and a 108 KB slice of dynamic shared memory
#define SS_XW_BIG_CAP 4096
#define SS_XW_BIG_LIST 2048
typedef SsXwSliceT<SS_XW_BIG_CAP, SS_XW_BIG_LIST, SS_XW_BIG_CAP> SsXwSliceBig;
// in between: up to 1024 candidates (two or three overlapping bodies of fluid), one warp per CTA, 27 KB of static shared memory ->
// 8 bricks in flight per SM instead of the big variant's 2
#define SS_XW_MID_CAP 1024
#define SS_XW_MID_LIST 640
typedef SsXwSliceT<SS_XW_MID_CAP, SS_XW_MID_LIST, SS_XW_MID_CAP> SsXwSliceMid;
#ifdef SS_HOST_EMUL
static thread_local __align__(16) unsigned char ss_dyn_smem[sizeof(SsXwSliceBig)];
#else
extern __shared__ __align__(16) unsigned char ss_dyn_smem[];
#endif

// AVX-path kernel (kernel.rs:343-378) of two radii as a pair; every element rounds like ss_kernel_avx
__device__ __forceinline__ ss_f2 ss_kernel_avx2(const SsDev &P, float ra, float rb) {
    const ss_f2 q = ss_mul2(ss_pack(ra, rb), ss_pack(P.a_hinv, P.a_hinv));
    float qa, qb;
    ss_unpack(q, qa, qb);
    const ss_f2 one_m = ss_fma2(q, ss_pack(-1.0f, -1.0f), ss_pack(1.0f, 1.0f));          // 1 - q, one rounding
    float va, vb;
    ss_unpack(one_m, va, vb);
    const ss_f2 v = ss_pack(fmaxf(va, 0.0f), fmaxf(vb, 0.0f));
    const ss_f2 v2 = ss_mul2(v, v);
    const ss_f2 v3 = ss_mul2(v2, v);
    const ss_f2 outer = ss_mul2(v3, ss_pack(P.a_s2, P.a_s2));
    ss_f2 inner = ss_fma2(v, ss_pack(-P.a_s6, -P.a_s6), ss_pack(P.a_sigma, P.a_sigma));  // fnmadd(v, 6 sigma, sigma)
    inner = ss_fma2(v2, ss_pack(P.a_s12, P.a_s12), inner);
    inner = ss_fma2(v3, ss_pack(-P.a_s6, -P.a_s6), inner);
    float ia, ib, oa, ob;
    ss_unpack(inner, ia, ib);
    ss_unpack(outer, oa, ob);
    return ss_pack(qa <= 0.5f ? ia : oa, qb <= 0.5f ? ib : ob);
}

// A flagged brick's candidate runs, one per lane (ss_xw_lookup), ready to be staged into the warp's slice.
struct SsXwRuns {
    uint32_t brick_lin;
    uint32_t need8;                    // sub-boxes (bits 2, 1, 0: upper half along x, y, z) with a flagged 2x4x4 box
    uint32_t run_a, run_len, run_dst;  // this lane's run: source record, length, destination slot
    uint32_t run_off;                  // run_a - run_dst (mod 2^32): source record of slot p is p + run_off
    int C;                             // candidates to stage; 0: the lookup finished the brick (nothing flagged, no candidate, or
                                       // more than CAP: sent to the fallback list)
};

// Looks up the runs of listed brick `work` (global loads and shuffles only, the slice is not touched).  Bricks that need no staging
// are finished here: without candidates the requested points get exact zeros, with more than CAP the brick goes to the fallback list.
template <int CAP>
__device__ __forceinline__ SsXwRuns ss_xw_lookup(const SsDev &P, const SsXwArgs &A, const uint32_t work, const int lane) {
    SsXwRuns R;
    R.C = 0; R.run_a = 0; R.run_len = 0; R.run_dst = 0; R.run_off = 0;
    const uint32_t brick_lin = A.bricks[work];
    R.brick_lin = brick_lin;
    const SsBrick B = ss_brick_from_lin(P, brick_lin);
    const int bx = B.bx, by = B.by, bz = B.bz, tile_idx = B.tile;
    // per-box flags of the brick: 16 bytes; sub-box (a, b, c) needs values when either of its two 2x4x4 boxes is flagged
    uint32_t need8 = 0;
    {
        const uint8_t f = lane < SS_LS_WARPS ? A.wflag[(size_t)brick_lin * SS_LS_WARPS + lane] : (uint8_t)0;
        const uint32_t fl = __ballot_sync(0xffffffffu, f != 0);          // bit (i2 * 4 + hb * 2 + hc), i2 = plane pair 0..3
        for (int b = 0; b < 8; ++b) {
            const int ha = (b >> 2) & 1, hbc = b & 3;
            if (fl & ((1u << ((2 * ha) * 4 + hbc)) | (1u << ((2 * ha + 1) * 4 + hbc)))) need8 |= 1u << b;
        }
    }
    R.need8 = need8;
    if (!need8) return R;
    const uint32_t tile_s = A.bins.tile_tab[tile_idx].s;

    // ---- candidate runs (FIX mode: no extension planes), one per lane (host guarantees <= 32 for this variant)
    const SsBrickBins K = ss_brick_bins(P, A.bins.brick_rng, bx, by, bz, false);
    uint32_t run_a, total;
    const uint32_t run_len = ss_brick_run(P, A.bins, tile_s, K, lane, run_a);
    const uint32_t run_dst = ss_warp_excl_scan(run_len, lane, total);
    const int C = (int)total;

    if (C == 0) {
        // nothing in reach: the exact value is 0 (the tile may hold markers from an earlier pass only if C > 0, so this is
        // defensive): store zeros for the requested sub-boxes
        float *const tile = A.tiles + (size_t)tile_idx * P.np * P.np * P.np;
        const SsSubLane L = ss_sub_lane(P, lane);
        for (int b = 0; b < 8; ++b) {
            if (!(need8 & (1u << b))) continue;
            const int pmax = P.np - 1;
            const int i = bx * 8 + 4 * ((b >> 2) & 1) + L.li, j = by * 8 + 4 * ((b >> 1) & 1) + L.lj, k = bz * 8 + 4 * (b & 1) + L.lk;
            if (i <= pmax && j <= pmax) { if (k <= pmax) tile[((size_t)i * P.np + j) * P.np + k] = 0.0f; if (k + 1 <= pmax) tile[((size_t)i * P.np + j) * P.np + k + 1] = 0.0f; }
        }
        return R;
    }
    if (C > CAP) {
        if (lane == 0) A.fallback[1 + atomicAdd(&A.fallback[0], 1u)] = brick_lin;
        return R;
    }
    R.run_a = run_a; R.run_len = run_len; R.run_dst = run_dst; R.run_off = run_a - run_dst; R.C = C;
    return R;
}

// Starts the bulk asynchronous copies (TMA engine) of the records of the runs R into the warp's slice; they complete on its
// mbarrier.  The slice was last read by this warp's ordinary accesses: order those before the async proxy's writes.
template <typename SLICE>
__device__ __forceinline__ void ss_xw_issue(SLICE &S, const SsXwArgs &A, const SsXwRuns &R, const int lane) {
    __syncwarp();
    ss_fence_proxy_async();
    if (lane == 0) ss_mbar_arrive_expect_tx(&S.mbar, (uint32_t)R.C * 16u);
    __syncwarp();
    if (R.run_len) ss_bulk_g2s(&S.rec[R.run_dst], A.bins.rec + R.run_a, R.run_len * 16u, &S.mbar);
    __syncwarp();
}

// Particle indices and remainder splits of up to SS_XW_GATHER * 32 slots, loaded into registers with every load in flight at once
// (ss_xw_gather), then written to the slice as sort keys and splits (ss_xw_put).  Lane l holds slots base + 32 w + l.  Slot p
// lies in the last run whose first slot is <= p (that run is never empty); a binary search over the lanes' runs finds it.
#define SS_XW_GATHER 16
struct SsXwKeys { uint32_t pid[SS_XW_GATHER]; int ks[SS_XW_GATHER]; };
__device__ __forceinline__ void ss_xw_gather(const SsXwArgs &A, const SsXwRuns &R, const int lane, const int base, SsXwKeys &G) {
#pragma unroll
    for (int w = 0; w < SS_XW_GATHER; ++w) {
        const uint32_t p = (uint32_t)(base + w * 32 + lane);
        int r = 0;
#pragma unroll
        for (int step = 16; step > 0; step >>= 1) {
            const uint32_t d = __shfl_sync(0xffffffffu, R.run_dst, r + step);
            if (d <= p) r += step;
        }
        const uint32_t a = p + __shfl_sync(0xffffffffu, R.run_off, r);
        G.pid[w] = 0; G.ks[w] = 0;
        if (p < (uint32_t)R.C) { G.pid[w] = A.bins.pidx[a]; G.ks[w] = A.bins.ksplit[a]; }
    }
}
template <typename SLICE>
__device__ __forceinline__ void ss_xw_put(SLICE &S, const SsXwRuns &R, const int lane, const int base, const SsXwKeys &G) {
#pragma unroll
    for (int w = 0; w < SS_XW_GATHER; ++w) {
        const int p = base + w * 32 + lane;
        if (p < R.C) {
            S.key[p] = ((unsigned long long)G.pid[w] << 32) | (unsigned long long)p;
            S.ks[p] = (uint16_t)max(G.ks[w], 0);
        }
    }
}

// Exact values of one brick whose C candidate records have landed in the slice and whose sort keys are sorted; returns the
// lane's in-support evaluations (COUNT).
template <bool GLOBAL, bool COUNT, int CAP, int LIST, typename SLICE, bool PHASES>
__device__ __forceinline__ unsigned ss_xw_brick(const SsDev &P, const SsXwArgs &A, SLICE &S, const SsXwRuns &R, const int lane,
                                                SsXpClock<PHASES> &clk) {
    const uint32_t brick_lin = R.brick_lin, need8 = R.need8;
    const int C = R.C;
    const SsBrick B = ss_brick_from_lin(P, brick_lin);
    const int bx = B.bx, by = B.by, bz = B.bz, tile_idx = B.tile;
    const SsTile T = A.bins.tile_tab[tile_idx];
    const bool sparse = GLOBAL || T.sparse != 0;
    float *const tile = A.tiles + (size_t)tile_idx * P.np * P.np * P.np;
    const SsSubLane L = ss_sub_lane(P, lane);

    const float cull2 = (GLOBAL ? P.rev2 : (sparse ? P.h2m : P.h2)) * 1.0001f;
    unsigned hits = 0;
    for (int b = 0; b < 8; ++b) {
        if (!(need8 & (1u << b))) continue;
        const SsSubBox X = ss_sub_box(P, T, bx, by, bz, b, L, sparse);
        if (!X.inside) continue;
        const int i = X.i, j = X.j, k = X.k, gi = X.gi, gj = X.gj, gk = X.gk, k1 = X.k1;
        const float gx = X.gx, gy = X.gy, gzA = X.gzA, gzB = X.gzB;
        // ---- candidates within the support of the sub-box, in ascending particle index
        int nlist = 0;
        bool overflow = false;
        for (int w = 0; w < ((C + 31) >> 5); ++w) {
            const int rnk = w * 32 + lane;
            bool keep = false;
            int slot = 0;
            if (rnk < C) {
                slot = (int)(S.key[rnk] & 0xffffu);
                const float4 r = S.rec[slot];
                keep = ss_axis_d2(r.x, X.bxl, X.bxh) + ss_axis_d2(r.y, X.byl, X.byh) + ss_axis_d2(r.z, X.bzl, X.bzh) < cull2;
            }
            const uint32_t mword = __ballot_sync(0xffffffffu, keep);
            const int pos = nlist + __popc(mword & ((1u << lane) - 1u));
            if (keep && pos < LIST) S.list[pos] = (uint16_t)slot;
            nlist += __popc(mword);
        }
        if (nlist > LIST) overflow = true;
        __syncwarp();
        clk.lap(SS_XP_LIST);
        if (overflow) {
            // pathological clustering: leave the whole brick to k_levelset (its flags are untouched; values written so far are exact)
            if (lane == 0) A.fallback[1 + atomicAdd(&A.fallback[0], 1u)] = brick_lin;
            return hits;
        }
        float phiA = 0.0f, phiB = 0.0f;
        if (GLOBAL) {
            for (int n = 0; n < nlist; ++n) {
                const float4 r = S.rec[S.list[n]];
                int im[3]; float d0[3];
                if (!ss_global_candidate(P, r, im, d0)) continue;                      // skipped particle (density_map.rs:645-656)
                ss_accumulate_global(P, r, im, d0, gi, gj, gk, phiA, hits);
                ss_accumulate_global(P, r, im, d0, gi, gj, gk + 1, phiB, hits);
            }
        } else if (sparse) {
            for (int n = 0; n < nlist; ++n) {
                const float4 r = S.rec[S.list[n]];
                ss_accumulate<true, false>(P, r, 0, k, gx, gy, gzA, phiA, hits);
                ss_accumulate<true, false>(P, r, 0, k + 1, gx, gy, gzB, phiB, hits);
            }
        } else if (nlist > 0) {
            // Software-pipelined: while candidate n is evaluated, candidate n + 1's record and split and candidate n + 2's list entry
            // are loaded, so no iteration waits on the list -> record -> split chain of shared-memory loads.  Past the end of the
            // list the loads repeat its last entry and are not used.
            const ss_f2 ngz = ss_pack(-gzA, -gzB);
            ss_f2 phi = ss_pack(0.0f, 0.0f);
            const int last = nlist - 1;
            int slot = S.list[0];
            float4 r = S.rec[slot];
            int ks = (int)S.ks[slot];
            slot = S.list[min(1, last)];
            for (int n = 0; n < nlist; ++n) {
                const float4 r_next = S.rec[slot];
                const int ks_next = (int)S.ks[slot];
                slot = S.list[min(n + 2, last)];
                const float dx = __fsub_rn(r.x, gx), dy = __fsub_rn(r.y, gy);
                const float t = __fmaf_rn(dx, dx, __fmul_rn(dy, dy));
                const ss_f2 dz = ss_add2(ss_pack(r.z, r.z), ngz);                      // r.z - gz, exact negation
                const ss_f2 d2 = ss_fma2(dz, dz, ss_pack(t, t));                       // fma(dz, dz, fma(dx, dx, dy * dy))
                float d2a, d2b;
                ss_unpack(d2, d2a, d2b);
                const bool inA = d2a < P.h2, inB = d2b < P.h2;
                if (__any_sync(0xffffffffu, inA || inB)) {
                    const ss_f2 wk = ss_kernel_avx2(P, __fsqrt_rn(d2a), __fsqrt_rn(d2b));
                    float wa, wb;
                    ss_unpack(wk, wa, wb);
                    wa = inA ? wa : 0.0f; wb = inB ? wb : 0.0f;                        // outside the support: exact zero term
                    if (COUNT) hits += (inA ? 1u : 0u) + (inB ? 1u : 0u);
                    if (ks > k1) {
                        phi = ss_fma2(ss_pack(wa, wb), ss_pack(r.w, r.w), phi);        // fmadd lanes (dense_subdomains.rs:1110-1114)
                    } else {
                        float pa, pb;
                        ss_unpack(phi, pa, pb);
                        pa = (k < ks) ? __fmaf_rn(wa, r.w, pa) : __fadd_rn(pa, __fmul_rn(wa, r.w));     // remainder lanes (:1117-1128)
                        pb = (k + 1 < ks) ? __fmaf_rn(wb, r.w, pb) : __fadd_rn(pb, __fmul_rn(wb, r.w));
                        phi = ss_pack(pa, pb);
                    }
                }
                r = r_next;
                ks = ks_next;
            }
            ss_unpack(phi, phiA, phiB);
        }
        clk.lap(SS_XP_FOLD);
        if (X.vA) tile[((size_t)i * P.np + j) * P.np + k] = phiA;
        if (X.vB) tile[((size_t)i * P.np + j) * P.np + k + 1] = phiB;
        __syncwarp();                                           // the list is rebuilt for the next sub-box
        clk.lap(SS_XP_STORE);
    }
    return hits;
}

__device__ __forceinline__ void ss_xw_count(const SsXwArgs &A, unsigned hits, const int lane) {
    unsigned long long np_ = hits;
    for (int o = 16; o > 0; o >>= 1) np_ += __shfl_xor_sync(0xffffffffu, np_, o);
    if (lane == 0 && np_ && A.pairs) atomicAdd(A.pairs, np_);
}

// One brick from lookup to stores, nothing overlapped (the one-warp tiers, CAP > 512).
template <bool GLOBAL, bool COUNT, int CAP, int LIST, typename SLICE>
__device__ __forceinline__ void ss_exact_brick(const SsDev &P, const SsXwArgs &A, SLICE &S, const uint32_t work, const int lane) {
    SsXpClock<false> clk;
    if (lane == 0) { ss_mbar_init(&S.mbar, 1); ss_mbar_fence_init(); }
    __syncwarp();
    const SsXwRuns R = ss_xw_lookup<CAP>(P, A, work, lane);
    if (!R.C) return;
    ss_xw_issue(S, A, R, lane);
    for (int base = 0; base < R.C; base += SS_XW_GATHER * 32) {
        SsXwKeys G;
        ss_xw_gather(A, R, lane, base, G);
        ss_xw_put(S, R, lane, base, G);
    }
    ss_sort_keys<true>(S.key, R.C);
    ss_mbar_wait(&S.mbar, 0);
    __syncwarp();
    const unsigned hits = ss_xw_brick<GLOBAL, COUNT, CAP, LIST>(P, A, S, R, lane, clk);
    if (COUNT) ss_xw_count(A, hits, lane);
}

// 512-candidate tier.  Persistent warps, like k_certify_warp: warp g of G starts with listed brick g and then takes the next unclaimed
// entry of the list (the counter A.taken, zero at launch), so the bricks in flight stay neighbours that share candidates in the
// L2; each brick's values depend on that brick only, whichever warp takes it.  Per brick the warp issues the record copies and the
// loads of the sort keys and splits, looks up the next brick's runs (a chain of dependent global loads: brick list, flags, tile
// table, brick ranges, bin table) while all of them are in flight, then writes and sorts the keys, waits for the records and
// evaluates.  One slice per warp: 15 warps per SM.
template <bool GLOBAL, bool COUNT, bool PHASES = false>
__global__ void __launch_bounds__(SS_XW_THREADS, 5)
k_exact_warp(SsDev P, SsXwArgs A) {
    static_assert(SS_XW_CAP <= SS_XW_GATHER * 32, "one gather holds every candidate of the 512-slot tier");
    __shared__ SsXwSlice s_slice[SS_XW_WARPS];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    SsXwSlice &S = s_slice[wib];
    const uint32_t stride = gridDim.x * SS_XW_WARPS;
    uint32_t work = blockIdx.x * SS_XW_WARPS + wib;
    if (work >= A.n_bricks) return;
    SsXpClock<PHASES> clk;
    clk.start();
    if (lane == 0) { ss_mbar_init(&S.mbar, 1); ss_mbar_fence_init(); }
    __syncwarp();                                                  // barrier initialised before anyone arrives / copies
    SsXwRuns R = ss_xw_lookup<SS_XW_CAP>(P, A, work, lane);
    clk.lap(SS_XP_LOOKUP);
    uint32_t phase = 0;
    unsigned hits = 0;
    unsigned long long bricks = 0;
    while (work < A.n_bricks) {
        SsXwKeys G;
        if (R.C) {
            ss_xw_issue(S, A, R, lane);
            ss_xw_gather(A, R, lane, 0, G);
        }
        clk.lap(SS_XP_STAGE);
        uint32_t next = 0;
        if (lane == 0) next = stride + atomicAdd(A.taken, 1u);
        next = __shfl_sync(0xffffffffu, next, 0);
        SsXwRuns Rn = R;
        Rn.C = 0;
        if (next < A.n_bricks) Rn = ss_xw_lookup<SS_XW_CAP>(P, A, next, lane);
        clk.lap(SS_XP_LOOKUP);
        if (R.C) {
            ss_xw_put(S, R, lane, 0, G);
            clk.lap(SS_XP_STAGE);
            ss_sort_keys<true>(S.key, R.C);
            clk.lap(SS_XP_SORT);
            ss_mbar_wait(&S.mbar, phase);
            phase ^= 1u;
            __syncwarp();
            clk.lap(SS_XP_COPY_WAIT);
            hits += ss_xw_brick<GLOBAL, COUNT, SS_XW_CAP, SS_XW_LIST>(P, A, S, R, lane, clk);
        }
        ++bricks;
        R = Rn;
        work = next;
    }
    if (COUNT) ss_xw_count(A, hits, lane);
    clk.flush(A.phases, bricks, lane);
}

// one warp per CTA: bricks with up to 1024 candidates
template <bool GLOBAL, bool COUNT>
__global__ void __launch_bounds__(32, 8)
k_exact_warp_mid(SsDev P, SsXwArgs A) {
    __shared__ SsXwSliceMid s_slice;
    if (blockIdx.x >= A.n_bricks) return;
    ss_exact_brick<GLOBAL, COUNT, SS_XW_MID_CAP, SS_XW_MID_LIST>(P, A, s_slice, blockIdx.x, (int)(threadIdx.x & 31));
}

// one warp per CTA, slice in dynamic shared memory (sizeof(SsXwSliceBig) bytes): bricks with up to 4096 candidates
template <bool GLOBAL, bool COUNT>
__global__ void __launch_bounds__(32, 2)
k_exact_warp_big(SsDev P, SsXwArgs A) {
    if (blockIdx.x >= A.n_bricks) return;
    ss_exact_brick<GLOBAL, COUNT, SS_XW_BIG_CAP, SS_XW_BIG_LIST>(P, A, *reinterpret_cast<SsXwSliceBig *>(ss_dyn_smem), blockIdx.x, (int)(threadIdx.x & 31));
}
