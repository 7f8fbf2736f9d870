// ss_density.cuh -- SPH particle densities, cell-cooperative kernel (sm_90a).  NOT the default; slower than k_density on the H100 (DESIGN.md section 6).
//
// An attempt to replace the thread-per-particle k_density (ss_kernels.cuh), whose warps leave many lanes idle
// (every lane walks its own 27 cell runs and its own hit list).  The pair test is only ~10 instructions, so the per-chunk bookkeeping
// of the cooperative scheme (index mapping, ballot, pool slot, overflow check) and the staging of nine short runs per cell can
// outweigh the lanes it keeps busy; it was slower than k_density where it was first measured.  Kept selectable (ss_context_set_density_variant 1 / 2) because it is
// bit-identical and documents the design space; the default stays k_density.  Reference semantics are unchanged
// (dense_subdomains.rs:496-646, neighborhood_search.rs:396-433, density_map.rs:169-185):
//     rho_i = m * (W(0) + sum_j W(|x_j - x_i|)),  j over the 26 adjacent h-cells in x-major order, then the own cell,
//     ascending particle index inside a cell, one f32 addition per neighbour in that order.
//
// One WARP owns one h-cell of one subdomain (persistent warps striding over the list of cells that hold a particle inside
// their subdomain's AABB):
//   1. lanes 0..26 look up the 27 candidate runs in the reference's visiting order; a shuffle scan lays them out back to back
//      and every non-empty run is moved into the warp's shared-memory slice by ONE bulk asynchronous copy (TMA engine)
//      completing on the warp's mbarrier -- the ~216 candidate positions are read from L2 once per cell, not once per particle;
//   2. per particle of the cell (warp-uniform loop): lane = candidate.  The squared distances are computed with the reference's
//      operation sequence; a ballot compacts the hits IN CANDIDATE ORDER into the particle's slice of a shared pool;
//   3. the kernel W(sqrt(d^2)) of every pooled hit is evaluated densely (lane = pool entry, all lanes busy, no divergence on
//      the 15 % hit rate);
//   4. lane = particle: the ordered f32 sum over its slice -- the only inherently serial part, now ~33 dependent additions
//      for up to 16 particles at a time.
// Cells with more candidates than the slice holds, and particles whose hit list does not fit the pool, take the
// thread-serial routine ss_density_entry (same arithmetic, same order).  Results are bit-identical to k_density by
// construction; tests compare both against the oracle and the reference fixtures.
#pragma once
#include "ss_sm90.cuh"

#define SS_DC_WARPS 4                  // cells in flight per CTA
#define SS_DC_CAP 320                  // candidates staged per cell (bulk fluid at h = 4 r: ~216)
#define SS_DC_POOL 640                 // hit pool of one round of particles, in floats
#define SS_DC_MAXP 16                  // particles per round
#define SS_DC_RESERVE 128              // free pool entries required before a particle starts (bulk: ~33 hits per particle)
#define SS_DC_CHUNK 32                 // consecutive cells a persistent warp takes at a time

struct __align__(16) SsDcSlice {
    float4 cand[SS_DC_CAP];            // staged candidate positions (x, y, z, particle index bits), visiting order
    float pool[SS_DC_POOL];            // d^2 of the hits, then W in place
    uint32_t ent[SS_DC_MAXP];          // membership entry of each particle of the round
    int base[SS_DC_MAXP];              // first pool entry of its slice
    int cnt[SS_DC_MAXP];               // hits (-1: list did not fit, thread-serial fallback)
    unsigned long long mbar;
    unsigned long long pad_;
};

#if defined(SS_HOST_EMUL) && defined(SS_DC_TRACE)      // which escape routes a test input takes (CPU executor, one-off builds only)
#define SS_DC_NOTE(what) do { if (lane == 0) fprintf(stderr, "[ss_density] %s\n", what); } while (0)
#else
#define SS_DC_NOTE(what) do { } while (0)
#endif

struct SsDcArgs {
    uint32_t m;                                        // membership entries
    const uint32_t *list, *list_off, *list_flag;       // compacted first entries of the listed cells; length = list_off[m-1] + list_flag[m-1]
    const uint32_t *key;                               // NS key of every entry (subdomain * ns_stride + cell)
    const float4 *spos;                                // NS-sorted positions
    const uint32_t *sub_flat, *off;                    // cell offsets (k_cell_offsets)
    float *rho;
    unsigned long long *nbr_count;                     // optional
};

// flag = 1 on the first entry of every h-cell run that holds at least one particle inside its subdomain's half-open AABB
// (aabb.rs:220-222): those are the cells with densities to compute
__global__ void k_density_cell_flags(SsDev P, uint32_t m, const uint32_t *__restrict__ key, const float4 *__restrict__ spos,
                                     const uint32_t *__restrict__ sub_flat, const uint32_t *__restrict__ off, uint32_t *__restrict__ flag) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= m) return;
    const uint32_t k = key[e];
    uint32_t f = 0;
    if (e == 0 || key[e - 1] != k) {
        const SsSubGeom g = ss_sub_geom(P, sub_flat[k / (uint32_t)P.ns_stride]);
        const uint32_t b = off[k + 1];
        for (uint32_t t = e; t < b && !f; ++t) {
            const float4 pi = spos[t];
            if ((pi.x >= g.smin[0] && pi.y >= g.smin[1] && pi.z >= g.smin[2]) && (pi.x < g.smax[0] && pi.y < g.smax[1] && pi.z < g.smax[2])) f = 1u;
        }
    }
    flag[e] = f;
}

// evaluates the pooled hits, sums them per particle in order, writes the densities of the round
__device__ __forceinline__ void ss_dc_flush(const SsDev &P, const SsDcArgs &A, SsDcSlice &S, const int lane, int &nround, int &total) {
    __syncwarp();
    for (int i = lane; i < total; i += 32) S.pool[i] = ss_kernel_scalar(P, __fsqrt_rn(S.pool[i]));
    __syncwarp();
    if (lane < nround) {
        const uint32_t e = S.ent[lane];
        const int cnt = S.cnt[lane];
        if (cnt >= 0) {
            float acc = ss_kernel_scalar(P, 0.0f);
            const float *w = S.pool + S.base[lane];
            for (int n = 0; n < cnt; ++n) acc = __fadd_rn(acc, w[n]);
            const uint32_t idx = __float_as_uint(A.spos[e].w);
            if (A.nbr_count) A.nbr_count[idx] = (unsigned long long)cnt;
            A.rho[idx] = __fmul_rn(acc, P.rest_mass);
        } else {
            ss_density_entry<false>(P, ss_walk_sub(P, e, A.key, A.sub_flat, A.off), A.spos, A.rho, A.nbr_count, (const unsigned long long *)nullptr, (uint32_t *)nullptr);
        }
    }
    __syncwarp();
    nround = 0; total = 0;
}

// TMA = true: the candidate runs are staged by bulk asynchronous copies (one per run, completing on the warp's mbarrier);
// TMA = false: by ordinary 16-byte loads, one run per step with lane = entry (no per-copy service time of the TMA unit, which
// bounds the kernel when the runs are only a few hundred bytes long).
template <bool TMA>
__global__ void __launch_bounds__(SS_DC_WARPS * 32)
k_density_cells(SsDev P, SsDcArgs A) {
    __shared__ SsDcSlice s_slice[SS_DC_WARPS];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    SsDcSlice &S = s_slice[wib];
    const uint32_t n_cells = A.list_off[A.m - 1] + A.list_flag[A.m - 1];
    const uint32_t n_warps = gridDim.x * SS_DC_WARPS;
    if (TMA) { if (lane == 0) { ss_mbar_init(&S.mbar, 1); ss_mbar_fence_init(); } }
    __syncwarp();
    uint32_t phase = 0;
    const uint32_t lt_mask = (1u << lane) - 1u;
    // persistent warps over chunks of SS_DC_CHUNK consecutive cells: neighbouring cells share their subdomain (geometry is
    // recomputed only when it changes) and their candidate runs (L2 locality)
    uint32_t s_cached = 0xffffffffu;
    SsSubGeom g{};
    SsNsGrid ns{};
    for (uint32_t w0 = (blockIdx.x * SS_DC_WARPS + wib) * SS_DC_CHUNK; w0 < n_cells; w0 += n_warps * SS_DC_CHUNK) {
      const uint32_t w1 = min(w0 + (uint32_t)SS_DC_CHUNK, n_cells);
      for (uint32_t w = w0; w < w1; ++w) {
        const uint32_t a0 = A.list[w];
        const uint32_t k = A.key[a0];
        const uint32_t s = k / (uint32_t)P.ns_stride, cell = k - s * (uint32_t)P.ns_stride;
        const int nown = (int)(A.off[k + 1] - a0);
        if (s != s_cached) { g = ss_sub_geom(P, A.sub_flat[s]); ns = ss_ns_grid(P, g); s_cached = s; }
        const int c0 = (int)cell / (P.nsD * P.nsD), c1 = ((int)cell / P.nsD) % P.nsD, c2 = (int)cell % P.nsD;

        // ---- candidate runs.  Visiting order: (-1,0,1)^3 x-major without the centre, then the own cell.  The three z-cells of one
        // (sx, sy) column have consecutive keys, so their entries are ONE contiguous run of the sorted array: 9 runs, lane = column.
        // Only the centre column is out of order (own cell last): it is staged as it lies and the order is restored by index
        // arithmetic (ss_dc_phys).
        uint32_t run_a = 0, run_len = 0, own_before = 0;
        if (lane < 9) {
            const int q0 = c0 + lane / 3 - 1, q1 = c1 + lane % 3 - 1;
            if (q0 >= 0 && q1 >= 0 && q0 < ns.nc[0] && q1 < ns.nc[1]) {
                const uint32_t kb = s * (uint32_t)P.ns_stride + (uint32_t)((q0 * P.nsD + q1) * P.nsD);
                run_a = A.off[kb + (uint32_t)max(c2 - 1, 0)];
                run_len = A.off[kb + (uint32_t)min(c2 + 1, ns.nc[2] - 1) + 1u] - run_a;
                if (lane == 4) own_before = a0 - run_a;         // entries of the cell (0, 0, -1): they precede the own cell in its run
            }
        }
        uint32_t incl = run_len;
        for (int o = 1; o < 16; o <<= 1) { const uint32_t n = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += n; }
        const uint32_t run_dst = incl - run_len;
        const int C = (int)__shfl_sync(0xffffffffu, incl, 8);
        // physical position of the own cell inside the staged array, and where it sits in the visiting order (at the end)
        const int own_phys = (int)(__shfl_sync(0xffffffffu, run_dst, 4) + __shfl_sync(0xffffffffu, own_before, 4));
        const int own_log = C - nown;

        if (C > SS_DC_CAP) {
            // dense cluster: thread-serial routine, lane = particle of the cell
            SS_DC_NOTE("oversized cell");
            for (int t = lane; t < nown; t += 32) {
                const float4 pi = A.spos[a0 + t];
                if ((pi.x >= g.smin[0] && pi.y >= g.smin[1] && pi.z >= g.smin[2]) && (pi.x < g.smax[0] && pi.y < g.smax[1] && pi.z < g.smax[2]))
                    ss_density_entry<false>(P, ss_walk_sub(P, a0 + t, A.key, A.sub_flat, A.off), A.spos, A.rho, A.nbr_count,
                                            (const unsigned long long *)nullptr, (uint32_t *)nullptr);
            }
            continue;
        }

        // ---- stage the runs
        if (TMA) {
            ss_fence_proxy_async();                                // the previous cell's reads of the slice precede these writes
            __syncwarp();
            if (lane == 0) ss_mbar_arrive_expect_tx(&S.mbar, (uint32_t)C * 16u);
            __syncwarp();
            if (run_len) ss_bulk_g2s(&S.cand[run_dst], A.spos + run_a, run_len * 16u, &S.mbar);
            __syncwarp();
            ss_mbar_wait(&S.mbar, phase);
            phase ^= 1u;
        } else {
            __syncwarp();                                          // the previous cell's reads of the slice are done
#pragma unroll
            for (int r = 0; r < 9; ++r) {
                const uint32_t a = __shfl_sync(0xffffffffu, run_a, r), len = __shfl_sync(0xffffffffu, run_len, r), dst = __shfl_sync(0xffffffffu, run_dst, r);
                for (uint32_t t = lane; t < len; t += 32) S.cand[dst + t] = A.spos[a + t];
            }
            __syncwarp();
        }

        // ---- per particle of the cell: ordered hit list (lane = candidate in VISITING order), pooled per round of particles
        int nround = 0, total = 0;
        for (int t = 0; t < nown; ++t) {
            const float4 pi = S.cand[own_phys + t];
            if (!((pi.x >= g.smin[0] && pi.y >= g.smin[1] && pi.z >= g.smin[2]) && (pi.x < g.smax[0] && pi.y < g.smax[1] && pi.z < g.smax[2]))) continue;
            if (nround == SS_DC_MAXP || total > SS_DC_POOL - SS_DC_RESERVE) { SS_DC_NOTE(nround == SS_DC_MAXP ? "round full" : "pool nearly full"); ss_dc_flush(P, A, S, lane, nround, total); }
            const int selfc = own_log + t;
            int cnt = 0;
            bool over = false;
            for (int cb = 0; cb < C; cb += 32) {
                const int c = cb + lane;
                bool hit = false;
                float d2 = 0.0f;
                if (c < C && c != selfc) {
                    // visiting order -> staged position: the own cell's entries are visited last but lie inside the centre column
                    const int cp = c < own_phys ? c : (c < own_log ? c + nown : own_phys + (c - own_log));
                    const float4 pj = S.cand[cp];
                    const float dx = __fsub_rn(pj.x, pi.x), dy = __fsub_rn(pj.y, pi.y), dz = __fsub_rn(pj.z, pi.z);
                    d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
                    hit = d2 < P.h2;
                }
                const uint32_t bal = __ballot_sync(0xffffffffu, hit);
                const int nh = __popc(bal);
                if (total + cnt + nh > SS_DC_POOL) { over = true; SS_DC_NOTE("pool overflow"); break; }
                if (hit) S.pool[total + cnt + __popc(bal & lt_mask)] = d2;
                cnt += nh;
            }
            if (lane == 0) { S.ent[nround] = a0 + (uint32_t)t; S.base[nround] = total; S.cnt[nround] = over ? -1 : cnt; }
            if (!over) total += cnt;
            ++nround;
        }
        ss_dc_flush(P, A, S, lane, nround, total);
      }
    }
}
