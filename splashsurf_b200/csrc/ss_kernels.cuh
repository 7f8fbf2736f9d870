// ss_kernels.cuh -- device kernels of the H100 reconstruct path (included once by ss_pipeline.cu).
//
// Pipeline (one GPU):
//   k_aabb                      particle bounding box                         (aabb.rs:28-52)
//   k_classify_count/fill       owner + ghost subdomain memberships           (dense_subdomains.rs:1810-1905)
//   [cub radix sort]            -> per-subdomain ascending particle lists     (dense_subdomains.rs:476-488)
//   k_ns_keys + [sort] + k_density   per-subdomain cell lists, SPH densities  (neighborhood_search.rs:345-438,
//                                                                              density_map.rs:150-186)
//   k_bin_keys + [sort] + k_records  splat bins (8^3-point bricks) + particle records
//   k_brick_worklist + k_levelset    ordered cubic-spline gather per grid point; certify pass, then
//   k_brick_classify + k_fixup_flags + k_levelset(FIX)  exact values next to the surface (dense_subdomains.rs:784-1213)
//   k_mc_count + [scan] + k_mc_verts + k_mc_tris  marching cubes over listed bricks (dense_subdomains.rs:1470-1568)
//   k_weld_* / k_compact_*      boundary-vertex de-duplication ("stitching")  (dense_subdomains.rs:1603-1749)
#pragma once
#include "ss_common.cuh"
#include "mc_lut.inc"

__constant__ signed char c_tri_table[256][16];
__constant__ unsigned char c_num_tris[256];
// local edge -> (origin corner offset, axis), uniform_grid.rs:822-871
__constant__ signed char c_edge_org[12][3] = { {0,0,0},{1,0,0},{0,1,0},{0,0,0},{0,0,1},{1,0,1},{0,1,1},{0,0,1},{0,0,0},{1,0,0},{1,1,0},{0,1,0} };
__constant__ signed char c_edge_axis[12] = { 0, 1, 0, 1, 0, 1, 0, 1, 2, 2, 2, 2 };

// ------------------------------------------------------------------ AABB ----
__device__ __forceinline__ int ss_f2ord(float f) { int i = __float_as_int(f); return i >= 0 ? i : i ^ 0x7fffffff; }
__host__ __device__ inline float ss_ord2f(int i) {
    int j = i >= 0 ? i : i ^ 0x7fffffff;
#ifdef __CUDA_ARCH__
    return __int_as_float(j);
#else
    float f; memcpy(&f, &j, 4); return f;
#endif
}

__global__ void k_aabb(const float *__restrict__ xyz, uint64_t n, int *__restrict__ out /* min3, max3 ordered ints */) {
    int mn[3] = { INT_MAX, INT_MAX, INT_MAX }, mx[3] = { INT_MIN, INT_MIN, INT_MIN };
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
#pragma unroll
        for (int d = 0; d < 3; ++d) { int v = ss_f2ord(xyz[3 * i + d]); mn[d] = min(mn[d], v); mx[d] = max(mx[d], v); }
    }
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        for (int o = 16; o > 0; o >>= 1) {
            mn[d] = min(mn[d], __shfl_xor_sync(0xffffffffu, mn[d], o));
            mx[d] = max(mx[d], __shfl_xor_sync(0xffffffffu, mx[d], o));
        }
    }
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
        for (int d = 0; d < 3; ++d) { atomicMin(&out[d], mn[d]); atomicMax(&out[3 + d], mx[d]); }
    }
}

// particle AABB filter (lib.rs:369-406): half-open contains_point
__global__ void k_filter_flags(const float *__restrict__ xyz, uint64_t n, float3 mn, float3 mx,
                               uint8_t *__restrict__ flag, uint32_t *__restrict__ flag32) {
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= n) return;
    float x = xyz[3 * i], y = xyz[3 * i + 1], z = xyz[3 * i + 2];
    int in = (x >= mn.x && y >= mn.y && z >= mn.z) && (x < mx.x && y < mx.y && z < mx.z);
    flag[i] = (uint8_t)in; flag32[i] = (uint32_t)in;
}
__global__ void k_filter_scatter(const float *__restrict__ xyz, uint64_t n, const uint8_t *__restrict__ flag,
                                 const uint32_t *__restrict__ off, float *__restrict__ out) {
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= n || !flag[i]) return;
    uint32_t o = off[i];
    out[3 * (uint64_t)o] = xyz[3 * i]; out[3 * (uint64_t)o + 1] = xyz[3 * i + 1]; out[3 * (uint64_t)o + 2] = xyz[3 * i + 2];
}

// ------------------------------------------------------------------ decomposition ----
// Visits every subdomain the particle belongs to (owner + ghosts), dense_subdomains.rs:1810-1905.
template <typename F>
__device__ __forceinline__ int ss_classify(const SsDev &P, float px, float py, float pz, F &&emit) {
    float p[3] = { px, py, pz };
    int ijk[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        ijk[d] = ss_cell_of(p[d], P.gmin[d], P.sub_size);
        if (ijk[d] < 0 || ijk[d] >= P.nsd[d]) return 0;
    }
    float minc[3], maxc[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) { minc[d] = ss_coord(P.gmin[d], ijk[d], P.sub_size); maxc[d] = ss_coord(P.gmin[d], ijk[d] + 1, P.sub_size); }
    const int r = P.srad;
    int cnt = 0;
    for (int i = -r; i <= r; ++i) for (int j = -r; j <= r; ++j) for (int k = -r; k <= r; ++k) {
        int st[3] = { i, j, k };
        bool ok = true;
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            int s = st[d];
            float off = (float)(abs(s) - 1);
            if (s > 0) ok = ok && (__fsub_rn(__fadd_rn(maxc[d], __fmul_rn(off, P.sub_size)), p[d]) < P.margin);
            else if (s < 0) ok = ok && (__fsub_rn(p[d], __fsub_rn(minc[d], __fmul_rn(off, P.sub_size))) < P.margin);
        }
        if (!ok) continue;
        int t0 = ijk[0] + i, t1 = ijk[1] + j, t2 = ijk[2] + k;
        if (t0 < 0 || t1 < 0 || t2 < 0 || t0 >= P.nsd[0] || t1 >= P.nsd[1] || t2 >= P.nsd[2]) continue;
        {   // partitioned run: this rank keeps only its slab (+ density halo) of subdomains
            const int ta = P.part_axis == 0 ? t0 : (P.part_axis == 1 ? t1 : t2);
            if (ta < P.keep_lo || ta >= P.keep_hi) continue;
        }
        emit(cnt, (t0 * P.nsd[1] + t1) * P.nsd[2] + t2);
        ++cnt;
    }
    return cnt;
}

__global__ void k_classify_count(SsDev P, const float *__restrict__ xyz, uint32_t n, uint32_t *__restrict__ cnt) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    cnt[i] = (uint32_t)ss_classify(P, xyz[3 * (uint64_t)i], xyz[3 * (uint64_t)i + 1], xyz[3 * (uint64_t)i + 2], [](int, int) {});
}
__global__ void k_classify_fill(SsDev P, const float *__restrict__ xyz, uint32_t n, const uint32_t *__restrict__ off,
                                uint32_t *__restrict__ sub_flat, uint32_t *__restrict__ pidx) {
    uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    uint32_t o = off[i];
    ss_classify(P, xyz[3 * (uint64_t)i], xyz[3 * (uint64_t)i + 1], xyz[3 * (uint64_t)i + 2],
                [&](int m, int flat) { sub_flat[o + m] = (uint32_t)flat; pidx[o + m] = i; });
}

// membership index -> compressed subdomain id: segment heads flagged, then scanned
__global__ void k_seg_flags(const uint32_t *__restrict__ keys, uint32_t m, uint32_t *__restrict__ flag) {
    uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= m) return;
    flag[e] = (e == 0 || keys[e] != keys[e - 1]) ? 1u : 0u;
}
// after inclusive scan of flags: cid[e] = scan[e]-1; records each segment's flat id and start
__global__ void k_seg_finish(const uint32_t *__restrict__ keys, uint32_t m, const uint32_t *__restrict__ incl,
                             uint32_t *__restrict__ cid, uint32_t *__restrict__ sub_flat, uint32_t *__restrict__ sub_off) {
    uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= m) return;
    uint32_t id = incl[e] - 1;
    cid[e] = id;
    if (e == 0 || keys[e] != keys[e - 1]) { sub_flat[id] = keys[e]; sub_off[id] = e; }
    if (e == m - 1) sub_off[id + 1] = m;
}

struct SsSubGeom { float smin[3], smax[3]; int ijk[3]; };
__device__ __forceinline__ SsSubGeom ss_sub_geom(const SsDev &P, uint32_t flat) {
    SsSubGeom g;
    int f = (int)flat;
    g.ijk[0] = f / (P.nsd[1] * P.nsd[2]);
    g.ijk[1] = (f - g.ijk[0] * P.nsd[1] * P.nsd[2]) / P.nsd[2];
    g.ijk[2] = f - g.ijk[0] * P.nsd[1] * P.nsd[2] - g.ijk[1] * P.nsd[2];
#pragma unroll
    for (int d = 0; d < 3; ++d) { g.smin[d] = ss_coord(P.gmin[d], g.ijk[d], P.sub_size); g.smax[d] = ss_coord(P.gmin[d], g.ijk[d] + 1, P.sub_size); }
    return g;
}

// neighbourhood-search grid of one subdomain: from_aabb(subdomain aabb grown by 1.5*margin, h)
// (dense_subdomains.rs:560-565, uniform_grid.rs:175-201)
struct SsNsGrid { float amin[3]; int nc[3]; };
__device__ __forceinline__ SsNsGrid ss_ns_grid(const SsDev &P, const SsSubGeom &g) {
    SsNsGrid ns;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        float mmin = __fsub_rn(g.smin[d], P.grow), mmax = __fadd_rn(g.smax[d], P.grow);
        ns.amin[d] = __fmul_rn(floorf(__fdiv_rn(mmin, P.h)), P.h);
        float ext = __fsub_rn(mmax, ns.amin[d]);
        int n = (int)ceilf(__fdiv_rn(ext, P.h));
        ns.nc[d] = n > 1 ? n : 1;
    }
    return ns;
}

// ------------------------------------------------------------------ density ----
// key = cid * ns_stride + NS cell (x-major flat, padded to nsD per dim)
__global__ void k_ns_keys(SsDev P, const float *__restrict__ xyz, uint32_t m, const uint32_t *__restrict__ cid,
                          const uint32_t *__restrict__ sub_flat, const uint32_t *__restrict__ pidx,
                          uint32_t *__restrict__ key, int *__restrict__ err) {
    uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= m) return;
    uint32_t s = cid[e], p = pidx[e];
    SsSubGeom g = ss_sub_geom(P, sub_flat[s]);
    SsNsGrid ns = ss_ns_grid(P, g);
    int c[3];
    bool bad = false;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        c[d] = ss_cell_of(xyz[3 * (uint64_t)p + d], ns.amin[d], P.h);
        if (c[d] < 0 || c[d] >= ns.nc[d] || ns.nc[d] > P.nsD) { bad = true; c[d] = 0; }
    }
    if (bad && P.aniso) { key[e] = 0xffffffffu; return; }   // wide anisotropic margin: no density neighbour of an owned particle
    if (bad) atomicExch(err, 1);   // reference: unwrap() panic "particle outside NS grid"
    key[e] = s * (uint32_t)P.ns_stride + (uint32_t)((c[0] * P.nsD + c[1]) * P.nsD + c[2]);
}

// Dense (start, end) tables over a sorted key array: start[key] = first entry of the run (table pre-filled with
// 0xffffffff = empty), end[key] = one past its last entry.  Keys >= nkeys (dropped entries) are ignored.
__global__ void k_mark_starts(const uint32_t *__restrict__ key, uint32_t m, uint32_t *__restrict__ start, uint32_t nkeys) {
    uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= m) return;
    uint32_t k = key[e];
    if (k >= nkeys) return;
    if (e == 0 || k != key[e - 1]) start[k] = e;
}
__global__ void k_run_counts(const uint32_t *__restrict__ key, uint32_t m, uint32_t *__restrict__ end, uint32_t nkeys) {
    uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= m) return;
    uint32_t k = key[e];
    if (k >= nkeys) return;
    if (e == m - 1 || k != key[e + 1]) end[k] = e + 1;
}

// Cell offsets over a sorted key array, for k = 0 .. nkeys: off[k] = the first entry whose key is >= k (m if there is none).
// Cell k holds the entries [off[k], off[k+1]), and a run of consecutive cells [klo, khi] the entries [off[klo], off[khi+1]).
// Launched over m + 1 threads: entry e writes the keys in (key[e-1], key[e]], clipped to nkeys, and thread m fills up to nkeys,
// so every slot is written once and the table needs no fill.  Keys >= nkeys (members k_ns_keys dropped) sort behind every cell
// and lie in none.
__global__ void k_cell_offsets(const uint32_t *__restrict__ key, uint32_t m, uint32_t *__restrict__ off, uint32_t nkeys) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e > m) return;
    const uint32_t hi = e < m ? min(key[e], nkeys) : nkeys;
    const uint32_t lo = e > 0 ? min(key[e - 1], nkeys) + 1u : 0u;
    for (uint32_t k = lo; k <= hi; ++k) off[k] = e;
}

__global__ void k_gather_pos(const float *__restrict__ xyz, const uint32_t *__restrict__ pidx, uint32_t m,
                             float4 *__restrict__ out) {
    uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= m) return;
    uint32_t p = pidx[e];
    out[e] = make_float4(xyz[3 * (uint64_t)p], xyz[3 * (uint64_t)p + 1], xyz[3 * (uint64_t)p + 2], __uint_as_float(p));
}

// Membership entries whose particle lies inside its subdomain's half-open AABB (aabb.rs:220-222): only those get a density.
// Roughly half of the entries are ghosts, so k_density runs over the compacted list of the others (full warps).
__global__ void k_density_flags(SsDev P, uint32_t m, const uint32_t *__restrict__ key, const float4 *__restrict__ spos,
                                const uint32_t *__restrict__ sub_flat, uint32_t *__restrict__ flag) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= m) return;
    if (key[e] == 0xffffffffu) { flag[e] = 0u; return; }       // dropped member (anisotropic margin, k_ns_keys)
    const uint32_t s = key[e] / (uint32_t)P.ns_stride;
    const float4 pi = spos[e];
    const SsSubGeom g = ss_sub_geom(P, sub_flat[s]);
    const bool inside = (pi.x >= g.smin[0] && pi.y >= g.smin[1] && pi.z >= g.smin[2]) &&
                        (pi.x < g.smax[0] && pi.y < g.smax[1] && pi.z < g.smax[2]);
    flag[e] = inside ? 1u : 0u;
}

// The neighbour cells of one entry as 12 runs of consecutive entries of the cell-sorted array, in the reference's visiting
// order (26 adjacent cells x-major, then the own cell; ascending index inside a cell).  The three z-cells of an (x, y) column
// have consecutive keys, so a column is one run:
//   runs 0-3: columns (-1,-1), (-1,0), (-1,1), (0,-1);   run 4: cell (0,0,-1);   run 5: cell (0,0,+1);
//   runs 6-9: columns (0,1), (1,-1), (1,0), (1,1);       runs 10, 11: the own cell before and after the entry itself.
// Cells outside [0, nc) per dimension are clipped, as the reference skips them.
#define SS_WALK_RUNS 12
struct SsWalk {
    const uint32_t *off;         // cell offsets (k_cell_offsets)
    uint32_t base;               // key of the grid's cell (0, 0, 0)
    uint32_t e;                  // the entry itself
    int sx, sy;                  // key strides of x and y (z: 1)
    int c[3], nc[3];             // own cell, cells per dimension
};

// per-subdomain grids: key = subdomain * ns_stride + x-major cell, padded to nsD per dimension
__device__ __forceinline__ SsWalk ss_walk_sub(const SsDev &P, const uint32_t e, const uint32_t *__restrict__ key,
                                              const uint32_t *__restrict__ sub_flat, const uint32_t *__restrict__ off) {
    const uint32_t k = key[e];
    const uint32_t s = k / (uint32_t)P.ns_stride, cell = k - s * (uint32_t)P.ns_stride;
    const SsNsGrid ns = ss_ns_grid(P, ss_sub_geom(P, sub_flat[s]));
    SsWalk W;
    W.off = off; W.base = s * (uint32_t)P.ns_stride; W.e = e; W.sx = P.nsD * P.nsD; W.sy = P.nsD;
    W.c[0] = (int)cell / W.sx; W.c[1] = ((int)cell / P.nsD) % P.nsD; W.c[2] = (int)cell % P.nsD;
    for (int d = 0; d < 3; ++d) W.nc[d] = ns.nc[d];
    return W;
}

// the global path's grid over the whole domain: key = x-major cell
__device__ __forceinline__ SsWalk ss_walk_global(const SsDev &P, const uint32_t e, const uint32_t *__restrict__ key, const uint32_t *__restrict__ off) {
    const int cell = (int)key[e];
    SsWalk W;
    W.off = off; W.base = 0; W.e = e; W.sx = P.g_ns_nc[1] * P.g_ns_nc[2]; W.sy = P.g_ns_nc[2];
    W.c[0] = cell / W.sx; W.c[1] = (cell / W.sy) % P.g_ns_nc[1]; W.c[2] = cell % W.sy;
    for (int d = 0; d < 3; ++d) W.nc[d] = P.g_ns_nc[d];
    return W;
}

// entries [t, b) of run r (empty: t == b)
__device__ __forceinline__ void ss_walk_run(const SsWalk &W, const int r, uint32_t &t, uint32_t &b) {
    if (r >= 10) {
        const uint32_t own = W.base + (uint32_t)(W.c[0] * W.sx + W.c[1] * W.sy + W.c[2]);
        if (r == 10) { t = W.off[own]; b = W.e; } else { t = W.e + 1u; b = W.off[own + 1]; }
        return;
    }
    const int j = r < 4 ? r : (r < 6 ? 4 : r - 1);                       // column, (-1,0,1)^2 x-major
    const int q0 = W.c[0] + j / 3 - 1, q1 = W.c[1] + j % 3 - 1;
    const int zlo = max(r == 5 ? W.c[2] + 1 : W.c[2] - 1, 0), zhi = min(r == 4 ? W.c[2] - 1 : W.c[2] + 1, W.nc[2] - 1);
    t = b = 0u;
    if (q0 < 0 || q1 < 0 || q0 >= W.nc[0] || q1 >= W.nc[1] || zlo > zhi) return;
    const uint32_t kb = W.base + (uint32_t)(q0 * W.sx + q1 * W.sy);
    t = W.off[kb + zlo]; b = W.off[kb + zhi + 1];
}

// d^2 = |xj - xi|^2 with the reference's operation order; visit(pj, dx, dy, dz, d2) if d^2 < h^2
template <typename F>
__device__ __forceinline__ void ss_nbr_pair(const SsDev &P, const float4 &pi, const float4 &pj, F &visit) {
    const float dx = __fsub_rn(pj.x, pi.x), dy = __fsub_rn(pj.y, pi.y), dz = __fsub_rn(pj.z, pi.z);
    const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
    if (d2 < P.h2) visit(pj, dx, dy, dz, d2);
}

// Neighbour walk of ONE entry (thread-serial): visit(pj, dx, dy, dz, d2) for every other particle with d^2 < h^2, in the
// reference's order, with dx = xj - xi.  Shared by the neighbour lists, the global path's densities, the fallback of the
// cell-cooperative density kernel (ss_density.cuh) and the anisotropy of a particle (ss_aniso.cuh).
template <typename F>
__device__ __forceinline__ void ss_nbr_walk(const SsDev &P, const SsWalk &W, const float4 &pi, const float4 *__restrict__ spos, F &&visit) {
    for (int r = 0; r < SS_WALK_RUNS; ++r) {
        uint32_t t, b;
        ss_walk_run(W, r, t, b);
        for (; t + 1u < b; t += 2u) {                                     // two independent loads in flight
            const float4 p0 = spos[t], p1 = spos[t + 1u];
            ss_nbr_pair(P, pi, p0, visit);
            ss_nbr_pair(P, pi, p1, visit);
        }
        if (t < b) ss_nbr_pair(P, pi, spos[t], visit);
    }
}

// The ordered neighbour sum of ONE entry (thread-serial), or with FILL its neighbour indices (global particle ids, in the
// reference's order) written into the CSR array prepared from the counts (Parameters::global_neighborhood_list,
// dense_subdomains.rs:617-639).
template <bool FILL>
__device__ __forceinline__ void ss_density_entry(const SsDev &P, const SsWalk &W, const float4 *__restrict__ spos, float *__restrict__ rho,
                                                 unsigned long long *__restrict__ nbr_count, const unsigned long long *__restrict__ nbr_off,
                                                 uint32_t *__restrict__ nbr_idx) {
    const float4 pi = spos[W.e];
    unsigned long long ncount = 0;
    const unsigned long long fill_base = FILL ? nbr_off[__float_as_uint(pi.w)] : 0ull;
    float acc = ss_kernel_scalar(P, 0.0f);
    ss_nbr_walk(P, W, pi, spos, [&](const float4 &pj, float, float, float, float d2) {
        if constexpr (FILL) nbr_idx[fill_base + ncount] = __float_as_uint(pj.w);
        else acc = __fadd_rn(acc, ss_kernel_scalar(P, __fsqrt_rn(d2)));
        ++ncount;
    });
    if (FILL) return;
    if (nbr_count) nbr_count[__float_as_uint(pi.w)] = ncount;
    rho[__float_as_uint(pi.w)] = __fmul_rn(acc, P.rest_mass);
}

// d^2 slots per thread of k_density's hit list (shared memory: SS_DENSITY_K * 4 B per thread)
#define SS_DENSITY_K 16
#define SS_DENSITY_BLOCK 128

// One thread per membership entry of the compacted list (entries with the particle inside its subdomain, ascending):
// rho = m * (W(0) + sum_j W(|xj - xi|)) with neighbours visited in the reference's order (neighborhood_search.rs:396-433,
// density_map.rs:169-185), plus the optional neighbour counts.  FILL = true writes the neighbour lists instead (thread-serial).
// The walk tests ~216 candidates for ~33 hits, so the kernel W(sqrt(d^2)) is not evaluated per candidate: every lane appends the
// d^2 of its hits to its list in shared memory (slot s of lane l at [32 s + l] of the warp's region: no bank conflicts), and when
// a lane's list may overflow in the next step the whole warp drains -- each lane folds its list into its sum in order, with all
// lanes converged.  The summation order is the visiting order, as in the reference.  The warp walks the 12 runs together,
// each run as long as its longest lane's, four candidates per step, and loads the next run's bounds while it walks the current one.
template <bool FILL>
__global__ void __launch_bounds__(SS_DENSITY_BLOCK)
k_density(SsDev P, uint32_t m, const uint32_t *__restrict__ list, const uint32_t *__restrict__ list_off, const uint32_t *__restrict__ list_flag,
          const uint32_t *__restrict__ key, const float4 *__restrict__ spos, const uint32_t *__restrict__ sub_flat, const uint32_t *__restrict__ off,
          float *__restrict__ rho, unsigned long long *__restrict__ nbr_count, const unsigned long long *__restrict__ nbr_off,
          uint32_t *__restrict__ nbr_idx) {
    const uint32_t n_list = list_off[m - 1] + list_flag[m - 1];
    const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x;
    if constexpr (FILL) {
        if (tid < n_list) ss_density_entry<true>(P, ss_walk_sub(P, list[tid], key, sub_flat, off), spos, rho, nbr_count, nbr_off, nbr_idx);
    } else {
        __shared__ float s_d2[SS_DENSITY_BLOCK * SS_DENSITY_K];
        if ((tid & ~31u) >= n_list) return;                               // whole warps only: the drains are warp-wide
        const bool live = tid < n_list;
        float *const slot = s_d2 + (threadIdx.x & ~31u) * SS_DENSITY_K + (threadIdx.x & 31u);
        SsWalk W{};
        float4 pi = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
        uint32_t t = 0u, b = 0u;
        if (live) {
            W = ss_walk_sub(P, list[tid], key, sub_flat, off);
            pi = spos[W.e];
            ss_walk_run(W, 0, t, b);
        }
        float acc = ss_kernel_scalar(P, 0.0f);
        int nl = 0;
        uint32_t ncount = 0;
        auto drain = [&]() {
            for (int s = 0; s < nl; ++s) acc = __fadd_rn(acc, ss_kernel_scalar(P, __fsqrt_rn(slot[32 * s])));
            ncount += (uint32_t)nl;
            nl = 0;
        };
        for (int r = 0; r < SS_WALK_RUNS; ++r) {
            uint32_t tn = 0u, bn = 0u;
            if (live && r + 1 < SS_WALK_RUNS) ss_walk_run(W, r + 1, tn, bn);
            while (__any_sync(0xffffffffu, t < b)) {
                if (t < b) {
                    // four candidates per step with their loads issued together; a hit's d^2 is stored unconditionally at
                    // the list's end and kept by advancing nl, so the step has no branches (nl <= K - 4 on entry)
                    const uint32_t last = b - t - 1u;
                    float4 q[4];
#pragma unroll
                    for (uint32_t i = 0; i < 4u; ++i) q[i] = spos[t + min(i, last)];
#pragma unroll
                    for (uint32_t i = 0; i < 4u; ++i) {
                        const float dx = __fsub_rn(q[i].x, pi.x), dy = __fsub_rn(q[i].y, pi.y), dz = __fsub_rn(q[i].z, pi.z);
                        const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
                        slot[32 * nl] = d2;
                        nl += (i <= last && d2 < P.h2) ? 1 : 0;
                    }
                    t += 4u;
                }
                if (__any_sync(0xffffffffu, nl > SS_DENSITY_K - 4)) drain();
            }
            t = tn; b = bn;
        }
        drain();
        if (!live) return;
        const uint32_t p = __float_as_uint(pi.w);
        if (nbr_count) nbr_count[p] = ncount;
        rho[p] = __fmul_rn(acc, P.rest_mass);
    }
}


// ---- global path: one neighbourhood-search grid over the whole domain (neighborhood_search.rs:148-230) ----
__global__ void k_ns_keys_global(SsDev P, const float *__restrict__ xyz, uint32_t n, uint32_t *__restrict__ key, uint32_t *__restrict__ idx,
                                 int *__restrict__ err) {
    uint32_t p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n) return;
    int c[3];
    bool bad = false;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        c[d] = ss_cell_of(xyz[3 * (uint64_t)p + d], P.g_ns_amin[d], P.h);
        if (c[d] < 0 || c[d] >= P.g_ns_nc[d]) { bad = true; c[d] = 0; }
    }
    if (bad) atomicExch(err, 1);
    key[p] = (uint32_t)((c[0] * P.g_ns_nc[1] + c[1]) * P.g_ns_nc[2] + c[2]);
    idx[p] = p;
}
template <bool FILL>
__global__ void __launch_bounds__(128)
k_density_global(SsDev P, uint32_t n, const uint32_t *__restrict__ key, const float4 *__restrict__ spos, const uint32_t *__restrict__ off,
                 float *__restrict__ rho, unsigned long long *__restrict__ nbr_count, const unsigned long long *__restrict__ nbr_off,
                 uint32_t *__restrict__ nbr_idx) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    ss_density_entry<FILL>(P, ss_walk_global(P, e, key, off), spos, rho, nbr_count, nbr_off, nbr_idx);
}

// ------------------------------------------------------------------ splat binning ----
// Bins are cubes of `be` cells (8 = one 8x8x8-point brick, unless h/c is large) of the subdomain tile plus a halo.
// Binning is only a conservative cull: a particle farther than h from every tile point is dropped (key 0xffffffff).
__global__ void k_bin_keys(SsDev P, const float *__restrict__ xyz, uint32_t m, const uint32_t *__restrict__ cid,
                           const uint32_t *__restrict__ sub_flat, const uint32_t *__restrict__ pidx,
                           const uint8_t *__restrict__ sub_owned, uint32_t *__restrict__ key) {
    uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= m) return;
    uint32_t s = cid[e], p = pidx[e];
    if (sub_owned && !sub_owned[s]) { key[e] = 0xffffffffu; return; }   // density-only halo subdomain
    SsSubGeom g = ss_sub_geom(P, sub_flat[s]);
    int b[3];
    bool drop = false;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        float u = (xyz[3 * (uint64_t)p + d] - g.smin[d]) * P.inv_c;        // local coordinate in cells
        if (u < -P.rr_cells || u > (float)P.S + P.rr_cells) drop = true;
        int bb = (int)floorf(u / (float)P.be) + P.nlo;
        bb = max(0, min(P.nbin - 1, bb));
        b[d] = bb;
    }
    key[e] = drop ? 0xffffffffu : s * (uint32_t)P.nbin_sub + (uint32_t)((b[0] * P.nbin + b[1]) * P.nbin + b[2]);
}

// particle record in bin-sorted order: (x, y, z, V = m / rho) + k_split of the AVX remainder lanes
__global__ void k_records(SsDev P, const float *__restrict__ xyz, const float *__restrict__ rho, uint32_t m,
                          const uint32_t *__restrict__ key, const uint32_t *__restrict__ pidx,
                          const uint32_t *__restrict__ sub_flat, float4 *__restrict__ rec, int *__restrict__ ksplit) {
    uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= m) return;
    uint32_t k = key[e];
    if (k == 0xffffffffu) return;
    uint32_t s = k / (uint32_t)P.nbin_sub, p = pidx[e];
    float x = xyz[3 * (uint64_t)p], y = xyz[3 * (uint64_t)p + 1], z = xyz[3 * (uint64_t)p + 2];
    float v = __fdiv_rn(P.rest_mass, rho[p]);                              // dense_subdomains.rs:1044
    rec[e] = make_float4(x, y, z, v);
    SsSubGeom g = ss_sub_geom(P, sub_flat[s]);
    // particle_influence_aabb along z (dense_subdomains.rs:660-693) and the 8-lane remainder (:1050-1051)
    int ck = ss_cell_of(z, g.smin[2], P.c);
    int lo = min(max(ck - P.R, 0), P.np);
    int up = max(min(ck + P.R + 2, P.np), 0);
    int rem = up > lo ? (up - lo) % 8 : 0;
    ksplit[e] = up - rem;
}

// ------------------------------------------------------------------ level set ----
#define SS_LS_THREADS 512
#define SS_LS_WARPS (SS_LS_THREADS / 32)
#define SS_LS_CAP 512            // candidates staged per brick; larger bricks take the slow exact path
#define SS_MARKER 3.0e38f        // "certified inside, exact value not computed" (always > threshold)

enum { SS_LS_EXACT_ALL = 0, SS_LS_CERTIFY = 1, SS_LS_FIX = 2 };

// per-tile constants of a batch, filled on the host (exact f32)
struct SsTile {
    int gbase[3];        // global point index of the tile's point (0,0,0): subdomain_ijk * S
    uint32_t s;          // compressed subdomain id
    uint32_t sparse;     // scalar-arithmetic subdomain (dense_subdomains.rs:1251, :1590) or simd disabled
    float smin[3];       // subdomain aabb.min (marching cubes vertex coordinates)
};

#include "ss_brick.cuh"

struct SsLsArgs {
    SsBins bins;
    const uint32_t *fix_bricks;  // SS_LS_FIX: list of flagged bricks (global brick index)
    const uint32_t *work_list;   // other modes: list of non-empty bricks to evaluate
    float *tiles;                // [batch][np^3]
    uint8_t *wflag;              // [batch][nb^3][16] warp boxes that need exact values (SS_LS_FIX)
    uint8_t *bstate;             // [batch][nb^3] 0: untouched (all zero), 1: every point certified inside, 2: has exact values
    unsigned long long *pairs;   // work counter (in-support evaluations), only with COUNT
    int mode;
};

// One exact accumulation step (the reference's arithmetic) of candidate `r` (x, y, z, V) into phi.
template <bool SPARSE, bool UNIFORM_FMA>
__device__ __forceinline__ void ss_accumulate(const SsDev &P, const float4 r, const int ks, const int k,
                                              const float gx, const float gy, const float gz, float &phi, unsigned &hits) {
    const float dx = __fsub_rn(r.x, gx), dy = __fsub_rn(r.y, gy), dz = __fsub_rn(r.z, gz);
    if (!SPARSE) {
        // dense_subdomains.rs:1071-1090 + :1110-1127
        const float d2 = __fmaf_rn(dz, dz, __fmaf_rn(dx, dx, __fmul_rn(dy, dy)));
        if (d2 < P.h2) {
            const float wgt = ss_kernel_avx(P, __fsqrt_rn(d2));
            if (UNIFORM_FMA) phi = __fmaf_rn(wgt, r.w, phi);
            else phi = (k < ks) ? __fmaf_rn(wgt, r.w, phi) : __fadd_rn(phi, __fmul_rn(wgt, r.w));
            ++hits;
        }
    } else {
        // dense_subdomains.rs:828-842 / :1181-1194
        const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
        if (d2 < P.h2m) {
            phi = __fadd_rn(phi, __fmul_rn(r.w, ss_kernel_scalar(P, __fsqrt_rn(d2))));
            ++hits;
        }
    }
}


// Global path (density_map.rs:677-736): the delta of stencil point n along an axis is built by n+1 sequential additions
// of the cell size to (min_supported_point - particle - cell_size); accepted when r^2 < kernel_evaluation_radius^2.
__device__ __forceinline__ void ss_accumulate_global(const SsDev &P, const float4 r, const int *imin, const float *dx0,
                                                     const int gi, const int gj, const int gk, float &phi, unsigned &hits) {
    const int nx = gi - imin[0], ny = gj - imin[1], nz = gk - imin[2];
    if ((unsigned)nx >= (unsigned)P.sup || (unsigned)ny >= (unsigned)P.sup || (unsigned)nz >= (unsigned)P.sup) return;
    float dx = dx0[0], dy = dx0[1], dz = dx0[2];
    for (int t = 0; t <= nx; ++t) dx = __fadd_rn(dx, P.c);
    for (int t = 0; t <= ny; ++t) dy = __fadd_rn(dy, P.c);
    for (int t = 0; t <= nz; ++t) dz = __fadd_rn(dz, P.c);
    const float rr = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
    if (rr < P.rev2) {
        phi = __fadd_rn(phi, __fmul_rn(r.w, ss_kernel_scalar(P, __fsqrt_rn(rr))));
        ++hits;
    }
}

// per candidate: allowed-domain test, first stencil point, start deltas (density_map.rs:645-697)
__device__ __forceinline__ bool ss_global_candidate(const SsDev &P, const float4 r, int *imin, float *dx0) {
    const float p[3] = { r.x, r.y, r.z };
    bool allowed = true;
#pragma unroll
    for (int d = 0; d < 3; ++d) allowed = allowed && (p[d] >= P.g_allow_min[d]) && (p[d] < P.g_allow_max[d]);
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const int cell = ss_cell_of(p[d], P.gmin[d], P.c);
        imin[d] = allowed ? cell - P.R : (1 << 30);          // never in range when the particle is skipped
        const float mp = ss_coord(P.gmin[d], cell - P.R, P.c);
        dx0[d] = __fsub_rn(__fsub_rn(mp, p[d]), P.c);
    }
    return allowed;
}

// A warp's set of grid points: origin + power-of-two dimensions (dx * dy * dz <= 32), clipped to the tile.
struct SsWarpBox { int i0, j0, k0, dx, dy, dz; };

// Everything a lane needs about its grid point and its warp's box.
struct SsLanePoint {
    int i, j, k, gi, gj, gk, k1;
    bool valid, warp_valid;
    float gx, gy, gz;                 // point coordinates (reference arithmetic)
    float bxl, bxh, byl, byh, bzl, bzh;   // warp box in world coordinates (culling only)
    size_t out_idx;
};
__device__ __forceinline__ SsLanePoint ss_lane_point(const SsDev &P, const SsTile &T, const SsWarpBox &W, int tile_idx, int lane, bool sparse) {
    SsLanePoint L;
    const int lk = lane & (W.dz - 1), lj = (lane / W.dz) & (W.dy - 1), li = lane / (W.dz * W.dy);
    L.i = W.i0 + li; L.j = W.j0 + lj; L.k = W.k0 + lk;
    L.valid = (li < W.dx) && (L.i < P.np) && (L.j < P.np) && (L.k < P.np);
    L.warp_valid = (W.i0 < P.np) && (W.j0 < P.np) && (W.k0 < P.np);
    L.gi = T.gbase[0] + L.i; L.gj = T.gbase[1] + L.j; L.gk = T.gbase[2] + L.k;
    // grid point coordinates from GLOBAL indices: x, y = mul then add, z fused in the AVX path
    // (dense_subdomains.rs:1068, :1101-1102); scalar path: point_coordinates (uniform_grid.rs:418-425)
    L.gx = ss_grid_xy(P, L.gi, 0);
    L.gy = ss_grid_xy(P, L.gj, 1);
    L.gz = ss_grid_z(P, L.gk, sparse);
    const int i1 = min(W.i0 + W.dx - 1, P.np - 1), j1 = min(W.j0 + W.dy - 1, P.np - 1), k1 = min(W.k0 + W.dz - 1, P.np - 1);
    L.k1 = k1;
    L.bxl = ss_grid_xy(P, T.gbase[0] + W.i0, 0); L.bxh = ss_grid_xy(P, T.gbase[0] + i1, 0);
    L.byl = ss_grid_xy(P, T.gbase[1] + W.j0, 1); L.byh = ss_grid_xy(P, T.gbase[1] + j1, 1);
    L.bzl = ss_grid_z(P, T.gbase[2] + W.k0, sparse); L.bzh = ss_grid_z(P, T.gbase[2] + k1, sparse);
    L.out_idx = (size_t)tile_idx * P.np * P.np * P.np + ((size_t)L.i * P.np + L.j) * P.np + L.k;
    return L;
}
__device__ __forceinline__ float ss_box_dist2(const SsLanePoint &L, const float4 r) {
    const float dx = fmaxf(fmaxf(L.bxl - r.x, r.x - L.bxh), 0.0f);
    const float dy = fmaxf(fmaxf(L.byl - r.y, r.y - L.byh), 0.0f);
    const float dz = fmaxf(fmaxf(L.bzl - r.z, r.z - L.bzh), 0.0f);
    return fmaf(dx, dx, fmaf(dy, dy, dz * dz));
}

// Certification of one warp box: true when every valid lane is provably inside (see k_levelset).
//
// Lower bound of the kernel shape f(q) = W(q h) / sigma as a cubic in s = q^2 (so no square root is needed):
//     g(s) = max(0, G0 + G1 s + G2 s^2 + G3 s^3) <= f(sqrt(s))   for all s >= 0
// (tools/fit_kernel_bound.py: linear program over a fine grid; g captures 94 % of the kernel's volume integral, zero at
// q = 0.755).  G0 carries an extra -1e-5 safety offset; the comparison keeps a 1e-4 relative margin on top.
#ifdef SS_EMUL_STATS   // work statistics of the certification sweep, CPU executor only (tools/certify_stats.py)
// per outcome o (0 certified in ring 0, 1 in ring 1, 2 not certified): [5 o + 0] boxes, [5 o + 1] words visited in ring 0,
// [5 o + 2] candidates evaluated in ring 0, [5 o + 3], [5 o + 4] same for ring 1
static std::atomic<unsigned long long> ss_emul_stats[15];
extern "C" void ss_emul_stats_read(unsigned long long *out, int reset) { for (int k = 0; k < 15; ++k) { out[k] = ss_emul_stats[k]; if (reset) ss_emul_stats[k] = 0; } }
#define SS_STATS_DECL unsigned long long st_[4] = { 0, 0, 0, 0 };
#define SS_STATS_WORD(ring, mword) do { st_[2 * (ring)] += 1; st_[2 * (ring) + 1] += __popc(mword); } while (0)
#define SS_STATS_DONE(outcome) do { if (lane == 0) { ss_emul_stats[5 * (outcome)] += 1; for (int q_ = 0; q_ < 4; ++q_) ss_emul_stats[5 * (outcome) + 1 + q_] += st_[q_]; } } while (0)
#else
#define SS_STATS_DECL
#define SS_STATS_WORD(ring, mword)
#define SS_STATS_DONE(outcome)
#endif
#define SS_G0 0.98199678f
#define SS_G1 -4.74153665f
#define SS_G2 8.78317336f
#define SS_G3 -6.1170936f
__device__ __forceinline__ bool ss_certify_box(const SsDev &P, const SsLanePoint &L, const float4 *s_rec, int C, int lane, int w0) {
    const float cert = (P.thr + fabsf(P.thr) * 1.0e-4f + 1.0e-30f) / P.a_sigma;     // compare the un-normalised sum
    const float inv_h2 = P.a_hinv * P.a_hinv;
    float sum = 0.0f;
    const int nwords = (C + 31) >> 5;
    SS_STATS_DECL
    // ring 0: candidates within 0.55 h of the warp box; only if some lane is still short, ring 1: 0.55 h .. 0.8 h.
    // Words are visited starting at the brick's own bin (closest particles first) and the warp stops as soon as every lane
    // has enough.
    float r_lo2 = -1.0f, r_hi2 = 0.3025f * P.h2;
    for (int ring = 0; ring < 2; ++ring) {
        for (int wi = 0; wi < nwords; ++wi) {
            int w = wi + w0; if (w >= nwords) w -= nwords;
            const int c = w * 32 + lane;
            bool keep = false;
            if (c < C) { const float db2 = ss_box_dist2(L, s_rec[c]); keep = (db2 < r_hi2) && !(db2 < r_lo2); }
            uint32_t mword = __ballot_sync(0xffffffffu, keep);
            SS_STATS_WORD(ring, mword);
            if (!mword) continue;
            while (mword) {
                const int cc = w * 32 + __ffs(mword) - 1;
                mword &= mword - 1;
                const float4 r = s_rec[cc];
                const float dx = r.x - L.gx, dy = r.y - L.gy, dz = r.z - L.gz;
                const float sq = fmaf(dx, dx, fmaf(dy, dy, dz * dz)) * inv_h2;
                const float g = fmaf(sq, fmaf(sq, fmaf(sq, SS_G3, SS_G2), SS_G1), SS_G0);
                sum = fmaf(fmaxf(g, 0.0f), r.w, sum);
            }
            // lanes outside the tile (clipped boxes) do not need a value
            if (__all_sync(0xffffffffu, !L.valid || (sum > cert))) { SS_STATS_DONE(ring); return true; }
        }
        r_lo2 = r_hi2; r_hi2 = 0.64f * P.h2;
    }
    SS_STATS_DONE(2);
    return false;
}

// Exact, ordered evaluation of one warp box from the sorted candidate keys; returns the lane's value.
template <bool GLOBAL>
__device__ __forceinline__ float ss_exact_box(const SsDev &P, const SsLanePoint &L, bool sparse, const float4 *s_rec, const int *s_ks,
                                              const unsigned long long *s_key, unsigned short *my_list, const int (*s_imin)[3],
                                              const float (*s_dx0)[3], int C, int lane, unsigned &hits) {
    const float cull2 = (GLOBAL ? P.rev2 : (sparse ? P.h2m : P.h2)) * 1.0001f;
    // per-warp compacted list (sorted order) of the candidates within h of the warp's point box
    int nlist = 0;
    bool all_fma = true;                                   // no lane of this warp in any candidate's remainder lanes
    const int nwords = (C + 31) >> 5;
    for (int w = 0; w < nwords; ++w) {
        const int rnk = w * 32 + lane;
        bool keep = false;
        int slot = 0;
        if (rnk < C) {
            slot = (int)(s_key[rnk] & 0xffffu);
            keep = ss_box_dist2(L, s_rec[slot]) < cull2;
            if (keep && s_ks[slot] <= L.k1) all_fma = false;
        }
        const uint32_t mword = __ballot_sync(0xffffffffu, keep);
        if (keep) my_list[nlist + __popc(mword & ((1u << lane) - 1u))] = (unsigned short)slot;
        nlist += __popc(mword);
    }
    all_fma = __all_sync(0xffffffffu, all_fma);
    __syncwarp();
    float phi = 0.0f;
    if (GLOBAL) {
        for (int n = 0; n < nlist; ++n) {
            const int slot = my_list[n];
            ss_accumulate_global(P, s_rec[slot], s_imin[slot], s_dx0[slot], L.gi, L.gj, L.gk, phi, hits);
        }
    } else if (sparse) {
        for (int n = 0; n < nlist; ++n) ss_accumulate<true, false>(P, s_rec[my_list[n]], 0, L.k, L.gx, L.gy, L.gz, phi, hits);
    } else if (all_fma) {
        for (int n = 0; n < nlist; ++n) ss_accumulate<false, true>(P, s_rec[my_list[n]], 0, L.k, L.gx, L.gy, L.gz, phi, hits);
    } else {
        for (int n = 0; n < nlist; ++n) { const int slot = my_list[n]; ss_accumulate<false, false>(P, s_rec[slot], s_ks[slot], L.k, L.gx, L.gy, L.gz, phi, hits); }
    }
    __syncwarp();
    return phi;
}

// Extension tasks: when the tile has 8 * (nb - 1) + 1 points per axis, the single point planes at index np - 1 are
// evaluated by the CTA of the last full brick (it already staged their candidates) instead of by 217 nearly idle
// CTAs per tile.  Task t of a brick with (ex, ey, ez) "last brick along x / y / z" flags:
//   0,1: x-face halves   2,3: y-face halves   4,5: z-face halves   6: xy-edge   7: xz-edge   8: yz-edge   9: corner
__device__ __forceinline__ bool ss_ext_task(int t, int bx, int by, int bz, bool ex, bool ey, bool ez, SsWarpBox &W, int &vbx, int &vby, int &vbz) {
    const int i0 = bx * 8, j0 = by * 8, k0 = bz * 8, iL = i0 + 8, jL = j0 + 8, kL = k0 + 8;
    vbx = bx; vby = by; vbz = bz;
    switch (t) {
        case 0: case 1: if (!ex) return false; W = SsWarpBox{ iL, j0 + 4 * t, k0, 1, 4, 8 }; vbx = bx + 1; return true;
        case 2: case 3: if (!ey) return false; W = SsWarpBox{ i0 + 4 * (t - 2), jL, k0, 4, 1, 8 }; vby = by + 1; return true;
        case 4: case 5: if (!ez) return false; W = SsWarpBox{ i0 + 4 * (t - 4), j0, kL, 4, 8, 1 }; vbz = bz + 1; return true;
        case 6: if (!(ex && ey)) return false; W = SsWarpBox{ iL, jL, k0, 1, 1, 8 }; vbx = bx + 1; vby = by + 1; return true;
        case 7: if (!(ex && ez)) return false; W = SsWarpBox{ iL, j0, kL, 1, 8, 1 }; vbx = bx + 1; vbz = bz + 1; return true;
        case 8: if (!(ey && ez)) return false; W = SsWarpBox{ i0, jL, kL, 8, 1, 1 }; vby = by + 1; vbz = bz + 1; return true;
        case 9: if (!(ex && ey && ez)) return false; W = SsWarpBox{ iL, jL, kL, 1, 1, 1 }; vbx = bx + 1; vby = by + 1; vbz = bz + 1; return true;
    }
    return false;
}
// virtual (index nb - 1) bricks covered by extension tasks: 0:x 1:y 2:z 3:xy 4:xz 5:yz 6:xyz  <- tasks
__device__ __forceinline__ int ss_ext_group(int t) { return t < 6 ? (t >> 1) : t - 3; }

// One CTA = one 8x8x8-point brick of one subdomain tile; one warp = a 2x4x4 point box; one lane = one point.
//
// Exact value of a point: phi = ordered fold over the subdomain's particles in ascending global index of
//     dense : phi = fma(W_avx(r), V, phi)  (or phi + W*V for the 8-lane remainder)   dense_subdomains.rs:1106-1128
//     sparse: phi = phi + V * W_scalar(r)                                            dense_subdomains.rs:1184-1194
// restricted to particles with d^2 < h^2 (dense) / d^2 < 1.01 h^2 (scalar).  Candidates come from the brick's
// neighbouring bins; each warp walks only the candidates within h of its own point box, in ascending index.
//
// Certification (SS_LS_CERTIFY): every term is >= 0, so the reference's value is >= any partial sum of its terms
// (up to ~1e-6 relative rounding).  A warp first sums -- with fast arithmetic, in any order -- the candidates
// near its box; if every lane already exceeds threshold * (1 + 1e-4) all its points are provably inside
// and only SS_MARKER is stored.  Otherwise the warp evaluates all its points exactly.  k_fixup_flags then finds
// marker points that touch an outside point (a surface-crossing edge needs both exact endpoints) and a second
// launch (SS_LS_FIX) evaluates those warp boxes exactly.
//
// Launch: SS_LS_CERTIFY / SS_LS_EXACT_ALL run over a work list of non-empty bricks (k_brick_worklist); with
// P.ext_bricks the list only holds bricks 0 .. nb-2 per axis and the last one also evaluates the np-1 planes
// (extension tasks).  SS_LS_FIX runs over the flagged bricks (any index, no extension).
// adds a warp's in-support evaluations to the work counter (COUNT instantiations)
__device__ __forceinline__ void ss_flush_hits(unsigned long long *pairs, unsigned hits, int lane) {
    unsigned long long np_ = hits;
    for (int o = 16; o > 0; o >>= 1) np_ += __shfl_xor_sync(0xffffffffu, np_, o);
    if (lane == 0 && np_) atomicAdd(pairs, np_);
}

template <bool COUNT, bool GLOBAL>
__global__ void __launch_bounds__(SS_LS_THREADS, 3)
k_levelset(SsDev P, SsLsArgs A) {
    __shared__ float4 s_rec[SS_LS_CAP];
    __shared__ int s_ks[SS_LS_CAP];
    __shared__ unsigned long long s_key[SS_LS_CAP];
    __shared__ unsigned short s_list[SS_LS_WARPS][SS_LS_CAP];
    __shared__ uint32_t s_rng[2][128];          // candidate runs (start, length)
    __shared__ uint32_t s_pre[129];
    __shared__ int s_ext_need[8];               // per virtual brick group: some extension warp needs exact values
    // global path only: per candidate the first stencil point index and the start value of the incremental deltas
    __shared__ int s_imin[GLOBAL ? SS_LS_CAP : 1][3];
    __shared__ float s_dx0[GLOBAL ? SS_LS_CAP : 1][3];

    const int nb = P.nb;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int mode = A.mode;
    const uint32_t brick_lin = (mode == SS_LS_FIX) ? A.fix_bricks[blockIdx.x] : A.work_list[blockIdx.x];
    const SsBrick B = ss_brick_from_lin(P, brick_lin);
    const int bx = B.bx, by = B.by, bz = B.bz, tile_idx = B.tile;
    const bool my_flag = (mode != SS_LS_FIX) || (A.wflag[(size_t)brick_lin * SS_LS_WARPS + warp] != 0);
    if (threadIdx.x < 8) s_ext_need[threadIdx.x] = 0;

    const SsTile T = A.bins.tile_tab[tile_idx];
    const bool sparse = GLOBAL || T.sparse != 0;

    // ---- candidate runs (+ the extension plane), one per thread
    const SsBrickBins K = ss_brick_bins(P, A.bins.brick_rng, bx, by, bz, P.ext_bricks && mode != SS_LS_FIX);
    const bool ex = K.ex, ey = K.ey, ez = K.ez;
    const int nyr = K.nyr;
    const int nruns = K.nruns;                   // host guarantees <= 128
    if ((int)threadIdx.x < nruns) {
        uint32_t a;
        const uint32_t len = ss_brick_run(P, A.bins, T.s, K, (int)threadIdx.x, a);
        s_rng[0][threadIdx.x] = a; s_rng[1][threadIdx.x] = len;
    }
    __syncthreads();
    if (warp == 0) {
        // exclusive prefix of the run lengths (<= 128 runs: 4 per lane)
        uint32_t v[4], tot = 0;
#pragma unroll
        for (int q = 0; q < 4; ++q) { int r = lane * 4 + q; v[q] = r < nruns ? s_rng[1][r] : 0; tot += v[q]; }
        uint32_t incl = tot;
        for (int o = 1; o < 32; o <<= 1) { uint32_t n = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += n; }
        uint32_t run = incl - tot;
#pragma unroll
        for (int q = 0; q < 4; ++q) { int r = lane * 4 + q; if (r < nruns) s_pre[r] = run; run += v[q]; }
        if (lane == 31) s_pre[128] = incl;
    }
    __syncthreads();
    const int C = (int)s_pre[128];
    if (C == 0) return;                          // tile is pre-zeroed: phi = 0 exactly (bstate stays 0)

    const SsWarpBox Wm = { bx * 8 + (warp >> 2) * 2, by * 8 + ((warp >> 1) & 1) * 4, bz * 8 + (warp & 1) * 4, 2, 4, 4 };
    SsWarpBox We = Wm;
    int vbx = bx, vby = by, vbz = bz;
    const bool has_ext = (ex || ey || ez) && warp < 10 && ss_ext_task(warp, bx, by, bz, ex, ey, ez, We, vbx, vby, vbz);
    unsigned hits = 0;

    if (C > SS_LS_CAP) {
        // ---- oversized brick (pathological clustering): every warp walks all candidates in ascending particle
        // index by repeated selection of the next-larger index.  O(C^2) but exact; no certification.
        for (int pass = 0; pass < 2; ++pass) {
            if (pass == 1 && !has_ext) break;
            const SsLanePoint L = ss_lane_point(P, T, pass ? We : Wm, tile_idx, lane, sparse);
            if (!L.warp_valid || (pass == 0 && !my_flag)) continue;
            float phi = 0.0f;
            long long last = -1;
            for (int done = 0; done < C; ++done) {
                unsigned long long best = ~0ull;
                for (int r = 0; r < nruns; ++r) {
                    uint32_t a = s_rng[0][r], len = s_rng[1][r];
                    for (uint32_t t = lane; t < len; t += 32) {
                        uint32_t pi = A.bins.pidx[a + t];
                        if ((long long)pi > last) { unsigned long long kk = ((unsigned long long)pi << 32) | (a + t); if (kk < best) best = kk; }
                    }
                }
                for (int o = 16; o > 0; o >>= 1) { unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o); if (other < best) best = other; }
                if (best == ~0ull) break;
                last = (long long)(best >> 32);
                uint32_t src = (uint32_t)(best & 0xffffffffu);
                float4 r = A.bins.rec[src];
                int ks = A.bins.ksplit[src];
                if (GLOBAL) { int im[3]; float d0[3]; if (ss_global_candidate(P, r, im, d0)) ss_accumulate_global(P, r, im, d0, L.gi, L.gj, L.gk, phi, hits); }
                else if (sparse) ss_accumulate<true, false>(P, r, ks, L.k, L.gx, L.gy, L.gz, phi, hits);
                else ss_accumulate<false, false>(P, r, ks, L.k, L.gx, L.gy, L.gz, phi, hits);
            }
            if (L.valid) A.tiles[L.out_idx] = phi;
        }
        if (mode != SS_LS_FIX && A.bstate) {
            if (threadIdx.x == 0) A.bstate[brick_lin] = 2;
            if (has_ext && lane == 0) A.bstate[(((size_t)tile_idx * nb + vbx) * nb + vby) * nb + vbz] = 2;
        }
        if (COUNT && A.pairs) ss_flush_hits(A.pairs, hits, lane);
        return;
    }

    // ---- stage candidates (bin order) in shared memory: one warp per run
    for (int r = warp; r < nruns; r += SS_LS_WARPS) {
        const uint32_t a = s_rng[0][r], len = s_rng[1][r], dst = s_pre[r];
        for (uint32_t t = lane; t < len; t += 32) {
            const uint32_t src = a + t;
            float4 rc = A.bins.rec[src];
            if (GLOBAL && !ss_global_candidate(P, rc, s_imin[dst + t], s_dx0[dst + t])) rc.w = 0.0f;   // skipped particle: no volume
            s_rec[dst + t] = rc; s_ks[dst + t] = A.bins.ksplit[src];
            s_key[dst + t] = ((unsigned long long)A.bins.pidx[src] << 32) | (dst + t);
        }
    }
    __syncthreads();

    // ---- certification of the warp's main box and (if any) its extension box
    // start the candidate sweep at the run that holds the brick's own bin
    int w0;
    {
        const int ox = min(max(ss_floor_div(8 * bx, P.be) + P.nlo - K.rx.x, 0), K.rx.y - K.rx.x), oy = min(max(ss_floor_div(8 * by, P.be) + P.nlo - K.ry.x, 0), nyr - 1);
        w0 = (int)(s_pre[ox * nyr + oy] >> 5);
        if (w0 >= ((C + 31) >> 5)) w0 = 0;
    }
    bool need_main, need_ext = false;
    {
        const SsLanePoint L = ss_lane_point(P, T, Wm, tile_idx, lane, sparse);
        need_main = L.warp_valid && my_flag;
        if (mode == SS_LS_CERTIFY && L.warp_valid) need_main = !ss_certify_box(P, L, s_rec, C, lane, w0);
    }
    if (has_ext) {
        const SsLanePoint L = ss_lane_point(P, T, We, tile_idx, lane, sparse);
        need_ext = L.warp_valid;
        if (mode == SS_LS_CERTIFY && L.warp_valid) need_ext = !ss_certify_box(P, L, s_rec, C, lane, w0);
        if (need_ext && lane == 0) s_ext_need[ss_ext_group(warp)] = 1;
    }
    const int main_need = __syncthreads_or(need_main ? 1 : 0);
    const int any_ext_need = s_ext_need[0] | s_ext_need[1] | s_ext_need[2] | s_ext_need[3] | s_ext_need[4] | s_ext_need[5] | s_ext_need[6];
    if (mode != SS_LS_FIX && A.bstate) {
        if (threadIdx.x == 0) A.bstate[brick_lin] = main_need ? 2 : 1;
        if (has_ext && lane == 0) A.bstate[(((size_t)tile_idx * nb + vbx) * nb + vby) * nb + vbz] = s_ext_need[ss_ext_group(warp)] ? 2 : 1;
    }
    const bool block_need = main_need || any_ext_need;
    if (!block_need) {
        if (mode == SS_LS_CERTIFY) {
            const SsLanePoint L = ss_lane_point(P, T, Wm, tile_idx, lane, sparse);
            if (L.valid) A.tiles[L.out_idx] = SS_MARKER;
            if (has_ext) { const SsLanePoint Le = ss_lane_point(P, T, We, tile_idx, lane, sparse); if (Le.valid) A.tiles[Le.out_idx] = SS_MARKER; }
        }
        return;
    }

    // ---- exact path: order the candidates by global particle index
    ss_sort_keys<false>(s_key, C);
    for (int pass = 0; pass < 2; ++pass) {
        if (pass == 1 && !has_ext) break;
        const SsLanePoint L = ss_lane_point(P, T, pass ? We : Wm, tile_idx, lane, sparse);
        if (!L.warp_valid) continue;
        const bool need = pass ? need_ext : need_main;
        if (!need) { if (mode == SS_LS_CERTIFY && L.valid) A.tiles[L.out_idx] = SS_MARKER; continue; }
        const float phi = ss_exact_box<GLOBAL>(P, L, sparse, s_rec, s_ks, s_key, s_list[warp], s_imin, s_dx0, C, lane, hits);
        if (L.valid) A.tiles[L.out_idx] = phi;
    }
    if (COUNT && A.pairs) ss_flush_hits(A.pairs, hits, lane);
}

// Work list of the level-set launch: one thread per brick; listed when any of its candidate bins holds particles
// (with extension bricks: bricks 0 .. nb-2 per axis, the last one looking one bin range further).
__global__ void k_brick_worklist(SsDev P, const SsTile *__restrict__ tile_tab, const int2 *__restrict__ brick_rng,
                                 const uint32_t *__restrict__ bin_start, uint32_t ntiles, uint32_t *__restrict__ flag) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    const uint32_t nb = (uint32_t)P.nb;
    if (b >= ntiles * nb * nb * nb) return;
    const SsBrick B = ss_brick_from_lin(P, b);
    if (P.ext_bricks && (B.bx == (int)nb - 1 || B.by == (int)nb - 1 || B.bz == (int)nb - 1)) { flag[b] = 0; return; }
    const SsBrickBins K = ss_brick_bins(P, brick_rng, B.bx, B.by, B.bz, P.ext_bricks != 0);
    const uint32_t s = tile_tab[B.tile].s;
    bool any = false;
    for (int X = K.rx.x; X <= K.rx.y && !any; ++X) for (int Y = K.ry.x; Y <= K.ry.y && !any; ++Y) {
        const uint32_t base = s * (uint32_t)P.nbin_sub + (uint32_t)((X * P.nbin + Y) * P.nbin);
        for (int Z = K.rz.x; Z <= K.rz.y; ++Z) if (bin_start[base + Z] != 0xffffffffu) { any = true; break; }
    }
    flag[b] = any ? 1u : 0u;
}

// ------------------------------------------------------------------ brick-indexed tile passes ----
// The passes below use the level-set grid (one CTA of 512 threads per 8x8x8-point brick, one thread per point) and the
// per-brick state the level-set kernel records, so that bricks in the bulk (all certified) or in the void (all zero) cost
// one state lookup instead of a sweep over their 512 grid points.
#define SS_TP_THREADS 512
__device__ __forceinline__ int ss_state_at(const SsDev &P, const uint8_t *__restrict__ bstate, const SsBrick &B, int dx, int dy, int dz) {
    const int x = B.bx + dx, y = B.by + dy, z = B.bz + dz;
    if (x < 0 || y < 0 || z < 0 || x >= P.nb || y >= P.nb || z >= P.nb) return -1;       // outside the tile: no constraint
    return bstate[(((size_t)B.tile * P.nb + x) * P.nb + y) * P.nb + z];
}
// the passes run over compacted lists of bricks: blockIdx.x -> list entry
__device__ __forceinline__ SsBrick ss_brick_of_block(const SsDev &P, const uint32_t *__restrict__ list) {
    return ss_brick_from_lin(P, list[blockIdx.x]);
}

// Classifies every brick of the batch from the states the level-set kernel recorded:
//   flag_mc : the brick can hold a surface-crossing edge or a triangle (not all 8 bricks its cells reach are uniformly
//             certified-inside or uniformly untouched)
//   flag_fix: the brick holds markers that may touch an outside point (it has exact values itself, or a face neighbour is
//             not fully certified)
__global__ void k_brick_classify(SsDev P, const uint8_t *__restrict__ bstate, uint32_t nbricks, uint32_t *__restrict__ flag_mc,
                                 uint32_t *__restrict__ flag_fix) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= nbricks) return;
    const SsBrick B = ss_brick_from_lin(P, b);
    const int st = bstate[b];
    bool uniform = (st == 0 || st == 1);
    if (uniform) {
#pragma unroll
        for (int q = 1; q < 8; ++q) { const int s2 = ss_state_at(P, bstate, B, q & 1, (q >> 1) & 1, (q >> 2) & 1); if (s2 != st && s2 != -1) uniform = false; }
    }
    flag_mc[b] = uniform ? 0u : 1u;
    bool fix = (st == 2);
    if (st == 1) {
        const int nbr[6][3] = { {1,0,0},{-1,0,0},{0,1,0},{0,-1,0},{0,0,1},{0,0,-1} };
#pragma unroll
        for (int q = 0; q < 6; ++q) { const int s2 = ss_state_at(P, bstate, B, nbr[q][0], nbr[q][1], nbr[q][2]); if (s2 != 1 && s2 != -1) fix = true; }
    }
    flag_fix[b] = fix ? 1u : 0u;
}
__global__ void k_compact_list(const uint32_t *__restrict__ flag, const uint32_t *__restrict__ off, uint32_t n, uint32_t *__restrict__ list) {
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b < n && flag[b]) list[off[b]] = b;
}
__device__ __forceinline__ bool ss_brick_point(const SsDev &P, const SsBrick &B, int &i, int &j, int &k, int &l) {
    i = B.bx * 8 + (threadIdx.x >> 6); j = B.by * 8 + ((threadIdx.x >> 3) & 7); k = B.bz * 8 + (threadIdx.x & 7);
    l = (i * P.np + j) * P.np + k;
    return i < P.np && j < P.np && k < P.np;
}
// block-wide exclusive scan of a small per-thread count; returns the thread's prefix, total in `total`
__device__ __forceinline__ uint32_t ss_block_excl_scan(uint32_t v, uint32_t &total) {
    __shared__ uint32_t s_w[SS_TP_THREADS / 32 + 1];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t incl = v;
    for (int o = 1; o < 32; o <<= 1) { uint32_t n = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += n; }
    if (lane == 31) s_w[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        uint32_t w = lane < SS_TP_THREADS / 32 ? s_w[lane] : 0, wi = w;
        for (int o = 1; o < SS_TP_THREADS / 32; o <<= 1) { uint32_t n = __shfl_up_sync(0xffffffffu, wi, o); if (lane >= o) wi += n; }
        if (lane < SS_TP_THREADS / 32) s_w[lane] = wi - w;
        if (lane == SS_TP_THREADS / 32 - 1) s_w[SS_TP_THREADS / 32] = wi;
    }
    __syncthreads();
    total = s_w[SS_TP_THREADS / 32];
    return s_w[warp] + incl - v;
}

// Marker points (certified inside, value unknown) that touch an outside point along a grid edge carry a
// surface-crossing edge, so they need their exact value: flag their warp box and list their brick for the
// SS_LS_FIX launch.  Only bricks that hold markers and are not surrounded by all-marker bricks are swept.
__global__ void __launch_bounds__(SS_TP_THREADS)
k_fixup_flags(SsDev P, const float *__restrict__ tiles, const uint32_t *__restrict__ list, uint8_t *__restrict__ wflag,
              uint32_t *__restrict__ brick_seen, uint32_t *__restrict__ fix_bricks, uint32_t *__restrict__ nfix /* [0]: bricks, [1]: points */) {
    const SsBrick B = ss_brick_of_block(P, list);
    int i, j, k, l;
    if (!ss_brick_point(P, B, i, j, k, l)) return;
    const int np = P.np;
    const float *phi = tiles + (size_t)B.tile * np * np * np;
    if (phi[l] != SS_MARKER) return;
    const float thr = P.thr;
    bool hit = false;
    if (i > 0) hit |= !(phi[l - np * np] > thr);
    if (i + 1 < np) hit |= !(phi[l + np * np] > thr);
    if (j > 0) hit |= !(phi[l - np] > thr);
    if (j + 1 < np) hit |= !(phi[l + np] > thr);
    if (k > 0) hit |= !(phi[l - 1] > thr);
    if (k + 1 < np) hit |= !(phi[l + 1] > thr);
    if (!hit) return;
    const int warp = (((i & 7) >> 1) << 2) | (((j & 7) >> 2) << 1) | ((k & 7) >> 2);
    wflag[(size_t)B.lin * SS_LS_WARPS + warp] = 1;
    if (atomicExch(&brick_seen[B.lin], 1u) == 0u) fix_bricks[atomicAdd(&nfix[0], 1u)] = B.lin;
    atomicAdd(&nfix[1], 1u);
}

// ------------------------------------------------------------------ marching cubes ----
// "Above" flag of a grid point.  Subdomain path: value > threshold (dense_subdomains.rs:1482).  Global path: a point with
// value >= threshold that has a neighbour below it is marked Above by the edge loop, every other point by value > threshold
// (narrow_band_extraction.rs:79-126, :179-184) -- the two differ only for value == threshold (neighbours inside the tile).
template <bool GLOBAL>
__device__ __forceinline__ bool ss_above(const float *__restrict__ phi, int l, int i, int j, int k, int np, float thr) {
    const float v = phi[l];
    if (v > thr) return true;
    if (!GLOBAL || v != thr) return false;
    bool below = false;
    if (i > 0) below |= phi[l - np * np] < thr;
    if (i + 1 < np) below |= phi[l + np * np] < thr;
    if (j > 0) below |= phi[l - np] < thr;
    if (j + 1 < np) below |= phi[l + np] < thr;
    if (k > 0) below |= phi[l - 1] < thr;
    if (k + 1 < np) below |= phi[l + 1] < thr;
    return below;
}
template <bool GLOBAL>
__device__ __forceinline__ int ss_case_index(const float *__restrict__ phi, int l, int i, int j, int k, int np, float thr) {
    int idx = ss_above<GLOBAL>(phi, l, i, j, k, np, thr) ? 1 : 0;                                   // corner 0 (0,0,0)
    idx |= ss_above<GLOBAL>(phi, l + np * np, i + 1, j, k, np, thr) ? 2 : 0;                        // corner 1 (1,0,0)
    idx |= ss_above<GLOBAL>(phi, l + np * np + np, i + 1, j + 1, k, np, thr) ? 4 : 0;               // corner 2 (1,1,0)
    idx |= ss_above<GLOBAL>(phi, l + np, i, j + 1, k, np, thr) ? 8 : 0;                             // corner 3 (0,1,0)
    idx |= ss_above<GLOBAL>(phi, l + 1, i, j, k + 1, np, thr) ? 16 : 0;                             // corner 4 (0,0,1)
    idx |= ss_above<GLOBAL>(phi, l + np * np + 1, i + 1, j, k + 1, np, thr) ? 32 : 0;               // corner 5 (1,0,1)
    idx |= ss_above<GLOBAL>(phi, l + np * np + np + 1, i + 1, j + 1, k + 1, np, thr) ? 64 : 0;      // corner 6 (1,1,1)
    idx |= ss_above<GLOBAL>(phi, l + np + 1, i, j + 1, k + 1, np, thr) ? 128 : 0;                   // corner 7 (0,1,1)
    return idx;
}
// does the edge between two grid values carry a vertex?
template <bool GLOBAL>
__device__ __forceinline__ bool ss_crossing(float a, float b, float thr) {
    return GLOBAL ? ((a >= thr) != (b >= thr))           // one end >= threshold, the other < (narrow_band_extraction.rs:79-102)
                  : ((a > thr) != (b > thr));            // endpoints on different sides (dense_subdomains.rs:1482)
}

// Pass 1 (over the bricks k_brick_classify listed): per tile point, which of its +x/+y/+z edges carry a vertex and how many
// triangles its cell emits; per brick the totals.  Unlisted bricks keep their pre-zeroed masks.
template <bool GLOBAL>
__global__ void __launch_bounds__(SS_TP_THREADS)
k_mc_count(SsDev P, const float *__restrict__ tiles, const uint32_t *__restrict__ list, uint8_t *__restrict__ vmask,
           uint32_t *__restrict__ vblk, uint32_t *__restrict__ tblk) {
    const SsBrick B = ss_brick_of_block(P, list);
    int i, j, k, l;
    const bool ok = ss_brick_point(P, B, i, j, k, l);
    const int np = P.np;
    uint32_t mask = 0, nt = 0;
    if (ok) {
        const float *phi = tiles + (size_t)B.tile * np * np * np;
        const float thr = P.thr;
        const float v0 = phi[l];
        if (i + 1 < np && ss_crossing<GLOBAL>(v0, phi[l + np * np], thr)) mask |= 1u;
        if (j + 1 < np && ss_crossing<GLOBAL>(v0, phi[l + np], thr)) mask |= 2u;
        if (k + 1 < np && ss_crossing<GLOBAL>(v0, phi[l + 1], thr)) mask |= 4u;
        if (mask) vmask[(size_t)B.tile * np * np * np + l] = (uint8_t)mask;
        if (i < P.S && j < P.S && k < P.S) nt = c_num_tris[ss_case_index<GLOBAL>(phi, l, i, j, k, np, thr)];
    }
    uint32_t packed = (nt << 16) | __popc(mask);            // <= 512*5 and 512*3: no overflow between halves
    for (int o = 16; o > 0; o >>= 1) packed += __shfl_xor_sync(0xffffffffu, packed, o);
    __shared__ uint32_t s_part[SS_TP_THREADS / 32];
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = packed;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t tot = 0;
        for (int w = 0; w < SS_TP_THREADS / 32; ++w) tot += s_part[w];
        vblk[blockIdx.x] = tot & 0xffffu; tblk[blockIdx.x] = tot >> 16;
    }
}

struct SsMcOut {
    float *verts;                 // [*][3]
    uint32_t *tris;               // [*][3]
    unsigned long long *vkeys;    // per provisional vertex: global edge key
    unsigned long long *bkeys;    // boundary list: key
    uint32_t *bids;               // boundary list: provisional vertex id
    uint32_t *bcount;             // boundary list length (atomic)
    uint32_t vbase, tbase;        // offsets of this batch in the global arrays
    uint32_t bcap;
};

// Pass 2: vertices on the edges owned by each point (dense_subdomains.rs:1498-1538); records the id of each
// point's first vertex in voff.
template <bool GLOBAL>
__global__ void __launch_bounds__(SS_TP_THREADS)
k_mc_verts(SsDev P, const float *__restrict__ tiles, const uint8_t *__restrict__ vmask, const uint32_t *__restrict__ vblk_off,
           const uint32_t *__restrict__ vblk, uint32_t *__restrict__ voff, const SsTile *__restrict__ tile_tab, const uint32_t *__restrict__ list,
           SsMcOut O) {
    if (vblk[blockIdx.x] == 0) return;
    const SsBrick B = ss_brick_of_block(P, list);
    int i, j, k, l;
    const bool ok = ss_brick_point(P, B, i, j, k, l);
    const int tile = B.tile;
    const int np = P.np;
    const size_t pt = (size_t)tile * np * np * np + l;
    const uint32_t mask = ok ? vmask[pt] : 0u;
    uint32_t total;
    const uint32_t pre = ss_block_excl_scan(__popc(mask), total);
    if (!mask) return;
    uint32_t vid = O.vbase + vblk_off[blockIdx.x] + pre;
    voff[pt] = vid;
    const float *phi = tiles + (size_t)tile * np * np * np;
    const SsTile T = tile_tab[tile];
    const float thr = P.thr;
    const float a = phi[l];
    const int o[3] = { i, j, k };
    float oc[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) oc[d] = ss_coord(T.smin[d], o[d], P.c);
#pragma unroll
    for (int ax = 0; ax < 3; ++ax) {
        if (!(mask & (1u << ax))) continue;
        const int stride = ax == 0 ? np * np : (ax == 1 ? np : 1);
        const float bval = phi[l + stride];
        float pos[3];
        if (!GLOBAL) {
            const float alpha = __fdiv_rn(__fsub_rn(thr, a), __fsub_rn(bval, a));      // dense_subdomains.rs:1516-1519
            const float one_m = __fsub_rn(1.0f, alpha);
#pragma unroll
            for (int d = 0; d < 3; ++d) {
                const float tc = (d == ax) ? ss_coord(T.smin[d], o[d] + 1, P.c) : oc[d];
                pos[d] = __fadd_rn(__fmul_rn(oc[d], one_m), __fmul_rn(tc, alpha));
            }
        } else {
            // narrow_band_extraction.rs:104-109: interpolate from the point >= threshold towards its neighbour below,
            // coordinates from the global grid
            const bool from_o = a >= thr;
            const float vp = from_o ? a : bval, vn = from_o ? bval : a;
            const float alpha = __fdiv_rn(__fsub_rn(thr, vp), __fsub_rn(vn, vp));
            const float one_m = __fsub_rn(1.0f, alpha);
#pragma unroll
            for (int d = 0; d < 3; ++d) {
                const float c0 = ss_coord(P.gmin[d], T.gbase[d] + o[d], P.c);
                const float c1 = (d == ax) ? ss_coord(P.gmin[d], T.gbase[d] + o[d] + 1, P.c) : c0;
                const float pc = from_o ? c0 : c1, nc = from_o ? c1 : c0;
                pos[d] = __fadd_rn(__fmul_rn(pc, one_m), __fmul_rn(nc, alpha));
            }
        }
        O.verts[3 * (size_t)vid] = pos[0]; O.verts[3 * (size_t)vid + 1] = pos[1]; O.verts[3 * (size_t)vid + 2] = pos[2];
        const unsigned long long key = ss_edge_key(T.gbase[0] + i, T.gbase[1] + j, T.gbase[2] + k, ax);
        O.vkeys[vid] = key;
        // boundary edge: an orthogonal coordinate on a tile face (uniform_grid.rs:332-338)
        bool boundary = false;
#pragma unroll
        for (int d = 0; d < 3; ++d) if (d != ax && (o[d] == 0 || o[d] == P.S)) boundary = true;
        if (boundary) {
            const uint32_t slot = atomicAdd(O.bcount, 1u);
            if (slot < O.bcap) { O.bkeys[slot] = key; O.bids[slot] = vid; }
        }
        ++vid;
    }
}

// Pass 3: triangles of the cell whose origin is each point (dense_subdomains.rs:1470-1552)
template <bool GLOBAL>
__global__ void __launch_bounds__(SS_TP_THREADS)
k_mc_tris(SsDev P, const float *__restrict__ tiles, const uint8_t *__restrict__ vmask, const uint32_t *__restrict__ tblk_off,
          const uint32_t *__restrict__ tblk, const uint32_t *__restrict__ voff, const uint32_t *__restrict__ list, SsMcOut O) {
    if (tblk[blockIdx.x] == 0) return;
    const SsBrick B = ss_brick_of_block(P, list);
    int i, j, k, l;
    const bool ok = ss_brick_point(P, B, i, j, k, l);
    const int tile = B.tile;
    const int np = P.np;
    const float *phi = tiles + (size_t)tile * np * np * np;
    int idx = 0, nt = 0;
    if (ok && i < P.S && j < P.S && k < P.S) { idx = ss_case_index<GLOBAL>(phi, l, i, j, k, np, P.thr); nt = c_num_tris[idx]; }
    uint32_t total;
    const uint32_t pre = ss_block_excl_scan((uint32_t)nt, total);
    if (!nt) return;
    uint32_t tid = O.tbase + tblk_off[blockIdx.x] + pre;
    const size_t tbase_pt = (size_t)tile * np * np * np;
    for (int q = 0; q < nt; ++q) {
#pragma unroll
        for (int mth = 0; mth < 3; ++mth) {
            const int le = c_tri_table[idx][3 * q + (2 - mth)];              // reversed triplet, lut.rs:338-342
            const int ax = c_edge_axis[le];
            const int lo = l + c_edge_org[le][0] * np * np + c_edge_org[le][1] * np + c_edge_org[le][2];
            const uint32_t below = vmask[tbase_pt + lo] & ((1u << ax) - 1u);
            O.tris[3 * (size_t)tid + mth] = voff[tbase_pt + lo] + __popc(below);
        }
        ++tid;
    }
}

// ------------------------------------------------------------------ SPH normals at the mesh vertices ----
// SphInterpolator::interpolate_normals (sph_interpolation.rs:82-133): n_i = normalize(sum_j V_j (x_j - x_i)/r * |grad W|(r))
// over particles with |x_j - x_i|^2 <= h^2, V_j = m_sphere / rho_j.  One thread per vertex; candidates are the bins of the
// tile the vertex lies in (every particle within h of a tile point is a member of that tile's subdomain).  The reference
// sums in R-tree traversal order; here: bin order (parity to rounding, not bit-exact).
struct SsNrmArgs {
    const float *verts; const unsigned long long *vkeys; uint32_t nv;
    const uint32_t *sub_flat; const uint8_t *sub_owned; uint32_t nsub;
    SsBins bins; const float *rho; float sphere_mass; float *normals;
};
__device__ __forceinline__ float ss_kernel_dq(const SsDev &P, float q) {          // kernel.rs:83-94, constant 3/(4 pi)
    const float k = __fdiv_rn(3.0f, __fmul_rn(4.0f, SS_PI_F));
    if (q < 1.0f) return __fmul_rn(k, __fadd_rn(__fmul_rn(-4.0f, q), __fmul_rn(__fmul_rn(3.0f, q), q)));
    else if (q < 2.0f) { const float x = __fsub_rn(2.0f, q); return __fmul_rn(__fmul_rn(-k, x), x); }
    return 0.0f;
}
__global__ void __launch_bounds__(128)
k_sph_normals(SsDev P, SsNrmArgs A) {
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= A.nv) return;
    const unsigned long long key = A.vkeys[v];
    const int g[3] = { (int)((key >> 42) & 0xfffff), (int)((key >> 22) & 0xfffff), (int)((key >> 2) & 0xfffff) };
    const float xi = A.verts[3 * (size_t)v], yi = A.verts[3 * (size_t)v + 1], zi = A.verts[3 * (size_t)v + 2];
    // find an active tile that contains the vertex' grid edge
    int t[3], found = -1;
    for (int combo = 0; combo < 8 && found < 0; ++combo) {
        bool ok = true;
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            int td = min(g[d] / P.S, P.nsd[d] - 1);
            if (combo & (1 << d)) { if (g[d] % P.S == 0 && td > 0) td -= 1; else ok = false; }
            t[d] = td;
        }
        if (!ok) continue;
        const uint32_t flat = (uint32_t)((t[0] * P.nsd[1] + t[1]) * P.nsd[2] + t[2]);
        uint32_t lo = 0, hi = A.nsub;
        while (lo < hi) { uint32_t mid = (lo + hi) >> 1; if (A.sub_flat[mid] < flat) lo = mid + 1; else hi = mid; }
        if (lo < A.nsub && A.sub_flat[lo] == flat && (!A.sub_owned || A.sub_owned[lo])) found = (int)lo;
    }
    float gx = 0.0f, gy = 0.0f, gz = 0.0f;
    if (found >= 0) {
        const float dqdr = __fdiv_rn(2.0f, P.h);
        // A brick's range covers the reach of its grid points, [8b - R, 8b + 7 + R); the vertex lies anywhere on its edge from lp
        // to lp + 1, so the upper end is taken from the brick of lp + 1 (which differs from lp's when lp % 8 == 7).
        int2 rng[3];
#pragma unroll
        for (int d = 0; d < 3; ++d) {
            const int lp = g[d] - t[d] * P.S;
            rng[d] = A.bins.brick_rng[min(lp >> 3, P.nb - 1)];
            rng[d].y = A.bins.brick_rng[min((lp + 1) >> 3, P.nb - 1)].y;
        }
        for (int X = rng[0].x; X <= rng[0].y; ++X) for (int Y = rng[1].x; Y <= rng[1].y; ++Y) {
            uint32_t a;
            const uint32_t len = ss_bin_column(P, A.bins.bin_start, A.bins.bin_end, (uint32_t)found, X, Y, rng[2].x, rng[2].y, a);
            for (uint32_t e = a; e < a + len; ++e) {
                const float4 r = A.bins.rec[e];
                const float dx = __fsub_rn(r.x, xi), dy = __fsub_rn(r.y, yi), dz = __fsub_rn(r.z, zi);
                const float d2 = __fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz));
                if (!(d2 <= P.h2)) continue;
                const float rr = __fsqrt_rn(d2);
                const float q = __fdiv_rn(__fadd_rn(rr, rr), P.h);
                const float gn = __fmul_rn(__fmul_rn(P.s_sigma, ss_kernel_dq(P, q)), dqdr);
                const float vol = __fdiv_rn(A.sphere_mass, A.rho[A.bins.pidx[e]]);
                gx = __fadd_rn(gx, __fmul_rn(__fmul_rn(__fdiv_rn(dx, rr), gn), vol));
                gy = __fadd_rn(gy, __fmul_rn(__fmul_rn(__fdiv_rn(dy, rr), gn), vol));
                gz = __fadd_rn(gz, __fmul_rn(__fmul_rn(__fdiv_rn(dz, rr), gn), vol));
            }
        }
    }
    const float nrm = __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(gx, gx), __fmul_rn(gy, gy)), __fmul_rn(gz, gz)));
    A.normals[3 * (size_t)v] = __fdiv_rn(gx, nrm); A.normals[3 * (size_t)v + 1] = __fdiv_rn(gy, nrm); A.normals[3 * (size_t)v + 2] = __fdiv_rn(gz, nrm);
}

// ------------------------------------------------------------------ stitching (weld) ----
// Sorted boundary list (key, provisional id): duplicates of a key map to the smallest id of the run.
__global__ void k_weld_runs(const unsigned long long *__restrict__ bkeys, const uint32_t *__restrict__ bids, uint32_t nb,
                            uint32_t *__restrict__ remap, uint32_t *__restrict__ keep) {
    uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= nb) return;
    if (e > 0 && bkeys[e] == bkeys[e - 1]) return;          // run heads only
    uint32_t best = bids[e];
    uint32_t f = e + 1;
    while (f < nb && bkeys[f] == bkeys[e]) { best = min(best, bids[f]); ++f; }
    for (uint32_t q = e; q < f; ++q) { uint32_t id = bids[q]; remap[id] = best; if (id != best) keep[id] = 0; }
}
__global__ void k_gather_keys(const unsigned long long *__restrict__ keys, const uint32_t *__restrict__ ids, uint32_t n,
                              unsigned long long *__restrict__ out) {
    uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e < n) out[e] = keys[ids[e]];
}
__global__ void k_iota_keep(uint32_t n, uint32_t *__restrict__ remap, uint32_t *__restrict__ keep) {
    uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    remap[e] = e; keep[e] = 1;
}
__global__ void k_compact_verts(uint32_t n, const uint32_t *__restrict__ keep, const uint32_t *__restrict__ newid,
                                const float *__restrict__ vin, const unsigned long long *__restrict__ kin,
                                float *__restrict__ vout, unsigned long long *__restrict__ kout) {
    uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n || !keep[e]) return;
    uint32_t o = newid[e];
    vout[3 * (size_t)o] = vin[3 * (size_t)e]; vout[3 * (size_t)o + 1] = vin[3 * (size_t)e + 1]; vout[3 * (size_t)o + 2] = vin[3 * (size_t)e + 2];
    kout[o] = kin[e];
}
__global__ void k_remap_tris(uint64_t n3, const uint32_t *__restrict__ remap, const uint32_t *__restrict__ newid,
                             uint32_t *__restrict__ tris) {
    uint64_t e = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (e >= n3) return;
    tris[e] = newid[remap[tris[e]]];
}
__global__ void k_tris_to_u64(uint64_t n3, const uint32_t *__restrict__ in, unsigned long long *__restrict__ out) {
    uint64_t e = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (e >= n3) return;
    out[e] = in[e];
}
