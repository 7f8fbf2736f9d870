// ss_levelset_mesh.cuh -- the surface of a level-set field meshed over a box at any cube size (ss_levelset_field_mesh_f32, DESIGN.md §16).
//
// The lattice is the field's grid origin gmin with spacing c; lattice point I (global index per axis) lies at (float)I * c rounded, then
// + gmin rounded (ss_grid_xy's formula), and gets the value evaluate() returns there.  The call's index range is cut into tiles of 64^3
// cells (65^3 points, the layout of ss_mc.cuh) and bricks of 8^3 points:
//   k_lm_groups     per field group (compressed subdomain, brick): whether its candidate bins hold a record
//   k_lm_tiles      per tile of the range, in chunks: whether some group with records can hold one of its points (tiles without are
//                   never materialised); k_lm_offset appends a chunk's listed tiles
//   k_lm_list       per brick of the batch's tiles: the same test -> the bricks to fold; k_lm_mc_flags adds their lower neighbours for
//                   marching cubes (a brick's cells reach into its upper neighbours)
//   k_lm_fold       warp per listed brick: the brick's points generated in place, keyed like k_field_keys; per distinct group key the
//                   group's candidates staged once (ss_stage_candidates with the field's range table) and folded by the lanes whose
//                   points carry that key, per batch of 32 points with k_field_fold's cull; groups above the slice send the brick to the
//                   4096-slot instantiation, then to k_lm_select (the selection walk), which take only the groups earlier tiers left
//   k_lm_mc_count / k_lm_mc_emit   the warp-per-brick marching cubes of ss_mc.cuh (row masks, column masks, 256-case table with the
//                   reversed triplet order, local vertex offsets) with the range's clip and the lattice's vertex endpoints
// Vertex endpoints: at c == cell the lattice is the field's grid, and the endpoints are those the reconstruction's marching cubes writes
// (ss_mc.cuh: subdomain corner smin + local index * c, smin = gmin + s * (c * S)), taken from the subdomain whose tile keeps the vertex
// when the reconstruction welds its copies (the lowest subdomain along every axis the edge does not run along), so the mesh is the
// reconstruction's raw mesh bit for bit; at any other c there are no subdomains and the endpoints are the lattice points themselves.
#pragma once

#define SS_LM_NB 9                     // bricks per tile axis: 65 points
#define SS_LM_WARPS 4                  // listed bricks per CTA of the default slice
#define SS_LM_TILE_CHUNK (1u << 22)    // tiles of the range tested per launch (k_lm_tiles)

struct SsLmGrid {
    float gmin[3];
    float c;                           // lattice spacing
    int Sb;                            // the field's subdomain size when c == cell (vertex endpoints), else 0
    float sub_size;                    // c * Sb
    int imin[3];                       // first lattice index of the range
    int npts[3];                       // lattice points of the range per axis
    int ntile[3];                      // tiles per axis
    float3 gmax;                       // the field's grid maximum
    const uint32_t *sub_flat;          // the field's subdomains with members, ascending flat index
    uint32_t nsub;
    const uint8_t *grp;                // [nsub][nb^3] 1: the group's candidate bins hold a record
    const uint32_t *tiles;             // the batch's tiles: linear index (tx * nty + ty) * ntz + tz over the range
};

// tile q of the batch: its tile coordinates and its points per axis (<= 65; fewer at the range's upper end)
struct SsLmTile { int t[3], lim[3]; };
__device__ __forceinline__ SsLmTile ss_lm_tile(const SsLmGrid &G, uint32_t lin) {
    SsLmTile T;
    T.t[2] = (int)(lin % (uint32_t)G.ntile[2]); lin /= (uint32_t)G.ntile[2];
    T.t[1] = (int)(lin % (uint32_t)G.ntile[1]); T.t[0] = (int)(lin / (uint32_t)G.ntile[1]);
#pragma unroll
    for (int d = 0; d < 3; ++d) T.lim[d] = min(65, G.npts[d] - 64 * T.t[d]);
    return T;
}

__device__ __forceinline__ float ss_lm_point(const SsLmGrid &G, int I, int d) { return __fadd_rn(__fmul_rn((float)I, G.c), G.gmin[d]); }

// Whether a field group with records can hold a point of the lattice box [I0, I1] (conservative): the cells of the box's points,
// clamped to the grid as k_field_keys clamps them, walked field brick by field brick.
__device__ bool ss_lm_reach(const SsDev &P, const SsLmGrid &G, const int (&I0)[3], const int (&I1)[3]) {
    int c0[3], c1[3];
    const float hi[3] = { G.gmax.x, G.gmax.y, G.gmax.z };
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const float x0 = ss_lm_point(G, I0[d], d), x1 = ss_lm_point(G, I1[d], d);
        if (x1 < P.gmin[d] || x0 > hi[d]) return false;
        const int last = P.nsd[d] * P.S - 1;
        c0[d] = x0 < P.gmin[d] ? 0 : min(max(ss_cell_of(x0, P.gmin[d], P.c), 0), last);
        c1[d] = x1 > hi[d] ? last : min(max(ss_cell_of(x1, P.gmin[d], P.c), 0), last);
    }
    const uint32_t nb3 = (uint32_t)(P.nb * P.nb * P.nb);
    // next cell of another field brick along an axis
    const auto next = [&](int cc) { const int sd = cc / P.S, lb = (cc - sd * P.S) >> 3; return min(sd * P.S + 8 * (lb + 1), (sd + 1) * P.S); };
    for (int cx = c0[0]; cx <= c1[0]; cx = next(cx)) {
        for (int cy = c0[1]; cy <= c1[1]; cy = next(cy)) {
            for (int cz = c0[2]; cz <= c1[2]; cz = next(cz)) {
                const int sd[3] = { cx / P.S, cy / P.S, cz / P.S };
                const uint32_t flat = (uint32_t)(((int64_t)sd[0] * P.nsd[1] + sd[1]) * P.nsd[2] + sd[2]);
                uint32_t lo = 0, up = G.nsub;
                while (lo < up) { const uint32_t mid = (lo + up) >> 1; if (G.sub_flat[mid] < flat) lo = mid + 1; else up = mid; }
                if (lo >= G.nsub || G.sub_flat[lo] != flat) continue;
                const int lb[3] = { (cx - sd[0] * P.S) >> 3, (cy - sd[1] * P.S) >> 3, (cz - sd[2] * P.S) >> 3 };
                if (G.grp[(size_t)lo * nb3 + (uint32_t)((lb[0] * P.nb + lb[1]) * P.nb + lb[2])]) return true;
            }
        }
    }
    return false;
}

__global__ void k_lm_groups(SsDev P, SsBins B, uint32_t ngroups, uint8_t *__restrict__ grp) {
    const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= ngroups) return;
    const uint32_t nb3 = (uint32_t)(P.nb * P.nb * P.nb), s = g / nb3, b = g - s * nb3;
    const SsBrickBins K = ss_brick_bins(P, B.brick_rng, (int)(b / (uint32_t)(P.nb * P.nb)), (int)(b / (uint32_t)P.nb % (uint32_t)P.nb), (int)(b % (uint32_t)P.nb), false);
    uint8_t any = 0;
    for (int r = 0; r < K.nruns && !any; ++r) { uint32_t a; if (ss_brick_run(P, B, s, K, r, a)) any = 1; }
    grp[g] = any;
}

// tiles t0 .. t0 + ntiles - 1 of the range
__global__ void k_lm_tiles(SsDev P, SsLmGrid G, uint32_t t0, uint32_t ntiles, uint32_t *__restrict__ flag) {
    const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= ntiles) return;
    const uint32_t t = t0 + q;
    const SsLmTile T = ss_lm_tile(G, t);
    int I0[3], I1[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) { I0[d] = G.imin[d] + 64 * T.t[d]; I1[d] = I0[d] + T.lim[d] - 1; }
    flag[q] = ss_lm_reach(P, G, I0, I1) ? 1u : 0u;
}

// a chunk's listed tiles (chunk-relative) as tiles of the range
__global__ void k_lm_offset(const uint32_t *__restrict__ in, uint32_t n, uint32_t t0, uint32_t *__restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = in[i] + t0;
}

// brick lin = (q * 9 + bx) * 9 + by) * 9 + bz of the batch: listed when a group with records can hold one of its points
__global__ void k_lm_list(SsDev P, SsLmGrid G, uint32_t nbricks, uint32_t *__restrict__ flag) {
    const uint32_t lin = blockIdx.x * blockDim.x + threadIdx.x;
    if (lin >= nbricks) return;
    const int b[3] = { (int)(lin / 81u % 9u), (int)(lin / 9u % 9u), (int)(lin % 9u) };
    const SsLmTile T = ss_lm_tile(G, G.tiles[lin / 729u]);
    int I0[3], I1[3];
    bool on = true;
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        on = on && 8 * b[d] < T.lim[d];
        I0[d] = G.imin[d] + 64 * T.t[d] + 8 * b[d]; I1[d] = G.imin[d] + 64 * T.t[d] + min(8 * b[d] + 7, T.lim[d] - 1);
    }
    flag[lin] = (on && ss_lm_reach(P, G, I0, I1)) ? 1u : 0u;
}

// marching cubes reads a brick whose own points or whose upper neighbours' points were folded
__global__ void k_lm_mc_flags(const uint32_t *__restrict__ fold, uint32_t nbricks, uint32_t *__restrict__ mc) {
    const uint32_t lin = blockIdx.x * blockDim.x + threadIdx.x;
    if (lin >= nbricks) return;
    const int bx = (int)(lin / 81u % 9u), by = (int)(lin / 9u % 9u), bz = (int)(lin % 9u);
    uint32_t f = 0;
    for (int q = 0; q < 8; ++q) {
        const int x = bx + (q & 1), y = by + ((q >> 1) & 1), z = bz + (q >> 2);
        if (x < 9 && y < 9 && z < 9) f |= fold[lin + (uint32_t)((x - bx) * 81 + (y - by) * 9 + (z - bz))];
    }
    mc[lin] = f;
}

struct SsLmFoldArgs {
    SsAnArgs A;                        // the mode's records; A.bins.brick_rng: the field's candidate ranges
    SsLmGrid G;
    const uint32_t *bricks;            // this launch's bricks
    uint32_t n_bricks;
    uint32_t done;                     // groups with at most this many candidates were folded by an earlier tier
    float *tiles;                      // [batch][65^3], zero-filled
    uint32_t *fallback;                // bricks left to the next tier: [0] = count, [1..] = brick
};

// lane's point of batch qq (0..15) of the brick: local indices in the tile, and whether it lies in the range
__device__ __forceinline__ bool ss_lm_local(const SsLmTile &T, int bx, int by, int bz, int qq, int lane, int (&l)[3]) {
    l[0] = 8 * bx + (qq >> 1); l[1] = 8 * by + 4 * (qq & 1) + (lane >> 3); l[2] = 8 * bz + (lane & 7);
    return l[0] < T.lim[0] && l[1] < T.lim[1] && l[2] < T.lim[2];
}

// The group keys of the brick's 512 points into s_pk (0xffffffff: no group, value 0).  Returns the brick's tile.
__device__ __forceinline__ SsLmTile ss_lm_keys(const SsDev &P, const SsLmFoldArgs &L, uint32_t lin, int (&b)[3], uint32_t *s_pk, int lane) {
    b[0] = (int)(lin / 81u % 9u); b[1] = (int)(lin / 9u % 9u); b[2] = (int)(lin % 9u);
    const SsLmTile T = ss_lm_tile(L.G, L.G.tiles[lin / 729u]);
    for (int qq = 0; qq < 16; ++qq) {
        int l[3];
        uint32_t k = 0xffffffffu;
        if (ss_lm_local(T, b[0], b[1], b[2], qq, lane, l)) {
            float p[3];
#pragma unroll
            for (int d = 0; d < 3; ++d) p[d] = ss_lm_point(L.G, L.G.imin[d] + 64 * T.t[d] + l[d], d);
            bool finite;
            k = ss_field_key(P, p, L.G.gmax, L.G.sub_flat, L.G.nsub, finite);
        }
        s_pk[qq * 32 + lane] = k;
    }
    __syncwarp();
    return T;
}

// the smallest key of the brick above `prev` (any key when `first`), 0xffffffff when none is left
__device__ __forceinline__ uint32_t ss_lm_next_key(const uint32_t *s_pk, uint32_t prev, bool first, int lane) {
    uint32_t m = 0xffffffffu;
    for (int qq = 0; qq < 16; ++qq) { const uint32_t k = s_pk[qq * 32 + lane]; if (k != 0xffffffffu && (first || k > prev) && k < m) m = k; }
    for (int o = 16; o > 0; o >>= 1) m = min(m, __shfl_xor_sync(0xffffffffu, m, o));
    return m;
}

// group key -> compressed subdomain and candidate bins
__device__ __forceinline__ uint32_t ss_lm_group(const SsDev &P, const SsLmFoldArgs &L, uint32_t key, SsBrickBins &K) {
    const uint32_t nb3 = (uint32_t)(P.nb * P.nb * P.nb), s = key / nb3, b = key - s * nb3;
    K = ss_brick_bins(P, L.A.bins.brick_rng, (int)(b / (uint32_t)(P.nb * P.nb)), (int)(b / (uint32_t)P.nb % (uint32_t)P.nb), (int)(b % (uint32_t)P.nb), false);
    return s;
}

template <class F, int CAP, int WARPS>
__global__ void __launch_bounds__(WARPS * 32)
k_lm_fold(SsDev P, SsLmFoldArgs L) {
    __shared__ unsigned long long s_key[WARPS][CAP];
    __shared__ uint16_t s_list[WARPS][CAP];
    __shared__ uint32_t s_pk[WARPS][512];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t work = blockIdx.x * WARPS + wib;
    if (work >= L.n_bricks) return;
    const uint32_t lin = L.bricks[work];
    int b[3];
    const SsLmTile T = ss_lm_keys(P, L, lin, b, s_pk[wib], lane);
    float *tile = L.tiles + (size_t)(lin / 729u) * (65 * 65 * 65);
    const float cull2 = P.h2 * 1.0001f;
    bool pushed = false, first = true;
    uint32_t key = 0;
    for (;;) {
        key = ss_lm_next_key(s_pk[wib], key, first, lane);
        first = false;
        if (key == 0xffffffffu) break;
        SsBrickBins K;
        const uint32_t s = ss_lm_group(P, L, key, K);
        __syncwarp();                                        // the previous group's keys and list are read
        const uint32_t C = ss_stage_candidates<CAP>(P, L.A.bins, s, K, s_key[wib], lane);
        if (C == 0 || C <= L.done) continue;                 // pre-zeroed / folded by an earlier tier
        if (C > (uint32_t)CAP) {
            if (lane == 0 && !pushed) L.fallback[1 + atomicAdd(&L.fallback[0], 1u)] = lin;
            pushed = true;
            continue;
        }
        for (int qq = 0; qq < 16; ++qq) {
            int l[3];
            const bool valid = ss_lm_local(T, b[0], b[1], b[2], qq, lane, l);
            const bool on = valid && s_pk[wib][qq * 32 + lane] == key;
            const unsigned act = __ballot_sync(0xffffffffu, on);
            if (!act) continue;
            float p[3];
#pragma unroll
            for (int d = 0; d < 3; ++d) p[d] = ss_lm_point(L.G, L.G.imin[d] + 64 * T.t[d] + l[d], d);
            // the batch's bounding box over its points of this group (other lanes take the first such lane's point)
            const int src = __ffs(act) - 1;
            const float x0 = __shfl_sync(0xffffffffu, p[0], src), y0 = __shfl_sync(0xffffffffu, p[1], src), z0 = __shfl_sync(0xffffffffu, p[2], src);
            float xl = on ? p[0] : x0, xh = xl, yl = on ? p[1] : y0, yh = yl, zl = on ? p[2] : z0, zh = zl;
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
                    const float4 r = L.A.bins.rec[(uint32_t)s_key[wib][rnk]];
                    keep = ss_axis_d2(r.x, xl, xh) + ss_axis_d2(r.y, yl, yh) + ss_axis_d2(r.z, zl, zh) < cull2;
                }
                const uint32_t mword = __ballot_sync(0xffffffffu, keep);
                if (keep) s_list[wib][nlist + __popc(mword & ((1u << lane) - 1u))] = (uint16_t)rnk;
                nlist += __popc(mword);
            }
            __syncwarp();
            typename F::Acc acc = F::zero();
            for (int n = 0; n < nlist; ++n) F::add(P, F::load(L.A, (uint32_t)s_key[wib][s_list[wib][n]]), p[0], p[1], p[2], acc);
            if (on) tile[((size_t)l[0] * 65 + l[1]) * 65 + l[2]] = F::value(P, acc);
            __syncwarp();                                    // the list is rebuilt for the next batch
        }
    }
}

// Groups above the largest slice: per batch of 32 points the candidates in ascending particle index by repeated selection.
template <class F>
__global__ void __launch_bounds__(32)
k_lm_select(SsDev P, SsLmFoldArgs L) {
    __shared__ uint32_t s_pk[512];
    if (blockIdx.x >= L.n_bricks) return;
    const int lane = threadIdx.x & 31;
    const uint32_t lin = L.bricks[blockIdx.x];
    int b[3];
    const SsLmTile T = ss_lm_keys(P, L, lin, b, s_pk, lane);
    float *tile = L.tiles + (size_t)(lin / 729u) * (65 * 65 * 65);
    bool first = true;
    uint32_t key = 0;
    for (;;) {
        key = ss_lm_next_key(s_pk, key, first, lane);
        first = false;
        if (key == 0xffffffffu) break;
        SsBrickBins K;
        const uint32_t s = ss_lm_group(P, L, key, K);
        const uint32_t C = ss_stage_candidates<0>(P, L.A.bins, s, K, nullptr, lane);      // the count only
        if (C <= L.done) continue;
        for (int qq = 0; qq < 16; ++qq) {
            int l[3];
            const bool valid = ss_lm_local(T, b[0], b[1], b[2], qq, lane, l);
            const bool on = valid && s_pk[qq * 32 + lane] == key;
            if (!__any_sync(0xffffffffu, on)) continue;
            float p[3];
#pragma unroll
            for (int d = 0; d < 3; ++d) p[d] = ss_lm_point(L.G, L.G.imin[d] + 64 * T.t[d] + l[d], d);
            typename F::Acc acc = F::zero();
            unsigned long long last = 0;
            bool fst = true;
            for (;;) {
                const unsigned long long best = ss_select_next(P, L.A.bins, s, K, last, fst, lane);
                if (best == ~0ull) break;
                last = best; fst = false;
                F::add(P, F::load(L.A, (uint32_t)best), p[0], p[1], p[2], acc);
            }
            if (on) tile[((size_t)l[0] * 65 + l[1]) * 65 + l[2]] = F::value(P, acc);
        }
    }
}

// ---- marching cubes over the batch's tiles (P: S = 64, np = 65, nb = 9, thr)

// a column's masks clipped to the tile's points of the range: no edge to a point past it, no cell with such a corner
__device__ __forceinline__ void ss_lm_clip(SsMwColumn &C, int i, int j, int oz, const SsLmTile &T) {
    if (i >= T.lim[0] || j >= T.lim[1]) { C.ex = C.ey = C.ez = C.cells = 0; return; }
    const int nz = T.lim[2] - oz;                                           // own points of the column in the range
    const uint32_t pts = nz >= 8 ? 0xffu : (nz > 0 ? (1u << nz) - 1u : 0u);
    const uint32_t zed = nz - 1 >= 8 ? 0xffu : (nz - 1 > 0 ? (1u << (nz - 1)) - 1u : 0u);
    if (i + 1 >= T.lim[0]) C.ex = 0;
    if (j + 1 >= T.lim[1]) C.ey = 0;
    C.ex &= pts; C.ey &= pts; C.ez &= zed;
    C.cells = (i + 1 >= T.lim[0] || j + 1 >= T.lim[1]) ? 0u : (C.cells & zed);
}

// coordinate of the lattice point with global index I along axis d as the vertex endpoint: blk is its subdomain when G.Sb > 0
__device__ __forceinline__ float ss_lm_end(const SsLmGrid &G, int I, int d, int blk) {
    if (G.Sb == 0) return ss_lm_point(G, I, d);
    return ss_coord(ss_coord(G.gmin[d], blk, G.sub_size), I - blk * G.Sb, G.c);
}

__global__ void __launch_bounds__(SS_MW_WARPS * 32)
k_lm_mc_count(SsDev P, SsLmGrid G, const float *__restrict__ tiles, const uint32_t *__restrict__ list, uint32_t n_list, uint8_t *__restrict__ vmask,
              uint32_t *__restrict__ voff, uint32_t *__restrict__ vblk, uint32_t *__restrict__ tblk) {
    __shared__ SsMwSlice s_slice[SS_MW_WARPS];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t w = blockIdx.x * SS_MW_WARPS + wib;
    if (w >= n_list) return;
    SsMwSlice &S = s_slice[wib];
    const SsBrick B = ss_brick_from_lin(P, list[w]);
    const SsLmTile T = ss_lm_tile(G, G.tiles[B.tile]);
    const int np = P.np, ox = B.bx * 8, oy = B.by * 8, oz = B.bz * 8;
    const size_t tbase = (size_t)B.tile * np * np * np;
    ss_mw_rows(P, tiles + tbase, ox, oy, oz, S, lane);
    SsMwColumn C[2];
    uint32_t nv[2], nt[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int col = lane + 32 * h, a = col >> 3, b = col & 7;
        C[h] = ss_mw_column(P, S, a, b, ox + a, oy + b, oz);
        ss_lm_clip(C[h], ox + a, oy + b, oz, T);
        nv[h] = __popc(C[h].ex) + __popc(C[h].ey) + __popc(C[h].ez);
        nt[h] = ss_mw_column_tris(C[h]);
    }
    uint32_t total;
    uint32_t pre = ss_mw_scan((nv[0] + nv[1]) | ((nt[0] + nt[1]) << 16), lane, total) & 0xffffu;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int col = lane + 32 * h, a = col >> 3, b = col & 7;
        const size_t pt0 = tbase + ((size_t)(ox + a) * np + (oy + b)) * np + oz;
        for (uint32_t m = C[h].ex | C[h].ey | C[h].ez; m; m &= m - 1u) {
            const int k = __ffs(m) - 1;
            const uint32_t mask = ((C[h].ex >> k) & 1u) | (((C[h].ey >> k) & 1u) << 1) | (((C[h].ez >> k) & 1u) << 2);
            vmask[pt0 + k] = (uint8_t)mask;
            voff[pt0 + k] = pre;
            pre += __popc(mask);
        }
    }
    if (lane == 0) { vblk[w] = total & 0xffffu; tblk[w] = total >> 16; }
}

__global__ void __launch_bounds__(SS_MW_WARPS * 32)
k_lm_mc_emit(SsDev P, SsLmGrid G, const float *__restrict__ tiles, const uint32_t *__restrict__ list, uint32_t n_list, const uint8_t *__restrict__ vmask,
             const uint32_t *__restrict__ voff, const uint32_t *__restrict__ vblk, const uint32_t *__restrict__ tblk,
             const uint32_t *__restrict__ vblk_off, const uint32_t *__restrict__ tblk_off, const uint32_t *__restrict__ flag_mc,
             const uint32_t *__restrict__ off_mc, SsMcOut O) {
    __shared__ SsMwSlice s_slice[SS_MW_WARPS];
    const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t w = blockIdx.x * SS_MW_WARPS + wib;
    if (w >= n_list) return;
    const uint32_t nvb = vblk[w], ntb = tblk[w];
    if (nvb == 0 && ntb == 0) return;
    SsMwSlice &S = s_slice[wib];
    const SsBrick B = ss_brick_from_lin(P, list[w]);
    const SsLmTile T = ss_lm_tile(G, G.tiles[B.tile]);
    const int np = P.np, nb = P.nb, ox = B.bx * 8, oy = B.by * 8, oz = B.bz * 8;
    const size_t tbase = (size_t)B.tile * np * np * np;
    const float *phi = tiles + tbase;
    if (lane < 8) {
        const int x = B.bx + (lane & 1), y = B.by + ((lane >> 1) & 1), z = B.bz + (lane >> 2);
        uint32_t base = 0;
        if (x < nb && y < nb && z < nb) {
            const uint32_t lin = (uint32_t)((((size_t)B.tile * nb + x) * nb + y) * nb + z);
            if (flag_mc[lin]) base = O.vbase + vblk_off[off_mc[lin]];
        }
        S.base[lane] = base;
    }
    ss_mw_rows(P, phi, ox, oy, oz, S, lane);
    SsMwColumn C[2];
    uint32_t nt[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int col = lane + 32 * h, a = col >> 3, b = col & 7;
        C[h] = ss_mw_column(P, S, a, b, ox + a, oy + b, oz);
        ss_lm_clip(C[h], ox + a, oy + b, oz, T);
        nt[h] = ss_mw_column_tris(C[h]);
    }
    if (nvb) {
        const float thr = P.thr;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int col = lane + 32 * h, a = col >> 3, b = col & 7;
            const int i = ox + a, j = oy + b;
            for (uint32_t m = C[h].ex | C[h].ey | C[h].ez; m; m &= m - 1u) {
                const int kk = __ffs(m) - 1, k = oz + kk;
                const int l = (i * np + j) * np + k;
                uint32_t vid = S.base[0] + voff[tbase + l];
                const float av = phi[l];
                const int o[3] = { i, j, k };
                int I[3];
#pragma unroll
                for (int d = 0; d < 3; ++d) I[d] = G.imin[d] + 64 * T.t[d] + o[d];
#pragma unroll
                for (int ax = 0; ax < 3; ++ax) {
                    const uint32_t em = ax == 0 ? C[h].ex : (ax == 1 ? C[h].ey : C[h].ez);
                    if (!((em >> kk) & 1u)) continue;
                    const int stride = ax == 0 ? np * np : (ax == 1 ? np : 1);
                    const float bval = phi[l + stride];
                    const float alpha = __fdiv_rn(__fsub_rn(thr, av), __fsub_rn(bval, av));
                    const float one_m = __fsub_rn(1.0f, alpha);
                    float pos[3];
#pragma unroll
                    for (int d = 0; d < 3; ++d) {
                        // the subdomain of the kept copy: along the edge the one holding it, across it the lowest holding the point
                        const int blk = G.Sb == 0 ? 0 : (d == ax ? I[d] / G.Sb : (I[d] > 0 ? (I[d] - 1) / G.Sb : 0));
                        const float ac = ss_lm_end(G, I[d], d, blk);
                        const float bc = d == ax ? ss_lm_end(G, I[d] + 1, d, blk) : ac;
                        pos[d] = __fadd_rn(__fmul_rn(ac, one_m), __fmul_rn(bc, alpha));
                    }
                    O.verts[3 * (size_t)vid] = pos[0]; O.verts[3 * (size_t)vid + 1] = pos[1]; O.verts[3 * (size_t)vid + 2] = pos[2];
                    const unsigned long long key = ss_edge_key(I[0], I[1], I[2], ax);
                    O.vkeys[vid] = key;
                    bool boundary = false;                           // an orthogonal coordinate on a tile face: welded across tiles
#pragma unroll
                    for (int d = 0; d < 3; ++d) if (d != ax && (o[d] == 0 || o[d] == 64)) boundary = true;
                    if (boundary) {
                        const uint32_t slot = atomicAdd(O.bcount, 1u);
                        if (slot < O.bcap) { O.bkeys[slot] = key; O.bids[slot] = vid; }
                    }
                    ++vid;
                }
            }
        }
    }
    if (ntb) {
        uint32_t total;
        uint32_t tid = O.tbase + tblk_off[w] + (ss_mw_scan((nt[0] + nt[1]) << 16, lane, total) >> 16);
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int col = lane + 32 * h, a = col >> 3, b = col & 7;
            const int i = ox + a, j = oy + b;
            for (uint32_t m = C[h].cells; m; m &= m - 1u) {
                const int kk = __ffs(m) - 1;
                const int idx = ss_mw_case(C[h], kk);
                const int ntc = c_num_tris[idx];
                const int l = (i * np + j) * np + oz + kk;
                for (int q = 0; q < ntc; ++q) {
#pragma unroll
                    for (int mth = 0; mth < 3; ++mth) {
                        const int le = c_tri_table[idx][3 * q + (2 - mth)];
                        const int ax = c_edge_axis[le];
                        const int da = c_edge_org[le][0], db = c_edge_org[le][1], dc = c_edge_org[le][2];
                        const int lo = l + da * np * np + db * np + dc;
                        const int qn = ((a + da) >> 3) | (((b + db) >> 3) << 1) | (((kk + dc) >> 3) << 2);
                        const uint32_t below = vmask[tbase + lo] & ((1u << ax) - 1u);
                        O.tris[3 * (size_t)tid + mth] = S.base[qn] + voff[tbase + lo] + __popc(below);
                    }
                    ++tid;
                }
            }
        }
    }
}
