// ss_brick.cuh -- a brick's candidates in the splat-bin table, one definition for every level-set kernel (k_levelset,
// certification, exact pass, anisotropic level set) and the particle queries: the bin table, brick decode, candidate bin ranges
// with the extension plane, bin-column runs and their warp-wide layout, the candidate key sort, and the lane geometry of a
// 4x4x4-point sub-box.
#pragma once

// The splat bins of a batch: per (subdomain, bin) key the run of records in bin-sorted order.
struct SsBins {
    const uint32_t *bin_start;   // [nsub * nbin_sub] run start or 0xffffffff
    const uint32_t *bin_end;     // [nsub * nbin_sub] run end
    const float4 *rec;           // bin-sorted records (x, y, z, V)
    const int *ksplit;           // bin-sorted AVX-remainder splits
    const uint32_t *pidx;        // bin-sorted particle indices
    const SsTile *tile_tab;      // [batch] per-tile constants (host-filled)
    const int2 *brick_rng;       // [nb] candidate bin range (lo, hi) of brick b along one axis
};

// brick of the batch from its linear index ((tile * nb + bx) * nb + by) * nb + bz
struct SsBrick { int tile, bx, by, bz; uint32_t lin; };
__device__ __forceinline__ SsBrick ss_brick_from_lin(const SsDev &P, uint32_t lin) {
    SsBrick B;
    B.lin = lin;
    uint32_t q = lin;
    B.bz = (int)(q % (uint32_t)P.nb); q /= (uint32_t)P.nb;
    B.by = (int)(q % (uint32_t)P.nb); q /= (uint32_t)P.nb;
    B.bx = (int)(q % (uint32_t)P.nb); B.tile = (int)(q / (uint32_t)P.nb);
    return B;
}

// Candidate bins of brick (bx, by, bz): per axis the bins overlapping [8 b - R, 8 b + 7 + R).  With `ext` (extension bricks) the
// last full brick along an axis (ex / ey / ez) also gathers the bins of the np - 1 plane.  Run r is the bin column
// (rx.x + r / nyr, ry.x + r % nyr, rz.x .. rz.y).
struct SsBrickBins { int2 rx, ry, rz; int nyr, nruns; bool ex, ey, ez; };
__device__ __forceinline__ SsBrickBins ss_brick_bins(const SsDev &P, const int2 *brick_rng, int bx, int by, int bz, bool ext) {
    SsBrickBins K;
    K.ex = ext && bx == P.nb - 2; K.ey = ext && by == P.nb - 2; K.ez = ext && bz == P.nb - 2;
    K.rx = brick_rng[bx]; K.ry = brick_rng[by]; K.rz = brick_rng[bz];
    if (K.ex) K.rx.y = brick_rng[bx + 1].y;
    if (K.ey) K.ry.y = brick_rng[by + 1].y;
    if (K.ez) K.rz.y = brick_rng[bz + 1].y;
    K.nyr = K.ry.y - K.ry.x + 1;
    K.nruns = (K.rx.y - K.rx.x + 1) * K.nyr;
    return K;
}

// The records of bin column (X, Y, z0 .. z1) of subdomain s in the bin tables (bin_start, bin_end): bins along z are contiguous in
// the sorted records, so the column is one run.  Returns its length (0: every bin is empty) and its first record in `start` (0 when
// empty).
__device__ __forceinline__ uint32_t ss_bin_column(const SsDev &P, const uint32_t *bin_start, const uint32_t *bin_end, uint32_t s, int X, int Y,
                                                  int z0, int z1, uint32_t &start) {
    uint32_t a = 0xffffffffu, b = 0;
    const uint32_t base = s * (uint32_t)P.nbin_sub + (uint32_t)((X * P.nbin + Y) * P.nbin);
    for (int Z = z0; Z <= z1; ++Z) {
        const uint32_t st = bin_start[base + Z];
        if (st != 0xffffffffu) { if (a == 0xffffffffu) a = st; b = bin_end[base + Z]; }
    }
    start = a == 0xffffffffu ? 0u : a;
    return a == 0xffffffffu ? 0u : b - a;
}
// run r of a brick of subdomain s (length 0 for r >= nruns)
__device__ __forceinline__ uint32_t ss_brick_run(const SsDev &P, const SsBins &B, uint32_t s, const SsBrickBins &K, int r, uint32_t &start) {
    start = 0;
    if (r >= K.nruns) return 0;
    return ss_bin_column(P, B.bin_start, B.bin_end, s, K.rx.x + r / K.nyr, K.ry.x + r % K.nyr, K.rz.x, K.rz.y, start);
}

// exclusive prefix of v over the lanes of the warp (where the lane's run goes); the warp's total in `total`
__device__ __forceinline__ uint32_t ss_warp_excl_scan(uint32_t v, int lane, uint32_t &total) {
    uint32_t incl = v;
    for (int o = 1; o < 32; o <<= 1) { const uint32_t n = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += n; }
    total = __shfl_sync(0xffffffffu, incl, 31);
    return incl - v;
}

// Sorts the n staged candidate keys ((pidx << 32) | payload) ascending in shared memory: pads them with ~0 to a power of two
// (>= 32), then runs a bitonic network, by one warp (WARP) or by the whole CTA.
template <bool WARP>
__device__ __forceinline__ void ss_sort_keys(unsigned long long *keys, int n) {
    const int t0 = WARP ? (int)(threadIdx.x & 31) : (int)threadIdx.x, nt = WARP ? 32 : (int)blockDim.x;
    int npow = 32;
    while (npow < n) npow <<= 1;
    for (int t = n + t0; t < npow; t += nt) keys[t] = ~0ull;
    if (WARP) __syncwarp(); else __syncthreads();
    for (int k = 2; k <= npow; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int t = t0; t < (npow >> 1); t += nt) {
                const int lo = ((t & ~(j - 1)) << 1) | (t & (j - 1));      // index with bit j clear
                const int hi = lo | j;
                const unsigned long long a = keys[lo], b = keys[hi];
                const bool up = ((lo & k) == 0);
                if ((a > b) == up) { keys[lo] = b; keys[hi] = a; }
            }
            if (WARP) __syncwarp(); else __syncthreads();
        }
    }
}

// Coordinate of the grid point with GLOBAL index g, by the reference's expressions: x, y mul then add, z fused unless `sparse`
// (dense_subdomains.rs:1068, :1101-1102; scalar: uniform_grid.rs:418-425).  Both are monotonic in g, so a box whose bounds come from
// the same expression contains every point it spans, however large the coordinates' rounding is against the cell size; the culls
// with a relative slack on h^2 rely on this.
__device__ __forceinline__ float ss_grid_xy(const SsDev &P, int g, int d) { return __fadd_rn(__fmul_rn((float)g, P.c), P.gmin[d]); }
__device__ __forceinline__ float ss_grid_z(const SsDev &P, int g, bool sparse) {
    return sparse ? __fadd_rn(P.gmin[2], __fmul_rn((float)g, P.c)) : __fmaf_rn((float)g, P.c, P.gmin[2]);
}

// lane -> its two grid points (li, lj, lk) and (li, lj, lk + 1) within a 4x4x4-point sub-box; pmax: the tile's last point index
struct SsSubLane { int li, lj, lk, pmax; };
__device__ __forceinline__ SsSubLane ss_sub_lane(const SsDev &P, int lane) { return SsSubLane{ lane >> 3, (lane >> 1) & 3, (lane & 1) * 2, P.np - 1 }; }

// A lane's share of the 4x4x4-point sub-box b of brick (bx, by, bz) (bits 2, 1, 0: upper half along x, y, z): the grid points
// (i, j, k) and (i, j, k + 1), whether they lie in the tile (vA, vB), their coordinates from GLOBAL indices -- x, y: mul then
// add, z: fused unless `sparse` (dense_subdomains.rs:1068, :1101-1102; scalar: uniform_grid.rs:418-425) -- and the sub-box in
// world coordinates (culling only).  `inside`: the sub-box starts inside the tile.
struct SsSubBox {
    bool inside, vA, vB;
    int i, j, k, gi, gj, gk, k1;
    float gx, gy, gzA, gzB;
    float bxl, bxh, byl, byh, bzl, bzh;
};
__device__ __forceinline__ SsSubBox ss_sub_box(const SsDev &P, const SsTile &T, int bx, int by, int bz, int b, const SsSubLane &L, bool sparse) {
    SsSubBox G;
    const int pmax = L.pmax;
    const int i0 = bx * 8 + 4 * ((b >> 2) & 1), j0 = by * 8 + 4 * ((b >> 1) & 1), k0 = bz * 8 + 4 * (b & 1);
    G.inside = i0 <= pmax && j0 <= pmax && k0 <= pmax;
    G.i = i0 + L.li; G.j = j0 + L.lj; G.k = k0 + L.lk;
    const bool row_ok = G.i <= pmax && G.j <= pmax;
    G.vA = row_ok && G.k <= pmax; G.vB = row_ok && G.k + 1 <= pmax;
    G.gi = T.gbase[0] + G.i; G.gj = T.gbase[1] + G.j; G.gk = T.gbase[2] + G.k;
    G.gx = ss_grid_xy(P, G.gi, 0);
    G.gy = ss_grid_xy(P, G.gj, 1);
    G.gzA = ss_grid_z(P, G.gk, sparse);
    G.gzB = ss_grid_z(P, G.gk + 1, sparse);
    const int i1 = min(i0 + 3, pmax), j1 = min(j0 + 3, pmax), k1 = min(k0 + 3, pmax);
    G.k1 = k1;
    G.bxl = ss_grid_xy(P, T.gbase[0] + i0, 0); G.bxh = ss_grid_xy(P, T.gbase[0] + i1, 0);
    G.byl = ss_grid_xy(P, T.gbase[1] + j0, 1); G.byh = ss_grid_xy(P, T.gbase[1] + j1, 1);
    G.bzl = ss_grid_z(P, T.gbase[2] + k0, sparse); G.bzh = ss_grid_z(P, T.gbase[2] + k1, sparse);
    return G;
}
