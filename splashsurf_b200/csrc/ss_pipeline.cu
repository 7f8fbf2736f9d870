// ss_pipeline.cu -- host orchestration + C ABI of the H100 reconstruct path (see include/splashsurf_b200.h).
//
// Host-side mirror of splashsurf_lib::reconstruct_surface_inplace (lib.rs:340-473) and
// reconstruction::reconstruct_surface_subdomain_grid (reconstruction.rs:17-62): parameter validation, grid
// derivation in exact f32 (lib.rs:476-516, dense_subdomains.rs:89-244), then the device pipeline.  There is
// no CPU fallback: without a CUDA device every entry point fails with SS_ERR_NO_DEVICE.
#include "../../include/splashsurf_b200.h"
#include "ss_kernels.cuh"
#include "ss_certify.cuh"
#include "ss_exact.cuh"
#include "ss_aniso.cuh"
#include "ss_averaged.cuh"
#include "ss_field.cuh"
#include "ss_raycast.cuh"
#include "ss_sdf.cuh"
#include "ss_density.cuh"
#include "ss_mc.cuh"
#include "ss_levelset_mesh.cuh"

#ifndef SS_HOST_EMUL               // (tests/emul/cuda_emul.h compiles this file with g++ to step the kernels on the CPU)
#include <cub/cub.cuh>
#endif
#include <cfloat>
#include <climits>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#include <algorithm>
#include <functional>
#include <memory>
#include <initializer_list>
#include <type_traits>

// ------------------------------------------------------------------ errors ----
static thread_local std::string g_last_error;
static int ss_fail(int code, const std::string &msg) { g_last_error = msg; return code; }

struct SsCudaError { cudaError_t e; const char *what; const char *file; int line; };
#define CK(call) do { cudaError_t _e = (call); if (_e != cudaSuccess) throw SsCudaError{ _e, #call, __FILE__, __LINE__ }; } while (0)

// Runs an entry's body and turns a failure it throws into the entry's status: a CUDA error is cleared from the runtime and
// reported with its call site, a failed device or host allocation as SS_ERR_OUT_OF_MEMORY.
template <typename F>
static int ss_guard(F &&body) {
    try {
        return body();
    } catch (const SsCudaError &err) {
        cudaGetLastError();
        char buf[512];
        snprintf(buf, sizeof(buf), "%s failed at %s:%d: %s", err.what, err.file, err.line, cudaGetErrorString(err.e));
        return ss_fail(err.e == cudaErrorMemoryAllocation ? SS_ERR_OUT_OF_MEMORY : SS_ERR_CUDA, buf);
    } catch (const std::bad_alloc &) {
        return ss_fail(SS_ERR_OUT_OF_MEMORY, "host allocation failed");
    }
}

// ------------------------------------------------------------------ device buffers ----
// Growth slack of the pooled buffers in eighths of the request: 1 (12.5 %) for whole-domain runs; partitioned (multi-GPU) runs use 4
// (50 %), because the slab plan -- and with it every per-rank size -- moves a little from frame to frame while it balances, and
// re-allocating the scratch costs far more than the memory it saves (each rank holds 1/N of the data anyway).
static int g_devbuf_slack_eighths = 1;
// A device allocation with one owner: freed when the owner goes, handed on with std::move / std::swap.
struct DevBuf {
    void *p = nullptr; size_t cap = 0;
    DevBuf() = default;
    DevBuf(DevBuf &&o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
    DevBuf &operator=(DevBuf &&o) noexcept {
        if (this != &o) { release(); p = o.p; cap = o.cap; o.p = nullptr; o.cap = 0; }
        return *this;
    }
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;
    ~DevBuf() { release(); }
    template <typename T> T *as() const { return (T *)p; }
    void ensure(size_t bytes) {
#ifdef SS_EMUL_GUARD                      // tests/emul: exact-size allocations in front of a guard page (overrun detection)
        if (bytes == cap && p) return;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        size_t want = bytes;
#else
        if (bytes <= cap) return;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        size_t want = bytes + (bytes / 8) * (size_t)g_devbuf_slack_eighths + 256;
#endif
        cudaError_t e = cudaMalloc(&p, want);
        if (e != cudaSuccess) { p = nullptr; throw SsCudaError{ e, "cudaMalloc", __FILE__, __LINE__ }; }
        cap = want;
    }
    // grow while preserving contents
    void grow_keep(size_t bytes, size_t used, cudaStream_t st) {
        if (bytes <= cap) return;
#ifdef SS_EMUL_GUARD
        size_t want = bytes;
#else
        size_t want = std::max(bytes + bytes / 4, cap * 2) + 256;
#endif
        void *q = nullptr;
        cudaError_t e = cudaMalloc(&q, want);
        if (e != cudaSuccess) throw SsCudaError{ e, "cudaMalloc", __FILE__, __LINE__ };
        if (p && used) CK(cudaMemcpyAsync(q, p, used, cudaMemcpyDeviceToDevice, st));
        if (p) { CK(cudaStreamSynchronize(st)); cudaFree(p); }
        p = q; cap = want;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
};

struct HostGrid { float mn[3], mx[3]; float cell; int64_t np[3], nc[3]; };

// State of the most recent reconstruction that the post-processing entries (ss_post.cuh) need, and their scratch.
struct PostScratch {
    int valid = 0;                   // the splat bins in the context scratch belong to frame `ss_context::frame`
    int partitioned = 0;
    SsDev D{};
    uint32_t nsub = 0, M = 0;
    float sphere_mass = 0.f;         // 4/3 pi r^3 rho0 (reconstruct.rs:1126-1129)
    DevBuf keys_a, keys_b, flag, scan, vals, out, tmpv;
};

struct ss_context {
    int device = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev[12];
    uint32_t max_tiles = 0;          // 0 = auto
    int64_t keep_tile_flat = -1;
    int64_t keep_raw_flat = -1;      // ss_context_keep_levelset_tile_raw (does not force exact evaluation)
    int ls_exact_all = 0;           // 1: evaluate every grid point exactly (no certification)
    int ls_variant = 2;              // 2 (default): warp-per-brick certification + exact kernels (ss_certify.cuh, ss_exact.cuh); 1: CTA-per-brick certification kernel; 0: fused k_levelset
    int count_pairs = 0;             // 1: count in-support evaluations (work model; slower)
    int exact_phases = 0;            // 1: time the phases of k_exact_warp into xphase (ss_context_set_exact_phases; slower)
    int density_variant = 0;         // 0 (default): thread-per-particle k_density; 1 / 2: cell-cooperative kernel (ss_density.cuh), candidates staged by bulk copies / 16-byte loads
    int mc_variant = 1;              // 1 (default): warp-per-brick marching cubes (count + emit) and fix-up sweep (ss_mc.cuh); 0: CTA-per-brick passes
    void *h_stage[2] = { nullptr, nullptr };   // page-locked staging buffers of the result copies (copy_out), allocated on first use
    size_t stage_bytes = (size_t)32 << 20;     // chunk size of the staged result copies (copies below 4 chunks are plain)
    cudaEvent_t ev_stage[2] = { nullptr, nullptr };
    int sm_count = 132;              // streaming multiprocessors of the device (persistent-kernel grid sizing)
    int sph_normals = 0;             // 1: SPH normals at the mesh vertices (sph_interpolation.rs:82-133)
    int an_on = 0;                   // 1: anisotropic kernels (ss_aniso.cuh) with the parameters `an`
    ss_anisotropy_f32 an{};
    int avg_on = 0;                  // 1: averaged-position surface (ss_averaged.cuh) with the parameters `avg`
    ss_averaged_surface_f32 avg{};
    int ac_on = 0;                   // 1: Jacobian correction of the averaged-position surface (SsAvgCorrFold) with `ac`
    ss_averaged_correction_f32 ac{};
    int rad_on = 0;                  // 1: per-particle radii of the averaged-position surface (SsAvgRadFold, SsAvgCorrRadFold),
    uint64_t rad_n = 0;              //    rad_n of them in av_radii
    cudaEvent_t ev_an[2] = { nullptr, nullptr };
    // reusable scratch
    DevBuf xyz, xyz_f, filt_flag, filt_flag32, filt_off, aabb, cnt, off, key_a, key_b, val_a, val_b, cid, cub_tmp,
        sub_flat, sub_off, sub_owned, gkey_a, gkey_b, gval_a, gval_b, flags, scan, spos, rho, tab_a, tab_b, rec, ksplit, tiles, vcnt,
        tcnt, vmask, voff, vblk_off, tblk_off, tile_tab, brick_rng, bstate, flag_ls, off_ls, list_ls, flag_mc, flag_fix, off_mc, off_fix, list_mc, list_fix, wflag, wstate, desc_ls, dflag, doff, dlist, fallback, fallback2, fallback3, pack_cnt, pack_off, brick_seen, fix_list, nflag, bkeys_a, bkeys_b, bids_a, bids_b, bcount, remap, keep, newid, err, pairs, xphase, xw_taken, an_det, an_grec;
    DevBuf av_radii, av_delta, av_rrec, av_chk;      // per-particle radii: the caller's copy, delta_j (filtered), per membership, check
    // level-set field queries (ss_field.cuh): points, group keys and caller indices (sorted and not), group starts, values, checks,
    // and the candidate bin ranges of a group
    DevBuf fld_pts, fld_key_a, fld_key_b, fld_idx_a, fld_idx_b, fld_flag, fld_off, fld_starts, fld_out, fld_chk, fld_rng, fld_grad, fld_hess, fld_curv;
    // ray casts (ss_raycast.cuh): the caller's origins, directions and t_max, per-ray state, results, checks and the keyed-ray count
    DevBuf ray_o, ray_d, ray_tmax, ray_state, ray_t, ray_pos, ray_val, ray_status, ray_grad, ray_chk, ray_hits;
    uint64_t launches = 0;
    uint64_t pack_n = 0; uint32_t pack_world = 0;   // ss_partition_pack_f32: count phase the scatter phase must match
    // result buffers handed to surfaces and returned by ss_surface_free (avoids cudaMalloc/cudaFree per frame,
    // the analogue of the reference's ReconstructionWorkspace, workspace.rs:12-79)
    DevBuf o_verts, o_tris, o_vkeys, o_rho, o_verts2, o_vkeys2, o_normals;
    uint64_t hint_nv = 0, hint_nt = 0, hint_bc = 0;
    uint64_t frame = 0;              // serial of the last call that rewrote the scratch
    PostScratch post;
};

#include <mutex>
#include <set>
static std::mutex g_ctx_mutex;
static std::set<ss_context *> g_live_contexts;

struct ss_surface {
    ss_context *owner = nullptr;
    int device = 0;
    uint64_t n_in = 0, n = 0, nv = 0, nt = 0, nsub = 0;
    int used_decomposition = 0;
    HostGrid grid{}, subgrid{};
    int S = 0;
    DevBuf verts, tris, vkeys, rho, normals, nbr_off, nbr_idx;
    DevBuf weights, adj_row, adj_idx, inc_row, inc_idx;      // post-processing: smoothing weights, vertex->vertex / vertex->triangle CSR
    DevBuf an_xbar, an_g;                                    // anisotropic mode: smoothed centres (n x 3), G entries (n x 6)
    int has_aniso = 0;
    float an_ms = 0.f;                                       // anisotropy stage (k_aniso), ms
    int has_normals = 0, has_neighbors = 0, has_weights = 0, has_adj = 0, has_inc = 0;
    uint64_t frame = 0;              // ss_context::frame of the reconstruction that produced this surface
    uint64_t n_neighbors = 0;
    std::vector<uint8_t> inside_aabb;
    std::vector<int64_t> sub_flat; std::vector<uint64_t> sub_count; std::vector<uint8_t> sub_sparse, sub_owned;
    uint64_t max_particles = 0;
    std::vector<float> tile;
    std::vector<float> tile_raw;     // ss_context_keep_levelset_tile_raw: the tile before the fix-up pass, and its per-brick states
    std::vector<uint8_t> tile_raw_bstate;
    ss_timings tm{};
    uint64_t ls_paths[SS_LSP_N] = {};                        // ss_surface_levelset_paths
    // level-set field (ss_levelset_field_create_f32): the level set's device constants, its fold, whether records were binned
    int fld = 0, fld_mode = 0, fld_ready = 0;
    SsDev fld_D{};
    uint32_t fld_nsub = 0;
    uint64_t fld_paths[3] = {};                              // groups of the last query per tier: 512, 4096, select
    // mesh of a level-set field (ss_levelset_field_mesh_f32): lattice spacing, index range, batches
    int lm = 0;
    float lm_cube = 0.0f;
    int64_t lm_imin[3] = {}, lm_imax[3] = {};
    uint64_t lm_batches = 0;
};

// ------------------------------------------------------------------ host grid math (exact f32) ----
// All expressions are single roundings in the order the reference evaluates them; `volatile` stores stop the
// host compiler from keeping excess precision or contracting (the TU is also built with -ffp-contract=off).
static inline float fmulr(float a, float b) { volatile float r = a * b; return r; }
static inline float faddr(float a, float b) { volatile float r = a + b; return r; }
static inline float fsubr(float a, float b) { volatile float r = a - b; return r; }
static inline float fdivr(float a, float b) { volatile float r = a / b; return r; }

static int grid_new(HostGrid &g, const float mn[3], const int64_t nc[3], float cell) {       // uniform_grid.rs:204-232
    for (int d = 0; d < 3; ++d) {
        g.mn[d] = mn[d]; g.nc[d] = nc[d]; g.np[d] = nc[d] + 1;
        g.mx[d] = faddr(mn[d], fmulr(cell, (float)nc[d]));
        if (!std::isfinite(g.mx[d])) return SS_ERR_REAL_TOO_SMALL;
    }
    g.cell = cell;
    return SS_OK;
}
static int grid_from_aabb(HostGrid &g, const float mn[3], const float mx[3], float cell) {   // uniform_grid.rs:175-201
    if (!(cell > 0.0f)) return SS_ERR_INVALID_CELL_SIZE;
    if (mn[0] == mx[0] && mn[1] == mx[1] && mn[2] == mx[2]) return SS_ERR_DEGENERATE_AABB;
    for (int d = 0; d < 3; ++d) if (!(mn[d] <= mx[d])) return SS_ERR_INCONSISTENT_AABB;
    float amin[3]; int64_t nc[3];
    for (int d = 0; d < 3; ++d) {
        amin[d] = fmulr(floorf(fdivr(mn[d], cell)), cell);
        float ncr = ceilf(fdivr(fsubr(mx[d], amin[d]), cell));
        if (!(ncr < 9.0e18f)) return SS_ERR_INDEX_TOO_SMALL;
        int64_t n = (int64_t)ncr;
        nc[d] = n > 1 ? n : 1;
    }
    return grid_new(g, amin, nc, cell);
}
static void grid_to_abi(const HostGrid &g, ss_grid_f32 *o) {
    for (int d = 0; d < 3; ++d) { o->aabb_min[d] = g.mn[d]; o->aabb_max[d] = g.mx[d]; o->points_per_dim[d] = g.np[d]; o->cells_per_dim[d] = g.nc[d]; }
    o->cell_size = g.cell;
}

static int validate_params(const ss_params_f32 *p) {
    if (!p) return ss_fail(SS_ERR_INVALID_PARAMETER, "params is NULL");
    if (!(p->cube_size > 0.0f)) return ss_fail(SS_ERR_INVALID_CELL_SIZE, "invalid cell size supplied, cell size has to be larger than zero");
    if (!(p->compact_support_radius > 0.0f)) return ss_fail(SS_ERR_INVALID_PARAMETER, "compact support radius has to be positive (search radius for neighborhood search has to be positive)");
    if (!(p->particle_radius > 0.0f)) return ss_fail(SS_ERR_INVALID_PARAMETER, "particle radius has to be positive");
    if (p->spatial_decomposition == 1 && p->subdomain_num_cubes_per_dim < 1) return ss_fail(SS_ERR_INVALID_PARAMETER, "subdomain_num_cubes_per_dim has to be >= 1");
    return SS_OK;
}

// ------------------------------------------------------------------ small launch helpers ----
static inline unsigned nblk(uint64_t n, unsigned t) { return (unsigned)((n + t - 1) / t); }
#ifndef SS_LAUNCH
#define SS_LAUNCH(kern, grid, block, stream, ...) kern<<<(grid), (block), 0, (stream)>>>(__VA_ARGS__)
#endif
#define LAUNCH(ctx, kern, grid, block, ...) do { SS_LAUNCH(kern, grid, block, (ctx)->stream, __VA_ARGS__); (ctx)->launches++; } while (0)
#ifndef SS_LAUNCH_DYN
#define SS_LAUNCH_DYN(kern, grid, block, smem, stream, ...) kern<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
#endif
#define LAUNCH_DYN(ctx, kern, grid, block, smem, ...) do { SS_LAUNCH_DYN(kern, grid, block, smem, (ctx)->stream, __VA_ARGS__); (ctx)->launches++; } while (0)

// Radix sort of n keys on bits [0, end_bit), carrying the values vin -> vout when given (V = void: keys only).
template <typename K, typename V = void>
static void cub_sort(ss_context *c, const K *kin, K *kout, uint32_t n, int end_bit, const V *vin = nullptr, V *vout = nullptr) {
    const auto cub_radix_sort = [&](void *tmp, size_t &bytes) {
        if constexpr (std::is_void<V>::value) return cub::DeviceRadixSort::SortKeys(tmp, bytes, kin, kout, (int)n, 0, end_bit, c->stream);
        else return cub::DeviceRadixSort::SortPairs(tmp, bytes, kin, kout, vin, vout, (int)n, 0, end_bit, c->stream);
    };
    size_t bytes = 0;
    CK(cub_radix_sort(nullptr, bytes));
    c->cub_tmp.ensure(bytes);
    CK(cub_radix_sort(c->cub_tmp.p, bytes));
    c->launches += 1 + (uint64_t)((end_bit + 7) / 8) * 2;   // upsweep/onesweep histogram + per-digit passes (approx.)
}
// Exclusive (or inclusive) prefix sum of n entries.
template <bool INCLUSIVE = false, typename In, typename Out>
static void cub_scan(ss_context *c, In in, Out out, uint64_t n) {
    const auto cub_device_scan = [&](void *tmp, size_t &bytes) {
        if constexpr (INCLUSIVE) return cub::DeviceScan::InclusiveSum(tmp, bytes, in, out, (int)n, c->stream);
        else return cub::DeviceScan::ExclusiveSum(tmp, bytes, in, out, (int)n, c->stream);
    };
    size_t bytes = 0;
    CK(cub_device_scan(nullptr, bytes));
    c->cub_tmp.ensure(bytes);
    CK(cub_device_scan(c->cub_tmp.p, bytes));
    c->launches += 2;
}
// Exclusive scan of n >= 1 entries, and the read-back of its total out[n - 1] + in[n - 1] into last[0] + last[1]: the caller adds
// them after its next synchronisation of the stream.
static void scan_with_total(ss_context *c, const uint32_t *in, uint32_t *out, uint32_t n, uint32_t last[2]) {
    cub_scan(c, in, out, n);
    CK(cudaMemcpyAsync(&last[0], out + (n - 1), 4, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaMemcpyAsync(&last[1], in + (n - 1), 4, cudaMemcpyDeviceToHost, c->stream));
}
// ... synchronised: returns the total
static uint64_t scan_total(ss_context *c, const uint32_t *in, uint32_t *out, uint32_t n) {
    uint32_t last[2] = { 0, 0 };
    scan_with_total(c, in, out, n, last);
    CK(cudaStreamSynchronize(c->stream));
    return (uint64_t)last[0] + last[1];
}
// Exclusive scan of n 0/1 flags and the list of the flagged indices (k_compact_list); `last` as in scan_with_total, if given.
static void scan_compact(ss_context *c, const uint32_t *flag, uint32_t *off, uint32_t n, uint32_t *list, uint32_t *last = nullptr) {
    if (last) scan_with_total(c, flag, off, n, last);
    else cub_scan(c, flag, off, n);
    LAUNCH(c, k_compact_list, nblk(n, 256), 256, flag, off, n, list);
}
static int bits_for(uint64_t maxval) { int b = 1; while (b < 64 && (maxval >> b)) ++b; return b; }

// ------------------------------------------------------------------ context ----
extern "C" int ss_abi_version(void) { return SS_ABI_VERSION; }
extern "C" const char *ss_last_error(void) { return g_last_error.c_str(); }

extern "C" int ss_context_create(int device, ss_context **out) {
    if (!out) return ss_fail(SS_ERR_INVALID_PARAMETER, "out is NULL");
    *out = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev == 0)
        return ss_fail(SS_ERR_NO_DEVICE, std::string("no CUDA device available (") + cudaGetErrorString(e) + "); this library has no CPU path");
    return ss_guard([&]() -> int {
        if (device < 0) CK(cudaGetDevice(&device));
        if (device >= ndev) return ss_fail(SS_ERR_INVALID_PARAMETER, "device index out of range");
        CK(cudaSetDevice(device));
        ss_context *c = new ss_context();
        c->device = device;
        CK(cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking));
#ifndef SS_HOST_EMUL
        CK(cudaDeviceGetAttribute(&c->sm_count, cudaDevAttrMultiProcessorCount, device));
#else
        c->sm_count = 3;
#endif
        for (auto &ev : c->ev) CK(cudaEventCreate(&ev));
        for (auto &ev : c->ev_stage) CK(cudaEventCreate(&ev));
        for (auto &ev : c->ev_an) CK(cudaEventCreate(&ev));
        {
            signed char table[256][16];
            ss_mc_unpack(table);
            CK(cudaMemcpyToSymbol(c_tri_table, table, sizeof(table)));
        }
        CK(cudaMemcpyToSymbol(c_num_tris, SS_MC_NUM_TRIS, sizeof(SS_MC_NUM_TRIS)));
        { std::lock_guard<std::mutex> lk(g_ctx_mutex); g_live_contexts.insert(c); }
        *out = c;
        return SS_OK;
    });
}

extern "C" void ss_context_destroy(ss_context *c) {
    if (!c) return;
    { std::lock_guard<std::mutex> lk(g_ctx_mutex); g_live_contexts.erase(c); }
    cudaSetDevice(c->device);
    cudaStreamSynchronize(c->stream);                  // the device buffers are freed with the context below
    for (auto &ev : c->ev) cudaEventDestroy(ev);
    for (auto &ev : c->ev_stage) if (ev) cudaEventDestroy(ev);
    for (auto &ev : c->ev_an) if (ev) cudaEventDestroy(ev);
    for (auto &h : c->h_stage) if (h) cudaFreeHost(h);
    cudaStreamDestroy(c->stream);
    delete c;
}

extern "C" int ss_context_keep_levelset_tile(ss_context *c, int64_t flat) { if (!c) return SS_ERR_INVALID_PARAMETER; c->keep_tile_flat = flat; return SS_OK; }
extern "C" int ss_context_keep_levelset_tile_raw(ss_context *c, int64_t flat) { if (!c) return SS_ERR_INVALID_PARAMETER; c->keep_raw_flat = flat; return SS_OK; }
extern "C" int ss_context_set_tile_batch(ss_context *c, uint32_t m) { if (!c) return SS_ERR_INVALID_PARAMETER; c->max_tiles = m; return SS_OK; }
extern "C" int ss_context_set_levelset_exact_everywhere(ss_context *c, int on) { if (!c) return SS_ERR_INVALID_PARAMETER; c->ls_exact_all = on ? 1 : 0; return SS_OK; }
extern "C" int ss_context_set_density_variant(ss_context *c, int v) {
    if (!c || v < 0 || v > 2) return ss_fail(SS_ERR_INVALID_PARAMETER, "density variant must be 0, 1 or 2");
    c->density_variant = v; return SS_OK;
}
extern "C" int ss_context_set_copy_chunk_bytes(ss_context *c, uint64_t bytes) {
    if (!c || bytes < 4096 || bytes > ((uint64_t)32 << 20) || (bytes & 3)) return ss_fail(SS_ERR_INVALID_PARAMETER, "copy chunk must be 4 KiB .. 32 MiB, a multiple of 4");
    c->stage_bytes = (size_t)bytes; return SS_OK;
}
extern "C" int ss_context_set_mc_variant(ss_context *c, int v) {
    if (!c || v < 0 || v > 1) return ss_fail(SS_ERR_INVALID_PARAMETER, "marching-cubes variant must be 0 or 1");
    c->mc_variant = v; return SS_OK;
}
extern "C" int ss_context_set_levelset_variant(ss_context *c, int v) {
    if (!c || v < 0 || v > 2) return ss_fail(SS_ERR_INVALID_PARAMETER, "level-set variant must be 0, 1 or 2");
    c->ls_variant = v; return SS_OK;
}
extern "C" int ss_context_set_compute_sph_normals(ss_context *c, int on) { if (!c) return SS_ERR_INVALID_PARAMETER; c->sph_normals = on ? 1 : 0; return SS_OK; }
extern "C" int ss_surface_copy_normals(const ss_surface *s, float *dst) {
    if (!s || !dst) return SS_ERR_INVALID_PARAMETER;
    if (!s->has_normals) return ss_fail(SS_ERR_INVALID_PARAMETER, "normals were not computed (ss_context_set_compute_sph_normals)");
    cudaSetDevice(s->device);
    cudaError_t e = cudaMemcpy(dst, s->normals.p, s->nv * 12, cudaMemcpyDeviceToHost);
    return e == cudaSuccess ? SS_OK : ss_fail(SS_ERR_CUDA, cudaGetErrorString(e));
}
extern "C" const float *ss_surface_device_normals(const ss_surface *s) { return (s && s->has_normals) ? s->normals.as<float>() : nullptr; }
extern "C" int ss_context_set_count_pairs(ss_context *c, int on) { if (!c) return SS_ERR_INVALID_PARAMETER; c->count_pairs = on ? 1 : 0; return SS_OK; }
static_assert(SS_XP_N == SS_EXACT_PHASES, "phases of the exact pass: kernel and header disagree");
extern "C" int ss_context_set_exact_phases(ss_context *c, int on) {
    if (!c) return SS_ERR_INVALID_PARAMETER;
    c->exact_phases = on ? 1 : 0;
    if (!on) return SS_OK;
    return ss_guard([&] {
        CK(cudaSetDevice(c->device));
        c->xphase.ensure((SS_XP_N + 1) * 8);
        CK(cudaMemset(c->xphase.p, 0, (SS_XP_N + 1) * 8));
        return SS_OK;
    });
}
extern "C" int ss_context_exact_phases(ss_context *c, uint64_t *out) {
    if (!c || !out) return SS_ERR_INVALID_PARAMETER;
    if (!c->xphase.p) return ss_fail(SS_ERR_INVALID_PARAMETER, "phase timing is off (ss_context_set_exact_phases)");
    cudaSetDevice(c->device);
    const cudaError_t e = cudaMemcpy(out, c->xphase.p, (SS_XP_N + 1) * 8, cudaMemcpyDeviceToHost);
    return e == cudaSuccess ? SS_OK : ss_fail(SS_ERR_CUDA, cudaGetErrorString(e));
}
extern "C" int ss_context_set_anisotropy_f32(ss_context *c, const ss_anisotropy_f32 *a) {
    if (!c) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL context");
    if (!a) { c->an_on = 0; return SS_OK; }
    if (!(a->smoothing >= 0.0f && a->smoothing <= 1.0f)) return ss_fail(SS_ERR_INVALID_PARAMETER, "anisotropy smoothing must lie in [0, 1]");
    if (!(a->max_stretch >= 1.0f) || !std::isfinite(a->max_stretch)) return ss_fail(SS_ERR_INVALID_PARAMETER, "anisotropy max_stretch must be finite and >= 1");
    c->an = *a; c->an_on = 1;
    return SS_OK;
}
extern "C" int ss_context_set_averaged_surface_f32(ss_context *c, const ss_averaged_surface_f32 *a) {
    if (!c) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL context");
    if (!a) { c->avg_on = 0; return SS_OK; }
    if (!(a->radius_factor > 0.0f) || !std::isfinite(a->radius_factor)) return ss_fail(SS_ERR_INVALID_PARAMETER, "averaged surface radius_factor must be finite and > 0");
    c->avg = *a; c->avg_on = 1;
    return SS_OK;
}
extern "C" int ss_context_set_averaged_correction_f32(ss_context *c, const ss_averaged_correction_f32 *a) {
    if (!c) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL context");
    if (!a) { c->ac_on = 0; return SS_OK; }
    if (!std::isfinite(a->t_low) || !std::isfinite(a->t_high) || !(a->t_low >= 0.0f) || !(a->t_low < a->t_high))
        return ss_fail(SS_ERR_INVALID_PARAMETER, "averaged surface correction: t_low and t_high must be finite with 0 <= t_low < t_high");
    c->ac = *a; c->ac_on = 1;
    return SS_OK;
}
extern "C" int ss_context_set_averaged_radii_f32(ss_context *c, const float *radii, uint64_t n) {
    if (!c) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL context");
    if (!radii) { c->rad_on = 0; c->rad_n = 0; return SS_OK; }
    if (n > 0xfffffff0ull) return ss_fail(SS_ERR_INDEX_TOO_SMALL, "more than 2^32 particle radii are not supported by one device");
    return ss_guard([&]() -> int {
        CK(cudaSetDevice(c->device));
        if (n) {
            // host or device memory, like the positions; copied, so the caller may free its array when this returns
            cudaPointerAttributes attr{};
            const cudaError_t e = cudaPointerGetAttributes(&attr, radii);
            const bool on_device = e == cudaSuccess && (attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged);
            if (e != cudaSuccess) cudaGetLastError();
            c->av_radii.ensure(n * 4);
            CK(cudaMemcpyAsync(c->av_radii.p, radii, n * 4, on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, c->stream));
            CK(cudaStreamSynchronize(c->stream));
        }
        c->rad_on = 1; c->rad_n = n;
        return SS_OK;
    });
}

// ------------------------------------------------------------------ stage: input, filter, AABB, grid ----
struct Prepared {
    const float *d_xyz = nullptr;   // filtered particles on device
    uint64_t n = 0;
    HostGrid grid{};
    float upload_ms = 0.f;
};

// Result copies device -> host.  A plain cudaMemcpy into PAGEABLE memory is staged by the driver and, into freshly allocated arrays
// (what a numpy front end hands in), page-faults single-threaded, far below PCIe speed for the 2.5 GB of a 50 M-particle result.  Large
// copies therefore go through two page-locked staging buffers at PCIe speed, and a few host threads scatter each chunk into the
// destination (parallel first touch) while the next chunk is in flight; `widen` turns u32 triangle indices into the reference's
// usize on the way (half the PCIe bytes of converting on the device).  Destinations that are page-locked already take one cudaMemcpy.
#include <thread>
#define SS_STAGE_BYTES_MAX ((size_t)32 << 20)
#define SS_STAGE_THREADS 8
static void scatter_chunk(char *dst, const char *stage, size_t n_src_bytes, bool widen) {
    const size_t nthreads = n_src_bytes >= ((size_t)1 << 20) ? SS_STAGE_THREADS : 1;
    auto work = [&](size_t t) {
        const size_t per = ((n_src_bytes / 4 + nthreads - 1) / nthreads) * 4;           // multiples of one 4-byte element
        const size_t lo = std::min(n_src_bytes, t * per), hi = std::min(n_src_bytes, lo + per);
        if (!widen) { memcpy(dst + lo, stage + lo, hi - lo); return; }
        const uint32_t *in = reinterpret_cast<const uint32_t *>(stage + lo);
        uint64_t *out = reinterpret_cast<uint64_t *>(dst) + lo / 4;
        for (size_t e = 0; e < (hi - lo) / 4; ++e) out[e] = in[e];
    };
    if (nthreads == 1) { work(0); return; }
    std::thread th[SS_STAGE_THREADS];
    for (size_t t = 1; t < nthreads; ++t) th[t] = std::thread(work, t);
    work(0);
    for (size_t t = 1; t < nthreads; ++t) th[t].join();
}
// The same staging for the upload of a large PAGEABLE particle array (a numpy array handed to the front end): host threads gather a
// chunk into a page-locked buffer while the previous chunk travels; page-locked inputs take one asynchronous copy.
static void upload_particles(ss_context *c, void *dst_dev, const void *src, size_t bytes, bool pinned_src) {
    const size_t chunk = c->stage_bytes;
    if (pinned_src || bytes < 4 * chunk) { CK(cudaMemcpyAsync(dst_dev, src, bytes, cudaMemcpyHostToDevice, c->stream)); return; }
    for (int q = 0; q < 2; ++q) if (!c->h_stage[q]) {
        if (cudaHostAlloc(&c->h_stage[q], SS_STAGE_BYTES_MAX, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); c->h_stage[q] = nullptr; }
    }
    if (!c->h_stage[0] || !c->h_stage[1]) { CK(cudaMemcpyAsync(dst_dev, src, bytes, cudaMemcpyHostToDevice, c->stream)); return; }
    const size_t nchunks = (bytes + chunk - 1) / chunk;
    for (size_t k = 0; k < nchunks; ++k) {
        const size_t off = k * chunk, n = std::min(chunk, bytes - off);
        if (k >= 2) CK(cudaEventSynchronize(c->ev_stage[k & 1]));     // the copy that last read this staging buffer is done
        scatter_chunk(static_cast<char *>(c->h_stage[k & 1]), static_cast<const char *>(src) + off, n, false);
        CK(cudaMemcpyAsync(static_cast<char *>(dst_dev) + off, c->h_stage[k & 1], n, cudaMemcpyHostToDevice, c->stream));
        CK(cudaEventRecord(c->ev_stage[k & 1], c->stream));
    }
    CK(cudaStreamSynchronize(c->stream));                             // the staging buffers are free again when this returns
}

static int prepare_particles(ss_context *c, const float *xyz, uint64_t n_in, const ss_params_f32 *p, Prepared &P,
                             std::vector<uint8_t> *inside_out, const ss_grid_f32 *given_grid = nullptr) {
    if (n_in > 0xfffffff0ull) return ss_fail(SS_ERR_INDEX_TOO_SMALL, "more than 2^32 particles are not supported by one device");
    const float *d_in = nullptr;
    cudaPointerAttributes attr{};
    bool on_device = false;
    bool pinned_host = false;
    if (xyz && n_in) {
        cudaError_t e = cudaPointerGetAttributes(&attr, xyz);
        if (e == cudaSuccess && (attr.type == cudaMemoryTypeDevice || attr.type == cudaMemoryTypeManaged)) on_device = true;
        else if (e == cudaSuccess && attr.type == cudaMemoryTypeHost) pinned_host = true;
        else cudaGetLastError();
    }
    CK(cudaEventRecord(c->ev[0], c->stream));
    if (on_device) d_in = xyz;
    else if (n_in) {
        c->xyz.ensure(n_in * 12);
        upload_particles(c, c->xyz.p, xyz, n_in * 12, pinned_host);
        d_in = c->xyz.as<float>();
    }
    CK(cudaEventRecord(c->ev[1], c->stream));
    P.d_xyz = d_in; P.n = n_in;
    // particle AABB filter, lib.rs:369-406
    if (p->has_particle_aabb && n_in) {
        c->filt_flag.ensure(n_in); c->filt_flag32.ensure(n_in * 4); c->filt_off.ensure(n_in * 4 + 4);
        float3 mn = make_float3(p->particle_aabb_min[0], p->particle_aabb_min[1], p->particle_aabb_min[2]);
        float3 mx = make_float3(p->particle_aabb_max[0], p->particle_aabb_max[1], p->particle_aabb_max[2]);
        LAUNCH(c, k_filter_flags, nblk(n_in, 256), 256, d_in, n_in, mn, mx, c->filt_flag.as<uint8_t>(), c->filt_flag32.as<uint32_t>());
        const uint64_t nf = scan_total(c, c->filt_flag32.as<uint32_t>(), c->filt_off.as<uint32_t>(), (uint32_t)n_in);
        c->xyz_f.ensure(std::max<uint64_t>(nf, 1) * 12);
        LAUNCH(c, k_filter_scatter, nblk(n_in, 256), 256, d_in, n_in, c->filt_flag.as<uint8_t>(), c->filt_off.as<uint32_t>(), c->xyz_f.as<float>());
        P.d_xyz = c->xyz_f.as<float>(); P.n = nf;
        if (inside_out) {
            inside_out->resize(n_in);
            CK(cudaMemcpyAsync(inside_out->data(), c->filt_flag.p, n_in, cudaMemcpyDeviceToHost, c->stream));
            CK(cudaStreamSynchronize(c->stream));
        }
    } else if (p->has_particle_aabb && inside_out) inside_out->clear();

    if (given_grid) {   // partitioned run: the grid of ALL particles was computed by the caller
        for (int d = 0; d < 3; ++d) { P.grid.mn[d] = given_grid->aabb_min[d]; P.grid.mx[d] = given_grid->aabb_max[d]; P.grid.np[d] = given_grid->points_per_dim[d]; P.grid.nc[d] = given_grid->cells_per_dim[d]; }
        P.grid.cell = given_grid->cell_size;
        return SS_OK;
    }
    // grid_for_reconstruction, lib.rs:476-516
    float mn[3], mx[3];
    if (p->has_particle_aabb) {
        for (int d = 0; d < 3; ++d) { mn[d] = p->particle_aabb_min[d]; mx[d] = p->particle_aabb_max[d]; }
    } else {
        if (P.n == 0) { for (int d = 0; d < 3; ++d) mn[d] = mx[d] = 0.0f; }   // Aabb3d::zeros(), aabb.rs:29-30
        else {
            c->aabb.ensure(6 * sizeof(int));
            int init[6] = { INT_MAX, INT_MAX, INT_MAX, INT_MIN, INT_MIN, INT_MIN };
            CK(cudaMemcpyAsync(c->aabb.p, init, sizeof(init), cudaMemcpyHostToDevice, c->stream));
            unsigned blocks = std::min<uint64_t>(nblk(P.n, 256), (uint64_t)c->sm_count * 16);
            LAUNCH(c, k_aabb, blocks, 256, P.d_xyz, P.n, c->aabb.as<int>());
            int res[6];
            CK(cudaMemcpyAsync(res, c->aabb.p, sizeof(res), cudaMemcpyDeviceToHost, c->stream));
            CK(cudaStreamSynchronize(c->stream));
            for (int d = 0; d < 3; ++d) { mn[d] = ss_ord2f(res[d]); mx[d] = ss_ord2f(res[3 + d]); }
        }
        for (int d = 0; d < 3; ++d) { mn[d] = fsubr(mn[d], p->particle_radius); mx[d] = faddr(mx[d], p->particle_radius); }
    }
    // compute_kernel_evaluation_radius, density_map.rs:551-580
    float half_cells = ceilf(fdivr(p->compact_support_radius, p->cube_size));
    float margin = fmulr(fmulr(p->cube_size, half_cells), faddr(1.0f, sqrtf(FLT_EPSILON)));
    for (int d = 0; d < 3; ++d) { mn[d] = fsubr(mn[d], margin); mx[d] = faddr(mx[d], margin); }
    int rc = grid_from_aabb(P.grid, mn, mx, p->cube_size);
    if (rc != SS_OK) return ss_fail(rc, rc == SS_ERR_DEGENERATE_AABB ? "degenerate AABB supplied, every dimension of the AABB has to have non-zero extents"
                                        : rc == SS_ERR_INCONSISTENT_AABB ? "inconsistent AABB supplied" : "grid construction failed");
    return SS_OK;
}

extern "C" int ss_grid_for_reconstruction_f32(ss_context *c, const float *xyz, uint64_t n, const ss_params_f32 *p, ss_grid_f32 *out) {
    if (!c || !out) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL argument");
    int rc = validate_params(p);
    if (rc) return rc;
    return ss_guard([&]() -> int {
        CK(cudaSetDevice(c->device));
        Prepared P;
        const int rc = prepare_particles(c, xyz, n, p, P, nullptr);
        if (rc) return rc;
        grid_to_abi(P.grid, out);
        return SS_OK;
    });
}


// ------------------------------------------------------------------ templated launch helpers ----
// f(G, C) with G, C std::integral_constant<bool, ...>: the GLOBAL x COUNT instantiation of a kernel for the runtime flags
template <typename F>
static void with_global_count(bool global, bool count, F &&f) {
    if (global) { if (count) f(std::true_type(), std::true_type()); else f(std::true_type(), std::false_type()); }
    else { if (count) f(std::false_type(), std::true_type()); else f(std::false_type(), std::false_type()); }
}

static void launch_levelset(ss_context *c, dim3 grid, const SsDev &D, const SsLsArgs &A, bool count, bool global) {
    with_global_count(global, count, [&](auto G, auto C) { LAUNCH(c, (k_levelset<C, G>), grid, SS_LS_THREADS, D, A); });
}

// the splat bins of the last binning stage (context scratch)
static SsBins context_bins(const ss_context *c) {
    SsBins B;
    B.bin_start = c->tab_a.as<uint32_t>(); B.bin_end = c->tab_b.as<uint32_t>(); B.rec = c->rec.as<float4>(); B.ksplit = c->ksplit.as<int>();
    B.pidx = c->val_a.as<uint32_t>(); B.tile_tab = c->tile_tab.as<SsTile>(); B.brick_rng = c->brick_rng.as<int2>();
    return B;
}

// Fallback cascade over a list of n bricks: tier t launches over the bricks tier t - 1 could not take, appending those it cannot
// take itself to `left` ([0] = count, [1..] = linear brick indices), the next tier's list.  The last tier takes every brick it gets
// (left = nullptr).  Stops when no brick is left.  received[t] accumulates the length of tier t's list.
typedef std::function<void(const uint32_t *list, uint32_t n, uint32_t *left)> SsTier;
static void run_cascade(ss_context *c, const uint32_t *list, uint32_t n, std::initializer_list<SsTier> tiers, uint64_t &ls_launches,
                        uint64_t *received) {
    DevBuf *const left_bufs[] = { &c->fallback, &c->fallback2, &c->fallback3 };
    size_t t = 0;
    for (const SsTier &tier : tiers) {
        if (!n) return;
        received[t] += n;
        if (++t == tiers.size()) { tier(list, n, nullptr); ++ls_launches; return; }
        DevBuf &left = *left_bufs[t - 1];
        left.ensure(((size_t)n + 1) * 4);
        CK(cudaMemsetAsync(left.p, 0, 4, c->stream));
        tier(list, n, left.as<uint32_t>());
        ++ls_launches;
        CK(cudaMemcpyAsync(&n, left.p, 4, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        list = left.as<uint32_t>() + 1;
    }
}

// in-place exclusive scan of the per-particle neighbour counts (n + 1 entries, last = 0) -> CSR offsets; returns the total
static uint64_t scan_neighbor_counts(ss_context *c, unsigned long long *cnt, uint64_t n) {
    cub_scan(c, cnt, cnt, n + 1);
    unsigned long long total = 0;
    CK(cudaMemcpyAsync(&total, cnt + n, 8, cudaMemcpyDeviceToHost, c->stream));
    CK(cudaStreamSynchronize(c->stream));
    return total;
}

// Work list of non-empty bricks for the level-set launch (k_brick_worklist + scan + compaction); returns its length.
static uint32_t build_worklist(ss_context *c, const SsDev &D, uint32_t ntiles) {
    const uint32_t nbr = ntiles * (uint32_t)(D.nb * D.nb * D.nb);
    c->flag_ls.ensure((size_t)nbr * 4); c->off_ls.ensure((size_t)nbr * 4 + 4); c->list_ls.ensure((size_t)nbr * 4);
    LAUNCH(c, k_brick_worklist, nblk(nbr, 256), 256, D, c->tile_tab.as<SsTile>(), c->brick_rng.as<int2>(), c->tab_a.as<uint32_t>(), ntiles, c->flag_ls.as<uint32_t>());
    uint32_t lc[2] = { 0, 0 };
    scan_compact(c, c->flag_ls.as<uint32_t>(), c->off_ls.as<uint32_t>(), nbr, c->list_ls.as<uint32_t>(), lc);
    CK(cudaStreamSynchronize(c->stream));
    return lc[0] + lc[1];
}

// Candidate bin range of each brick along one axis (bins overlapping [8b - R, 8b + 7 + R)) -> c->brick_rng.
static void upload_brick_ranges(ss_context *c, const SsDev &D) {
    std::vector<int2> h_rng(D.nb);
    for (int bb = 0; bb < D.nb; ++bb) {
        h_rng[bb].x = std::max(ss_floor_div(8 * bb - D.R, D.be) + D.nlo, 0);
        h_rng[bb].y = std::min(ss_floor_div(8 * bb + 6 + D.R, D.be) + D.nlo, D.nbin - 1);
    }
    c->brick_rng.ensure((size_t)D.nb * sizeof(int2));
    CK(cudaMemcpyAsync(c->brick_rng.p, h_rng.data(), (size_t)D.nb * sizeof(int2), cudaMemcpyHostToDevice, c->stream));
    CK(cudaStreamSynchronize(c->stream));
}

// Candidate bin range of a level-set field's point group along one axis (ss_field.cuh): the bins overlapping [8b - R, 8b + 8 + R),
// because a point of brick b lies anywhere in the cells 8b .. 8b + 7 -> c->fld_rng.
static void upload_field_brick_ranges(ss_context *c, const SsDev &D) {
    std::vector<int2> h_rng(D.nb);
    for (int bb = 0; bb < D.nb; ++bb) {
        h_rng[bb].x = std::max(ss_floor_div(8 * bb - D.R, D.be) + D.nlo, 0);
        h_rng[bb].y = std::min(ss_floor_div(8 * bb + 7 + D.R, D.be) + D.nlo, D.nbin - 1);
    }
    c->fld_rng.ensure((size_t)D.nb * sizeof(int2));
    CK(cudaMemcpyAsync(c->fld_rng.p, h_rng.data(), (size_t)D.nb * sizeof(int2), cudaMemcpyHostToDevice, c->stream));
    CK(cudaStreamSynchronize(c->stream));
}

// (i, j, k) of the flat index f of a subdomain in a grid of nsd subdomains (k fastest).
static void subdomain_ijk(int64_t f, const int64_t nsd[3], int64_t ijk[3]) {
    ijk[0] = f / (nsd[1] * nsd[2]); ijk[1] = (f - ijk[0] * nsd[1] * nsd[2]) / nsd[2]; ijk[2] = f - ijk[0] * nsd[1] * nsd[2] - ijk[1] * nsd[2];
}

// The tile of subdomain ijk (S cubes per axis, `sub_size` = c * S): its first global grid point and lower corner.
static SsTile make_tile(const int64_t ijk[3], int64_t S, const float gmin[3], float sub_size, uint32_t s, bool sparse) {
    SsTile T{};
    for (int d = 0; d < 3; ++d) { T.gbase[d] = (int)(ijk[d] * S); T.smin[d] = faddr(gmin[d], fmulr((float)ijk[d], sub_size)); }
    T.s = s; T.sparse = sparse ? 1u : 0u;
    return T;
}

// kernel.rs:327-336 (AVX-path constants) and :61-66 (scalar normalisation), evaluated in f32 like the reference
static void fill_kernel_consts(SsDev &D, float h) {
    D.a_hinv = fdivr(1.0f, h);
    float rrr = fmulr(fmulr(h, h), h);
    D.a_sigma = fdivr(8.0f, fmulr(SS_PI_F, rrr));
    D.a_s2 = fmulr(2.0f, D.a_sigma); D.a_s6 = fmulr(6.0f, D.a_sigma); D.a_s12 = fmulr(12.0f, D.a_sigma);
    D.s_sigma = fdivr(8.0f, rrr);
    D.s_c_inner = fdivr(3.0f, fmulr(2.0f, SS_PI_F));
    D.s_c_outer = fdivr(1.0f, fmulr(4.0f, SS_PI_F));
    D.s_two_thirds = fdivr(2.0f, 3.0f);
}
// splat bins: cubes of `be` cells; a brick (8 points) gathers the bins overlapping [8b - R, 8b + 7 + R)
static void fill_bins(SsDev &D, float cs) {
    D.nb = (D.np + 7) / 8;
    D.ext_bricks = (D.nb >= 2 && D.np == 8 * (D.nb - 1) + 1) ? 1 : 0;
    D.be = 8 * std::max(1, (7 + 2 * D.R + 39) / 40);
    D.nlo = (D.R + D.be - 1) / D.be;
    D.nbin = ss_floor_div(D.S + D.R, D.be) + D.nlo + 1;
    D.nbin_sub = D.nbin * D.nbin * D.nbin;
    D.inv_c = (float)(1.0 / (double)cs);
    D.rr_cells = (float)D.R + 0.01f;
}
// Tiles of S cubes of size cs, kernel of compact support h: the grid, kernel and bin constants of the level set (dense_subdomains.rs:89-244)
static void fill_tile_geometry(SsDev &D, float cs, int64_t S, float h, float rest_mass) {
    D.c = cs; D.h = h; D.h2 = fmulr(h, h); D.h2m = fmulr(D.h2, 1.01f); D.rest_mass = rest_mass;
    D.sub_size = fmulr(cs, (float)S); D.S = (int)S; D.np = (int)S + 1; D.np_magic = (uint32_t)(4294967296ull / (uint64_t)D.np) + 1u;
    D.R = (int)ceilf(fdivr(h, cs));
    fill_kernel_consts(D, h);
    fill_bins(D, cs);
}
// Membership (ghost) margin of the subdomain decomposition for a kernel reach r: ceil(r / cs) cubes plus 1 % (dense_subdomains.rs:89-244)
static float member_margin(float r, float cs) { return fmulr(fmulr(ceilf(fdivr(r, cs)), cs), 1.01f); }
// D.margin and the number of subdomains it spans, D.srad (D.sub_size set)
static int set_member_margin(SsDev &D, float margin) {
    D.margin = margin;
    D.srad = (int)ceilf(fdivr(margin, D.sub_size));
    if (D.srad > 8) return ss_fail(SS_ERR_INVALID_PARAMETER, "ghost margin spans more than 8 subdomains; increase subdomain_num_cubes_per_dim");
    return SS_OK;
}

// ------------------------------------------------------------------ the subdomain-grid pipeline ----
struct Partition {
    int enabled = 0;
    int axis = 0;
    int64_t own_lo = 0, own_hi = 0;     // owned subdomain index range along `axis`
    int64_t halo = 0;                   // extra subdomain layers kept for densities only
    uint64_t global_max_particles = 0;  // max particles per subdomain over ALL ranks (0: use the local maximum)
    int stop_after_decomposition = 0;   // only report the local maximum (out->max_particles)
    uint64_t (*max_reduce)(uint64_t local_max, void *user) = nullptr;   // all-reduce(MAX) of the local maximum across ranks
    void *max_reduce_user = nullptr;
    // SphInterpolator entry (ss_sph_interpolator_create_f32): densities supplied by the caller; stop after the particle bins are built
    const float *given_rho = nullptr;
    float given_mass = 0.0f;
    // level-set field (ss_levelset_field_create_f32): the context's level set up to its records in the splat bins; no level set, no mesh
    int field = 0;
};

// SPH densities (and optional CSR neighbour lists) of the filtered particles: per-subdomain cell lists on the h-lattice with
// ordered neighbour sums (dense_subdomains.rs:496-646), or one cell list over the whole domain in global mode.
static int stage_densities(ss_context *c, const SsDev &D, const float *d_xyz, uint64_t n, uint32_t M, uint32_t nsub, uint64_t g_ns_cells,
                           bool global_mode, bool want_nbrs, ss_surface *out, float *d_rho) {
    cudaStream_t st = c->stream;
    if ((uint64_t)nsub * (uint64_t)D.ns_stride >= 0xffffffffull || (uint64_t)nsub * (uint64_t)D.nbin_sub >= 0xffffffffull)
        return ss_fail(SS_ERR_INDEX_TOO_SMALL, "too many non-empty subdomains for 32-bit cell keys");
    c->err.ensure(4);
    CK(cudaMemsetAsync(c->err.p, 0, 4, st));
    // membership arrays: cid (compressed subdomain), val_b (particle); keys -> key_a, sorted -> key_b? key_b is in use
    // (flat ids are no longer needed after cid): reuse key_b as sort output, val_a as sorted payload.
    if (!global_mode) {
    LAUNCH(c, k_ns_keys, nblk(M, 256), 256, D, d_xyz, M, c->cid.as<uint32_t>(), c->sub_flat.as<uint32_t>(), c->val_b.as<uint32_t>(),
           c->key_a.as<uint32_t>(), c->err.as<int>());
    const uint64_t ns_keys = (uint64_t)nsub * D.ns_stride;
    // anisotropic mode: members outside the neighbourhood-search grid carry key 0xffffffff and sort behind every cell
    cub_sort(c, c->key_a.as<uint32_t>(), c->key_b.as<uint32_t>(), M, D.aniso ? 32 : bits_for(ns_keys), c->val_b.as<uint32_t>(), c->val_a.as<uint32_t>());
    c->tab_a.ensure((ns_keys + 1) * 4);                  // cell offsets
    LAUNCH(c, k_cell_offsets, nblk((uint64_t)M + 1, 256), 256, c->key_b.as<uint32_t>(), M, c->tab_a.as<uint32_t>(), (uint32_t)ns_keys);
    c->spos.ensure((size_t)M * 16);
    LAUNCH(c, k_gather_pos, nblk(M, 256), 256, d_xyz, c->val_a.as<uint32_t>(), M, c->spos.as<float4>());
    unsigned long long *d_ncnt = nullptr;
    if (want_nbrs) { out->nbr_off.ensure((n + 1) * 8); d_ncnt = out->nbr_off.as<unsigned long long>(); CK(cudaMemsetAsync(d_ncnt, 0, (n + 1) * 8, st)); }
    // entries with the particle inside the subdomain (every particle is inside at most one: <= n of them), compacted
    c->dflag.ensure((size_t)M * 4); c->doff.ensure((size_t)M * 4 + 4); c->dlist.ensure(std::max<uint64_t>(n, 1) * 4);
    if (c->density_variant >= 1 && !want_nbrs && !D.aniso) {
        // cell-cooperative kernel (ss_density.cuh): one warp per h-cell that holds a particle inside its subdomain (<= n cells), persistent grid
        LAUNCH(c, k_density_cell_flags, nblk(M, 256), 256, D, M, c->key_b.as<uint32_t>(), c->spos.as<float4>(), c->sub_flat.as<uint32_t>(),
               c->tab_a.as<uint32_t>(), c->dflag.as<uint32_t>());
        scan_compact(c, c->dflag.as<uint32_t>(), c->doff.as<uint32_t>(), M, c->dlist.as<uint32_t>());
        SsDcArgs DA{};
        DA.m = M; DA.list = c->dlist.as<uint32_t>(); DA.list_off = c->doff.as<uint32_t>(); DA.list_flag = c->dflag.as<uint32_t>();
        DA.key = c->key_b.as<uint32_t>(); DA.spos = c->spos.as<float4>(); DA.sub_flat = c->sub_flat.as<uint32_t>();
        DA.off = c->tab_a.as<uint32_t>(); DA.rho = d_rho; DA.nbr_count = nullptr;
        const unsigned grid = (unsigned)std::min<uint64_t>((uint64_t)c->sm_count * 7u, ((uint64_t)n + SS_DC_WARPS - 1) / SS_DC_WARPS);
        if (c->density_variant == 1) LAUNCH(c, k_density_cells<true>, std::max(grid, 1u), SS_DC_WARPS * 32, D, DA);
        else LAUNCH(c, k_density_cells<false>, std::max(grid, 1u), SS_DC_WARPS * 32, D, DA);
    } else {
    LAUNCH(c, k_density_flags, nblk(M, 256), 256, D, M, c->key_b.as<uint32_t>(), c->spos.as<float4>(), c->sub_flat.as<uint32_t>(), c->dflag.as<uint32_t>());
    scan_compact(c, c->dflag.as<uint32_t>(), c->doff.as<uint32_t>(), M, c->dlist.as<uint32_t>());
    LAUNCH(c, k_density<false>, nblk(n, SS_DENSITY_BLOCK), SS_DENSITY_BLOCK, D, M, c->dlist.as<uint32_t>(), c->doff.as<uint32_t>(), c->dflag.as<uint32_t>(),
           c->key_b.as<uint32_t>(), c->spos.as<float4>(), c->sub_flat.as<uint32_t>(),
           c->tab_a.as<uint32_t>(), d_rho, d_ncnt, (const unsigned long long *)nullptr, (uint32_t *)nullptr);
    }
    if (want_nbrs) {
        const uint64_t total = scan_neighbor_counts(c, d_ncnt, n);
        out->nbr_idx.ensure(std::max<uint64_t>(total, 1) * 4);
        LAUNCH(c, k_density<true>, nblk(n, SS_DENSITY_BLOCK), SS_DENSITY_BLOCK, D, M, c->dlist.as<uint32_t>(), c->doff.as<uint32_t>(), c->dflag.as<uint32_t>(),
               c->key_b.as<uint32_t>(), c->spos.as<float4>(), c->sub_flat.as<uint32_t>(),
               c->tab_a.as<uint32_t>(), d_rho, (unsigned long long *)nullptr, (const unsigned long long *)d_ncnt, out->nbr_idx.as<uint32_t>());
        out->has_neighbors = 1; out->n_neighbors = total;
    }
    } else {
        // one cell list over the whole domain; particles (not memberships) are the entries
        const uint32_t n32 = (uint32_t)n;
        c->gkey_a.ensure((size_t)n32 * 4); c->gkey_b.ensure((size_t)n32 * 4); c->gval_a.ensure((size_t)n32 * 4); c->gval_b.ensure((size_t)n32 * 4);
        LAUNCH(c, k_ns_keys_global, nblk(n32, 256), 256, D, d_xyz, n32, c->gkey_a.as<uint32_t>(), c->gval_a.as<uint32_t>(), c->err.as<int>());
        cub_sort(c, c->gkey_a.as<uint32_t>(), c->gkey_b.as<uint32_t>(), n32, bits_for(g_ns_cells), c->gval_a.as<uint32_t>(), c->gval_b.as<uint32_t>());
        c->tab_a.ensure((g_ns_cells + 1) * 4);            // cell offsets
        LAUNCH(c, k_cell_offsets, nblk((uint64_t)n32 + 1, 256), 256, c->gkey_b.as<uint32_t>(), n32, c->tab_a.as<uint32_t>(), (uint32_t)g_ns_cells);
        c->spos.ensure((size_t)n32 * 16);
        LAUNCH(c, k_gather_pos, nblk(n32, 256), 256, d_xyz, c->gval_b.as<uint32_t>(), n32, c->spos.as<float4>());
        unsigned long long *d_ncnt = nullptr;
        if (want_nbrs) { out->nbr_off.ensure((n + 1) * 8); d_ncnt = out->nbr_off.as<unsigned long long>(); CK(cudaMemsetAsync(d_ncnt, 0, (n + 1) * 8, st)); }
        LAUNCH(c, k_density_global<false>, nblk(n32, 128), 128, D, n32, c->gkey_b.as<uint32_t>(), c->spos.as<float4>(), c->tab_a.as<uint32_t>(),
               d_rho, d_ncnt, (const unsigned long long *)nullptr, (uint32_t *)nullptr);
        if (want_nbrs) {
            const uint64_t total = scan_neighbor_counts(c, d_ncnt, n);
            out->nbr_idx.ensure(std::max<uint64_t>(total, 1) * 4);
            LAUNCH(c, k_density_global<true>, nblk(n32, 128), 128, D, n32, c->gkey_b.as<uint32_t>(), c->spos.as<float4>(), c->tab_a.as<uint32_t>(),
                   d_rho, (unsigned long long *)nullptr, (const unsigned long long *)d_ncnt, out->nbr_idx.as<uint32_t>());
            out->has_neighbors = 1; out->n_neighbors = total;
        }
    }
    return SS_OK;
}

// Splat bins: memberships sorted by (subdomain, 8^3-point brick bin) + the particle records (x, y, z, V) the level set gathers.
// val_b still holds the membership particle indices in subdomain order (stable input for the bin sort).
// Anisotropic mode: d_xyz are the smoothed centres and `an_g` / `an_det` the per-particle G entries and determinants; the records
// then carry V det G and the G entries go to c->an_grec.  `record_event` = false: a re-binning that is not part of the stage time.
// Per-particle radii of the averaged surface: `av_delta` (delta_j per filtered particle) goes to c->av_rrec per membership.
static int stage_binning(ss_context *c, const SsDev &D, const float *d_xyz, const float *d_rho, uint32_t M, uint32_t nsub, bool partitioned,
                         const float *an_g = nullptr, const float *an_det = nullptr, bool record_event = true, const float *av_delta = nullptr) {
    cudaStream_t st = c->stream;
    LAUNCH(c, k_bin_keys, nblk(M, 256), 256, D, d_xyz, M, c->cid.as<uint32_t>(), c->sub_flat.as<uint32_t>(), c->val_b.as<uint32_t>(),
           partitioned ? c->sub_owned.as<uint8_t>() : nullptr, c->key_a.as<uint32_t>());
    cub_sort(c, c->key_a.as<uint32_t>(), c->key_b.as<uint32_t>(), M, 32, c->val_b.as<uint32_t>(), c->val_a.as<uint32_t>());
    const uint64_t bin_keys = (uint64_t)nsub * D.nbin_sub;
    c->tab_a.ensure(bin_keys * 4); c->tab_b.ensure(bin_keys * 4);
    CK(cudaMemsetAsync(c->tab_a.p, 0xff, bin_keys * 4, st));
    LAUNCH(c, k_mark_starts, nblk(M, 256), 256, c->key_b.as<uint32_t>(), M, c->tab_a.as<uint32_t>(), (uint32_t)bin_keys);
    LAUNCH(c, k_run_counts, nblk(M, 256), 256, c->key_b.as<uint32_t>(), M, c->tab_b.as<uint32_t>(), (uint32_t)bin_keys);
    c->rec.ensure((size_t)M * 16); c->ksplit.ensure((size_t)M * 4);
    LAUNCH(c, k_records, nblk(M, 256), 256, D, d_xyz, d_rho, M, c->key_b.as<uint32_t>(), c->val_a.as<uint32_t>(),
           c->sub_flat.as<uint32_t>(), c->rec.as<float4>(), c->ksplit.as<int>());
    if (an_g) {
        c->an_grec.ensure((size_t)M * 32);
        LAUNCH(c, k_records_aniso, nblk(M, 256), 256, M, c->key_b.as<uint32_t>(), c->val_a.as<uint32_t>(), an_g, an_det, c->rec.as<float4>(),
               c->an_grec.as<float4>());
    }
    if (av_delta) {
        c->av_rrec.ensure((size_t)M * 4);
        LAUNCH(c, k_records_radius, nblk(M, 256), 256, M, c->key_b.as<uint32_t>(), c->val_a.as<uint32_t>(), av_delta, c->av_rrec.as<float>());
    }
    int h_err = 0;
    CK(cudaMemcpyAsync(&h_err, c->err.p, 4, cudaMemcpyDeviceToHost, st));
    if (record_event) CK(cudaEventRecord(c->ev[5], st));
    CK(cudaStreamSynchronize(st));
    if (h_err) return ss_fail(SS_ERR_INVALID_PARAMETER, "particle outside of its subdomain's neighbourhood-search grid (reference: panic)");
    return SS_OK;
}


// Exact values for the flagged boxes of `n_bricks` listed bricks.  Variant 2: warp-per-brick kernel (ss_exact.cuh), bricks it
// cannot take come back in a fallback list and go through k_levelset (SS_LS_FIX) like in the other variants.
// received: the cascade's tier counters in ss_surface::ls_paths (exact or fix-up pass).
static void launch_exact(ss_context *c, const SsDev &D, const SsLsArgs &F, uint32_t n_bricks, bool global_mode, uint64_t &ls_launches,
                         uint64_t *received) {
    if (!n_bricks) return;
    const bool count = c->count_pairs != 0;
    if (c->ls_variant != 2) { launch_levelset(c, dim3(n_bricks), D, F, count, global_mode); ++ls_launches; return; }
    const auto args = [&](const uint32_t *list, uint32_t n, uint32_t *left) {
        SsXwArgs X{};
        X.bins = F.bins; X.bricks = list; X.n_bricks = n; X.wflag = F.wflag; X.tiles = F.tiles; X.fallback = left; X.pairs = F.pairs;
        X.taken = c->xw_taken.as<uint32_t>();
        X.phases = c->exact_phases ? c->xphase.as<unsigned long long>() : nullptr;
        return X;
    };
    // dense clusters: the same kernel with one warp per CTA and a larger slice -- up to 1024 candidates per brick (27 KB, static),
    // then up to 4096 (108 KB of dynamic shared memory); beyond that k_levelset's O(C^2) selection path (extreme clustering only)
    run_cascade(c, F.fix_bricks, n_bricks, {
        [&](const uint32_t *list, uint32_t n, uint32_t *left) {
            // persistent warps: one wave of CTAs (15 warps per SM), fewer when the list is short; the counter hands out the rest
            const unsigned grid = (unsigned)std::min<uint64_t>((uint64_t)c->sm_count * 5, (n + SS_XW_WARPS - 1) / SS_XW_WARPS);
            c->xw_taken.ensure(4);
            CK(cudaMemsetAsync(c->xw_taken.p, 0, 4, c->stream));
            if (c->exact_phases && !global_mode && !count) LAUNCH(c, (k_exact_warp<false, false, true>), grid, SS_XW_THREADS, D, args(list, n, left));
            else with_global_count(global_mode, count, [&](auto G, auto C) { LAUNCH(c, (k_exact_warp<G, C>), grid, SS_XW_THREADS, D, args(list, n, left)); });
        },
        [&](const uint32_t *list, uint32_t n, uint32_t *left) {
            with_global_count(global_mode, count, [&](auto G, auto C) { LAUNCH(c, (k_exact_warp_mid<G, C>), n, 32, D, args(list, n, left)); });
        },
        [&](const uint32_t *list, uint32_t n, uint32_t *left) {
            with_global_count(global_mode, count, [&](auto G, auto C) {
#ifndef SS_HOST_EMUL
                CK(cudaFuncSetAttribute(k_exact_warp_big<G, C>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SsXwSliceBig)));
#endif
                LAUNCH_DYN(c, (k_exact_warp_big<G, C>), n, 32, sizeof(SsXwSliceBig), D, args(list, n, left));
            });
        },
        [&](const uint32_t *list, uint32_t n, uint32_t *) {
            SsLsArgs G = F;
            G.fix_bricks = list;
            launch_levelset(c, dim3(n), D, G, count, global_mode);
        },
    }, ls_launches, received);
}

// Warp-per-brick level set of one batch for the fold F (anisotropic kernels, ss_aniso.cuh, or the averaged-position surface with
// or without its Jacobian correction and per-particle radii, ss_averaged.cuh): work list of non-empty bricks without extension tasks (the single-point
// planes of the last brick are bricks of their own), the 512-slot slice, then the 4096-slot slice, then selection.  Every listed brick gets state 2 (exact values).
// Returns the length of the work list.
template <class F>
static uint32_t launch_fold_levelset(ss_context *c, const SsDev &D, uint32_t nbatch, const float4 *grec, const float *rrec, uint64_t &ls_launches,
                                     uint64_t *received) {
    SsDev Dw = D;
    Dw.ext_bricks = 0;
    const uint32_t n_work = build_worklist(c, Dw, nbatch);
    const auto args = [&](const uint32_t *list, uint32_t n, uint32_t *left, uint8_t *bstate) {
        SsAnArgs A{};
        A.bins = context_bins(c); A.grec = grec; A.rrec = rrec; A.bricks = list; A.n_bricks = n; A.tiles = c->tiles.as<float>();
        A.bstate = bstate; A.fallback = left;
        return A;
    };
    run_cascade(c, c->list_ls.as<uint32_t>(), n_work, {
        [&](const uint32_t *list, uint32_t n, uint32_t *left) {
            LAUNCH(c, (k_fold_levelset<F, SS_AN_CAP, SS_AN_WARPS>), (n + SS_AN_WARPS - 1) / SS_AN_WARPS, SS_AN_WARPS * 32, Dw, args(list, n, left, c->bstate.as<uint8_t>()));
        },
        [&](const uint32_t *list, uint32_t n, uint32_t *left) { LAUNCH(c, (k_fold_levelset<F, SS_AN_BIG_CAP, 1>), n, 32, Dw, args(list, n, left, nullptr)); },
        [&](const uint32_t *list, uint32_t n, uint32_t *left) { LAUNCH(c, k_fold_select<F>, n, 32, Dw, args(list, n, left, nullptr)); },
    }, ls_launches, received);
    return n_work;
}

// Level set of one batch of tiles: work list, certification + exact values (fused kernel, or variant 1: certification kernel +
// exact pass), brick classification, fix-up sweep.  Leaves the tiles, the per-brick states and the marching-cubes brick list
// (c->list_mc, *n_mc_out entries) in the context scratch.
static int levelset_batch(ss_context *c, const SsDev &D, uint32_t nbatch, unsigned nbricks, bool exact_all, int certify_runs, bool global_mode,
                          bool averaged, ss_surface *out, uint64_t &ls_launches, uint64_t &fix_points, uint32_t *n_mc_out, int raw_q) {
    cudaStream_t st = c->stream;
    SsLsArgs A{};
    A.bins = context_bins(c); A.tiles = c->tiles.as<float>();
    A.pairs = c->count_pairs ? c->pairs.as<unsigned long long>() : nullptr;
    A.mode = exact_all ? SS_LS_EXACT_ALL : SS_LS_CERTIFY;
    A.wflag = nullptr; A.fix_bricks = nullptr; A.bstate = c->bstate.as<uint8_t>();
    uint64_t *const paths = out->ls_paths;
    const bool folded = D.aniso || averaged;            // warp-per-brick fold cascade, exact values only
    const float *const rrec = c->av_rrec.as<float>();    // per-particle radii (c->rad_on): delta_j per membership
    const uint32_t n_work = D.aniso ? launch_fold_levelset<SsAnisoFold>(c, D, nbatch, c->an_grec.as<float4>(), nullptr, ls_launches, paths + SS_LSP_ANISO_512)
                          : averaged && c->rad_on && c->ac_on ? launch_fold_levelset<SsAvgCorrRadFold>(c, D, nbatch, nullptr, rrec, ls_launches, paths + SS_LSP_AVG_512)
                          : averaged && c->rad_on ? launch_fold_levelset<SsAvgRadFold>(c, D, nbatch, nullptr, rrec, ls_launches, paths + SS_LSP_AVG_512)
                          : averaged && c->ac_on ? launch_fold_levelset<SsAvgCorrFold>(c, D, nbatch, nullptr, nullptr, ls_launches, paths + SS_LSP_AVG_512)
                          : averaged ? launch_fold_levelset<SsAvgFold>(c, D, nbatch, nullptr, nullptr, ls_launches, paths + SS_LSP_AVG_512)
                          : build_worklist(c, D, nbatch);
    A.work_list = c->list_ls.as<uint32_t>();
    const bool split_certify = !folded && c->ls_variant >= 1 && !exact_all && certify_runs <= 32;
    if (n_work && !split_certify && !folded) {
        launch_levelset(c, dim3(n_work), D, A, c->count_pairs != 0, global_mode); ++ls_launches;
        paths[SS_LSP_CERT_FUSED] += n_work;
    }
    if (n_work && split_certify) {
        // variant 1 (ss_certify.cuh): certification kernel, then the exact pass over the boxes it could not certify
        const uint32_t nbr_c = nbatch * nbricks;
        c->wstate.ensure((size_t)nbr_c * SS_LS_WARPS); c->wflag.ensure((size_t)nbr_c * SS_LS_WARPS); c->desc_ls.ensure((size_t)n_work * 16);
        c->flag_fix.ensure((size_t)nbr_c * 4); c->off_fix.ensure((size_t)nbr_c * 4 + 4); c->fix_list.ensure((size_t)nbr_c * 4);
        CK(cudaMemsetAsync(c->wstate.p, 0, (size_t)nbr_c * SS_LS_WARPS, st));
        LAUNCH(c, k_compact_desc, nblk(nbr_c, 256), 256, D, c->flag_ls.as<uint32_t>(), c->off_ls.as<uint32_t>(), nbr_c, c->desc_ls.as<uint4>());
        SsCertArgs CA{};
        CA.bins = A.bins; CA.work_desc = c->desc_ls.as<uint4>(); CA.tiles = A.tiles; CA.wstate = c->wstate.as<uint8_t>();
        if (c->ls_variant == 2) {
            // warp-per-brick certification: TMA-staged candidates, paired FP32 (ss_certify.cuh, variant 2)
            SsCwArgs W{};
            W.bins = A.bins; W.work_desc = c->desc_ls.as<uint4>(); W.n_work = n_work; W.tiles = A.tiles; W.wstate = c->wstate.as<uint8_t>();
            W.evals = c->count_pairs ? c->pairs.as<unsigned long long>() + 1 : nullptr;
            c->nflag.ensure(8);                                  // work-list counter of the persistent warps (the fix-up sweep re-zeroes it)
            CK(cudaMemsetAsync(c->nflag.p, 0, 4, st));
            W.taken = c->nflag.as<uint32_t>();
            // the bound runs in coordinates scaled by cs = 2^-e, h cs in [1, 2): the coefficients are O(1) at every h (G3 / h^6
            // in absolute units leaves the f32 range outside about 1e-6 < h < 1e6), and the scaling is exact in f32
            const int e = std::ilogb(D.h);
            const double hs = std::ldexp((double)D.h, -e), ih2 = 1.0 / (hs * hs);
            W.cs = std::ldexp(1.0f, -e);
            W.g1 = (float)((double)SS_G1 * ih2); W.g2 = (float)((double)SS_G2 * ih2 * ih2); W.g3 = (float)((double)SS_G3 * ih2 * ih2 * ih2);
            W.r0sq = 0.3025f * D.h2; W.r1sq = 0.58f * D.h2;
            const bool cw_small = certify_runs <= 16;            // at most 4 candidate bins per axis (3 + the extension plane)
            // persistent warps: one wave of CTAs (20 warps per SM), fewer when the work list is short
            const unsigned grid_s = (unsigned)std::min<uint64_t>((uint64_t)c->sm_count * (20 / SS_CW_WARPS_S), (n_work + SS_CW_WARPS_S - 1) / SS_CW_WARPS_S);
            const unsigned grid_l = (unsigned)std::min<uint64_t>((uint64_t)c->sm_count * (20 / SS_CW_WARPS_L), (n_work + SS_CW_WARPS_L - 1) / SS_CW_WARPS_L);
            with_global_count(global_mode, c->count_pairs != 0, [&](auto G, auto C) {
                if (cw_small) LAUNCH(c, (k_certify_warp<G, C, SS_CW_CAP_S, SS_CW_WARPS_S>), grid_s, SS_CW_WARPS_S * 32, D, W);
                else LAUNCH(c, (k_certify_warp<G, C, SS_CW_CAP_L, SS_CW_WARPS_L>), grid_l, SS_CW_WARPS_L * 32, D, W);
            });
            paths[cw_small ? SS_LSP_CERT_WARP_384 : SS_LSP_CERT_WARP_576] += n_work;
        } else {
            if (global_mode) LAUNCH(c, k_certify<true>, n_work, SS_LS_THREADS, D, CA);
            else LAUNCH(c, k_certify<false>, n_work, SS_LS_THREADS, D, CA);
            paths[SS_LSP_CERT_CTA] += n_work;
        }
        ++ls_launches;
        LAUNCH(c, k_wstate_reduce, nblk(nbr_c, 256), 256, c->wstate.as<uint8_t>(), nbr_c, c->bstate.as<uint8_t>(), c->flag_fix.as<uint32_t>(),
               c->wflag.as<uint8_t>());
        uint32_t ln[2] = { 0, 0 };
        scan_compact(c, c->flag_fix.as<uint32_t>(), c->off_fix.as<uint32_t>(), nbr_c, c->fix_list.as<uint32_t>(), ln);
        CK(cudaStreamSynchronize(st));
        if (ln[0] + ln[1]) {
            SsLsArgs F = A;
            F.mode = SS_LS_FIX; F.wflag = c->wflag.as<uint8_t>(); F.fix_bricks = c->fix_list.as<uint32_t>();
            launch_exact(c, D, F, ln[0] + ln[1], global_mode, ls_launches, paths + SS_LSP_EXACT_512);
        }
    }
    out->tm.bricks_levelset += n_work;
    if (raw_q >= 0) {
        // raw tap (ss_context_keep_levelset_tile_raw): tile q as certification and exact pass left it -- markers where the sweep
        // certified, before the fix-up pass replaces the ones next to outside points -- and its per-brick states
        const size_t np3 = (size_t)D.np * D.np * D.np;
        out->tile_raw.resize(np3); out->tile_raw_bstate.resize(nbricks);
        CK(cudaMemcpyAsync(out->tile_raw.data(), c->tiles.as<float>() + (size_t)raw_q * np3, np3 * 4, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(out->tile_raw_bstate.data(), c->bstate.as<uint8_t>() + (size_t)raw_q * nbricks, nbricks, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
    }
    // bricks that can carry surface (for marching cubes) / markers next to outside points (for the fix-up sweep)
    const uint32_t nbr_b = nbatch * nbricks;
    c->flag_mc.ensure((size_t)nbr_b * 4); c->flag_fix.ensure((size_t)nbr_b * 4); c->off_mc.ensure((size_t)nbr_b * 4 + 4); c->off_fix.ensure((size_t)nbr_b * 4 + 4);
    c->list_mc.ensure((size_t)nbr_b * 4); c->list_fix.ensure((size_t)nbr_b * 4);
    LAUNCH(c, k_brick_classify, nblk(nbr_b, 256), 256, D, c->bstate.as<uint8_t>(), nbr_b, c->flag_mc.as<uint32_t>(), c->flag_fix.as<uint32_t>());
    uint32_t lc[4] = { 0, 0, 0, 0 };
    scan_compact(c, c->flag_mc.as<uint32_t>(), c->off_mc.as<uint32_t>(), nbr_b, c->list_mc.as<uint32_t>(), &lc[0]);
    scan_compact(c, c->flag_fix.as<uint32_t>(), c->off_fix.as<uint32_t>(), nbr_b, c->list_fix.as<uint32_t>(), &lc[2]);
    if (c->ls_variant == 2 && split_certify && !global_mode)       // the tiles were not zero-filled: untouched bricks a later pass can read
        LAUNCH(c, k_zero_untouched, nblk((uint64_t)nbr_b * 32, 256), 256, D, c->bstate.as<uint8_t>(), c->flag_mc.as<uint32_t>(), c->flag_fix.as<uint32_t>(),
               nbr_b, c->tiles.as<float>());
    CK(cudaStreamSynchronize(st));
    const uint32_t n_mc = lc[0] + lc[1], n_fixscan = lc[2] + lc[3];
    out->tm.bricks_total += nbr_b; out->tm.bricks_mc += n_mc; out->tm.bricks_fixscan += n_fixscan;
    if (!exact_all && n_fixscan) {
        // exact values for certified points that turn out to lie on a surface-crossing edge
        const size_t nbr = (size_t)nbatch * nbricks;
        c->wflag.ensure(nbr * SS_LS_WARPS); c->brick_seen.ensure(nbr * 4); c->fix_list.ensure(nbr * 4); c->nflag.ensure(8);
        CK(cudaMemsetAsync(c->wflag.p, 0, nbr * SS_LS_WARPS, st));
        CK(cudaMemsetAsync(c->brick_seen.p, 0, nbr * 4, st));
        CK(cudaMemsetAsync(c->nflag.p, 0, 8, st));
        if (c->mc_variant == 1 && !global_mode)
            LAUNCH(c, k_fixup_flags_warp, (n_fixscan + SS_MW_WARPS - 1) / SS_MW_WARPS, SS_MW_WARPS * 32, D, c->tiles.as<float>(), c->list_fix.as<uint32_t>(), n_fixscan,
                   c->wflag.as<uint8_t>(), c->fix_list.as<uint32_t>(), c->nflag.as<uint32_t>());
        else
        LAUNCH(c, k_fixup_flags, n_fixscan, SS_TP_THREADS, D, c->tiles.as<float>(), c->list_fix.as<uint32_t>(), c->wflag.as<uint8_t>(),
               c->brick_seen.as<uint32_t>(), c->fix_list.as<uint32_t>(), c->nflag.as<uint32_t>());
        uint32_t nfl[2] = { 0, 0 };
        CK(cudaMemcpyAsync(nfl, c->nflag.p, 8, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        if (nfl[0]) {
            A.mode = SS_LS_FIX; A.wflag = c->wflag.as<uint8_t>(); A.fix_bricks = c->fix_list.as<uint32_t>();
            if (split_certify) launch_exact(c, D, A, nfl[0], global_mode, ls_launches, paths + SS_LSP_FIXUP_512);
            else { launch_levelset(c, dim3(nfl[0]), D, A, c->count_pairs != 0, global_mode); ++ls_launches; }
            fix_points += nfl[1];
        }
    }
    *n_mc_out = n_mc;
    return SS_OK;
}

// Marching cubes over the listed bricks of one batch: count, scan the brick totals, emit vertices, emit triangles; appends to
// the surface's mesh buffers and to the boundary-vertex list.
static int marching_cubes_batch(ss_context *c, const SsDev &D, bool global_mode, uint32_t n_mc, ss_surface *out, uint64_t &vtotal, uint64_t &ttotal) {
    cudaStream_t st = c->stream;
    const bool warp_mc = c->mc_variant == 1 && !global_mode;       // ss_mc.cuh: one warp per brick, count + emit
    uint32_t lv[2] = { 0, 0 }, lt[2] = { 0, 0 };                  // vertex / triangle totals of the batch
    if (n_mc) {
        if (warp_mc) LAUNCH(c, k_mc_count_warp, (n_mc + SS_MW_WARPS - 1) / SS_MW_WARPS, SS_MW_WARPS * 32, D, c->tiles.as<float>(), c->list_mc.as<uint32_t>(), n_mc,
                            c->vmask.as<uint8_t>(), c->voff.as<uint32_t>(), c->vcnt.as<uint32_t>(), c->tcnt.as<uint32_t>());
        else if (global_mode) LAUNCH(c, k_mc_count<true>, n_mc, SS_TP_THREADS, D, c->tiles.as<float>(), c->list_mc.as<uint32_t>(), c->vmask.as<uint8_t>(), c->vcnt.as<uint32_t>(), c->tcnt.as<uint32_t>());
        else LAUNCH(c, k_mc_count<false>, n_mc, SS_TP_THREADS, D, c->tiles.as<float>(), c->list_mc.as<uint32_t>(), c->vmask.as<uint8_t>(), c->vcnt.as<uint32_t>(), c->tcnt.as<uint32_t>());
        scan_with_total(c, c->vcnt.as<uint32_t>(), c->vblk_off.as<uint32_t>(), n_mc, lv);
        scan_with_total(c, c->tcnt.as<uint32_t>(), c->tblk_off.as<uint32_t>(), n_mc, lt);
    }
    uint32_t bc = 0;
    CK(cudaMemcpyAsync(&bc, c->bcount.p, 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    const uint64_t bv = (uint64_t)lv[0] + lv[1], bt = (uint64_t)lt[0] + lt[1];
    if (vtotal + bv >= 0xfffffff0ull || ttotal + bt >= 0xfffffff0ull) return ss_fail(SS_ERR_INDEX_TOO_SMALL, "mesh too large for 32-bit vertex / triangle ids");
    if (bv || bt) {
        out->verts.grow_keep((vtotal + bv) * 12, vtotal * 12, st);
        out->vkeys.grow_keep((vtotal + bv) * 8, vtotal * 8, st);
        out->tris.grow_keep((ttotal + bt) * 12, ttotal * 12, st);
        // boundary list can hold at most every vertex of the batch
        c->bkeys_a.grow_keep(((size_t)bc + bv) * 8, (size_t)bc * 8, st);
        c->bids_a.grow_keep(((size_t)bc + bv) * 4, (size_t)bc * 4, st);
        SsMcOut O{};
        O.verts = out->verts.as<float>(); O.tris = out->tris.as<uint32_t>(); O.vkeys = out->vkeys.as<unsigned long long>();
        O.bkeys = c->bkeys_a.as<unsigned long long>(); O.bids = c->bids_a.as<uint32_t>(); O.bcount = c->bcount.as<uint32_t>();
        O.vbase = (uint32_t)vtotal; O.tbase = (uint32_t)ttotal; O.bcap = (uint32_t)std::min<size_t>((size_t)bc + bv, 0xffffffffu);
        if (warp_mc) {
            LAUNCH(c, k_mc_emit_warp, (n_mc + SS_MW_WARPS - 1) / SS_MW_WARPS, SS_MW_WARPS * 32, D, c->tiles.as<float>(), c->list_mc.as<uint32_t>(), n_mc,
                   c->vmask.as<uint8_t>(), c->voff.as<uint32_t>(), c->vcnt.as<uint32_t>(), c->tcnt.as<uint32_t>(), c->vblk_off.as<uint32_t>(),
                   c->tblk_off.as<uint32_t>(), c->flag_mc.as<uint32_t>(), c->off_mc.as<uint32_t>(), c->tile_tab.as<SsTile>(), O);
        } else if (global_mode) {
            LAUNCH(c, k_mc_verts<true>, n_mc, SS_TP_THREADS, D, c->tiles.as<float>(), c->vmask.as<uint8_t>(), c->vblk_off.as<uint32_t>(),
                   c->vcnt.as<uint32_t>(), c->voff.as<uint32_t>(), c->tile_tab.as<SsTile>(), c->list_mc.as<uint32_t>(), O);
            LAUNCH(c, k_mc_tris<true>, n_mc, SS_TP_THREADS, D, c->tiles.as<float>(), c->vmask.as<uint8_t>(), c->tblk_off.as<uint32_t>(),
                   c->tcnt.as<uint32_t>(), c->voff.as<uint32_t>(), c->list_mc.as<uint32_t>(), O);
        } else {
            LAUNCH(c, k_mc_verts<false>, n_mc, SS_TP_THREADS, D, c->tiles.as<float>(), c->vmask.as<uint8_t>(), c->vblk_off.as<uint32_t>(),
                   c->vcnt.as<uint32_t>(), c->voff.as<uint32_t>(), c->tile_tab.as<SsTile>(), c->list_mc.as<uint32_t>(), O);
            LAUNCH(c, k_mc_tris<false>, n_mc, SS_TP_THREADS, D, c->tiles.as<float>(), c->vmask.as<uint8_t>(), c->tblk_off.as<uint32_t>(),
                   c->tcnt.as<uint32_t>(), c->voff.as<uint32_t>(), c->list_mc.as<uint32_t>(), O);
        }
        vtotal += bv; ttotal += bt;
    }
    return SS_OK;
}

// Welds the vertices that carry the same MC edge key: c->bkeys_a holds the keys of the `bc` candidate vertices `ids`.  The kept
// vertices of verts / keys (nv) go to nverts / nkeys in order, the nt triangles are renumbered in place; returns how many are kept.
static uint64_t weld_vertices(ss_context *c, const uint32_t *ids, uint32_t bc, const float *verts, const unsigned long long *keys, uint64_t nv,
                              uint32_t *tris, uint64_t nt, DevBuf &nverts, DevBuf &nkeys) {
    c->bkeys_b.ensure((size_t)bc * 8); c->bids_b.ensure((size_t)bc * 4);
    cub_sort(c, c->bkeys_a.as<unsigned long long>(), c->bkeys_b.as<unsigned long long>(), bc, 64, ids, c->bids_b.as<uint32_t>());
    c->remap.ensure(nv * 4); c->keep.ensure(nv * 4); c->newid.ensure(nv * 4 + 4);
    LAUNCH(c, k_iota_keep, nblk(nv, 256), 256, (uint32_t)nv, c->remap.as<uint32_t>(), c->keep.as<uint32_t>());
    LAUNCH(c, k_weld_runs, nblk(bc, 256), 256, c->bkeys_b.as<unsigned long long>(), c->bids_b.as<uint32_t>(), bc,
           c->remap.as<uint32_t>(), c->keep.as<uint32_t>());
    const uint64_t nv_final = scan_total(c, c->keep.as<uint32_t>(), c->newid.as<uint32_t>(), (uint32_t)nv);
    nverts.ensure(std::max<uint64_t>(nv, 1) * 12); nkeys.ensure(std::max<uint64_t>(nv, 1) * 8);
    LAUNCH(c, k_compact_verts, nblk(nv, 256), 256, (uint32_t)nv, c->keep.as<uint32_t>(), c->newid.as<uint32_t>(), verts, keys,
           nverts.as<float>(), nkeys.as<unsigned long long>());
    if (nt) LAUNCH(c, k_remap_tris, nblk(nt * 3, 256), 256, nt * 3, c->remap.as<uint32_t>(), c->newid.as<uint32_t>(), tris);
    return nv_final;
}

// Stitching: weld duplicated boundary vertices (same MC edge key), compact the vertices, remap the triangle indices.
static int weld_boundary_vertices(ss_context *c, ss_surface *out, uint64_t vtotal, uint64_t ttotal, uint64_t &nv_final_out, uint32_t &bc_out) {
    cudaStream_t st = c->stream;
    uint32_t bc = 0;
    CK(cudaMemcpyAsync(&bc, c->bcount.p, 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    uint64_t nv_final = vtotal;
    if (vtotal && bc) {
        // compact into the context's spare mesh buffers, which keep the pre-weld buffers for the next frame
        nv_final = weld_vertices(c, c->bids_a.as<uint32_t>(), bc, out->verts.as<float>(), out->vkeys.as<unsigned long long>(), vtotal,
                                 out->tris.as<uint32_t>(), ttotal, c->o_verts2, c->o_vkeys2);
        CK(cudaStreamSynchronize(st));
        std::swap(out->verts, c->o_verts2); std::swap(out->vkeys, c->o_vkeys2);
    }
    nv_final_out = nv_final; bc_out = bc;
    return SS_OK;
}

// Per-particle radii of the averaged surface (DESIGN.md §12.2): checks all n_in radii of the context (0 < radius_factor * r_j < h,
// one read-back of the count and the first offending index), then delta_j = radius_factor * r_j - R_s of the particles the
// particle-AABB filter kept (prepare_particles left its flags and offsets in the context scratch) into c->av_delta.
static int prepare_radii(ss_context *c, const ss_params_f32 *p, uint64_t n_in, float factor, float h, float rs) {
    if (!n_in) return SS_OK;
    cudaStream_t st = c->stream;
    const float *radii = c->av_radii.as<float>();
    c->av_chk.ensure(8);
    const uint32_t init[2] = { 0u, 0xffffffffu };
    uint32_t chk[2];
    CK(cudaMemcpyAsync(c->av_chk.p, init, 8, cudaMemcpyHostToDevice, st));
    LAUNCH(c, k_radii_check, nblk(n_in, 256), 256, radii, n_in, factor, h, c->av_chk.as<uint32_t>());
    CK(cudaMemcpyAsync(chk, c->av_chk.p, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (chk[0]) {
        char msg[240];
        snprintf(msg, sizeof msg, "averaged surface radii: radius_factor * radius must be finite and lie in (0, compact support radius); "
                 "%u of %llu radii are not, the first at index %u", chk[0], (unsigned long long)n_in, chk[1]);
        return ss_fail(SS_ERR_INVALID_PARAMETER, msg);
    }
    const bool filtered = p->has_particle_aabb != 0;
    c->av_delta.ensure(n_in * 4);
    LAUNCH(c, k_radii_delta, nblk(n_in, 256), 256, radii, n_in, filtered ? c->filt_flag.as<uint8_t>() : nullptr,
           filtered ? c->filt_off.as<uint32_t>() : nullptr, factor, rs, c->av_delta.as<float>());
    return SS_OK;
}

static int run_subdomain_grid(ss_context *c, const Prepared &PP, const ss_params_f32 *p, ss_surface *out, const Partition &part = Partition(),
                              bool global_mode = false) {
    const uint64_t n = PP.n;
    const float *d_xyz = PP.d_xyz;
    cudaStream_t st = c->stream;

    // ---- initialize_parameters, dense_subdomains.rs:89-244
    // global path (reconstruction.rs:65-194): tiles of 64 cells are an implementation detail, the arithmetic is global
    const int64_t S = global_mode ? 64 : (int64_t)p->subdomain_num_cubes_per_dim;
    const float h = p->compact_support_radius, cs = p->cube_size;
    const float r2 = faddr(p->particle_radius, p->particle_radius);
    const float rest_mass = fmulr(fmulr(fmulr(r2, r2), r2), p->rest_density);
    const float ns_margin = global_mode ? fmulr(cs, ceilf(fdivr(h, cs)) + 2.0f)      // stencil reach (R + 1 cells) + slack
                                        : member_margin(h, cs);
    // anisotropic kernels (ss_aniso.cuh): a kernel centre moves up to smoothing * h < h from its particle, so memberships need a
    // margin of 2h; the neighbourhood-search grids and cell lists stay on the standard margin (bit-identical densities)
    const bool aniso = c->an_on && !global_mode && !part.enabled && !part.given_rho;
    // averaged-position surface (ss_averaged.cuh): kernel centres at the particles, standard margins and bins; surface f = h - R_s
    const bool averaged = c->avg_on && !global_mode && !part.enabled && !part.given_rho;
    const float margin = aniso ? member_margin(fmulr(2.0f, h), cs) : ns_margin;
    int64_t nsd[3], ncg[3];
    for (int d = 0; d < 3; ++d) { nsd[d] = (PP.grid.nc[d] + S - 1) / S; ncg[d] = nsd[d] * S; }
    HostGrid gg, sg;
    int rc = grid_new(gg, PP.grid.mn, ncg, cs);
    if (rc) return ss_fail(rc, "global marching cubes grid construction failed");
    const float sub_size = fmulr(cs, (float)S);
    rc = grid_new(sg, gg.mn, nsd, sub_size);
    if (rc) return ss_fail(rc, "subdomain grid construction failed");
    out->grid = global_mode ? PP.grid : gg; out->subgrid = sg; out->S = (int)S;

    for (int d = 0; d < 3; ++d) {
        if (gg.np[d] >= (1 << 20)) return ss_fail(SS_ERR_INDEX_TOO_SMALL, "more than 2^20 grid points per dimension are not supported by the device path");
    }
    if ((double)nsd[0] * (double)nsd[1] * (double)nsd[2] >= 2147483647.0) return ss_fail(SS_ERR_INDEX_TOO_SMALL, "too many subdomain slots");
    if (S > 1024) return ss_fail(SS_ERR_INDEX_TOO_SMALL, "subdomain_num_cubes_per_dim > 1024 is not supported");
    {
        // Far from the origin f32 grid coordinates round by a visible fraction of a cell.  The splat bins place a particle by its
        // cell with no slack for that rounding (DESIGN.md 4.3).  The limit ulp / c <= 1/64 is a tested one, not a derived bound:
        // up to it the device matches the oracle and the oracle matches the reference's binary; at 1/32 the latter pin fails.
        double amax = 0.0;
        for (int d = 0; d < 3; ++d) amax = std::max({ amax, std::fabs((double)gg.mn[d]), std::fabs((double)gg.mx[d]) });
        const double ulp = std::ldexp(1.0, std::ilogb(std::max(amax, 1e-30)) - 23);
        if (ulp > (double)cs / 64.0) {
            char msg[200];
            snprintf(msg, sizeof msg, "grid coordinates up to %.6g round by %.3g cells (ulp / cube size > 1/64): too far from the origin for the "
                     "device level set at this cube size; translate the particles towards the origin", amax, ulp / (double)cs);
            return ss_fail(SS_ERR_REAL_TOO_SMALL, msg);
        }
    }

    SsDev D{};
    for (int d = 0; d < 3; ++d) { D.gmin[d] = gg.mn[d]; D.nsd[d] = (int)nsd[d]; }
    fill_tile_geometry(D, cs, S, h, rest_mass);
    rc = set_member_margin(D, margin);
    if (rc) return rc;
    D.thr = p->iso_surface_threshold; D.grow = fmulr(ns_margin, 1.5f);
    if (averaged) {
        // DESIGN.md §12: 0 < R_s < h, so that t = h - R_s > 0 and a point no particle reaches (f = 0) lies outside
        const float rs = fmulr(c->avg.radius_factor, p->particle_radius);
        if (!(rs > 0.0f && rs < h) || !std::isfinite(rs))
            return ss_fail(SS_ERR_INVALID_PARAMETER, "averaged surface: radius_factor * particle_radius must lie in (0, compact support radius)");
        D.thr = fsubr(h, rs);
        D.av_rs = rs; D.av_low = c->ac.t_low; D.av_high = c->ac.t_high;     // read by SsAvgCorrFold only (DESIGN.md §12.1)
        if (c->rad_on) {
            rc = prepare_radii(c, p, out->n_in, c->avg.radius_factor, h, rs);
            if (rc) return rc;
        }
    }
    D.nsD = (int)ceil(((double)S * cs + 3.0 * (double)ns_margin) / (double)h) + 3;
    D.ns_stride = D.nsD * D.nsD * D.nsD;
    D.simd = p->enable_simd ? 1 : 0;
    D.gmode = global_mode ? 1 : 0;
    D.aniso = aniso ? 1 : 0;
    D.an_lambda = c->an.smoothing; D.an_kr = c->an.max_stretch; D.an_min_nb = c->an.min_neighbors;
    uint64_t g_ns_cells = 0;
    if (global_mode) {
        HostGrid ns;
        int rcn = grid_from_aabb(ns, PP.grid.mn, PP.grid.mx, h);                       // neighborhood_search.rs:172-173
        if (rcn) return ss_fail(SS_ERR_INVALID_PARAMETER, "failed to construct grid for neighborhood search");
        for (int d = 0; d < 3; ++d) { D.g_ns_amin[d] = ns.mn[d]; D.g_ns_nc[d] = (int)ns.nc[d]; }
        g_ns_cells = (uint64_t)ns.nc[0] * ns.nc[1] * ns.nc[2];
        if (g_ns_cells >= (1ull << 28)) return ss_fail(SS_ERR_INDEX_TOO_SMALL, "domain too large for the global (non-decomposed) path");
        const float half_real = ceilf(fdivr(h, cs));
        const float rev = fmulr(fmulr(cs, half_real), faddr(1.0f, sqrtf(FLT_EPSILON)));   // density_map.rs:575-576
        D.rev2 = fmulr(rev, rev); D.sup = 2 * D.R + 2;
        for (int d = 0; d < 3; ++d) { D.g_allow_min[d] = fsubr(PP.grid.mn[d], -rev); D.g_allow_max[d] = faddr(PP.grid.mx[d], -rev); }
        bool degen = D.g_allow_min[0] == D.g_allow_max[0] && D.g_allow_min[1] == D.g_allow_max[1] && D.g_allow_min[2] == D.g_allow_max[2];
        bool cons = D.g_allow_min[0] <= D.g_allow_max[0] && D.g_allow_min[1] <= D.g_allow_max[1] && D.g_allow_min[2] <= D.g_allow_max[2];
        if (degen || !cons) return ss_fail(SS_ERR_INVALID_DOMAIN, "the allowed domain of particles is inconsistent/degenerate (DensityMapError::InvalidDomain)");
    }
    D.part_axis = part.enabled ? part.axis : 0;
    D.keep_lo = part.enabled ? (int)std::max<int64_t>(part.own_lo - part.halo, 0) : 0;
    D.keep_hi = part.enabled ? (int)std::min<int64_t>(part.own_hi + part.halo, nsd[D.part_axis]) : (int)nsd[0];
    if (!part.enabled) { D.part_axis = 0; D.keep_lo = 0; D.keep_hi = (int)nsd[0]; }
    int certify_runs = 0;              // upper bound of the candidate runs of a brick (variant 1 keeps one per lane)
    {
        int per_axis = ss_floor_div(6 + D.R, D.be) - ss_floor_div(-D.R, D.be) + 2;
        if (per_axis * per_axis > 128) return ss_fail(SS_ERR_INVALID_PARAMETER, "internal: too many candidate bin runs per brick");
        certify_runs = per_axis * per_axis;
    }
    out->ls_paths[SS_LSP_GLOBAL] = global_mode ? 1 : 0; out->ls_paths[SS_LSP_COUNT_PAIRS] = c->count_pairs ? 1 : 0;
    out->ls_paths[SS_LSP_R] = (uint64_t)D.R; out->ls_paths[SS_LSP_BIN_CELLS] = (uint64_t)D.be;

    const bool want_nbrs = p->global_neighborhood_list != 0 && !part.enabled;
    CK(cudaEventRecord(c->ev[2], st));
    out->nv = out->nt = 0; out->nsub = 0;
    out->owner = c;
    c->post.valid = 0; out->frame = ++c->frame;
    out->rho = std::move(c->o_rho); out->verts = std::move(c->o_verts); out->tris = std::move(c->o_tris); out->vkeys = std::move(c->o_vkeys);
    out->rho.ensure(std::max<uint64_t>(n, 1) * 4);
    float *d_rho = out->rho.as<float>();
    CK(cudaMemsetAsync(d_rho, 0, std::max<uint64_t>(n, 1) * 4, st));
    if (aniso) {
        out->an_xbar.ensure(std::max<uint64_t>(n, 1) * 12); out->an_g.ensure(std::max<uint64_t>(n, 1) * 24); c->an_det.ensure(std::max<uint64_t>(n, 1) * 4);
        if (n) LAUNCH(c, k_aniso_init, nblk(n, 256), 256, d_xyz, (uint32_t)n, out->an_xbar.as<float>(), out->an_g.as<float>(), c->an_det.as<float>());
        out->has_aniso = 1;
    }
    // Early end without a mesh: the remaining stage events are recorded (the entries read the stage times).  NOTE (multi-GPU): the
    // max-reduce callback is a collective -- every rank must call it exactly once per reconstruction, also ranks that received no
    // particles or own no subdomain.
    const auto finish_early = [&](bool reduce) {
        for (int e = 3; e <= 9; ++e) CK(cudaEventRecord(c->ev[e], st));
        CK(cudaStreamSynchronize(st));
        if (reduce && part.enabled && part.max_reduce) part.max_reduce(0, part.max_reduce_user);
        return SS_OK;
    };
    if (part.field) {
        out->fld = 1; out->fld_D = D;
        out->fld_mode = aniso ? SS_FLD_ANISO : !averaged ? SS_FLD_SPH
                      : c->ac_on ? (c->rad_on ? SS_FLD_AVG_CORR_RAD : SS_FLD_AVG_CORR) : (c->rad_on ? SS_FLD_AVG_RAD : SS_FLD_AVG);
    }
    if (n == 0) return finish_early(true);

    // ---- decomposition: memberships (owner + ghosts), stable sort by subdomain
    c->cnt.ensure(n * 4); c->off.ensure(n * 4 + 4);
    LAUNCH(c, k_classify_count, nblk(n, 256), 256, D, d_xyz, (uint32_t)n, c->cnt.as<uint32_t>());
    const uint64_t M64 = scan_total(c, c->cnt.as<uint32_t>(), c->off.as<uint32_t>(), (uint32_t)n);
    if (M64 >= 0xfffffff0ull) return ss_fail(SS_ERR_INDEX_TOO_SMALL, "more than 2^32 subdomain memberships");
    const uint32_t M = (uint32_t)M64;
    if (M == 0) return finish_early(true);
    c->key_a.ensure((size_t)M * 4); c->key_b.ensure((size_t)M * 4); c->val_a.ensure((size_t)M * 4); c->val_b.ensure((size_t)M * 4);
    LAUNCH(c, k_classify_fill, nblk(n, 256), 256, D, d_xyz, (uint32_t)n, c->off.as<uint32_t>(), c->key_a.as<uint32_t>(), c->val_a.as<uint32_t>());
    const uint64_t nslots = (uint64_t)nsd[0] * nsd[1] * nsd[2];
    cub_sort(c, c->key_a.as<uint32_t>(), c->key_b.as<uint32_t>(), M, bits_for(nslots), c->val_a.as<uint32_t>(), c->val_b.as<uint32_t>());
    // key_b = flat subdomain per membership (sorted), val_b = particle index (ascending inside a subdomain)
    c->flags.ensure((size_t)M * 4); c->scan.ensure((size_t)M * 4); c->cid.ensure((size_t)M * 4);
    LAUNCH(c, k_seg_flags, nblk(M, 256), 256, c->key_b.as<uint32_t>(), M, c->flags.as<uint32_t>());
    cub_scan<true>(c, c->flags.as<const uint32_t>(), c->scan.as<uint32_t>(), M);
    uint32_t nsub = 0;
    CK(cudaMemcpyAsync(&nsub, c->scan.as<uint32_t>() + (M - 1), 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    c->sub_flat.ensure((size_t)nsub * 4); c->sub_off.ensure((size_t)(nsub + 1) * 4);
    LAUNCH(c, k_seg_finish, nblk(M, 256), 256, c->key_b.as<uint32_t>(), M, c->scan.as<uint32_t>(), c->cid.as<uint32_t>(),
           c->sub_flat.as<uint32_t>(), c->sub_off.as<uint32_t>());
    std::vector<uint32_t> h_flat(nsub), h_off(nsub + 1);
    CK(cudaMemcpyAsync(h_flat.data(), c->sub_flat.p, (size_t)nsub * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(h_off.data(), c->sub_off.p, (size_t)(nsub + 1) * 4, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    // sparse classification, dense_subdomains.rs:1242-1251, :1590
    uint64_t maxp = 0;
    for (uint32_t s = 0; s < nsub; ++s) maxp = std::max<uint64_t>(maxp, h_off[s + 1] - h_off[s]);
    out->max_particles = maxp;
    if (part.enabled && part.max_reduce) maxp = std::max<uint64_t>(maxp, part.max_reduce(maxp, part.max_reduce_user));
    if (part.enabled && part.global_max_particles) maxp = std::max<uint64_t>(maxp, part.global_max_particles);
    const uint64_t sparse_limit = std::max<uint64_t>(maxp / 20, 100);
    out->nsub = nsub; out->sub_flat.resize(nsub); out->sub_count.resize(nsub); out->sub_sparse.resize(nsub);
    std::vector<uint8_t> h_owned(nsub, 1);
    std::vector<uint32_t> owned_list;
    owned_list.reserve(nsub);
    for (uint32_t s = 0; s < nsub; ++s) {
        out->sub_flat[s] = h_flat[s]; out->sub_count[s] = h_off[s + 1] - h_off[s];
        out->sub_sparse[s] = (!global_mode && out->sub_count[s] <= sparse_limit) ? 1 : 0;
        if (part.enabled) {
            int64_t ijk[3];
            subdomain_ijk(h_flat[s], nsd, ijk);
            h_owned[s] = (ijk[part.axis] >= part.own_lo && ijk[part.axis] < part.own_hi) ? 1 : 0;
        }
        if (h_owned[s]) owned_list.push_back(s);
    }
    out->sub_owned = h_owned;
    if (part.enabled && part.stop_after_decomposition) return finish_early(false);   // (the max-reduce ran above)
    c->sub_owned.ensure(nsub);
    CK(cudaMemcpyAsync(c->sub_owned.p, h_owned.data(), nsub, cudaMemcpyHostToDevice, st));
    CK(cudaEventRecord(c->ev[3], st));

    if (part.given_rho) {
        // SphInterpolator::new (sph_interpolation.rs:40-80): the caller's densities and the particle bins the queries of ss_post.cuh walk;
        // no density pass, no level set, no mesh
        c->err.ensure(4);
        CK(cudaMemsetAsync(c->err.p, 0, 4, st));
        CK(cudaMemcpyAsync(d_rho, part.given_rho, (size_t)n * 4, cudaMemcpyDefault, st));
        CK(cudaEventRecord(c->ev[4], st));
        rc = stage_binning(c, D, d_xyz, d_rho, M, nsub, false);
        if (rc) return rc;
        c->post.D = D; c->post.nsub = nsub; c->post.M = M; c->post.partitioned = 0; c->post.sphere_mass = part.given_mass; c->post.valid = 1;
        for (int e = 6; e <= 9; ++e) CK(cudaEventRecord(c->ev[e], st));
        CK(cudaStreamSynchronize(st));
        return SS_OK;
    }

    // ---- densities, then the splat bins
    rc = stage_densities(c, D, d_xyz, n, M, nsub, g_ns_cells, global_mode, want_nbrs, out, d_rho);
    if (rc) return rc;
    if (aniso) {
        // x_bar, G, det G of every particle in its owning subdomain, over the density stage's list and cell tables
        CK(cudaEventRecord(c->ev_an[0], st));
        LAUNCH(c, k_aniso, nblk(n, 128), 128, D, M, c->dlist.as<uint32_t>(), c->doff.as<uint32_t>(), c->dflag.as<uint32_t>(),
               c->key_b.as<uint32_t>(), c->spos.as<float4>(), c->sub_flat.as<uint32_t>(), c->tab_a.as<uint32_t>(),
               out->an_xbar.as<float>(), out->an_g.as<float>(), c->an_det.as<float>());
        CK(cudaEventRecord(c->ev_an[1], st));
    }
    CK(cudaEventRecord(c->ev[4], st));
    if (aniso) rc = stage_binning(c, D, out->an_xbar.as<float>(), d_rho, M, nsub, false, out->an_g.as<float>(), c->an_det.as<float>());
    else rc = stage_binning(c, D, d_xyz, d_rho, M, nsub, part.enabled != 0, nullptr, nullptr, true,
                            averaged && c->rad_on ? c->av_delta.as<float>() : nullptr);
    if (rc) return rc;
    if (part.field) {
        // the records of the level set stay in the scratch for ss_levelset_field_at_f32 (DESIGN.md §13)
        if ((uint64_t)nsub * (uint64_t)(D.nb * D.nb * D.nb) >= 0xffffffffull)
            return ss_fail(SS_ERR_INDEX_TOO_SMALL, "too many non-empty subdomains for 32-bit point group keys");
        upload_field_brick_ranges(c, D);
        out->fld_nsub = nsub; out->fld_ready = 1;
        for (int e = 6; e <= 9; ++e) CK(cudaEventRecord(c->ev[e], st));
        CK(cudaStreamSynchronize(st));
        return SS_OK;
    }

    // ---- level set + marching cubes over batches of subdomain tiles
    const size_t np3 = (size_t)D.np * D.np * D.np;
    const unsigned nbricks = (unsigned)(D.nb * D.nb * D.nb);
    const size_t per_tile = np3 * (4 + 4 + 1) + (size_t)nbricks * (SS_LS_WARPS + 8 + 1 + 16) + 256;
    // as many tiles per batch as fit a third of the free memory (fewer host synchronisations per frame); the brick index
    // tile * nb^3 + ... must stay below 2^31
    const uint32_t nown = (uint32_t)owned_list.size();
    // The tile buffers of the previous frame are reused whenever they hold all tiles or at least half of what a fresh
    // allocation would get: the amount of free memory wobbles from frame to frame (result buffers in flight), and re-allocating
    // tens of GB is slow.  The free memory is only queried when the buffers do not hold all tiles: cudaMemGetInfo takes a
    // device-wide lock, and with an `nvidia-smi -lms 200` sampler running beside the process (bench.py's clock record) it can
    // stall here on every step the sampler's query falls into (tile_setup in the timings).
    const size_t have_tiles = std::min(c->tiles.cap / (np3 * 4), std::min(c->voff.cap / (np3 * 4), c->vmask.cap / np3));
    size_t max_tiles;
    if (c->max_tiles) max_tiles = c->max_tiles;
    else if (have_tiles >= nown && have_tiles) max_tiles = have_tiles;
    else {
        size_t free_b = 0, total_b = 0;
        CK(cudaMemGetInfo(&free_b, &total_b));
        const size_t reusable = c->tiles.cap + c->voff.cap + c->vmask.cap;
        const size_t want_tiles = std::max<size_t>(1, ((free_b + reusable) / 3) / per_tile);
        max_tiles = (have_tiles >= want_tiles / 2 && have_tiles) ? have_tiles : want_tiles;
    }
    max_tiles = std::min<size_t>(max_tiles, std::max<size_t>(1, (size_t)0x7fffffff / nbricks / 2));
    max_tiles = std::min<size_t>(max_tiles, std::max<uint32_t>(nown, 1));
    const size_t nblk_max = max_tiles * nbricks;
    c->tiles.ensure(max_tiles * np3 * 4); c->voff.ensure(max_tiles * np3 * 4); c->vmask.ensure(max_tiles * np3);
    c->vcnt.ensure(nblk_max * 4 + 4); c->tcnt.ensure(nblk_max * 4 + 4); c->vblk_off.ensure(nblk_max * 4 + 4); c->tblk_off.ensure(nblk_max * 4 + 4);
    c->tile_tab.ensure(max_tiles * sizeof(SsTile)); c->bstate.ensure(nblk_max);
    c->bcount.ensure(4); c->pairs.ensure(16);
    CK(cudaMemsetAsync(c->bcount.p, 0, 4, st));
    CK(cudaMemsetAsync(c->pairs.p, 0, 16, st));
    upload_brick_ranges(c, D);
    std::vector<SsTile> h_tiles(max_tiles);
    uint64_t vtotal = 0, ttotal = 0;
    size_t bcap = std::max<size_t>(1 << 16, c->hint_bc + c->hint_bc / 8);
    c->bkeys_a.ensure(bcap * 8); c->bids_a.ensure(bcap * 4);
    size_t vcap = std::max<size_t>(1 << 16, c->hint_nv + c->hint_nv / 8), tcap = std::max<size_t>(1 << 17, c->hint_nt + c->hint_nt / 8);
    out->verts.ensure(vcap * 12); out->vkeys.ensure(vcap * 8); out->tris.ensure(tcap * 12);
    float ls_ms = 0.f, mc_ms = 0.f, setup_ms = 0.f;
    uint64_t ls_launches = 0, fix_points = 0;
    out->tile.clear(); out->tile_raw.clear(); out->tile_raw_bstate.clear();
    const bool exact_all = c->ls_exact_all || c->keep_tile_flat >= 0 || aniso || averaged;
    for (uint32_t s0 = 0; s0 < nown; s0 += (uint32_t)max_tiles) {
        const uint32_t nbatch = std::min<uint32_t>((uint32_t)max_tiles, nown - s0);
        for (uint32_t q = 0; q < nbatch; ++q) {
            const uint32_t sid = owned_list[s0 + q];
            int64_t ijk[3];
            subdomain_ijk(h_flat[sid], nsd, ijk);
            h_tiles[q] = make_tile(ijk, S, gg.mn, sub_size, sid, out->sub_sparse[sid] || !D.simd);
        }
        CK(cudaMemcpyAsync(c->tile_tab.p, h_tiles.data(), (size_t)nbatch * sizeof(SsTile), cudaMemcpyHostToDevice, st));
        // level-set variant 2 writes every value a later pass reads (markers, exact values, exact zeros) and fills the untouched
        // bricks next to listed ones itself (k_zero_untouched): no zero-fill of the tiles (16 GB at 50 M particles)
        const bool lazy_zero = c->ls_variant == 2 && !exact_all && certify_runs <= 32 && !global_mode;
        if (!lazy_zero) CK(cudaMemsetAsync(c->tiles.p, 0, (size_t)nbatch * np3 * 4, st));
        CK(cudaMemsetAsync(c->bstate.p, 0, (size_t)nbatch * nbricks, st));
        // edge masks: the CTA-per-brick marching-cubes passes read the mask of every point of a listed brick (zero = no vertex); the
        // warp-per-brick passes only read masks their count pass wrote, so they need no zero-fill (4 GB at 50 M particles)
        if (global_mode || c->mc_variant != 1) CK(cudaMemsetAsync(c->vmask.p, 0, (size_t)nbatch * np3, st));
        CK(cudaEventRecord(c->ev[10], st));
        {   // set-up time of this batch: from the end of binning (first batch) / of the previous batch's marching cubes to here
            CK(cudaEventSynchronize(c->ev[10]));
            float su = 0.f;
            CK(cudaEventElapsedTime(&su, s0 == 0 ? c->ev[5] : c->ev[6], c->ev[10]));
            setup_ms += su;
        }
        uint32_t n_mc = 0;
        int raw_q = -1;
        if (c->keep_raw_flat >= 0)
            for (uint32_t q = 0; q < nbatch; ++q) if ((int64_t)h_flat[owned_list[s0 + q]] == c->keep_raw_flat) raw_q = (int)q;
        rc = levelset_batch(c, D, nbatch, nbricks, exact_all, certify_runs, global_mode, averaged, out, ls_launches, fix_points, &n_mc, raw_q);
        if (rc) return rc;
        CK(cudaEventRecord(c->ev[11], st));
        // optional parity tap
        if (c->keep_tile_flat >= 0) {
            for (uint32_t q = 0; q < nbatch; ++q) if ((int64_t)h_flat[owned_list[s0 + q]] == c->keep_tile_flat) {
                out->tile.resize(np3);
                CK(cudaMemcpyAsync(out->tile.data(), c->tiles.as<float>() + (size_t)q * np3, np3 * 4, cudaMemcpyDeviceToHost, st));
                CK(cudaStreamSynchronize(st));
            }
        }
        rc = marching_cubes_batch(c, D, global_mode, n_mc, out, vtotal, ttotal);
        if (rc) return rc;
        CK(cudaEventRecord(c->ev[6], st));
        CK(cudaEventSynchronize(c->ev[6]));
        float a = 0.f, b = 0.f;
        CK(cudaEventElapsedTime(&a, c->ev[10], c->ev[11]));
        CK(cudaEventElapsedTime(&b, c->ev[11], c->ev[6]));
        ls_ms += a; mc_ms += b;
    }
    CK(cudaEventRecord(c->ev[7], st));

    // ---- stitching
    uint64_t nv_final = vtotal;
    uint32_t bc = 0;
    rc = weld_boundary_vertices(c, out, vtotal, ttotal, nv_final, bc);
    if (rc) return rc;
    out->nv = nv_final; out->nt = ttotal;
    c->hint_nv = vtotal; c->hint_nt = ttotal; c->hint_bc = bc;
    if (aniso) {
        // SPH normals and the [bins] post-processing entries use the isotropic kernel at the particle positions: bin them again
        rc = stage_binning(c, D, d_xyz, d_rho, M, nsub, false, nullptr, nullptr, /*record_event=*/false);
        if (rc) return rc;
    }
    {
        // the splat bins stay in the scratch until the next call on this context: ss_post.cuh queries them
        const float r3p = fmulr(fmulr(p->particle_radius, p->particle_radius), p->particle_radius);
        c->post.D = D; c->post.nsub = nsub; c->post.M = M; c->post.partitioned = part.enabled;
        c->post.sphere_mass = fmulr(fmulr(fmulr(4.0f, 1.04719755119659774615f), r3p), p->rest_density);
        c->post.valid = 1;
    }
    if (c->sph_normals && nv_final) {
        // SPH normals at the vertices (pipeline post-processing step, splashsurf/src/reconstruct.rs:1287-1294); sphere rest mass
        // 4/3 pi r^3 rho0 as in reconstruct.rs:1126-1129
        out->normals = std::move(c->o_normals);
        out->normals.ensure(nv_final * 12);
        SsNrmArgs NA{};
        NA.verts = out->verts.as<float>(); NA.vkeys = out->vkeys.as<unsigned long long>(); NA.nv = (uint32_t)nv_final;
        NA.sub_flat = c->sub_flat.as<uint32_t>(); NA.sub_owned = part.enabled ? c->sub_owned.as<uint8_t>() : nullptr; NA.nsub = nsub;
        NA.bins = context_bins(c); NA.rho = d_rho;
        const float r3 = fmulr(fmulr(p->particle_radius, p->particle_radius), p->particle_radius);
        const float frac_pi_3 = 1.04719755119659774615f;
        NA.sphere_mass = fmulr(fmulr(fmulr(4.0f, frac_pi_3), r3), p->rest_density);
        NA.normals = out->normals.as<float>();
        LAUNCH(c, k_sph_normals, nblk(nv_final, 128), 128, D, NA);
        out->has_normals = 1;
    }
    CK(cudaEventRecord(c->ev[8], st));
    CK(cudaEventRecord(c->ev[9], st));
    CK(cudaStreamSynchronize(st));

    // ---- timings
    ss_timings &T = out->tm;
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, c->ev[2], c->ev[3])); T.decomposition = ms;
    CK(cudaEventElapsedTime(&ms, c->ev[3], aniso ? c->ev_an[0] : c->ev[4])); T.density = ms;
    if (aniso) { CK(cudaEventElapsedTime(&ms, c->ev_an[0], c->ev_an[1])); out->an_ms = ms; }
    CK(cudaEventElapsedTime(&ms, c->ev[4], c->ev[5])); T.binning = ms;
    T.levelset = ls_ms; T.marching_cubes = mc_ms; T.tile_setup = setup_ms;
    CK(cudaEventElapsedTime(&ms, c->ev[7], c->ev[8])); T.stitching = ms;
    T.levelset_launches = ls_launches; T.levelset_fixup_points = fix_points;
    unsigned long long h_pairs[2] = { 0, 0 };
    CK(cudaMemcpy(h_pairs, c->pairs.p, 16, cudaMemcpyDeviceToHost));
    T.levelset_pairs = (double)h_pairs[0]; T.levelset_cert_evals = (double)h_pairs[1];
    return SS_OK;
}

// The frame of an entry that creates a surface: body(s) runs on a fresh surface of context c, which goes to *out when body returns
// SS_OK and is freed when it returns an error or throws.  The surface records the kernel launches of the call.
template <typename F>
static int with_new_surface(ss_context *c, ss_surface **out, F &&body) {
    ss_surface *s = nullptr;
    const int rc = ss_guard([&]() -> int {
        CK(cudaSetDevice(c->device));
        s = new ss_surface();
        s->device = c->device;
        c->launches = 0;
        const int rc = body(s);
        s->tm.kernel_launches = c->launches;
        return rc;
    });
    if (rc) ss_surface_free(s);
    else *out = s;
    return rc;
}

// times of the upload, of the AABB and grid, and of the whole device pass of a reconstruction
static void front_timings(const ss_context *c, ss_surface *s) {
    float ms = 0.f;
    CK(cudaEventElapsedTime(&ms, c->ev[0], c->ev[1])); s->tm.upload = ms;
    CK(cudaEventElapsedTime(&ms, c->ev[1], c->ev[2])); s->tm.aabb_and_grid = ms;
    CK(cudaEventElapsedTime(&ms, c->ev[1], c->ev[9])); s->tm.total_device = ms;
}

// ------------------------------------------------------------------ stage-level entry: one level-set tile ----
// density_grid_loop_auto / density_grid_loop_scalar (dense_subdomains.rs:715-847, both `pub`): the level-set tile of
// ONE subdomain from an explicit particle list (in list order == ascending index) and explicit densities.
__global__ void k_iota2(uint32_t n, uint32_t *__restrict__ a, uint32_t *__restrict__ zero) {
    uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= n) return;
    a[e] = e; zero[e] = 0;
}
extern "C" int ss_levelset_tile_f32(ss_context *c, const float *xyz, const float *rho, uint64_t n, const float global_min[3],
                                    float cube_size, const int64_t subdomain_ijk[3], uint32_t S, float h, float rest_mass,
                                    int mode, float *tile_out) {
    if (!c || !tile_out || !global_min || !subdomain_ijk || (n && (!xyz || !rho))) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL argument");
    if (!(cube_size > 0.0f) || !(h > 0.0f) || S < 1 || S > 1024) return ss_fail(SS_ERR_INVALID_PARAMETER, "bad tile parameters");
    if (n >= 0x7fffffffull) return ss_fail(SS_ERR_INDEX_TOO_SMALL, "too many particles");
    for (int d = 0; d < 3; ++d) if (subdomain_ijk[d] < 0 || subdomain_ijk[d] > 1000) return ss_fail(SS_ERR_INVALID_PARAMETER, "subdomain_ijk out of range");
    return ss_guard([&]() -> int {
        CK(cudaSetDevice(c->device));
        cudaStream_t st = c->stream;
        c->post.valid = 0; ++c->frame;                       // this entry rewrites the bins in the scratch
        SsDev D{};
        for (int d = 0; d < 3; ++d) { D.gmin[d] = global_min[d]; D.nsd[d] = (int)subdomain_ijk[d] + 1; }
        fill_tile_geometry(D, cube_size, S, h, rest_mass);
        D.simd = mode == 0 ? 1 : 0;
        const size_t np3 = (size_t)D.np * D.np * D.np;
        c->tiles.ensure(np3 * 4);
        CK(cudaMemsetAsync(c->tiles.p, 0, np3 * 4, st));
        if (n) {
            const uint32_t M = (uint32_t)n;
            const uint32_t flat = (uint32_t)((subdomain_ijk[0] * D.nsd[1] + subdomain_ijk[1]) * D.nsd[2] + subdomain_ijk[2]);
            c->xyz.ensure(n * 12); c->rho.ensure(n * 4);
            CK(cudaMemcpyAsync(c->xyz.p, xyz, n * 12, cudaMemcpyDefault, st));
            CK(cudaMemcpyAsync(c->rho.p, rho, n * 4, cudaMemcpyDefault, st));
            c->key_a.ensure((size_t)M * 4); c->key_b.ensure((size_t)M * 4); c->val_a.ensure((size_t)M * 4); c->val_b.ensure((size_t)M * 4);
            c->cid.ensure((size_t)M * 4); c->sub_flat.ensure(4); c->err.ensure(4);
            LAUNCH(c, k_iota2, nblk(M, 256), 256, M, c->val_b.as<uint32_t>(), c->cid.as<uint32_t>());
            CK(cudaMemcpyAsync(c->sub_flat.p, &flat, 4, cudaMemcpyHostToDevice, st));
            CK(cudaMemsetAsync(c->err.p, 0, 4, st));
            const int rc = stage_binning(c, D, c->xyz.as<float>(), c->rho.as<float>(), M, 1, false, nullptr, nullptr, /*record_event=*/false);
            if (rc) return rc;
            const SsTile T = make_tile(subdomain_ijk, S, global_min, D.sub_size, 0, !D.simd);
            c->tile_tab.ensure(sizeof(SsTile));
            CK(cudaMemcpyAsync(c->tile_tab.p, &T, sizeof(SsTile), cudaMemcpyHostToDevice, st));
            upload_brick_ranges(c, D);
            SsLsArgs A{};
            A.bins = context_bins(c); A.tiles = c->tiles.as<float>();
            A.pairs = nullptr; A.wflag = nullptr; A.fix_bricks = nullptr; A.bstate = nullptr; A.mode = SS_LS_EXACT_ALL;
            const uint32_t n_work = build_worklist(c, D, 1);
            A.work_list = c->list_ls.as<uint32_t>();
            if (n_work) launch_levelset(c, dim3(n_work), D, A, false, false);
            CK(cudaStreamSynchronize(st));
        }
        CK(cudaMemcpyAsync(tile_out, c->tiles.p, np3 * 4, cudaMemcpyDefault, st));
        CK(cudaStreamSynchronize(st));
        return SS_OK;
    });
}

// ------------------------------------------------------------------ multi-GPU: plan statistics + halo packing ----
// Slab plan input: particles per subdomain layer along the partition axis + occupancy of every subdomain slot (work model of
// distributed.py: particles + a fixed cost per occupied tile).  Owner cells are computed in plain f32: the plan only balances.
__global__ void k_part_stats(const float *__restrict__ xyz, uint32_t n, float3 gmin, float inv_sub, int3 nsd, int axis,
                             uint32_t *__restrict__ hist, uint32_t *__restrict__ occ) {
    __shared__ uint32_t s_hist[1024];
    const int nax = axis == 0 ? nsd.x : (axis == 1 ? nsd.y : nsd.z);
    for (int t = threadIdx.x; t < nax && t < 1024; t += blockDim.x) s_hist[t] = 0;
    __syncthreads();
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int ix = min(max((int)floorf((xyz[3 * (uint64_t)i] - gmin.x) * inv_sub), 0), nsd.x - 1);
        const int iy = min(max((int)floorf((xyz[3 * (uint64_t)i + 1] - gmin.y) * inv_sub), 0), nsd.y - 1);
        const int iz = min(max((int)floorf((xyz[3 * (uint64_t)i + 2] - gmin.z) * inv_sub), 0), nsd.z - 1);
        const int ia = axis == 0 ? ix : (axis == 1 ? iy : iz);
        if (ia < 1024) atomicAdd(&s_hist[ia], 1u); else atomicAdd(&hist[ia], 1u);
        occ[(ix * nsd.y + iy) * nsd.z + iz] = 1u;
    }
    __syncthreads();
    for (int t = threadIdx.x; t < nax && t < 1024; t += blockDim.x) if (s_hist[t]) atomicAdd(&hist[t], s_hist[t]);
}
extern "C" int ss_partition_stats_f32(ss_context *c, const float *xyz, uint64_t n, const ss_grid_f32 *grid, uint32_t S, int axis,
                                      uint32_t *hist, uint32_t *occ) {
    if (!c || !grid || !hist || !occ || (n && !xyz) || axis < 0 || axis > 2 || S < 1) return ss_fail(SS_ERR_INVALID_PARAMETER, "bad argument");
    if (n >= 0xfffffff0ull) return ss_fail(SS_ERR_INDEX_TOO_SMALL, "too many particles");
    return ss_guard([&]() -> int {
        CK(cudaSetDevice(c->device));
        int3 nsd;
        nsd.x = (int)((grid->cells_per_dim[0] + S - 1) / S); nsd.y = (int)((grid->cells_per_dim[1] + S - 1) / S); nsd.z = (int)((grid->cells_per_dim[2] + S - 1) / S);
        const int nax = axis == 0 ? nsd.x : (axis == 1 ? nsd.y : nsd.z);
        CK(cudaMemsetAsync(hist, 0, (size_t)nax * 4, c->stream));
        CK(cudaMemsetAsync(occ, 0, (size_t)nsd.x * nsd.y * nsd.z * 4, c->stream));
        if (n) {
            const float sub = fmulr(grid->cell_size, (float)S);
            const unsigned blocks = (unsigned)std::min<uint64_t>(nblk(n, 256), (uint64_t)c->sm_count * 8);
            LAUNCH(c, k_part_stats, blocks, 256, xyz, (uint32_t)n, make_float3(grid->aabb_min[0], grid->aabb_min[1], grid->aabb_min[2]), 1.0f / sub, nsd, axis, hist, occ);
        }
        CK(cudaStreamSynchronize(c->stream));
        return SS_OK;
    });
}

// Plan statistics with the EXACT classifier: `members[slot]` = number of particles of this rank's input that are members (owner or
// ghost, dense_subdomains.rs:1810-1905) of subdomain `slot` -- summed over the ranks this is the subdomain's population, so the
// global maximum (sparse rule, dense_subdomains.rs:1242-1251) is known BEFORE any rank decomposes: the runner needs neither the
// decomposition pre-pass nor the callback.  `hist` as in ss_partition_stats_f32 (owner layer counts, for the balance only).
__global__ void k_part_members(SsDev P, const float *__restrict__ xyz, uint32_t n, int axis, uint32_t *__restrict__ hist, uint32_t *__restrict__ members) {
    __shared__ uint32_t s_hist[1024];
    const int nax = P.nsd[axis];
    for (int t = threadIdx.x; t < nax && t < 1024; t += blockDim.x) s_hist[t] = 0;
    __syncthreads();
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float px = xyz[3 * (uint64_t)i], py = xyz[3 * (uint64_t)i + 1], pz = xyz[3 * (uint64_t)i + 2];
        const float pc = axis == 0 ? px : (axis == 1 ? py : pz);
        const int ia = min(max(ss_cell_of(pc, P.gmin[axis], P.sub_size), 0), nax - 1);
        if (ia < 1024) atomicAdd(&s_hist[ia], 1u); else atomicAdd(&hist[ia], 1u);
        ss_classify(P, px, py, pz, [&](int, int flat) { atomicAdd(&members[flat], 1u); });
    }
    __syncthreads();
    for (int t = threadIdx.x; t < nax && t < 1024; t += blockDim.x) if (s_hist[t]) atomicAdd(&hist[t], s_hist[t]);
}
extern "C" int ss_partition_members_f32(ss_context *c, const float *xyz, uint64_t n, const ss_params_f32 *p, const ss_grid_f32 *grid, int axis,
                                        uint32_t *hist, uint32_t *members) {
    if (!c || !grid || !hist || !members || (n && !xyz) || axis < 0 || axis > 2) return ss_fail(SS_ERR_INVALID_PARAMETER, "bad argument");
    int rc = validate_params(p);
    if (rc) return rc;
    if (n >= 0xfffffff0ull) return ss_fail(SS_ERR_INDEX_TOO_SMALL, "too many particles");
    return ss_guard([&]() -> int {
        CK(cudaSetDevice(c->device));
        const int64_t S = (int64_t)p->subdomain_num_cubes_per_dim;
        const float h = p->compact_support_radius, cs = p->cube_size;
        SsDev D{};
        D.sub_size = fmulr(cs, (float)S);
        const int rc = set_member_margin(D, member_margin(h, cs));
        if (rc) return rc;
        uint64_t nslots = 1;
        for (int d = 0; d < 3; ++d) { D.gmin[d] = grid->aabb_min[d]; D.nsd[d] = (int)((grid->cells_per_dim[d] + S - 1) / S); nslots *= (uint64_t)D.nsd[d]; }
        if (nslots >= 2147483647ull) return ss_fail(SS_ERR_INDEX_TOO_SMALL, "too many subdomain slots");
        D.part_axis = 0; D.keep_lo = 0; D.keep_hi = 0x7fffffff;
        CK(cudaMemsetAsync(hist, 0, (size_t)D.nsd[axis] * 4, c->stream));
        CK(cudaMemsetAsync(members, 0, (size_t)nslots * 4, c->stream));
        if (n) {
            const unsigned blocks = (unsigned)std::min<uint64_t>(nblk(n, 256), (uint64_t)c->sm_count * 8);
            LAUNCH(c, k_part_members, blocks, 256, D, xyz, (uint32_t)n, axis, hist, members);
        }
        CK(cudaStreamSynchronize(c->stream));
        return SS_OK;
    });
}

// Halo packing: destination d takes the particles with lo[d] <= coordinate < hi[d] along the partition axis (one particle may
// go to several destinations), ascending particle index preserved inside every destination.  One warp walks a chunk of
// SS_PACK_CHUNK particles in index order; pass 0 counts per (destination, chunk), an exclusive scan over the destination-major
// count table gives every chunk its output offset, pass 1 scatters.
#define SS_PACK_CHUNK 2048
#define SS_PACK_MAXW 64
struct SsPackIv { double lo[SS_PACK_MAXW], hi[SS_PACK_MAXW]; };
template <bool SCATTER>
__global__ void k_part_pack(const float *__restrict__ xyz, uint32_t n, int axis, SsPackIv iv, int world, uint32_t nchunks,
                            uint32_t *__restrict__ table /* [world][nchunks]: counts in, offsets for SCATTER */, float *__restrict__ send) {
    const uint32_t chunk = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    const int lane = threadIdx.x & 31;
    if (chunk >= nchunks) return;
    const uint32_t first = chunk * SS_PACK_CHUNK, last = min(first + SS_PACK_CHUNK, n);
    for (int d = 0; d < world; ++d) {
        const double lo = iv.lo[d], hi = iv.hi[d];
        uint32_t run = SCATTER ? table[(size_t)d * nchunks + chunk] : 0u;
        for (uint32_t base = first; base < last; base += 32) {
            const uint32_t i = base + lane;
            bool in = false;
            float x = 0.f, y = 0.f, z = 0.f;
            if (i < last) {
                x = xyz[3 * (uint64_t)i]; y = xyz[3 * (uint64_t)i + 1]; z = xyz[3 * (uint64_t)i + 2];
                const double cax = (double)(axis == 0 ? x : (axis == 1 ? y : z));
                in = cax >= lo && cax < hi;
            }
            const uint32_t bal = __ballot_sync(0xffffffffu, in);
            if (SCATTER && in) {
                const uint64_t o = (uint64_t)run + __popc(bal & ((1u << lane) - 1u));
                send[3 * o] = x; send[3 * o + 1] = y; send[3 * o + 2] = z;
            }
            run += __popc(bal);
        }
        if (!SCATTER && lane == 0) table[(size_t)d * nchunks + chunk] = run;
    }
}
// Two-phase: send == NULL counts (counts_out[world], host) and leaves the offset table in the context; the second call with a
// device buffer of sum(counts) * 3 floats scatters.  xyz is DEVICE memory.
extern "C" int ss_partition_pack_f32(ss_context *c, const float *xyz, uint64_t n, int axis, const double *lo, const double *hi, uint32_t world,
                                     uint64_t *counts_out, float *send) {
    if (!c || !lo || !hi || !counts_out || (n && !xyz) || axis < 0 || axis > 2 || world < 1 || world > SS_PACK_MAXW) return ss_fail(SS_ERR_INVALID_PARAMETER, "bad argument");
    if (n >= 0xfffffff0ull) return ss_fail(SS_ERR_INDEX_TOO_SMALL, "too many particles");
    return ss_guard([&]() -> int {
        CK(cudaSetDevice(c->device));
        cudaStream_t st = c->stream;
        const uint32_t nchunks = (uint32_t)((n + SS_PACK_CHUNK - 1) / SS_PACK_CHUNK);
        for (uint32_t d = 0; d < world; ++d) counts_out[d] = 0;
        if (!n) return SS_OK;
        SsPackIv iv{};
        for (uint32_t d = 0; d < world; ++d) { iv.lo[d] = lo[d]; iv.hi[d] = hi[d]; }
        const size_t tab = (size_t)world * nchunks;
        c->pack_cnt.ensure(tab * 4); c->pack_off.ensure(tab * 4 + 4);
        const unsigned blocks = nblk((uint64_t)nchunks * 32, 128);
        if (!send) {
            LAUNCH(c, k_part_pack<false>, blocks, 128, xyz, (uint32_t)n, axis, iv, (int)world, nchunks, c->pack_cnt.as<uint32_t>(), (float *)nullptr);
            uint32_t h_last[2] = { 0, 0 };
            scan_with_total(c, c->pack_cnt.as<uint32_t>(), c->pack_off.as<uint32_t>(), (uint32_t)tab, h_last);
            std::vector<uint32_t> h_off(world);
            for (uint32_t d = 0; d < world; ++d) CK(cudaMemcpyAsync(&h_off[d], c->pack_off.as<uint32_t>() + (size_t)d * nchunks, 4, cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
            const uint64_t total = (uint64_t)h_last[0] + h_last[1];
            for (uint32_t d = 0; d < world; ++d) counts_out[d] = (d + 1 < world ? h_off[d + 1] : total) - h_off[d];
            c->pack_n = n; c->pack_world = world;
        } else {
            if (c->pack_n != n || c->pack_world != world) return ss_fail(SS_ERR_INVALID_PARAMETER, "ss_partition_pack_f32: scatter phase without a matching count phase");
            LAUNCH(c, k_part_pack<true>, blocks, 128, xyz, (uint32_t)n, axis, iv, (int)world, nchunks, c->pack_off.as<uint32_t>(), send);
            CK(cudaStreamSynchronize(st));
            c->pack_n = 0;
        }
        return SS_OK;
    });
}

// ------------------------------------------------------------------ multi-GPU: one rank's slab of subdomains ----
static int reconstruct_partition_impl(ss_context *c, const float *xyz, uint64_t n_in, const ss_params_f32 *p, const ss_grid_f32 *grid,
                                      int axis, int64_t own_lo, int64_t own_hi, int64_t halo, uint64_t global_max_particles,
                                      int stop_after_decomposition, uint64_t (*max_reduce)(uint64_t, void *), void *user, ss_surface **out);
extern "C" int ss_reconstruct_partition_f32(ss_context *c, const float *xyz, uint64_t n_in, const ss_params_f32 *p, const ss_grid_f32 *grid,
                                            int axis, int64_t own_lo, int64_t own_hi, int64_t halo, uint64_t global_max_particles,
                                            int stop_after_decomposition, ss_surface **out) {
    return reconstruct_partition_impl(c, xyz, n_in, p, grid, axis, own_lo, own_hi, halo, global_max_particles, stop_after_decomposition, nullptr, nullptr, out);
}
extern "C" int ss_reconstruct_partition_cb_f32(ss_context *c, const float *xyz, uint64_t n_in, const ss_params_f32 *p, const ss_grid_f32 *grid,
                                               int axis, int64_t own_lo, int64_t own_hi, int64_t halo,
                                               uint64_t (*max_reduce)(uint64_t local_max, void *user), void *user, ss_surface **out) {
    return reconstruct_partition_impl(c, xyz, n_in, p, grid, axis, own_lo, own_hi, halo, 0, 0, max_reduce, user, out);
}
struct ReduceOnce {
    uint64_t (*fn)(uint64_t, void *); void *user; bool done = false;
    static uint64_t call(uint64_t v, void *self) { ReduceOnce *r = (ReduceOnce *)self; r->done = true; return r->fn(v, r->user); }
    ~ReduceOnce() { if (fn && !done) { done = true; fn(0, user); } }
};
static int reconstruct_partition_impl(ss_context *c, const float *xyz, uint64_t n_in, const ss_params_f32 *p, const ss_grid_f32 *grid,
                                      int axis, int64_t own_lo, int64_t own_hi, int64_t halo, uint64_t global_max_particles,
                                      int stop_after_decomposition, uint64_t (*max_reduce)(uint64_t, void *), void *user, ss_surface **out) {
    // The max-reduce callback is a collective: it runs exactly once on EVERY exit path below (argument errors, error returns and
    // CUDA failures included), so that a rank that fails cannot leave the others blocked in their all-reduce.
    ReduceOnce once{ max_reduce, user };
    if (!c || !out || !grid) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL argument");
    *out = nullptr;
    int rc = validate_params(p);
    if (rc) return rc;
    if (p->has_particle_aabb) return ss_fail(SS_ERR_UNSUPPORTED, "filter particles before partitioning (particle_aabb is applied by the caller)");
    if (c->an_on) return ss_fail(SS_ERR_UNSUPPORTED, "anisotropic kernels are not available on partitioned (multi-GPU) reconstructions");
    if (c->avg_on) return ss_fail(SS_ERR_UNSUPPORTED, "the averaged-position surface is not available on partitioned (multi-GPU) reconstructions");
    if (c->ac_on) return ss_fail(SS_ERR_INVALID_PARAMETER, "the Jacobian correction applies to the averaged-position surface, which is off");
    if (c->rad_on) return ss_fail(SS_ERR_INVALID_PARAMETER, "per-particle radii apply to the averaged-position surface, which is off");
    if (p->spatial_decomposition != 1) return ss_fail(SS_ERR_INVALID_PARAMETER, "partitioned reconstruction requires the subdomain grid");
    if (axis < 0 || axis > 2 || own_lo < 0 || own_hi < own_lo || halo < 0) return ss_fail(SS_ERR_INVALID_PARAMETER, "bad partition");
    if (n_in && !xyz) return ss_fail(SS_ERR_INVALID_PARAMETER, "xyz is NULL");
    return with_new_surface(c, out, [&](ss_surface *s) -> int {
        s->n_in = n_in;
        Prepared P;
        g_devbuf_slack_eighths = 4;
        int rc = prepare_particles(c, xyz, n_in, p, P, nullptr, grid);
        if (rc) return rc;
        s->n = P.n; s->grid = P.grid; s->used_decomposition = 1;
        Partition part;
        part.enabled = 1; part.axis = axis; part.own_lo = own_lo; part.own_hi = own_hi; part.halo = halo;
        part.global_max_particles = global_max_particles; part.stop_after_decomposition = stop_after_decomposition;
        part.max_reduce = max_reduce ? &ReduceOnce::call : nullptr; part.max_reduce_user = &once;
        rc = run_subdomain_grid(c, P, p, s, part);
        if (rc) return rc;
        front_timings(c, s);
        return SS_OK;
    });
}
extern "C" uint64_t ss_surface_max_subdomain_particles(const ss_surface *s) { return s ? s->max_particles : 0; }

// Welds vertices that carry the same MC edge key (duplicates on faces between ranks' slabs) in a concatenation of
// per-rank meshes.  All pointers are DEVICE memory: verts nv x 3 f32, keys nv u64 (as produced per vertex by
// ss_surface_device_vertex_keys), tris nt x 3 u32 (already offset to the concatenated numbering).  `cand` lists the
// n_cand vertex ids that may have duplicates.  Compacts verts/keys in place, rewrites tris, returns the new count.
extern "C" int ss_weld_meshes(ss_context *c, float *verts, unsigned long long *keys, uint64_t nv, uint32_t *tris, uint64_t nt,
                              const uint32_t *cand, uint64_t n_cand, uint64_t *nv_out) {
    if (!c || !nv_out) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL argument");
    *nv_out = nv;
    if (!nv || !n_cand) return SS_OK;
    if (nv >= 0xfffffff0ull || n_cand >= 0x7fffffffull) return ss_fail(SS_ERR_INDEX_TOO_SMALL, "mesh too large");
    return ss_guard([&]() -> int {
        CK(cudaSetDevice(c->device));
        cudaStream_t st = c->stream;
        const uint32_t bc = (uint32_t)n_cand;
        c->bkeys_a.ensure((size_t)bc * 8);
        LAUNCH(c, k_gather_keys, nblk(bc, 256), 256, keys, cand, bc, c->bkeys_a.as<unsigned long long>());
        DevBuf nverts, nkeys;                                // compacted copies, written back over verts / keys
        const uint64_t nv_final = weld_vertices(c, cand, bc, verts, keys, nv, tris, nt, nverts, nkeys);
        CK(cudaMemcpyAsync(verts, nverts.p, nv_final * 12, cudaMemcpyDeviceToDevice, st));
        CK(cudaMemcpyAsync(keys, nkeys.p, nv_final * 8, cudaMemcpyDeviceToDevice, st));
        CK(cudaStreamSynchronize(st));
        *nv_out = nv_final;
        return SS_OK;
    });
}
extern "C" const unsigned long long *ss_surface_device_vertex_keys(const ss_surface *s) { return s ? s->vkeys.as<unsigned long long>() : nullptr; }
extern "C" int ss_surface_copy_subdomain_owned(const ss_surface *s, uint8_t *dst) {
    if (!s || !dst) return SS_ERR_INVALID_PARAMETER;
    for (uint64_t q = 0; q < s->nsub; ++q) dst[q] = s->sub_owned.empty() ? 1 : s->sub_owned[q];
    return SS_OK;
}

// ------------------------------------------------------------------ public entry ----
// The context's per-particle radii against the call's particle count (before the level set is built)
static int check_radii_setting(const ss_context *c, uint64_t n_in) {
    if (c->rad_on && !c->avg_on) return ss_fail(SS_ERR_INVALID_PARAMETER, "per-particle radii apply to the averaged-position surface, which is off");
    if (c->rad_on && c->rad_n != n_in) {
        char msg[160];
        snprintf(msg, sizeof msg, "averaged surface radii: %llu radii for %llu particles", (unsigned long long)c->rad_n, (unsigned long long)n_in);
        return ss_fail(SS_ERR_INVALID_PARAMETER, msg);
    }
    return SS_OK;
}
// The context's opt-in level sets combine: anisotropy excludes the averaged surface, the correction requires it
static int check_level_set_modes(const ss_context *c) {
    if (c->an_on && c->avg_on) return ss_fail(SS_ERR_INVALID_PARAMETER, "anisotropic kernels and the averaged-position surface are exclusive");
    if (c->ac_on && !c->avg_on) return ss_fail(SS_ERR_INVALID_PARAMETER, "the Jacobian correction applies to the averaged-position surface, which is off");
    return SS_OK;
}

extern "C" int ss_reconstruct_surface_f32(ss_context *c, const float *xyz, uint64_t n_in, const ss_params_f32 *p, ss_surface **out) {
    if (!c || !out) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL argument");
    *out = nullptr;
    int rc = validate_params(p);
    if (rc) return rc;
    if (n_in && !xyz) return ss_fail(SS_ERR_INVALID_PARAMETER, "xyz is NULL");
    rc = check_radii_setting(c, n_in);
    if (rc) return rc;
    return with_new_surface(c, out, [&](ss_surface *s) -> int {
        s->n_in = n_in;
        Prepared P;
        int rc = prepare_particles(c, xyz, n_in, p, P, &s->inside_aabb);
        if (rc) return rc;
        s->n = P.n; s->grid = P.grid;
        // decomposition decision, lib.rs:421-464
        int use_dec = 0;
        rc = check_level_set_modes(c);
        if (rc) return rc;
        if (c->avg_on) {
            // averaged-position surface: subdomain path only, always decomposed (no auto-disable)
            if (p->spatial_decomposition != 1) return ss_fail(SS_ERR_UNSUPPORTED, "the averaged-position surface requires the subdomain grid (spatial_decomposition = UniformGrid)");
            use_dec = 1;
        } else if (c->an_on) {
            // anisotropic kernels: subdomain path only, always decomposed (no auto-disable)
            if (p->spatial_decomposition != 1) return ss_fail(SS_ERR_UNSUPPORTED, "anisotropic kernels require the subdomain grid (spatial_decomposition = UniformGrid)");
            use_dec = 1;
        } else if (p->spatial_decomposition == 1) {
            if (p->auto_disable) {
                int64_t mc = std::max(P.grid.nc[0], std::max(P.grid.nc[1], P.grid.nc[2]));
                uint32_t with_margin = (uint32_t)(1.2 * (double)p->subdomain_num_cubes_per_dim);
                use_dec = (uint64_t)mc > (uint64_t)with_margin;
            } else use_dec = 1;
        }
        s->used_decomposition = use_dec;
        rc = run_subdomain_grid(c, P, p, s, Partition(), /*global_mode=*/!use_dec);
        if (rc) return rc;
        front_timings(c, s);
        return SS_OK;
    });
}

// a result buffer of a freed surface goes back to the context's pool when the pool's is smaller (or missing)
static void give_back(DevBuf &slot, DevBuf &buf) {
    if (buf.p && (!slot.p || slot.cap < buf.cap)) slot = std::move(buf);
}
extern "C" void ss_surface_free(ss_surface *s) {
    if (!s) return;
    cudaSetDevice(s->device);
    {
        std::lock_guard<std::mutex> lk(g_ctx_mutex);
        if (s->owner && g_live_contexts.count(s->owner)) {
            ss_context *c = s->owner;
            give_back(c->o_verts, s->verts); give_back(c->o_tris, s->tris); give_back(c->o_vkeys, s->vkeys); give_back(c->o_rho, s->rho);
            give_back(c->o_normals, s->normals);
        }
    }
    delete s;                                          // frees the buffers the pool did not take
}

// ------------------------------------------------------------------ accessors ----
extern "C" uint64_t ss_surface_num_vertices(const ss_surface *s) { return s ? s->nv : 0; }
extern "C" uint64_t ss_surface_num_triangles(const ss_surface *s) { return s ? s->nt : 0; }
extern "C" uint64_t ss_surface_num_particles(const ss_surface *s) { return s ? s->n : 0; }
extern "C" uint64_t ss_surface_num_subdomains(const ss_surface *s) { return s ? s->nsub : 0; }
extern "C" int ss_surface_used_decomposition(const ss_surface *s) { return s ? s->used_decomposition : 0; }
extern "C" int ss_surface_grid(const ss_surface *s, ss_grid_f32 *o) { if (!s || !o) return SS_ERR_INVALID_PARAMETER; grid_to_abi(s->grid, o); return SS_OK; }
extern "C" int ss_surface_subdomain_grid(const ss_surface *s, ss_grid_f32 *o) {
    if (!s || !o) return SS_ERR_INVALID_PARAMETER;
    if (!s->used_decomposition) return ss_fail(SS_ERR_INVALID_PARAMETER, "no subdomain grid: decomposition was not used");
    grid_to_abi(s->subgrid, o); return SS_OK;
}
static int copy_out(const ss_surface *s, void *dst, const void *src, size_t bytes, bool widen = false) {
    if (!s || (!dst && bytes)) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL argument");
    if (!bytes) return SS_OK;
    cudaSetDevice(s->device);
    ss_context *c = nullptr;
    {
        std::lock_guard<std::mutex> lk(g_ctx_mutex);
        if (s->owner && g_live_contexts.count(s->owner)) c = s->owner;
    }
    bool pinned_dst = false;
    {
        cudaPointerAttributes at;
        if (cudaPointerGetAttributes(&at, dst) == cudaSuccess) pinned_dst = at.type == cudaMemoryTypeHost || at.type == cudaMemoryTypeManaged;
        else cudaGetLastError();
    }
    const size_t SS_STAGE_BYTES = c ? c->stage_bytes : SS_STAGE_BYTES_MAX;                // chunk size (tests shrink it)
    if (!c || (pinned_dst && !widen) || bytes < 4 * SS_STAGE_BYTES) {
        if (!widen) {
            cudaError_t e = cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost);
            if (e != cudaSuccess) return ss_fail(SS_ERR_CUDA, cudaGetErrorString(e));
            return SS_OK;
        }
        std::vector<uint32_t> tmp(bytes / 4);
        cudaError_t e = cudaMemcpy(tmp.data(), src, bytes, cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) return ss_fail(SS_ERR_CUDA, cudaGetErrorString(e));
        scatter_chunk(static_cast<char *>(dst), reinterpret_cast<const char *>(tmp.data()), bytes, true);
        return SS_OK;
    }
    return ss_guard([&]() -> int {
        for (int q = 0; q < 2; ++q) if (!c->h_stage[q]) {
            if (cudaHostAlloc(&c->h_stage[q], SS_STAGE_BYTES_MAX, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); c->h_stage[q] = nullptr; }
        }
        if (!c->h_stage[0] || !c->h_stage[1]) {                      // cannot page-lock: the plain copy still works
            if (widen) { std::vector<uint32_t> tmp(bytes / 4); CK(cudaMemcpy(tmp.data(), src, bytes, cudaMemcpyDeviceToHost)); scatter_chunk(static_cast<char *>(dst), reinterpret_cast<const char *>(tmp.data()), bytes, true); }
            else CK(cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost));
            return SS_OK;
        }
        cudaStream_t st = c->stream;
        const size_t nchunks = (bytes + SS_STAGE_BYTES - 1) / SS_STAGE_BYTES;
        auto issue = [&](size_t k) {
            const size_t off = k * SS_STAGE_BYTES, n = std::min(SS_STAGE_BYTES, bytes - off);
            CK(cudaMemcpyAsync(c->h_stage[k & 1], static_cast<const char *>(src) + off, n, cudaMemcpyDeviceToHost, st));
            CK(cudaEventRecord(c->ev_stage[k & 1], st));
        };
        issue(0);
        for (size_t k = 0; k < nchunks; ++k) {
            if (k + 1 < nchunks) issue(k + 1);                       // its staging buffer was scattered in the previous iteration
            CK(cudaEventSynchronize(c->ev_stage[k & 1]));
            const size_t off = k * SS_STAGE_BYTES, n = std::min(SS_STAGE_BYTES, bytes - off);
            scatter_chunk(static_cast<char *>(dst) + (widen ? 2 * off : off), static_cast<const char *>(c->h_stage[k & 1]), n, widen);
        }
        return SS_OK;
    });
}
extern "C" int ss_surface_copy_vertices(const ss_surface *s, float *dst) { return copy_out(s, dst, s ? s->verts.p : nullptr, s ? s->nv * 12 : 0); }
extern "C" int ss_surface_copy_triangles_u32(const ss_surface *s, uint32_t *dst) { return copy_out(s, dst, s ? s->tris.p : nullptr, s ? s->nt * 12 : 0); }
extern "C" int ss_surface_copy_triangles_u64(const ss_surface *s, uint64_t *dst) {      /* usize like the reference: widened on the host */
    if (!s || (!dst && s->nt)) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL argument");
    return copy_out(s, dst, s->tris.p, s->nt * 12, true);
}
extern "C" int ss_surface_copy_particle_densities(const ss_surface *s, float *dst) { return copy_out(s, dst, s ? s->rho.p : nullptr, s ? s->n * 4 : 0); }
extern "C" int ss_surface_copy_particle_inside_aabb(const ss_surface *s, uint8_t *dst) {
    if (!s || !dst) return SS_ERR_INVALID_PARAMETER;
    if (s->inside_aabb.empty()) return ss_fail(SS_ERR_INVALID_PARAMETER, "no particle AABB was specified");
    memcpy(dst, s->inside_aabb.data(), s->inside_aabb.size());
    return SS_OK;
}
// Page-locked host memory for callers without a CUDA binding of their own (the Python mirror's reusable result buffers): device ->
// host copies into it run at PCIe speed and touch no fresh pages.
extern "C" void *ss_host_alloc_pinned(uint64_t bytes) {
    void *p = nullptr;
    if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); return nullptr; }
    return p;
}
extern "C" void ss_host_free_pinned(void *p) { if (p) cudaFreeHost(p); }
extern "C" const float *ss_surface_device_vertices(const ss_surface *s) { return s ? s->verts.as<float>() : nullptr; }
extern "C" const uint32_t *ss_surface_device_triangles(const ss_surface *s) { return s ? s->tris.as<uint32_t>() : nullptr; }
extern "C" const float *ss_surface_device_densities(const ss_surface *s) { return s ? s->rho.as<float>() : nullptr; }

extern "C" int ss_surface_copy_vertex_edge_keys(const ss_surface *s, int64_t *dst) {
    if (!s || (!dst && s->nv)) return SS_ERR_INVALID_PARAMETER;
    std::vector<unsigned long long> k(s->nv);
    int rc = copy_out(s, k.data(), s->vkeys.p, s->nv * 8);
    if (rc) return rc;
    for (uint64_t v = 0; v < s->nv; ++v) {
        dst[4 * v] = (int64_t)((k[v] >> 42) & 0xfffff); dst[4 * v + 1] = (int64_t)((k[v] >> 22) & 0xfffff);
        dst[4 * v + 2] = (int64_t)((k[v] >> 2) & 0xfffff); dst[4 * v + 3] = (int64_t)(k[v] & 3);
    }
    return SS_OK;
}
extern "C" int ss_surface_copy_subdomains(const ss_surface *s, int64_t *flat, uint64_t *count, uint8_t *sparse) {
    if (!s) return SS_ERR_INVALID_PARAMETER;
    for (uint64_t q = 0; q < s->nsub; ++q) {
        if (flat) flat[q] = s->sub_flat[q];
        if (count) count[q] = s->sub_count[q];
        if (sparse) sparse[q] = s->sub_sparse[q];
    }
    return SS_OK;
}
extern "C" int ss_surface_copy_levelset_tile(const ss_surface *s, float *dst) {
    if (!s || !dst) return SS_ERR_INVALID_PARAMETER;
    if (s->tile.empty()) return ss_fail(SS_ERR_INVALID_PARAMETER, "no level-set tile was kept (ss_context_keep_levelset_tile)");
    memcpy(dst, s->tile.data(), s->tile.size() * 4);
    return SS_OK;
}
extern "C" int ss_surface_copy_levelset_tile_raw(const ss_surface *s, float *tile, uint8_t *brick_state) {
    if (!s) return SS_ERR_INVALID_PARAMETER;
    if (s->tile_raw.empty()) return ss_fail(SS_ERR_INVALID_PARAMETER, "no raw level-set tile was kept (ss_context_keep_levelset_tile_raw)");
    if (tile) memcpy(tile, s->tile_raw.data(), s->tile_raw.size() * 4);
    if (brick_state) memcpy(brick_state, s->tile_raw_bstate.data(), s->tile_raw_bstate.size());
    return SS_OK;
}
extern "C" uint64_t ss_surface_num_neighbors(const ss_surface *s) { return (s && s->has_neighbors) ? s->n_neighbors : 0; }
extern "C" int ss_surface_copy_neighbor_lists(const ss_surface *s, uint64_t *offsets, uint32_t *indices) {
    if (!s) return SS_ERR_INVALID_PARAMETER;
    if (!s->has_neighbors) return ss_fail(SS_ERR_INVALID_PARAMETER, "neighbor lists were not requested (Parameters::global_neighborhood_list)");
    int rc = SS_OK;
    if (offsets) rc = copy_out(s, offsets, s->nbr_off.p, (s->n + 1) * 8);
    if (!rc && indices) rc = copy_out(s, indices, s->nbr_idx.p, s->n_neighbors * 4);
    return rc;
}
extern "C" int ss_surface_timings(const ss_surface *s, ss_timings *o) { if (!s || !o) return SS_ERR_INVALID_PARAMETER; *o = s->tm; return SS_OK; }
extern "C" int ss_surface_levelset_paths(const ss_surface *s, uint64_t *out, int n) {
    if (!s) return -SS_ERR_INVALID_PARAMETER;
    for (int i = 0; i < std::min(n, (int)SS_LSP_N); ++i) out[i] = s->ls_paths[i];
    return SS_LSP_N;
}
extern "C" float ss_surface_anisotropy_ms(const ss_surface *s) { return (s && s->has_aniso) ? s->an_ms : 0.0f; }
extern "C" int ss_surface_copy_anisotropy(const ss_surface *s, float *xbar, float *g) {
    if (!s) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL surface");
    if (!s->has_aniso) return ss_fail(SS_ERR_INVALID_PARAMETER, "the surface was not reconstructed with anisotropic kernels");
    int rc = xbar ? copy_out(s, xbar, s->an_xbar.p, s->n * 12) : SS_OK;
    if (rc == SS_OK && g) rc = copy_out(s, g, s->an_g.p, s->n * 24);
    return rc;
}

// ------------------------------------------------------------------ level-set field at arbitrary points ----
// DESIGN.md §13.  The handle is a surface without a mesh: the context's level set (standard, anisotropic or averaged, with the
// context's settings) up to its records in the splat bins, which live in the context's scratch until the next reconstruction,
// interpolator or field on that context.  Always decomposed: the grid, the densities, the filter and the refusals are those of
// ss_reconstruct_surface_f32 with the subdomain grid.
extern "C" int ss_levelset_field_create_f32(ss_context *c, const float *xyz, uint64_t n_in, const ss_params_f32 *p, ss_surface **out) {
    if (!c || !out) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL argument");
    *out = nullptr;
    int rc = validate_params(p);
    if (rc) return rc;
    if (p->subdomain_num_cubes_per_dim < 1) return ss_fail(SS_ERR_INVALID_PARAMETER, "subdomain_num_cubes_per_dim has to be >= 1");
    if (n_in && !xyz) return ss_fail(SS_ERR_INVALID_PARAMETER, "xyz is NULL");
    rc = check_radii_setting(c, n_in);
    if (rc) return rc;
    return with_new_surface(c, out, [&](ss_surface *s) -> int {
        s->n_in = n_in;
        Prepared P;
        int rc = prepare_particles(c, xyz, n_in, p, P, &s->inside_aabb);
        if (rc) return rc;
        s->n = P.n; s->grid = P.grid; s->used_decomposition = 1;
        rc = check_level_set_modes(c);
        if (rc) return rc;
        Partition opt;
        opt.field = 1;
        rc = run_subdomain_grid(c, P, p, s, opt, /*global_mode=*/false);
        if (rc) return rc;
        front_timings(c, s);
        return SS_OK;
    });
}

// context of a field whose records are still in place (nullptr + error otherwise)
static ss_context *field_context(const ss_surface *f, int *rc) {
    *rc = SS_OK;
    if (!f || !f->fld) { *rc = ss_fail(SS_ERR_INVALID_PARAMETER, "not a level-set field (ss_levelset_field_create_f32)"); return nullptr; }
    ss_context *c = f->owner;
    {
        std::lock_guard<std::mutex> lk(g_ctx_mutex);
        if (!c || !g_live_contexts.count(c)) { *rc = ss_fail(SS_ERR_INVALID_PARAMETER, "the context of this level-set field was destroyed"); return nullptr; }
    }
    if (c->frame != f->frame) {
        *rc = ss_fail(SS_ERR_INVALID_PARAMETER, "the records of this level-set field are gone: use it before the next reconstruction / interpolator / field on its context");
        return nullptr;
    }
    return c;
}

// The point groups of one query through the tiers of the fold F: 512-slot slice, 4096-slot slice, selection.
template <class F>
static void field_fold(ss_context *c, const SsDev &D, const SsFieldArgs &Q0, uint32_t n_groups, uint64_t *received) {
    uint64_t launches = 0;
    const auto args = [&](const uint32_t *list, uint32_t n, uint32_t *left) {
        SsFieldArgs Q = Q0;
        Q.groups = list; Q.n_groups = n; Q.fallback = left;
        return Q;
    };
    run_cascade(c, nullptr, n_groups, {
        [&](const uint32_t *list, uint32_t n, uint32_t *left) {
            LAUNCH(c, (k_field_fold<F, SS_AN_CAP, SS_FLD_WARPS>), (n + SS_FLD_WARPS - 1) / SS_FLD_WARPS, SS_FLD_WARPS * 32, D, args(list, n, left));
        },
        [&](const uint32_t *list, uint32_t n, uint32_t *left) { LAUNCH(c, (k_field_fold<F, SS_AN_BIG_CAP, 1>), n, 32, D, args(list, n, left)); },
        [&](const uint32_t *list, uint32_t n, uint32_t *left) { LAUNCH(c, k_field_select<F>, n, 32, D, args(list, n, left)); },
    }, launches, received);
}

// The field at m device-resident points `pts` into `out` (and, with `grad`, the gradient fold into grad, pre-zeroed; with `grad` and
// `hess`, the Hessian fold into both, pre-zeroed): keys, sort, group starts, then the cascade of the mode's value, gradient or
// Hessian fold.  Uses the context's query scratch (fld_key_*, fld_idx_*, fld_flag, fld_off, fld_starts, fld_chk), never the field's
// records.  Returns the refusal of a non-finite point.
static int field_run(ss_surface *f, ss_context *c, const float *pts, uint32_t m32, float *out, float *grad, float *hess = nullptr) {
    cudaStream_t st = c->stream;
    const SsDev &D = f->fld_D;
    c->fld_chk.ensure(8);
    c->fld_key_a.ensure((size_t)m32 * 4); c->fld_key_b.ensure((size_t)m32 * 4); c->fld_idx_a.ensure((size_t)m32 * 4); c->fld_idx_b.ensure((size_t)m32 * 4);
    uint32_t chk[2] = { 0xffffffffu, 0u };
    CK(cudaMemcpyAsync(c->fld_chk.p, chk, 8, cudaMemcpyHostToDevice, st));
    const uint32_t nsub = f->fld_ready ? f->fld_nsub : 0u;            // no records: every point is 0
    LAUNCH(c, k_field_keys, nblk(m32, 256), 256, D, pts, m32, make_float3(f->grid.mx[0], f->grid.mx[1], f->grid.mx[2]),
           c->sub_flat.as<uint32_t>(), nsub, c->fld_key_a.as<uint32_t>(), c->fld_idx_a.as<uint32_t>(), out, c->fld_chk.as<uint32_t>());
    CK(cudaMemcpyAsync(chk, c->fld_chk.p, 8, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    if (chk[0] != 0xffffffffu) {
        char msg[160];
        snprintf(msg, sizeof msg, "level-set field: point %u has a non-finite coordinate", chk[0]);
        return ss_fail(SS_ERR_INVALID_PARAMETER, msg);
    }
    const uint32_t nin = chk[1];
    if (!nin) return SS_OK;
    cub_sort(c, c->fld_key_a.as<uint32_t>(), c->fld_key_b.as<uint32_t>(), m32, 32, c->fld_idx_a.as<uint32_t>(), c->fld_idx_b.as<uint32_t>());
    c->fld_flag.ensure((size_t)nin * 4); c->fld_off.ensure((size_t)nin * 4 + 4); c->fld_starts.ensure((size_t)nin * 4 + 4);
    LAUNCH(c, k_field_starts, nblk(nin, 256), 256, c->fld_key_b.as<uint32_t>(), nin, c->fld_flag.as<uint32_t>());
    uint32_t lc[2] = { 0, 0 };
    scan_compact(c, c->fld_flag.as<uint32_t>(), c->fld_off.as<uint32_t>(), nin, c->fld_starts.as<uint32_t>(), lc);
    CK(cudaStreamSynchronize(st));
    const uint32_t n_groups = lc[0] + lc[1];
    CK(cudaMemcpyAsync(c->fld_starts.as<uint32_t>() + n_groups, &nin, 4, cudaMemcpyHostToDevice, st));
    SsFieldArgs Q{};
    Q.A.bins = context_bins(c); Q.A.bins.brick_rng = c->fld_rng.as<int2>();
    Q.A.grec = c->an_grec.as<float4>(); Q.A.rrec = c->av_rrec.as<float>();
    Q.pts = pts; Q.key = c->fld_key_b.as<uint32_t>(); Q.idx = c->fld_idx_b.as<uint32_t>();
    Q.starts = c->fld_starts.as<uint32_t>(); Q.out = out;
    if (hess) {
        Q.grad = grad; Q.hess = hess;
        switch (f->fld_mode) {
        case SS_FLD_ANISO: field_fold<SsAnisoHessFold>(c, D, Q, n_groups, f->fld_paths); break;
        case SS_FLD_AVG: field_fold<SsAvgHessFold>(c, D, Q, n_groups, f->fld_paths); break;
        case SS_FLD_AVG_RAD: field_fold<SsAvgRadHessFold>(c, D, Q, n_groups, f->fld_paths); break;
        default: field_fold<SsSphHessFold>(c, D, Q, n_groups, f->fld_paths); break;
        }
    } else if (grad) {
        Q.grad = grad;
        switch (f->fld_mode) {
        case SS_FLD_ANISO: field_fold<SsAnisoGradFold>(c, D, Q, n_groups, f->fld_paths); break;
        case SS_FLD_AVG: field_fold<SsAvgGradFold>(c, D, Q, n_groups, f->fld_paths); break;
        case SS_FLD_AVG_RAD: field_fold<SsAvgRadGradFold>(c, D, Q, n_groups, f->fld_paths); break;
        default: field_fold<SsSphGradFold>(c, D, Q, n_groups, f->fld_paths); break;
        }
    } else {
        switch (f->fld_mode) {
        case SS_FLD_ANISO: field_fold<SsAnisoFold>(c, D, Q, n_groups, f->fld_paths); break;
        case SS_FLD_AVG: field_fold<SsAvgFold>(c, D, Q, n_groups, f->fld_paths); break;
        case SS_FLD_AVG_CORR: field_fold<SsAvgCorrFold>(c, D, Q, n_groups, f->fld_paths); break;
        case SS_FLD_AVG_RAD: field_fold<SsAvgRadFold>(c, D, Q, n_groups, f->fld_paths); break;
        case SS_FLD_AVG_CORR_RAD: field_fold<SsAvgCorrRadFold>(c, D, Q, n_groups, f->fld_paths); break;
        default: field_fold<SsSphFold>(c, D, Q, n_groups, f->fld_paths); break;
        }
    }
    return SS_OK;
}

// What one field query returns beside the values
enum FieldQuery { FQ_VALUE, FQ_GRADIENT, FQ_HESSIAN, FQ_CURVATURE };

// One query of ss_levelset_field_at_f32, ss_levelset_field_gradient_at_f32 (grads: [m][3]), ss_levelset_field_hessian_at_f32 (grads,
// hess: [m][6]) or ss_levelset_field_curvature_at_f32 (curv: [m][2]; gradients and Hessians in the context's buffers): the caller's
// points copied to the device, field_run, the curvature epilogue, the results copied back.
static int field_query(ss_surface *f, const float *points, uint64_t m, float *out, FieldQuery kind, float *grads, float *hess, float *curv) {
    int rc; ss_context *c = field_context(f, &rc);
    if (!c) return rc;
    if (m && (!points || !out || ((kind == FQ_GRADIENT || kind == FQ_HESSIAN) && !grads) || (kind == FQ_HESSIAN && !hess) ||
              (kind == FQ_CURVATURE && !curv)))
        return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL argument");
    if (m >= 0x7fffffffull) return ss_fail(SS_ERR_INDEX_TOO_SMALL, "too many points for one call");
    if (kind == FQ_GRADIENT && (f->fld_mode == SS_FLD_AVG_CORR || f->fld_mode == SS_FLD_AVG_CORR_RAD))
        return ss_fail(SS_ERR_UNSUPPORTED, "level-set field: the Jacobian-corrected averaged surface has no gradient (DESIGN.md 13.1)");
    if (kind >= FQ_HESSIAN && (f->fld_mode == SS_FLD_AVG_CORR || f->fld_mode == SS_FLD_AVG_CORR_RAD))
        return ss_fail(SS_ERR_UNSUPPORTED, "level-set field: the Jacobian-corrected averaged surface has no Hessian or curvature (DESIGN.md 13.2)");
    for (uint64_t &q : f->fld_paths) q = 0;
    if (!m) return SS_OK;
    return ss_guard([&]() -> int {
        CK(cudaSetDevice(c->device));
        cudaStream_t st = c->stream;
        const uint32_t m32 = (uint32_t)m;
        c->fld_pts.ensure((size_t)m32 * 12); c->fld_out.ensure((size_t)m32 * 4);
        if (kind != FQ_VALUE) {
            c->fld_grad.ensure((size_t)m32 * 12);
            CK(cudaMemsetAsync(c->fld_grad.p, 0, (size_t)m32 * 12, st));       // points without candidates: gradient 0
        }
        if (kind >= FQ_HESSIAN) {
            c->fld_hess.ensure((size_t)m32 * 24);
            CK(cudaMemsetAsync(c->fld_hess.p, 0, (size_t)m32 * 24, st));       // and Hessian 0
        }
        CK(cudaMemcpyAsync(c->fld_pts.p, points, (size_t)m32 * 12, cudaMemcpyDefault, st));
        const int rc = field_run(f, c, c->fld_pts.as<float>(), m32, c->fld_out.as<float>(), kind != FQ_VALUE ? c->fld_grad.as<float>() : nullptr,
                                 kind >= FQ_HESSIAN ? c->fld_hess.as<float>() : nullptr);
        if (rc) return rc;
        CK(cudaMemcpyAsync(out, c->fld_out.p, (size_t)m32 * 4, cudaMemcpyDefault, st));
        if (kind == FQ_GRADIENT || kind == FQ_HESSIAN) CK(cudaMemcpyAsync(grads, c->fld_grad.p, (size_t)m32 * 12, cudaMemcpyDefault, st));
        if (kind == FQ_HESSIAN) CK(cudaMemcpyAsync(hess, c->fld_hess.p, (size_t)m32 * 24, cudaMemcpyDefault, st));
        if (kind == FQ_CURVATURE) {
            c->fld_curv.ensure((size_t)m32 * 8);
            LAUNCH(c, k_field_curvature, nblk(m32, 256), 256, c->fld_grad.as<float>(), c->fld_hess.as<float>(), m32, c->fld_curv.as<float>());
            CK(cudaMemcpyAsync(curv, c->fld_curv.p, (size_t)m32 * 8, cudaMemcpyDefault, st));
        }
        CK(cudaStreamSynchronize(st));
        return SS_OK;
    });
}

extern "C" int ss_levelset_field_at_f32(ss_surface *f, const float *points, uint64_t m, float *out) {
    return field_query(f, points, m, out, FQ_VALUE, nullptr, nullptr, nullptr);
}

extern "C" int ss_levelset_field_gradient_at_f32(ss_surface *f, const float *points, uint64_t m, float *values, float *gradients) {
    return field_query(f, points, m, values, FQ_GRADIENT, gradients, nullptr, nullptr);
}

extern "C" int ss_levelset_field_hessian_at_f32(ss_surface *f, const float *points, uint64_t m, float *values, float *gradients, float *hessians) {
    return field_query(f, points, m, values, FQ_HESSIAN, gradients, hessians, nullptr);
}

extern "C" int ss_levelset_field_curvature_at_f32(ss_surface *f, const float *points, uint64_t m, float *values, float *curvatures) {
    return field_query(f, points, m, values, FQ_CURVATURE, nullptr, nullptr, curvatures);
}

extern "C" int ss_levelset_field_threshold_f32(const ss_surface *f, float *threshold) {
    if (!f || !f->fld || !threshold) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL argument or not a level-set field");
    *threshold = f->fld_D.thr;
    return SS_OK;
}

extern "C" int ss_levelset_field_paths(const ss_surface *f, uint64_t out[3]) {
    if (!f || !f->fld || !out) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL argument or not a level-set field");
    for (int t = 0; t < 3; ++t) out[t] = f->fld_paths[t];
    return SS_OK;
}

// ------------------------------------------------------------------ first crossings along rays ----
// DESIGN.md §15.  Rounds of k_ray_keys, the key sort and group starts of a field query, and the cascade of k_ray_fold / k_ray_select
// with the mode's value fold, until every ray is done; then the gradient fold at the hits through field_run.
template <class F>
static void ray_fold(ss_context *c, const SsDev &D, const SsRayArgs &Q0, uint32_t n_groups, uint64_t *received) {
    uint64_t launches = 0;
    const auto args = [&](const uint32_t *list, uint32_t n, uint32_t *left) {
        SsRayArgs Q = Q0;
        Q.F.groups = list; Q.F.n_groups = n; Q.F.fallback = left;
        return Q;
    };
    run_cascade(c, nullptr, n_groups, {
        [&](const uint32_t *list, uint32_t n, uint32_t *left) {
            LAUNCH(c, (k_ray_fold<F, SS_AN_CAP, SS_FLD_WARPS>), (n + SS_FLD_WARPS - 1) / SS_FLD_WARPS, SS_FLD_WARPS * 32, D, args(list, n, left));
        },
        [&](const uint32_t *list, uint32_t n, uint32_t *left) { LAUNCH(c, (k_ray_fold<F, SS_AN_BIG_CAP, 1>), n, 32, D, args(list, n, left)); },
        [&](const uint32_t *list, uint32_t n, uint32_t *left) { LAUNCH(c, k_ray_select<F>, n, 32, D, args(list, n, left)); },
    }, launches, received);
}

extern "C" int ss_levelset_field_raycast_f32(ss_surface *f, const float *origins, const float *directions, const float *t_max, uint64_t m,
                                             float step, uint32_t refine, float *t, float *positions, float *values, int8_t *status,
                                             float *gradients, uint64_t *rounds) {
    int rc; ss_context *c = field_context(f, &rc);
    if (!c) return rc;
    if (rounds) *rounds = 0;
    if (m && (!origins || !directions || !t || !positions || !values || !status)) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL argument");
    if (!(std::isfinite(step) && step > 0.0f)) return ss_fail(SS_ERR_INVALID_PARAMETER, "level-set raycast: step has to be finite and > 0");
    if (refine > 64) return ss_fail(SS_ERR_INVALID_PARAMETER, "level-set raycast: refine has to lie in [0, 64]");
    if (m >= 0x7fffffffull) return ss_fail(SS_ERR_INDEX_TOO_SMALL, "too many rays for one call");
    if (gradients && (f->fld_mode == SS_FLD_AVG_CORR || f->fld_mode == SS_FLD_AVG_CORR_RAD))
        return ss_fail(SS_ERR_UNSUPPORTED, "level-set field: the Jacobian-corrected averaged surface has no gradient (DESIGN.md 13.1)");
    for (uint64_t &q : f->fld_paths) q = 0;
    if (!m) return SS_OK;
    return ss_guard([&]() -> int {
        CK(cudaSetDevice(c->device));
        cudaStream_t st = c->stream;
        const SsDev &D = f->fld_D;
        const uint32_t m32 = (uint32_t)m;
        c->ray_o.ensure((size_t)m32 * 12); c->ray_d.ensure((size_t)m32 * 12); c->ray_state.ensure((size_t)m32 * sizeof(SsRay));
        c->ray_t.ensure((size_t)m32 * 4); c->ray_pos.ensure((size_t)m32 * 12); c->ray_val.ensure((size_t)m32 * 4); c->ray_status.ensure(m32);
        c->ray_chk.ensure(16);
        CK(cudaMemcpyAsync(c->ray_o.p, origins, (size_t)m32 * 12, cudaMemcpyDefault, st));
        CK(cudaMemcpyAsync(c->ray_d.p, directions, (size_t)m32 * 12, cudaMemcpyDefault, st));
        if (t_max) {
            c->ray_tmax.ensure((size_t)m32 * 4);
            CK(cudaMemcpyAsync(c->ray_tmax.p, t_max, (size_t)m32 * 4, cudaMemcpyDefault, st));
        }
        SsRayOut O{ c->ray_t.as<float>(), c->ray_pos.as<float>(), c->ray_val.as<float>(), c->ray_status.as<int8_t>() };
        uint32_t chk[4] = { 0xffffffffu, 0xffffffffu, 0xffffffffu, 0u };
        CK(cudaMemcpyAsync(c->ray_chk.p, chk, 16, cudaMemcpyHostToDevice, st));
        LAUNCH(c, k_ray_init, nblk(m32, 256), 256, c->ray_o.as<float>(), c->ray_d.as<float>(), t_max ? c->ray_tmax.as<float>() : nullptr, m32, step,
               c->ray_state.as<SsRay>(), O, c->ray_chk.as<uint32_t>());
        CK(cudaMemcpyAsync(chk, c->ray_chk.p, 16, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        static const char *const what[3] = { "has a non-finite origin or direction", "has a zero direction, or a step / |direction| of 0 or not finite",
                                             "has a NaN or negative t_max" };
        for (int q = 0; q < 3; ++q) {
            if (chk[q] == 0xffffffffu) continue;
            char msg[200];
            snprintf(msg, sizeof msg, "level-set raycast: ray %u %s", chk[q], what[q]);
            return ss_fail(SS_ERR_INVALID_PARAMETER, msg);
        }
        SsRayArgs Q{};
        Q.F.A.bins = context_bins(c); Q.F.A.bins.brick_rng = c->fld_rng.as<int2>();
        Q.F.A.grec = c->an_grec.as<float4>(); Q.F.A.rrec = c->av_rrec.as<float>();
        Q.rays = c->ray_state.as<SsRay>(); Q.O = O;
        Q.gmax = make_float3(f->grid.mx[0], f->grid.mx[1], f->grid.mx[2]);
        Q.sub_flat = c->sub_flat.as<uint32_t>(); Q.nsub = f->fld_ready ? f->fld_nsub : 0u;   // no records: every point is 0
        Q.refine = refine;
        c->fld_key_a.ensure((size_t)m32 * 4); c->fld_key_b.ensure((size_t)m32 * 4); c->fld_idx_a.ensure((size_t)m32 * 4); c->fld_idx_b.ensure((size_t)m32 * 4);
        c->fld_chk.ensure(8);
        uint64_t nround = 0;
        for (;;) {
            // one round: the keyed rays' count (the round's synchronisation), their groups, the cascade
            CK(cudaMemsetAsync(c->fld_chk.p, 0, 4, st));
            LAUNCH(c, k_ray_keys, nblk(m32, 256), 256, D, Q, m32, c->fld_key_a.as<uint32_t>(), c->fld_idx_a.as<uint32_t>(), c->fld_chk.as<uint32_t>());
            uint32_t nact = 0;
            CK(cudaMemcpyAsync(&nact, c->fld_chk.p, 4, cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
            if (!nact) break;
            ++nround;
            cub_sort(c, c->fld_key_a.as<uint32_t>(), c->fld_key_b.as<uint32_t>(), nact, 32, c->fld_idx_a.as<uint32_t>(), c->fld_idx_b.as<uint32_t>());
            c->fld_flag.ensure((size_t)nact * 4); c->fld_off.ensure((size_t)nact * 4 + 4); c->fld_starts.ensure((size_t)nact * 4 + 4);
            LAUNCH(c, k_field_starts, nblk(nact, 256), 256, c->fld_key_b.as<uint32_t>(), nact, c->fld_flag.as<uint32_t>());
            uint32_t lc[2] = { 0, 0 };
            scan_compact(c, c->fld_flag.as<uint32_t>(), c->fld_off.as<uint32_t>(), nact, c->fld_starts.as<uint32_t>(), lc);
            CK(cudaStreamSynchronize(st));
            const uint32_t n_groups = lc[0] + lc[1];
            CK(cudaMemcpyAsync(c->fld_starts.as<uint32_t>() + n_groups, &nact, 4, cudaMemcpyHostToDevice, st));
            Q.F.key = c->fld_key_b.as<uint32_t>(); Q.F.idx = c->fld_idx_b.as<uint32_t>(); Q.F.starts = c->fld_starts.as<uint32_t>();
            switch (f->fld_mode) {
            case SS_FLD_ANISO: ray_fold<SsAnisoFold>(c, D, Q, n_groups, f->fld_paths); break;
            case SS_FLD_AVG: ray_fold<SsAvgFold>(c, D, Q, n_groups, f->fld_paths); break;
            case SS_FLD_AVG_CORR: ray_fold<SsAvgCorrFold>(c, D, Q, n_groups, f->fld_paths); break;
            case SS_FLD_AVG_RAD: ray_fold<SsAvgRadFold>(c, D, Q, n_groups, f->fld_paths); break;
            case SS_FLD_AVG_CORR_RAD: ray_fold<SsAvgCorrRadFold>(c, D, Q, n_groups, f->fld_paths); break;
            default: ray_fold<SsSphFold>(c, D, Q, n_groups, f->fld_paths); break;
            }
        }
        if (rounds) *rounds = nround;
        CK(cudaMemcpyAsync(t, c->ray_t.p, (size_t)m32 * 4, cudaMemcpyDefault, st));
        CK(cudaMemcpyAsync(positions, c->ray_pos.p, (size_t)m32 * 12, cudaMemcpyDefault, st));
        CK(cudaMemcpyAsync(values, c->ray_val.p, (size_t)m32 * 4, cudaMemcpyDefault, st));
        CK(cudaMemcpyAsync(status, c->ray_status.p, m32, cudaMemcpyDefault, st));
        if (gradients) {
            // the gradient fold at the hits, packed, then scattered: gradient(position) bit for bit, NaN where there is no hit
            c->ray_grad.ensure((size_t)m32 * 12);
            LAUNCH(c, k_ray_fill_nan, nblk((uint64_t)m32 * 3, 256), 256, c->ray_grad.as<float>(), (uint64_t)m32 * 3);
            c->fld_flag.ensure((size_t)m32 * 4); c->fld_off.ensure((size_t)m32 * 4 + 4);
            c->ray_hits.ensure((size_t)m32 * 4);
            LAUNCH(c, k_ray_hit_flags, nblk(m32, 256), 256, c->ray_status.as<int8_t>(), m32, c->fld_flag.as<uint32_t>());
            uint32_t lc[2] = { 0, 0 };
            scan_compact(c, c->fld_flag.as<uint32_t>(), c->fld_off.as<uint32_t>(), m32, c->ray_hits.as<uint32_t>(), lc);
            CK(cudaStreamSynchronize(st));
            const uint32_t nh = lc[0] + lc[1];
            if (nh) {
                c->fld_pts.ensure((size_t)nh * 12); c->fld_out.ensure((size_t)nh * 4); c->fld_grad.ensure((size_t)nh * 12);
                CK(cudaMemsetAsync(c->fld_grad.p, 0, (size_t)nh * 12, st));           // points without candidates: gradient 0
                LAUNCH(c, k_ray_gather, nblk(nh, 256), 256, c->ray_hits.as<uint32_t>(), nh, c->ray_pos.as<float>(), c->fld_pts.as<float>());
                const int rc = field_run(f, c, c->fld_pts.as<float>(), nh, c->fld_out.as<float>(), c->fld_grad.as<float>());
                if (rc) return rc;
                LAUNCH(c, k_ray_scatter_hits, nblk(nh, 256), 256, c->ray_hits.as<uint32_t>(), nh, c->fld_grad.as<float>(), c->ray_grad.as<float>());
            }
            CK(cudaMemcpyAsync(gradients, c->ray_grad.p, (size_t)m32 * 12, cudaMemcpyDefault, st));
        }
        CK(cudaStreamSynchronize(st));
        return SS_OK;
    });
}

// ------------------------------------------------------------------ narrow-band signed distance grid ----
// DESIGN.md §14.  The result owns its device buffers: it outlives later queries, reconstructions and the field itself.
struct ss_sdf {
    int device = 0;
    uint64_t nl = 0;                 // listed bricks
    int64_t nb[3] = { 0, 0, 0 };     // bricks per axis
    float B = 0.0f;                  // background
    uint64_t paths[2] = { 0, 0 };    // candidate bricks through the shared slice, through the global walk
    uint64_t passes = 0, pairs = 0;  // slabs with candidates, and their (brick, triangle) pairs
    DevBuf coords, values, inside;   // [nl][3] int32, [nl][512] float, [nb0 nb1 nb2] uint8
};

// The working set of one pass: its (brick, triangle) pairs (16 bytes each in keys and values) and its bricks (up to 2 KB of distances
// each, 16 KB of query points, keys and values per listed brick), also bounded by the free device memory.  A call runs as many passes
// as its mesh needs.
#define SS_SDF_PASS_BRICKS (1ull << 19)
static uint64_t g_sdf_pass_pairs = 1ull << 27;
extern "C" void ss_sdf_set_pass_pairs(uint64_t pairs) { g_sdf_pass_pairs = pairs ? std::min<uint64_t>(pairs, 0x7ffffffeull) : (1ull << 27); }

extern "C" int ss_levelset_field_sdf_f32(ss_surface *f, const float *vertices, uint64_t nv, const uint32_t *triangles, uint64_t nt,
                                         uint32_t band, ss_sdf **out) {
    if (!out) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL argument");
    *out = nullptr;
    int rc; ss_context *c = field_context(f, &rc);
    if (!c) return rc;
    if ((nv && !vertices) || (nt && !triangles)) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL argument");
    if (band < 1 || band > 8) return ss_fail(SS_ERR_INVALID_PARAMETER, "signed distance: band must lie in [1, 8] cells");
    if (nv >= (1ull << 32)) return ss_fail(SS_ERR_INDEX_TOO_SMALL, "signed distance: 2^32 or more vertices");
    if (nt >= 0x7fffffffull) return ss_fail(SS_ERR_INDEX_TOO_SMALL, "signed distance: too many triangles for one call");
    SsSdfGrid G{};
    uint64_t nbtot = 1;
    for (int d = 0; d < 3; ++d) {
        G.gmin[d] = f->grid.mn[d];
        G.np[d] = (int)f->grid.np[d];
        G.nb[d] = (int)((f->grid.np[d] + 7) / 8);
        nbtot *= (uint64_t)G.nb[d];
    }
    G.c = f->grid.cell;
    { volatile float b = (float)band * G.c; G.B = b; volatile float r = G.B + G.c; G.reach = r; }
    if (nbtot >= 0x7fffffffull) return ss_fail(SS_ERR_INDEX_TOO_SMALL, "signed distance: too many bricks in the grid");
    std::unique_ptr<ss_sdf> R(new ss_sdf());
    R->device = c->device; R->B = G.B;
    for (int d = 0; d < 3; ++d) R->nb[d] = G.nb[d];
    rc = ss_guard([&]() -> int {
        CK(cudaSetDevice(c->device));
        cudaStream_t st = c->stream;
        const uint32_t nt32 = (uint32_t)nt;
        // own buffers throughout: the context scratch holds the field's records
        DevBuf verts, tris, chk, cnt, off, hist, key_a, key_b, val_a, val_b, flag, scan, starts, dist, listed, lpaths, list, pts, fv;
        verts.ensure(nv * 12); tris.ensure((size_t)nt32 * 12); chk.ensure(16); lpaths.ensure(8); hist.ensure((size_t)G.nb[0] * 8);
        if (nv) CK(cudaMemcpyAsync(verts.p, vertices, nv * 12, cudaMemcpyDefault, st));
        if (nt32) CK(cudaMemcpyAsync(tris.p, triangles, (size_t)nt32 * 12, cudaMemcpyDefault, st));
        unsigned long long hchk[2] = { ~0ull, ~0ull };
        CK(cudaMemcpyAsync(chk.p, hchk, 16, cudaMemcpyHostToDevice, st));
        CK(cudaMemsetAsync(lpaths.p, 0, 8, st));
        CK(cudaMemsetAsync(hist.p, 0, (size_t)G.nb[0] * 8, st));
        if (nv) LAUNCH(c, k_sdf_check_verts, nblk(nv, 256), 256, verts.as<float>(), nv, chk.as<unsigned long long>());
        // candidate bricks per brick column over the whole grid, and the index check
        if (nt32) LAUNCH(c, k_sdf_count, nblk(nt32, 256), 256, G, verts.as<float>(), nv, tris.as<uint32_t>(), nt32, 0, G.nb[0],
                         (unsigned long long *)nullptr, hist.as<unsigned long long>(), chk.as<unsigned long long>());
        std::vector<unsigned long long> col((size_t)G.nb[0]);
        CK(cudaMemcpyAsync(col.data(), hist.p, (size_t)G.nb[0] * 8, cudaMemcpyDeviceToHost, st));
        CK(cudaMemcpyAsync(hchk, chk.p, 16, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        char msg[200];
        if (hchk[0] != ~0ull) {
            snprintf(msg, sizeof msg, "signed distance: vertex %llu has a non-finite coordinate", hchk[0]);
            return ss_fail(SS_ERR_INVALID_PARAMETER, msg);
        }
        if (hchk[1] != ~0ull) {
            snprintf(msg, sizeof msg, "signed distance: triangle %llu has a vertex index >= the number of vertices (%llu)", hchk[1], (unsigned long long)nv);
            return ss_fail(SS_ERR_INVALID_PARAMETER, msg);
        }
        // Passes over slabs of whole brick columns, ascending (the listed bricks stay in ascending order): a slab grows while its pairs
        // stay within the pair bound and its bricks within SS_SDF_PASS_BRICKS; one column is the least a pass takes.
        const uint64_t col_bricks = (uint64_t)G.nb[1] * (uint64_t)G.nb[2];
        // a pass holds about 36 bytes per pair (keys, values, flags, scan, starts, sort scratch) and 25 KB per brick (distances, then
        // query points, keys, indices and values of its listed bricks): both bounds also stay within a third of the free memory each
        size_t free_b = 0, total_b = 0;
        CK(cudaMemGetInfo(&free_b, &total_b));
        const uint64_t max_pairs = std::max<uint64_t>(1, std::min<uint64_t>(g_sdf_pass_pairs, free_b / 3 / 36));
        const uint64_t max_bricks = std::max<uint64_t>(1, std::min<uint64_t>(SS_SDF_PASS_BRICKS, free_b / 3 / 25600));
        int bx0 = 0;
        while (bx0 < G.nb[0]) {
            int bx1 = bx0 + 1;
            uint64_t np_s = col[bx0];
            while (bx1 < G.nb[0] && np_s + col[bx1] <= max_pairs && (uint64_t)(bx1 + 1 - bx0) * col_bricks <= max_bricks) np_s += col[bx1++];
            const int sx0 = bx0;
            bx0 = bx1;
            if (!np_s) continue;
            if (np_s >= 0x7fffffffull) return ss_fail(SS_ERR_INDEX_TOO_SMALL, "signed distance: one brick column has 2^31 or more (brick, triangle) pairs");
            ++R->passes;
            R->pairs += np_s;
            const uint32_t np32 = (uint32_t)np_s;
            cnt.ensure((size_t)nt32 * 8); off.ensure((size_t)nt32 * 8);
            LAUNCH(c, k_sdf_count, nblk(nt32, 256), 256, G, verts.as<float>(), nv, tris.as<uint32_t>(), nt32, sx0, bx1, cnt.as<unsigned long long>(),
                   (unsigned long long *)nullptr, chk.as<unsigned long long>());
            cub_scan(c, cnt.as<unsigned long long>(), off.as<unsigned long long>(), nt32);
            key_a.ensure((size_t)np32 * 4); key_b.ensure((size_t)np32 * 4); val_a.ensure((size_t)np32 * 4); val_b.ensure((size_t)np32 * 4);
            LAUNCH(c, k_sdf_emit, nblk(nt32, 256), 256, G, verts.as<float>(), tris.as<uint32_t>(), nt32, sx0, bx1, off.as<unsigned long long>(),
                   key_a.as<uint32_t>(), val_a.as<uint32_t>());
            cub_sort(c, key_a.as<uint32_t>(), key_b.as<uint32_t>(), np32, bits_for(nbtot - 1), val_a.as<uint32_t>(), val_b.as<uint32_t>());
            flag.ensure((size_t)np32 * 4); scan.ensure((size_t)np32 * 4); starts.ensure((size_t)np32 * 4 + 4);
            LAUNCH(c, k_field_starts, nblk(np32, 256), 256, key_b.as<uint32_t>(), np32, flag.as<uint32_t>());
            uint32_t lc[2] = { 0, 0 };
            scan_compact(c, flag.as<uint32_t>(), scan.as<uint32_t>(), np32, starts.as<uint32_t>(), lc);
            CK(cudaStreamSynchronize(st));
            const uint32_t ncand = lc[0] + lc[1];
            CK(cudaMemcpyAsync(starts.as<uint32_t>() + ncand, &np32, 4, cudaMemcpyHostToDevice, st));
            dist.ensure((size_t)ncand * 512 * 4); listed.ensure((size_t)ncand * 4);
            SsSdfArgs A{};
            A.G = G; A.verts = verts.as<float>(); A.tris = tris.as<uint32_t>(); A.key = key_b.as<uint32_t>(); A.val = val_b.as<uint32_t>();
            A.starts = starts.as<uint32_t>(); A.ncand = ncand; A.dist = dist.as<float>(); A.listed = listed.as<uint32_t>(); A.paths = lpaths.as<uint32_t>();
            LAUNCH(c, (k_sdf_brick<SS_SDF_WARPS, SS_SDF_CAP>), nblk(ncand, SS_SDF_WARPS), SS_SDF_WARPS * 32, A);
            list.ensure((size_t)ncand * 4); scan.ensure((size_t)ncand * 4);
            uint32_t ll[2] = { 0, 0 };
            scan_compact(c, listed.as<uint32_t>(), scan.as<uint32_t>(), ncand, list.as<uint32_t>(), ll);
            CK(cudaStreamSynchronize(st));
            const uint32_t nl = ll[0] + ll[1];
            if (!nl) continue;
            // this pass's listed bricks: coordinates, then distances with the field's sign, appended to the result
            if ((uint64_t)nl * 512 >= 0x7fffffffull) return ss_fail(SS_ERR_INDEX_TOO_SMALL, "signed distance: one brick column lists 2^22 or more bricks");
            const uint32_t m32 = nl * 512u;
            R->coords.grow_keep((R->nl + nl) * 12, R->nl * 12, st); R->values.grow_keep((R->nl + nl) * 2048, R->nl * 2048, st);
            pts.ensure((size_t)m32 * 12); fv.ensure((size_t)m32 * 4);
            LAUNCH(c, k_sdf_points, nblk(m32, 256), 256, G, key_b.as<uint32_t>(), starts.as<uint32_t>(), list.as<uint32_t>(), nl, 0u,
                   pts.as<float>(), R->coords.as<int32_t>() + 3 * R->nl);
            int rc = field_run(f, c, pts.as<float>(), m32, fv.as<float>(), nullptr);
            if (rc) return rc;
            LAUNCH(c, k_sdf_sign, nblk(m32, 256), 256, G, f->fld_D.thr, dist.as<float>(), key_b.as<uint32_t>(), starts.as<uint32_t>(),
                   list.as<uint32_t>(), nl, 0u, fv.as<float>(), R->values.as<float>() + 512 * R->nl, (uint8_t *)nullptr);
            R->nl += nl;
        }
        uint32_t hp[2] = { 0, 0 };
        CK(cudaMemcpyAsync(hp, lpaths.p, 8, cudaMemcpyDeviceToHost, st));
        // the inside flag of every brick: the field at its first point
        const uint32_t nb32 = (uint32_t)nbtot;
        R->inside.ensure(nbtot);
        pts.ensure((size_t)nb32 * 12); fv.ensure((size_t)nb32 * 4);
        LAUNCH(c, k_sdf_points, nblk(nb32, 256), 256, G, key_b.as<uint32_t>(), starts.as<uint32_t>(), list.as<uint32_t>(), 0u, nb32,
               pts.as<float>(), (int32_t *)nullptr);
        int rc = field_run(f, c, pts.as<float>(), nb32, fv.as<float>(), nullptr);
        if (rc) return rc;
        LAUNCH(c, k_sdf_sign, nblk(nb32, 256), 256, G, f->fld_D.thr, dist.as<float>(), key_b.as<uint32_t>(), starts.as<uint32_t>(), list.as<uint32_t>(),
               0u, nb32, fv.as<float>(), (float *)nullptr, R->inside.as<uint8_t>());
        CK(cudaStreamSynchronize(st));
        R->paths[0] = hp[0]; R->paths[1] = hp[1];
        return SS_OK;
    });
    if (rc) return rc;
    *out = R.release();
    return SS_OK;
}

extern "C" uint64_t ss_sdf_num_bricks(const ss_sdf *s) { return s ? s->nl : 0; }

extern "C" int ss_sdf_info(const ss_sdf *s, int64_t bricks_per_dim[3], float *background) {
    if (!s) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL signed distance grid");
    if (bricks_per_dim) for (int d = 0; d < 3; ++d) bricks_per_dim[d] = s->nb[d];
    if (background) *background = s->B;
    return SS_OK;
}

extern "C" int ss_sdf_copy_f32(const ss_sdf *s, int32_t *brick_coords, float *values, uint8_t *brick_inside) {
    if (!s) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL signed distance grid");
    return ss_guard([&]() -> int {
        CK(cudaSetDevice(s->device));
        if (brick_coords && s->nl) CK(cudaMemcpy(brick_coords, s->coords.p, s->nl * 12, cudaMemcpyDefault));
        if (values && s->nl) CK(cudaMemcpy(values, s->values.p, s->nl * 2048, cudaMemcpyDefault));
        if (brick_inside) CK(cudaMemcpy(brick_inside, s->inside.p, (size_t)(s->nb[0] * s->nb[1] * s->nb[2]), cudaMemcpyDefault));
        return SS_OK;
    });
}

extern "C" int ss_sdf_passes(const ss_sdf *s, uint64_t out[2]) {
    if (!s || !out) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL argument");
    out[0] = s->passes; out[1] = s->pairs;
    return SS_OK;
}

extern "C" int ss_sdf_paths(const ss_sdf *s, uint64_t out[2]) {
    if (!s || !out) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL argument");
    out[0] = s->paths[0]; out[1] = s->paths[1];
    return SS_OK;
}

extern "C" void ss_sdf_free(ss_sdf *s) {
    if (!s) return;
    cudaSetDevice(s->device);
    delete s;
}

// ------------------------------------------------------------------ the field's surface as a mesh ----
// DESIGN.md §16.  Tiles of 64^3 lattice cells in batches; per batch: listing, the cascade of k_lm_fold / k_lm_select into zero-filled
// tiles, marching cubes; the weld by global edge key at the end.  The result owns its mesh; the field's records are only read.
static uint32_t g_lm_batch_tiles = 0;          // 0: as many tiles per batch as fit a third of the free device memory
extern "C" void ss_levelset_mesh_set_batch_tiles(uint32_t tiles) { g_lm_batch_tiles = tiles; }

// The listed bricks of a batch through the tiers of run_cascade: 512-slot slice, 4096-slot slice, selection walk.  A brick goes on with
// all its groups; each tier folds only the groups with more candidates than the previous tier's slice (paths: bricks per tier).
template <class F>
static void lm_fold(ss_context *c, const SsDev &D, const SsLmFoldArgs &L0, const uint32_t *list, uint32_t n, uint64_t *paths) {
    uint64_t launches = 0;
    const auto args = [&](const uint32_t *l, uint32_t m, uint32_t *left, uint32_t done) {
        SsLmFoldArgs L = L0;
        L.bricks = l; L.n_bricks = m; L.fallback = left; L.done = done;
        return L;
    };
    run_cascade(c, list, n, {
        [&](const uint32_t *l, uint32_t m, uint32_t *left) {
            LAUNCH(c, (k_lm_fold<F, SS_AN_CAP, SS_LM_WARPS>), (m + SS_LM_WARPS - 1) / SS_LM_WARPS, SS_LM_WARPS * 32, D, args(l, m, left, 0));
        },
        [&](const uint32_t *l, uint32_t m, uint32_t *left) { LAUNCH(c, (k_lm_fold<F, SS_AN_BIG_CAP, 1>), m, 32, D, args(l, m, left, SS_AN_CAP)); },
        [&](const uint32_t *l, uint32_t m, uint32_t *left) { LAUNCH(c, k_lm_select<F>, m, 32, D, args(l, m, left, SS_AN_BIG_CAP)); },
    }, launches, paths);
}

extern "C" int ss_levelset_field_mesh_f32(ss_surface *f, const float *aabb_min, const float *aabb_max, float cube_size, ss_surface **out) {
    if (!out) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL argument");
    *out = nullptr;
    int rc; ss_context *c = field_context(f, &rc);
    if (!c) return rc;
    if ((aabb_min == nullptr) != (aabb_max == nullptr)) return ss_fail(SS_ERR_INVALID_PARAMETER, "level-set mesh: give both aabb_min and aabb_max, or neither");
    if (!std::isfinite(cube_size)) return ss_fail(SS_ERR_INVALID_PARAMETER, "level-set mesh: the cube size has to be finite");
    if (aabb_min) {
        for (int d = 0; d < 3; ++d) {
            if (!std::isfinite(aabb_min[d]) || !std::isfinite(aabb_max[d])) return ss_fail(SS_ERR_INVALID_PARAMETER, "level-set mesh: the box has to be finite");
            if (!(aabb_min[d] <= aabb_max[d])) return ss_fail(SS_ERR_INVALID_PARAMETER, "level-set mesh: aabb_min has to be <= aabb_max");
        }
    }
    const SsDev &D = f->fld_D;
    if (!(D.thr >= 0.0f))
        return ss_fail(SS_ERR_UNSUPPORTED, "level-set mesh: a negative threshold would put the points no particle reaches inside (DESIGN.md 16)");
    const float cell = f->grid.cell, cs = cube_size > 0.0f ? cube_size : cell;
    // the index range per axis, float64 arithmetic on the f32 values
    int64_t lo[3], hi[3];
    bool empty = false;
    for (int d = 0; d < 3; ++d) {
        const double top = cs == cell ? (double)f->grid.nc[d] : std::ceil((double)f->grid.nc[d] * (double)cell / (double)cs);
        double l = 0.0, h = top;
        if (aabb_min) {
            l = std::max(l, std::floor(((double)aabb_min[d] - (double)f->grid.mn[d]) / (double)cs));
            h = std::min(h, std::ceil(((double)aabb_max[d] - (double)f->grid.mn[d]) / (double)cs));
        }
        if (l > h) { empty = true; lo[d] = hi[d] = 0; continue; }
        if (h > (double)((1 << 20) - 1)) return ss_fail(SS_ERR_INDEX_TOO_SMALL, "level-set mesh: lattice index above 2^20 - 1 (the marching-cubes edge key)");
        lo[d] = (int64_t)l; hi[d] = (int64_t)h;
    }
    for (uint64_t &q : f->fld_paths) q = 0;
    return with_new_surface(c, out, [&](ss_surface *s) -> int {
        cudaStream_t st = c->stream;
        s->owner = c; s->frame = f->frame; s->S = 64; s->lm = 1; s->lm_cube = cs;
        s->grid = f->grid; s->grid.cell = cs;
        for (int d = 0; d < 3; ++d) { s->lm_imin[d] = lo[d]; s->lm_imax[d] = hi[d]; }
        const uint32_t nsub = f->fld_ready ? f->fld_nsub : 0u;
        SsLmGrid G{};
        uint64_t ntt = 1;
        for (int d = 0; d < 3; ++d) {
            G.gmin[d] = f->grid.mn[d]; G.imin[d] = (int)lo[d]; G.npts[d] = (int)(hi[d] - lo[d] + 1);
            G.ntile[d] = (int)((hi[d] - lo[d] + 63) / 64);
            ntt *= (uint64_t)G.ntile[d];
        }
        if (empty || !nsub || !ntt) return SS_OK;                       // no cell, or no record: the empty mesh
        if (ntt >= 0x7fffffffull) return ss_fail(SS_ERR_INDEX_TOO_SMALL, "level-set mesh: 2^31 or more tiles in the range");
        G.c = cs; G.Sb = cs == cell ? D.S : 0; G.sub_size = G.Sb ? fmulr(cs, (float)G.Sb) : 0.0f;
        G.gmax = make_float3(f->grid.mx[0], f->grid.mx[1], f->grid.mx[2]);
        G.sub_flat = c->sub_flat.as<uint32_t>(); G.nsub = nsub;
        // groups with records, tiles that can hold a nonzero point
        const uint32_t nb3 = (uint32_t)(D.nb * D.nb * D.nb), ngroups = nsub * nb3, ntt32 = (uint32_t)ntt;
        SsBins bins = context_bins(c); bins.brick_rng = c->fld_rng.as<int2>();
        DevBuf grp, tflag, toff, tchunk, tlist, fflag, foff, flist, mflag, moff, mlist, tiles, voff, vmask, vcnt, tcnt, vblk_off, tblk_off;
        grp.ensure(ngroups);
        LAUNCH(c, k_lm_groups, nblk(ngroups, 256), 256, D, bins, ngroups, grp.as<uint8_t>());
        G.grp = grp.as<uint8_t>();
        // in chunks of SS_LM_TILE_CHUNK tiles: 12 bytes per tile of the chunk, then 4 per tile that can hold a nonzero point
        const uint32_t chunk = std::min<uint32_t>(ntt32, SS_LM_TILE_CHUNK);
        tflag.ensure((size_t)chunk * 4); toff.ensure((size_t)chunk * 4 + 4); tchunk.ensure((size_t)chunk * 4);
        uint32_t ntl = 0;
        for (uint32_t t0 = 0; t0 < ntt32; t0 += chunk) {
            const uint32_t nc = std::min<uint32_t>(chunk, ntt32 - t0);
            LAUNCH(c, k_lm_tiles, nblk(nc, 128), 128, D, G, t0, nc, tflag.as<uint32_t>());
            uint32_t lt[2] = { 0, 0 };
            scan_compact(c, tflag.as<uint32_t>(), toff.as<uint32_t>(), nc, tchunk.as<uint32_t>(), lt);
            CK(cudaStreamSynchronize(st));
            const uint32_t k = lt[0] + lt[1];
            if (!k) continue;
            tlist.grow_keep(((size_t)ntl + k) * 4, (size_t)ntl * 4, st);
            LAUNCH(c, k_lm_offset, nblk(k, 256), 256, tchunk.as<uint32_t>(), k, t0, tlist.as<uint32_t>() + ntl);
            ntl += k;
        }
        if (!ntl) return SS_OK;
        // batch size: a third of the free memory (values, vertex offsets and masks per point, six lists per brick)
        const size_t np3 = 65ull * 65 * 65, per_tile = np3 * 9 + 729ull * 40 + 256;
        size_t free_b = 0, total_b = 0;
        CK(cudaMemGetInfo(&free_b, &total_b));
        size_t max_tiles = std::max<size_t>(1, free_b / 3 / per_tile);
        if (g_lm_batch_tiles) max_tiles = std::min<size_t>(max_tiles, g_lm_batch_tiles);
        max_tiles = std::min<size_t>(max_tiles, ntl);
        const size_t nbr_max = max_tiles * 729;
        tiles.ensure(max_tiles * np3 * 4); voff.ensure(max_tiles * np3 * 4); vmask.ensure(max_tiles * np3);
        for (DevBuf *b : { &fflag, &foff, &flist, &mflag, &moff, &mlist, &vcnt, &tcnt, &vblk_off, &tblk_off }) b->ensure(nbr_max * 4 + 4);
        SsDev Pm = D;                                                   // the tile layout of marching cubes
        Pm.S = 64; Pm.np = 65; Pm.nb = SS_LM_NB; Pm.np_magic = (uint32_t)(4294967296ull / 65ull) + 1u;
        SsLmFoldArgs L{};
        L.A.bins = bins; L.A.grec = c->an_grec.as<float4>(); L.A.rrec = c->av_rrec.as<float>();
        L.tiles = tiles.as<float>();
        s->verts.ensure(1 << 16); s->vkeys.ensure(1 << 16); s->tris.ensure(1 << 16);
        c->bkeys_a.ensure(1 << 16); c->bids_a.ensure(1 << 16); c->bcount.ensure(4);
        CK(cudaMemsetAsync(c->bcount.p, 0, 4, st));
        uint64_t vtotal = 0, ttotal = 0;
        for (uint32_t t0 = 0; t0 < ntl; t0 += (uint32_t)max_tiles) {
            const uint32_t nbatch = std::min<uint32_t>((uint32_t)max_tiles, ntl - t0), nbr = nbatch * 729u;
            G.tiles = tlist.as<uint32_t>() + t0; L.G = G;
            CK(cudaMemsetAsync(tiles.p, 0, (size_t)nbatch * np3 * 4, st));
            LAUNCH(c, k_lm_list, nblk(nbr, 128), 128, D, G, nbr, fflag.as<uint32_t>());
            LAUNCH(c, k_lm_mc_flags, nblk(nbr, 256), 256, fflag.as<uint32_t>(), nbr, mflag.as<uint32_t>());
            uint32_t lf[2] = { 0, 0 }, lm[2] = { 0, 0 };
            scan_compact(c, fflag.as<uint32_t>(), foff.as<uint32_t>(), nbr, flist.as<uint32_t>(), lf);
            scan_compact(c, mflag.as<uint32_t>(), moff.as<uint32_t>(), nbr, mlist.as<uint32_t>(), lm);
            CK(cudaStreamSynchronize(st));
            const uint32_t nf = lf[0] + lf[1], n_mc = lm[0] + lm[1];
            ++s->lm_batches;
            switch (f->fld_mode) {
            case SS_FLD_ANISO: lm_fold<SsAnisoFold>(c, D, L, flist.as<uint32_t>(), nf, f->fld_paths); break;
            case SS_FLD_AVG: lm_fold<SsAvgFold>(c, D, L, flist.as<uint32_t>(), nf, f->fld_paths); break;
            case SS_FLD_AVG_CORR: lm_fold<SsAvgCorrFold>(c, D, L, flist.as<uint32_t>(), nf, f->fld_paths); break;
            case SS_FLD_AVG_RAD: lm_fold<SsAvgRadFold>(c, D, L, flist.as<uint32_t>(), nf, f->fld_paths); break;
            case SS_FLD_AVG_CORR_RAD: lm_fold<SsAvgCorrRadFold>(c, D, L, flist.as<uint32_t>(), nf, f->fld_paths); break;
            default: lm_fold<SsSphFold>(c, D, L, flist.as<uint32_t>(), nf, f->fld_paths); break;
            }
            if (!n_mc) continue;
            // marching cubes of the batch, appended to the result (as marching_cubes_batch)
            LAUNCH(c, k_lm_mc_count, (n_mc + SS_MW_WARPS - 1) / SS_MW_WARPS, SS_MW_WARPS * 32, Pm, G, tiles.as<float>(), mlist.as<uint32_t>(), n_mc,
                   vmask.as<uint8_t>(), voff.as<uint32_t>(), vcnt.as<uint32_t>(), tcnt.as<uint32_t>());
            uint32_t lv[2] = { 0, 0 }, ltr[2] = { 0, 0 }, bc = 0;
            scan_with_total(c, vcnt.as<uint32_t>(), vblk_off.as<uint32_t>(), n_mc, lv);
            scan_with_total(c, tcnt.as<uint32_t>(), tblk_off.as<uint32_t>(), n_mc, ltr);
            CK(cudaMemcpyAsync(&bc, c->bcount.p, 4, cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
            const uint64_t bv = (uint64_t)lv[0] + lv[1], bt = (uint64_t)ltr[0] + ltr[1];
            if (vtotal + bv >= 0xfffffff0ull || ttotal + bt >= 0xfffffff0ull) return ss_fail(SS_ERR_INDEX_TOO_SMALL, "mesh too large for 32-bit vertex / triangle ids");
            if (!bv && !bt) continue;
            s->verts.grow_keep((vtotal + bv) * 12, vtotal * 12, st);
            s->vkeys.grow_keep((vtotal + bv) * 8, vtotal * 8, st);
            s->tris.grow_keep((ttotal + bt) * 12, ttotal * 12, st);
            c->bkeys_a.grow_keep(((size_t)bc + bv) * 8, (size_t)bc * 8, st);
            c->bids_a.grow_keep(((size_t)bc + bv) * 4, (size_t)bc * 4, st);
            SsMcOut O{};
            O.verts = s->verts.as<float>(); O.tris = s->tris.as<uint32_t>(); O.vkeys = s->vkeys.as<unsigned long long>();
            O.bkeys = c->bkeys_a.as<unsigned long long>(); O.bids = c->bids_a.as<uint32_t>(); O.bcount = c->bcount.as<uint32_t>();
            O.vbase = (uint32_t)vtotal; O.tbase = (uint32_t)ttotal; O.bcap = (uint32_t)std::min<size_t>((size_t)bc + bv, 0xffffffffu);
            LAUNCH(c, k_lm_mc_emit, (n_mc + SS_MW_WARPS - 1) / SS_MW_WARPS, SS_MW_WARPS * 32, Pm, G, tiles.as<float>(), mlist.as<uint32_t>(), n_mc,
                   vmask.as<uint8_t>(), voff.as<uint32_t>(), vcnt.as<uint32_t>(), tcnt.as<uint32_t>(), vblk_off.as<uint32_t>(), tblk_off.as<uint32_t>(),
                   mflag.as<uint32_t>(), moff.as<uint32_t>(), O);
            vtotal += bv; ttotal += bt;
        }
        uint64_t nv_final = vtotal;
        uint32_t bc = 0;
        rc = weld_boundary_vertices(c, s, vtotal, ttotal, nv_final, bc);
        if (rc) return rc;
        s->nv = nv_final; s->nt = ttotal;
        CK(cudaStreamSynchronize(st));
        return SS_OK;
    });
}

extern "C" int ss_levelset_mesh_info(const ss_surface *m, float *cube_size, int64_t index_min[3], int64_t index_max[3], uint64_t *batches) {
    if (!m || !m->lm) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL argument or not a level-set mesh (ss_levelset_field_mesh_f32)");
    if (cube_size) *cube_size = m->lm_cube;
    for (int d = 0; d < 3; ++d) { if (index_min) index_min[d] = m->lm_imin[d]; if (index_max) index_max[d] = m->lm_imax[d]; }
    if (batches) *batches = m->lm_batches;
    return SS_OK;
}

#include "ss_post.cuh"
#include "ss_meshproc.inc"
#include "ss_meshio.inc"
