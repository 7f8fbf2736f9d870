// ss_post.cuh -- mesh post-processing on the device (SURVEY.md 8f; splashsurf/src/reconstruct.rs:1094-1391).
// Included at the end of ss_pipeline.cu (needs ss_context / ss_surface and the launch helpers).
//
//   SPH interpolation of per-particle quantities to the mesh vertices      sph_interpolation.rs:210-258
//   smoothing weights from distance-weighted neighbour counts              reconstruct.rs:1159-1258
//   weighted Laplacian smoothing of the vertices                           postprocessing.rs:17-53
//   SPH / area-weighted vertex normals at the (smoothed) vertices          sph_interpolation.rs:82-133, mesh.rs:799-906
//   Laplacian smoothing of the normal field                                postprocessing.rs:56-97
//
// The particle queries reuse the splat bins of the reconstruction that produced the surface (they stay in the context's
// scratch until the next call on that context).  All results are sums whose order differs from the reference's (R-tree
// and hash-map order there): parity is to f32 round-off (tests: 2e-5 relative), not bit-exact.
#pragma once

// ------------------------------------------------------------------ particle queries over the splat bins ----
struct SsQuery {
    const uint32_t *sub_flat; uint32_t nsub;      // compressed -> flat subdomain index (ascending)
    const uint32_t *bin_start, *bin_end;          // [nsub * nbin_sub]
    const uint32_t *pidx;                         // bin-sorted particle indices
    const float4 *rec;                            // bin-sorted (x, y, z, V)
    const float *rho;                             // per particle density
    float sphere_mass;                            // 4/3 pi r^3 rho0 (reconstruct.rs:1126-1129)
};

// flat index of the subdomain tile that contains x (clamped to the grid)
__device__ __forceinline__ uint32_t ss_tile_of_position(const SsDev &P, const float x[3]) {
    int t[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) t[d] = min(max((int)floorf((x[d] - P.gmin[d]) / P.sub_size), 0), P.nsd[d] - 1);
    return (uint32_t)((t[0] * P.nsd[1] + t[1]) * P.nsd[2] + t[2]);
}

// visit(e, rec[e]) for every binned particle of the tile containing x whose bin overlaps the ball of radius h around x.
// The tile's bins hold every particle within the ghost margin (>= h) of the tile, hence every particle within h of x.
template <typename F>
__device__ __forceinline__ void ss_particles_near(const SsDev &P, const SsQuery &Q, const float x[3], F &&visit) {
    const uint32_t flat = ss_tile_of_position(P, x);
    uint32_t lo = 0, hi = Q.nsub;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (Q.sub_flat[mid] < flat) lo = mid + 1; else hi = mid; }
    if (lo >= Q.nsub || Q.sub_flat[lo] != flat) return;          // no particle within the ghost margin of this tile
    const SsSubGeom g = ss_sub_geom(P, flat);
    const float reach = P.h * P.inv_c * 1.0001f + 0.001f;        // h in cells, with slack
    int b0[3], b1[3];
#pragma unroll
    for (int d = 0; d < 3; ++d) {
        const float u = (x[d] - g.smin[d]) * P.inv_c;
        b0[d] = min(max((int)floorf((u - reach) / (float)P.be) + P.nlo, 0), P.nbin - 1);
        b1[d] = min(max((int)floorf((u + reach) / (float)P.be) + P.nlo, 0), P.nbin - 1);
    }
    for (int X = b0[0]; X <= b1[0]; ++X) for (int Y = b0[1]; Y <= b1[1]; ++Y) {
        uint32_t a;
        const uint32_t len = ss_bin_column(P, Q.bin_start, Q.bin_end, lo, X, Y, b0[2], b1[2], a);
        for (uint32_t e = a; e < a + len; ++e) visit(e, Q.rec[e]);
    }
}

__device__ __forceinline__ float ss_dist2(const float4 r, const float x[3], float &dx, float &dy, float &dz) {
    dx = r.x - x[0]; dy = r.y - x[1]; dz = r.z - x[2];
    return dx * dx + dy * dy + dz * dz;
}

// Distance-weighted neighbour count per particle (reconstruct.rs:1190-1205): sum over j != i, d^2 < h^2 of
// 1 - clamp(d^2 / h^2, 0, 1).  One thread per bin entry; the entry of the tile that contains the particle does the work.
__global__ void __launch_bounds__(128)
k_pp_weighted_ncount(SsDev P, SsQuery Q, const uint32_t *__restrict__ bin_key, uint32_t m, float *__restrict__ wnc) {
    const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
    if (e >= m) return;
    const uint32_t key = bin_key[e];
    if (key == 0xffffffffu) return;
    const uint32_t s = key / (uint32_t)P.nbin_sub;
    const float4 me = Q.rec[e];
    const float x[3] = { me.x, me.y, me.z };
    if (Q.sub_flat[s] != ss_tile_of_position(P, x)) return;
    const uint32_t i = Q.pidx[e];
    float sum = 0.0f;
    ss_particles_near(P, Q, x, [&](uint32_t e2, const float4 r) {
        float dx, dy, dz;
        const float d2 = ss_dist2(r, x, dx, dy, dz);
        if (d2 < P.h2 && Q.pidx[e2] != i) sum += 1.0f - fminf(fmaxf(d2 / P.h2, 0.0f), 1.0f);
    });
    wnc[i] = sum;
}

// SPH interpolation of a DIM-component particle quantity to points (sph_interpolation.rs:210-258).
template <int DIM>
__global__ void __launch_bounds__(128)
k_pp_interpolate(SsDev P, SsQuery Q, const float *__restrict__ pts, uint32_t npts, const float *__restrict__ values,
                 int correction, float *__restrict__ out) {
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= npts) return;
    const float x[3] = { pts[3 * (size_t)v], pts[3 * (size_t)v + 1], pts[3 * (size_t)v + 2] };
    float acc[DIM], corr = 0.0f;
#pragma unroll
    for (int k = 0; k < DIM; ++k) acc[k] = 0.0f;
    ss_particles_near(P, Q, x, [&](uint32_t e, const float4 r) {
        float dx, dy, dz;
        const float d2 = ss_dist2(r, x, dx, dy, dz);
        if (!(d2 <= P.h2)) return;
        const uint32_t j = Q.pidx[e];
        const float w = (Q.sphere_mass / Q.rho[j]) * ss_kernel_scalar(P, sqrtf(d2));
#pragma unroll
        for (int k = 0; k < DIM; ++k) acc[k] += values[(size_t)j * DIM + k] * w;
        corr += w;
    });
    // sph_interpolation.rs:252-254: enable * (1 / correction) + (1 - enable).  No particle in range: 0 * inf = NaN with or without the
    // correction, like in the reference
    const float en = correction ? 1.0f : 0.0f;
    const float f = en * (1.0f / corr) + (1.0f - en);
#pragma unroll
    for (int k = 0; k < DIM; ++k) out[(size_t)v * DIM + k] = acc[k] * f;
}

// SPH normals at arbitrary points (the vertices after smoothing): same arithmetic as k_sph_normals, position-based query.
__global__ void __launch_bounds__(128)
k_pp_sph_normals(SsDev P, SsQuery Q, const float *__restrict__ pts, uint32_t npts, float *__restrict__ normals) {
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v >= npts) return;
    const float x[3] = { pts[3 * (size_t)v], pts[3 * (size_t)v + 1], pts[3 * (size_t)v + 2] };
    const float dqdr = 2.0f / P.h;
    float gx = 0.0f, gy = 0.0f, gz = 0.0f;
    ss_particles_near(P, Q, x, [&](uint32_t e, const float4 r) {
        float dx, dy, dz;
        const float d2 = ss_dist2(r, x, dx, dy, dz);
        if (!(d2 <= P.h2)) return;
        const float rr = sqrtf(d2);
        const float gn = P.s_sigma * ss_kernel_dq(P, (rr + rr) / P.h) * dqdr;
        const float vol = Q.sphere_mass / Q.rho[Q.pidx[e]];
        gx += (dx / rr) * gn * vol; gy += (dy / rr) * gn * vol; gz += (dz / rr) * gn * vol;
    });
    const float nrm = sqrtf(gx * gx + gy * gy + gz * gz);
    normals[3 * (size_t)v] = gx / nrm; normals[3 * (size_t)v + 1] = gy / nrm; normals[3 * (size_t)v + 2] = gz / nrm;
}

// reconstruct.rs:1220-1231: x = min(max(n, 0) / normalization, 1); smooth step 6 x^5 - 15 x^4 + 10 x^3
__global__ void k_pp_smoothstep(uint32_t n, const float *__restrict__ wnn, float normalization, float *__restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float x = fminf(fmaxf(wnn[i], 0.0f) / normalization, 1.0f);
    const float x3 = x * x * x, x4 = x3 * x, x5 = x4 * x;
    out[i] = x5 * 6.0f - x4 * 15.0f + x3 * 10.0f;
}

// ------------------------------------------------------------------ mesh connectivity (CSR) ----
// vertex -> vertex: the 6 directed pairs of every triangle as (a << 32 | b), sorted, duplicates dropped
// (mesh.rs:290-306; neighbours end up in ascending order instead of first-appearance order).
__global__ void k_pp_edge_keys(const uint32_t *__restrict__ tris, uint32_t nt, unsigned long long *__restrict__ keys) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nt) return;
    const uint32_t v[3] = { tris[3 * (size_t)t], tris[3 * (size_t)t + 1], tris[3 * (size_t)t + 2] };
    int o = 0;
#pragma unroll
    for (int a = 0; a < 3; ++a)
#pragma unroll
        for (int b = 0; b < 3; ++b) {
            if (a == b) continue;
            keys[6 * (size_t)t + o] = (v[a] == v[b]) ? ~0ull : (((unsigned long long)v[a] << 32) | v[b]);
            ++o;
        }
}
// vertex -> incident triangle: (vertex << 32 | triangle)
__global__ void k_pp_corner_keys(const uint32_t *__restrict__ tris, uint32_t nt, unsigned long long *__restrict__ keys) {
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= nt) return;
#pragma unroll
    for (int a = 0; a < 3; ++a) keys[3 * (size_t)t + a] = ((unsigned long long)tris[3 * (size_t)t + a] << 32) | t;
}
__global__ void k_pp_flag_unique(const unsigned long long *__restrict__ keys, uint32_t n, uint32_t *__restrict__ flag) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const unsigned long long key = keys[k];
    flag[k] = (key != ~0ull && (k == 0 || keys[k - 1] != key)) ? 1u : 0u;
}
__global__ void k_pp_compact_low(const unsigned long long *__restrict__ keys, const uint32_t *__restrict__ flag,
                                 const uint32_t *__restrict__ off, uint32_t n, uint32_t *__restrict__ out) {
    const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < n && flag[k]) out[off[k]] = (uint32_t)(keys[k] & 0xffffffffull);
}
// row[v] = number of kept keys with high word < v, for v = 0 .. nv (lower bound in the sorted keys)
__global__ void k_pp_row_offsets(const unsigned long long *__restrict__ keys, const uint32_t *__restrict__ off, uint32_t n,
                                 uint32_t total, uint32_t nv, uint32_t *__restrict__ row) {
    const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
    if (v > nv) return;
    const unsigned long long want = (unsigned long long)v << 32;
    uint32_t lo = 0, hi = n;
    while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (keys[mid] < want) lo = mid + 1; else hi = mid; }
    row[v] = lo < n ? off[lo] : total;
}

// ------------------------------------------------------------------ smoothing ----
// One iteration of postprocessing.rs:31-51 after the buffer swap: `cur` holds the vertices of two iterations ago (read at i
// only, then overwritten), `prev` those of the previous iteration (read at the neighbours).
__global__ void k_pp_laplacian(uint32_t nv, float *__restrict__ cur, const float *__restrict__ prev, const uint32_t *__restrict__ row,
                               const uint32_t *__restrict__ adj, const float *__restrict__ weights, float beta) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nv) return;
    const float be = beta * (weights ? weights[i] : 1.0f);
    const uint32_t a = row[i], b = row[i + 1];
    float sx = 0.0f, sy = 0.0f, sz = 0.0f;
    for (uint32_t k = a; k < b; ++k) { const size_t j = adj[k]; sx += prev[3 * j]; sy += prev[3 * j + 1]; sz += prev[3 * j + 2]; }
    if (b > a) { const float n = (float)(b - a); sx /= n; sy /= n; sz /= n; }
    const float om = 1.0f - be;
    cur[3 * (size_t)i] = cur[3 * (size_t)i] * om + sx * be;
    cur[3 * (size_t)i + 1] = cur[3 * (size_t)i + 1] * om + sy * be;
    cur[3 * (size_t)i + 2] = cur[3 * (size_t)i + 2] * om + sz * be;
}
// postprocessing.rs:74-85: n_i = normalize(sum of the neighbours' normals)
__global__ void k_pp_smooth_normals(uint32_t nv, const float *__restrict__ in, float *__restrict__ out, const uint32_t *__restrict__ row,
                                    const uint32_t *__restrict__ adj) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nv) return;
    float sx = 0.0f, sy = 0.0f, sz = 0.0f;
    for (uint32_t k = row[i]; k < row[i + 1]; ++k) { const size_t j = adj[k]; sx += in[3 * j]; sy += in[3 * j + 1]; sz += in[3 * j + 2]; }
    const float nrm = sqrtf(sx * sx + sy * sy + sz * sz);
    out[3 * (size_t)i] = sx / nrm; out[3 * (size_t)i + 1] = sy / nrm; out[3 * (size_t)i + 2] = sz / nrm;
}
// mesh.rs:812-821 + :899-905: sum over the incident triangles of cross(v1 - v0, v2 - v1), normalised
__global__ void k_pp_area_normals(uint32_t nv, const float *__restrict__ verts, const uint32_t *__restrict__ tris,
                                  const uint32_t *__restrict__ row, const uint32_t *__restrict__ inc, float *__restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nv) return;
    float sx = 0.0f, sy = 0.0f, sz = 0.0f;
    for (uint32_t k = row[i]; k < row[i + 1]; ++k) {
        const size_t t = inc[k];
        const size_t i0 = tris[3 * t], i1 = tris[3 * t + 1], i2 = tris[3 * t + 2];
        const float ax = verts[3 * i1] - verts[3 * i0], ay = verts[3 * i1 + 1] - verts[3 * i0 + 1], az = verts[3 * i1 + 2] - verts[3 * i0 + 2];
        const float bx = verts[3 * i2] - verts[3 * i1], by = verts[3 * i2 + 1] - verts[3 * i1 + 1], bz = verts[3 * i2 + 2] - verts[3 * i1 + 2];
        sx += ay * bz - az * by; sy += az * bx - ax * bz; sz += ax * by - ay * bx;
    }
    const float nrm = sqrtf(sx * sx + sy * sy + sz * sz);
    out[3 * (size_t)i] = sx / nrm; out[3 * (size_t)i + 1] = sy / nrm; out[3 * (size_t)i + 2] = sz / nrm;
}

// ------------------------------------------------------------------ host side ----
#ifndef SS_POST_KERNELS_ONLY          // (tests/emul steps the kernels above on the CPU and skips the rest)
// Sorted unique low words per high word: row[nv + 1], idx[total].  `keys_a` holds n keys on entry (destroyed).
static uint32_t pp_build_csr(ss_context *c, uint32_t n, uint32_t nv, int key_bits, DevBuf &row, DevBuf &idx) {
    cudaStream_t st = c->stream;
    PostScratch &S = c->post;
    if (n == 0) {                                   // vertices without triangles: empty adjacency lists, like the reference
        row.ensure(((size_t)nv + 1) * 4); idx.ensure(4);
        CK(cudaMemsetAsync(row.p, 0, ((size_t)nv + 1) * 4, st));
        return 0;
    }
    S.keys_b.ensure((size_t)n * 8); S.flag.ensure((size_t)n * 4); S.scan.ensure((size_t)n * 4 + 4);
    cub_sort(c, S.keys_a.as<unsigned long long>(), S.keys_b.as<unsigned long long>(), n, key_bits);
    LAUNCH(c, k_pp_flag_unique, nblk(n, 256), 256, S.keys_b.as<unsigned long long>(), n, S.flag.as<uint32_t>());
    const uint32_t total = (uint32_t)scan_total(c, S.flag.as<uint32_t>(), S.scan.as<uint32_t>(), n);
    row.ensure(((size_t)nv + 1) * 4); idx.ensure(std::max<size_t>(total, 1) * 4);
    LAUNCH(c, k_pp_compact_low, nblk(n, 256), 256, S.keys_b.as<unsigned long long>(), S.flag.as<uint32_t>(), S.scan.as<uint32_t>(), n,
           idx.as<uint32_t>());
    LAUNCH(c, k_pp_row_offsets, nblk((uint64_t)nv + 1, 256), 256, S.keys_b.as<unsigned long long>(), S.scan.as<uint32_t>(), n, total, nv,
           row.as<uint32_t>());
    return total;
}

static void pp_vertex_adjacency(ss_context *c, ss_surface *s) {          // vertex -> vertex
    if (s->has_adj) return;
    const uint32_t nt = (uint32_t)s->nt, nv = (uint32_t)s->nv;
    c->post.keys_a.ensure((size_t)nt * 6 * 8);
    if (nt) LAUNCH(c, k_pp_edge_keys, nblk(nt, 256), 256, s->tris.as<uint32_t>(), nt, c->post.keys_a.as<unsigned long long>());
    pp_build_csr(c, nt * 6, nv, 64, s->adj_row, s->adj_idx);             // 64 bits: the degenerate-pair sentinel sorts last
    s->has_adj = 1;
}
static void pp_vertex_triangles(ss_context *c, ss_surface *s) {          // vertex -> incident triangles
    if (s->has_inc) return;
    const uint32_t nt = (uint32_t)s->nt, nv = (uint32_t)s->nv;
    c->post.keys_a.ensure((size_t)nt * 3 * 8);
    if (nt) LAUNCH(c, k_pp_corner_keys, nblk(nt, 256), 256, s->tris.as<uint32_t>(), nt, c->post.keys_a.as<unsigned long long>());
    pp_build_csr(c, nt * 3, nv, 32 + bits_for(nv), s->inc_row, s->inc_idx);
    s->has_inc = 1;
}

// common argument / state checks; returns the owning context or nullptr (error already recorded)
static ss_context *pp_context(ss_surface *s, bool need_bins, int *rc) {
    *rc = SS_OK;
    if (!s) { *rc = ss_fail(SS_ERR_INVALID_PARAMETER, "NULL surface"); return nullptr; }
    ss_context *c = s->owner;
    {
        std::lock_guard<std::mutex> lk(g_ctx_mutex);
        if (!c || !g_live_contexts.count(c)) { *rc = ss_fail(SS_ERR_INVALID_PARAMETER, "the context of this surface was destroyed"); return nullptr; }
    }
    if (s->nv >= 0x7fffffffull || s->nt * 6 >= 0x7fffffffull) { *rc = ss_fail(SS_ERR_INDEX_TOO_SMALL, "mesh too large for device post-processing"); return nullptr; }
    if (need_bins && s->nv) {                     // (an empty mesh needs no particle query)
        if (c->post.partitioned) { *rc = ss_fail(SS_ERR_UNSUPPORTED, "particle queries are not available on a partitioned (multi-GPU) surface"); return nullptr; }
        if (!c->post.valid || c->frame != s->frame) {
            *rc = ss_fail(SS_ERR_INVALID_PARAMETER, "the particle bins of this surface are gone: call the post-processing entry before the next reconstruction on its context");
            return nullptr;
        }
    }
    return c;
}
static SsQuery pp_query(const ss_context *c, const ss_surface *s) {
    SsQuery Q{};
    Q.sub_flat = c->sub_flat.as<uint32_t>(); Q.nsub = c->post.nsub;
    Q.bin_start = c->tab_a.as<uint32_t>(); Q.bin_end = c->tab_b.as<uint32_t>(); Q.pidx = c->val_a.as<uint32_t>();
    Q.rec = c->rec.as<float4>(); Q.rho = s->rho.as<float>(); Q.sphere_mass = c->post.sphere_mass;
    return Q;
}

// SphInterpolator::interpolate_scalar_quantity / interpolate_vector_quantity at the mesh vertices (sph_interpolation.rs:141-258;
// pipeline hook reconstruct.rs:1345-1391).  values: [num_particles * dim] (filtered particles, host or device), out: [nv * dim].
extern "C" int ss_surface_interpolate_quantity_f32(ss_surface *s, const float *values, uint32_t dim, int first_order_correction, float *out) {
    int rc; ss_context *c = pp_context(s, true, &rc);
    if (!c) return rc;
    if (!values || !out || (dim != 1 && dim != 3)) return ss_fail(SS_ERR_INVALID_PARAMETER, "values/out must be non-NULL and dim 1 or 3");
    if (!s->nv) return SS_OK;
    return ss_guard([&]() -> int {
        CK(cudaSetDevice(c->device));
        cudaStream_t st = c->stream;
        const uint32_t nv = (uint32_t)s->nv;
        c->post.vals.ensure(std::max<size_t>(s->n, 1) * dim * 4); c->post.out.ensure((size_t)nv * dim * 4);
        CK(cudaMemcpyAsync(c->post.vals.p, values, (size_t)s->n * dim * 4, cudaMemcpyDefault, st));
        const SsQuery Q = pp_query(c, s);
        if (dim == 1) LAUNCH(c, k_pp_interpolate<1>, nblk(nv, 128), 128, c->post.D, Q, s->verts.as<float>(), nv, c->post.vals.as<float>(), first_order_correction, c->post.out.as<float>());
        else LAUNCH(c, k_pp_interpolate<3>, nblk(nv, 128), 128, c->post.D, Q, s->verts.as<float>(), nv, c->post.vals.as<float>(), first_order_correction, c->post.out.as<float>());
        CK(cudaMemcpyAsync(out, c->post.out.p, (size_t)nv * dim * 4, cudaMemcpyDefault, st));
        CK(cudaStreamSynchronize(st));
        return SS_OK;
    });
}

// ------------------------------------------------------------------ SphInterpolator at arbitrary points ----
// splashsurf_lib::sph_interpolation::SphInterpolator (sph_interpolation.rs:22-258; Python class pysplashsurf.SphInterpolator): particles,
// their densities, the rest mass and the compact support radius define the interpolator; quantities and normals are then evaluated at any
// set of points.  The handle is a surface without a mesh whose particle bins live in the context's scratch: like the [bins] entries above it
// has to be used before the next reconstruction (or interpolator) on the same context.
extern "C" int ss_sph_interpolator_create_f32(ss_context *c, const float *xyz, uint64_t n, const float *densities, float particle_rest_mass,
                                              float compact_support_radius, ss_surface **out) {
    if (!c || !out) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL argument");
    *out = nullptr;
    if (n && (!xyz || !densities)) return ss_fail(SS_ERR_INVALID_PARAMETER, "xyz / densities is NULL");
    if (!(compact_support_radius > 0.0f) || !std::isfinite(compact_support_radius)) return ss_fail(SS_ERR_INVALID_PARAMETER, "compact_support_radius must be positive");
    // the bins only have to cover a ball of radius h around any query point: cubes of h / 2, subdomain tiles of 64 cubes
    ss_params_f32 p{};
    p.particle_radius = compact_support_radius * 0.25f; p.rest_density = 1000.0f; p.compact_support_radius = compact_support_radius;
    p.cube_size = compact_support_radius * 0.5f; p.iso_surface_threshold = 0.6f; p.enable_multi_threading = 1; p.enable_simd = 1;
    p.spatial_decomposition = 1; p.subdomain_num_cubes_per_dim = 64; p.auto_disable = 0;
    return with_new_surface(c, out, [&](ss_surface *s) -> int {
        s->n_in = n;
        Prepared P;
        int rc = prepare_particles(c, xyz, n, &p, P, nullptr);
        if (rc) return rc;
        s->n = P.n; s->grid = P.grid; s->used_decomposition = 1;
        Partition opt;
        opt.given_rho = densities; opt.given_mass = particle_rest_mass;
        return run_subdomain_grid(c, P, &p, s, opt, /*global_mode=*/false);
    });
}

__global__ void k_pp_fill(uint32_t n, float value, float *__restrict__ out) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) out[i] = value;
}

// context of an interpolator handle whose bins are still in place (nullptr + error otherwise); *empty: no particle at all
static ss_context *pp_interpolator_context(ss_surface *s, bool *empty, int *rc) {
    *rc = SS_OK; *empty = false;
    if (!s) { *rc = ss_fail(SS_ERR_INVALID_PARAMETER, "NULL interpolator"); return nullptr; }
    ss_context *c = s->owner;
    {
        std::lock_guard<std::mutex> lk(g_ctx_mutex);
        if (!c || !g_live_contexts.count(c)) { *rc = ss_fail(SS_ERR_INVALID_PARAMETER, "the context of this interpolator was destroyed"); return nullptr; }
    }
    if (c->frame != s->frame) {
        *rc = ss_fail(SS_ERR_INVALID_PARAMETER, "the particle bins of this interpolator are gone: use it before the next reconstruction / interpolator on its context");
        return nullptr;
    }
    *empty = !c->post.valid;                         // no particle (or none inside the grid): every sum is empty
    return c;
}

// SphInterpolator::interpolate_scalar_quantity / interpolate_vector_quantity (sph_interpolation.rs:141-258) at `m` points.
// values: [num_particles * dim], points: [m * 3], out: [m * dim]; host or device pointers.
extern "C" int ss_sph_interpolate_quantity_at_f32(ss_surface *s, const float *values, uint32_t dim, const float *points, uint64_t m,
                                                  int first_order_correction, float *out) {
    int rc; bool empty; ss_context *c = pp_interpolator_context(s, &empty, &rc);
    if (!c) return rc;
    if ((dim != 1 && dim != 3) || (m && (!points || !out)) || (s->n && !values)) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL argument or dim not 1 / 3");
    if (m >= 0x7fffffffull) return ss_fail(SS_ERR_INDEX_TOO_SMALL, "too many interpolation points for one call");
    if (!m) return SS_OK;
    return ss_guard([&]() -> int {
        CK(cudaSetDevice(c->device));
        cudaStream_t st = c->stream;
        const uint32_t np = (uint32_t)m;
        c->post.out.ensure((size_t)np * dim * 4);
        if (empty) {
            // no particle at all: every point sees an empty sum, and the reference's correction factor enable * (1 / 0) + (1 - enable) is
            // NaN whether the correction is enabled or not (sph_interpolation.rs:252-254)
            LAUNCH(c, k_pp_fill, nblk((uint64_t)np * dim, 256), 256, np * dim, nanf(""), c->post.out.as<float>());
        } else {
            c->post.vals.ensure(std::max<size_t>(s->n, 1) * dim * 4); c->post.tmpv.ensure((size_t)np * 12);
            CK(cudaMemcpyAsync(c->post.vals.p, values, (size_t)s->n * dim * 4, cudaMemcpyDefault, st));
            CK(cudaMemcpyAsync(c->post.tmpv.p, points, (size_t)np * 12, cudaMemcpyDefault, st));
            const SsQuery Q = pp_query(c, s);
            if (dim == 1) LAUNCH(c, k_pp_interpolate<1>, nblk(np, 128), 128, c->post.D, Q, c->post.tmpv.as<float>(), np, c->post.vals.as<float>(), first_order_correction, c->post.out.as<float>());
            else LAUNCH(c, k_pp_interpolate<3>, nblk(np, 128), 128, c->post.D, Q, c->post.tmpv.as<float>(), np, c->post.vals.as<float>(), first_order_correction, c->post.out.as<float>());
        }
        CK(cudaMemcpyAsync(out, c->post.out.p, (size_t)np * dim * 4, cudaMemcpyDefault, st));
        CK(cudaStreamSynchronize(st));
        return SS_OK;
    });
}

// SphInterpolator::interpolate_normals (sph_interpolation.rs:82-133) at `m` points: normalised SPH gradient of the indicator function
// (NaN where no particle is within the support, like the reference's normalisation of a zero vector).
extern "C" int ss_sph_interpolate_normals_at_f32(ss_surface *s, const float *points, uint64_t m, float *out) {
    int rc; bool empty; ss_context *c = pp_interpolator_context(s, &empty, &rc);
    if (!c) return rc;
    if (m && (!points || !out)) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL argument");
    if (m >= 0x7fffffffull) return ss_fail(SS_ERR_INDEX_TOO_SMALL, "too many interpolation points for one call");
    if (!m) return SS_OK;
    return ss_guard([&]() -> int {
        CK(cudaSetDevice(c->device));
        cudaStream_t st = c->stream;
        const uint32_t np = (uint32_t)m;
        c->post.out.ensure((size_t)np * 12);
        if (empty) LAUNCH(c, k_pp_fill, nblk((uint64_t)np * 3, 256), 256, np * 3, nanf(""), c->post.out.as<float>());
        else {
            c->post.tmpv.ensure((size_t)np * 12);
            CK(cudaMemcpyAsync(c->post.tmpv.p, points, (size_t)np * 12, cudaMemcpyDefault, st));
            LAUNCH(c, k_pp_sph_normals, nblk(np, 128), 128, c->post.D, pp_query(c, s), c->post.tmpv.as<float>(), np, c->post.out.as<float>());
        }
        CK(cudaMemcpyAsync(out, c->post.out.p, (size_t)np * 12, cudaMemcpyDefault, st));
        CK(cudaStreamSynchronize(st));
        return SS_OK;
    });
}

// ------------------------------------------------------------------ stand-alone neighbourhood search ----
// splashsurf_lib::neighborhood_search::neighborhood_search_spatial_hashing_parallel (neighborhood_search.rs:444-588; the Python function of
// the same name): per particle the indices of all other particles with squared distance < search_radius^2.  The global path's cell-list
// stage does the work: cells of `search_radius` on the lattice of UniformGrid::from_aabb(domain, search_radius) (:172-173), 27 cells per
// particle.  The lists come back through ss_surface_num_neighbors / ss_surface_copy_neighbor_lists (order inside a list: cell order, then
// ascending index; the reference's order depends on its hash map).  A particle outside of the domain is an error (reference: panic).
extern "C" int ss_neighborhood_search_f32(ss_context *c, const float *xyz, uint64_t n, const float domain_min[3], const float domain_max[3],
                                          float search_radius, ss_surface **out) {
    if (!c || !out || !domain_min || !domain_max) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL argument");
    *out = nullptr;
    if (n && !xyz) return ss_fail(SS_ERR_INVALID_PARAMETER, "xyz is NULL");
    if (!(search_radius > 0.0f) || !std::isfinite(search_radius)) return ss_fail(SS_ERR_INVALID_PARAMETER, "search radius must be positive (reference: panic)");
    HostGrid ns;
    int rcn = grid_from_aabb(ns, domain_min, domain_max, search_radius);
    if (rcn) return ss_fail(rcn, "failed to construct grid for neighborhood search: degenerate or inconsistent domain (reference: panic)");
    const uint64_t cells = (uint64_t)ns.nc[0] * ns.nc[1] * ns.nc[2];
    if (ns.nc[0] >= (1 << 20) || ns.nc[1] >= (1 << 20) || ns.nc[2] >= (1 << 20) || cells >= (1ull << 28))
        return ss_fail(SS_ERR_INDEX_TOO_SMALL, "domain too large for the cell list of the neighbourhood search");
    ss_params_f32 p{};
    p.particle_radius = search_radius * 0.25f; p.rest_density = 1000.0f; p.compact_support_radius = search_radius; p.cube_size = search_radius;
    p.iso_surface_threshold = 0.6f; p.enable_multi_threading = 1; p.enable_simd = 1;
    ss_grid_f32 g{};                                    // only keeps prepare_particles from reducing a bounding box nobody needs
    for (int d = 0; d < 3; ++d) { g.aabb_min[d] = ns.mn[d]; g.aabb_max[d] = ns.mx[d]; g.points_per_dim[d] = ns.np[d]; g.cells_per_dim[d] = ns.nc[d]; }
    g.cell_size = search_radius;
    return with_new_surface(c, out, [&](ss_surface *s) -> int {
        s->n_in = n;
        Prepared P;
        int rc = prepare_particles(c, xyz, n, &p, P, nullptr, &g);
        if (rc) return rc;
        s->n = P.n; s->grid = ns;
        s->owner = c; c->post.valid = 0; s->frame = ++c->frame;
        cudaStream_t st = c->stream;
        s->rho = std::move(c->o_rho);
        s->rho.ensure(std::max<uint64_t>(n, 1) * 4);
        s->nbr_off.ensure((n + 1) * 8);
        if (n == 0) {
            CK(cudaMemsetAsync(s->nbr_off.p, 0, 8, st));
            CK(cudaStreamSynchronize(st));
            s->has_neighbors = 1; s->n_neighbors = 0;
            return SS_OK;
        }
        SsDev D{};
        D.h = search_radius; D.h2 = fmulr(search_radius, search_radius); D.c = search_radius; D.rest_mass = 1.0f; D.gmode = 1;
        fill_kernel_consts(D, search_radius);
        for (int d = 0; d < 3; ++d) { D.g_ns_amin[d] = ns.mn[d]; D.g_ns_nc[d] = (int)ns.nc[d]; D.gmin[d] = ns.mn[d]; }
        rc = stage_densities(c, D, P.d_xyz, n, 0, 0, cells, /*global_mode=*/true, /*want_nbrs=*/true, s, s->rho.as<float>());
        if (rc) return rc;
        int h_err = 0;
        CK(cudaMemcpyAsync(&h_err, c->err.p, 4, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        if (h_err) return ss_fail(SS_ERR_INVALID_PARAMETER, "particle outside of the domain of the neighbourhood search (reference: panic)");
        return SS_OK;
    });
}

// ------------------------------------------------------------------ marching cubes on caller-supplied level-set tiles ----
// marching_cubes::triangulate_density_map (marching_cubes.rs:61-127 with narrow_band_extraction.rs / triangulation.rs; the Python function
// pysplashsurf.marching_cubes on a dense array): the global path's marching-cubes kernels on level-set values the caller provides.
// The values come as tiles of 65^3 points (64^3 cells; neighbouring tiles share their face planes), tile t covering the global points
// tile_ijk[t] * 64 .. + 64 per axis -- the layout the level-set stage produces.  Vertices are welded across tiles by their global edge
// key (ss_surface_copy_vertex_edge_keys).  Cells beyond the caller's array have to be padded by the caller (the Python front end repeats
// the border values and drops the triangles of the padded cells afterwards).
extern "C" int ss_marching_cubes_tiles_f32(ss_context *c, const float *tiles, uint32_t ntiles, const int32_t *tile_ijk, const float grid_min[3],
                                           float cube_size, float iso_surface_threshold, ss_surface **out) {
    if (!c || !out || !grid_min) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL argument");
    *out = nullptr;
    if (ntiles && (!tiles || !tile_ijk)) return ss_fail(SS_ERR_INVALID_PARAMETER, "tiles / tile_ijk is NULL");
    if (!(cube_size > 0.0f) || !std::isfinite(cube_size)) return ss_fail(SS_ERR_INVALID_CELL_SIZE, "cube size must be positive");
    SsDev D{};
    D.S = 64; D.np = 65; D.np_magic = (uint32_t)(4294967296ull / (uint64_t)D.np) + 1u;
    D.c = cube_size; D.thr = iso_surface_threshold; D.gmode = 1; D.R = 1; D.simd = 1;
    D.sub_size = fmulr(cube_size, 64.0f);
    for (int d = 0; d < 3; ++d) { D.gmin[d] = grid_min[d]; D.nsd[d] = 1; }
    fill_bins(D, cube_size);
    const size_t np3 = (size_t)D.np * D.np * D.np;
    const uint64_t nbricks = (uint64_t)D.nb * D.nb * D.nb;
    if ((uint64_t)ntiles * nbricks >= 0x7fffffffull) return ss_fail(SS_ERR_INDEX_TOO_SMALL, "too many tiles for one call");
    std::vector<SsTile> h_tiles(ntiles);
    for (uint32_t t = 0; t < ntiles; ++t) {
        int64_t ijk[3];
        for (int d = 0; d < 3; ++d) {
            ijk[d] = tile_ijk[3 * (size_t)t + d];
            if (ijk[d] < 0 || ijk[d] * 64 + 64 >= (1 << 20)) return ss_fail(SS_ERR_INDEX_TOO_SMALL, "tile index out of range (2^20 grid points per dimension)");
        }
        h_tiles[t] = make_tile(ijk, 64, grid_min, D.sub_size, t, true);
    }
    return with_new_surface(c, out, [&](ss_surface *s) -> int {
        cudaStream_t st = c->stream;
        s->owner = c; s->S = 64;
        c->post.valid = 0; s->frame = ++c->frame;
        for (int d = 0; d < 3; ++d) { s->grid.mn[d] = s->grid.mx[d] = grid_min[d]; s->grid.np[d] = s->grid.nc[d] = 0; }
        s->grid.cell = cube_size;
        s->verts = std::move(c->o_verts); s->tris = std::move(c->o_tris); s->vkeys = std::move(c->o_vkeys);
        s->verts.ensure(1 << 16); s->vkeys.ensure(1 << 16); s->tris.ensure(1 << 16);
        uint64_t vtotal = 0, ttotal = 0, nv_final = 0;
        uint32_t bc = 0;
        if (ntiles) {
            const uint32_t n_mc = (uint32_t)(ntiles * nbricks);
            c->tiles.ensure((size_t)ntiles * np3 * 4); c->voff.ensure((size_t)ntiles * np3 * 4); c->vmask.ensure((size_t)ntiles * np3);
            c->vcnt.ensure((size_t)n_mc * 4 + 4); c->tcnt.ensure((size_t)n_mc * 4 + 4); c->vblk_off.ensure((size_t)n_mc * 4 + 4); c->tblk_off.ensure((size_t)n_mc * 4 + 4);
            c->tile_tab.ensure((size_t)ntiles * sizeof(SsTile)); c->list_mc.ensure((size_t)n_mc * 4); c->bcount.ensure(4);
            c->bkeys_a.ensure(1 << 16); c->bids_a.ensure(1 << 16);
            CK(cudaMemcpyAsync(c->tiles.p, tiles, (size_t)ntiles * np3 * 4, cudaMemcpyDefault, st));
            CK(cudaMemcpyAsync(c->tile_tab.p, h_tiles.data(), (size_t)ntiles * sizeof(SsTile), cudaMemcpyHostToDevice, st));
            CK(cudaMemsetAsync(c->vmask.p, 0, (size_t)ntiles * np3, st));
            CK(cudaMemsetAsync(c->bcount.p, 0, 4, st));
            LAUNCH(c, k_iota2, nblk(n_mc, 256), 256, n_mc, c->list_mc.as<uint32_t>(), c->vcnt.as<uint32_t>());      // every brick of every tile
            CK(cudaStreamSynchronize(st));                                                                          // h_tiles is read by the copy above
            int rc = marching_cubes_batch(c, D, /*global_mode=*/true, n_mc, s, vtotal, ttotal);
            if (rc) return rc;
            nv_final = vtotal;
            rc = weld_boundary_vertices(c, s, vtotal, ttotal, nv_final, bc);
            if (rc) return rc;
        }
        s->nv = nv_final; s->nt = ttotal;
        CK(cudaStreamSynchronize(st));
        return SS_OK;
    });
}

// Smoothing weights of the mesh vertices (reconstruct.rs:1159-1258): distance-weighted neighbour count per particle,
// SPH-interpolated (with correction) to the vertices, normalised and passed through the smooth-step.  The weights stay on
// the device for ss_surface_laplacian_smoothing_f32; wnn_out / weights_out ([nv], optional) receive copies
// (the "wnn" and "sw" attributes of the reference).
extern "C" int ss_surface_compute_smoothing_weights_f32(ss_surface *s, float normalization, float *wnn_out, float *weights_out) {
    int rc; ss_context *c = pp_context(s, true, &rc);
    if (!c) return rc;
    if (!s->nv) return SS_OK;
    return ss_guard([&]() -> int {
        CK(cudaSetDevice(c->device));
        cudaStream_t st = c->stream;
        const uint32_t nv = (uint32_t)s->nv;
        const SsQuery Q = pp_query(c, s);
        c->post.vals.ensure(std::max<size_t>(s->n, 1) * 4); c->post.out.ensure((size_t)nv * 4); s->weights.ensure((size_t)nv * 4);
        CK(cudaMemsetAsync(c->post.vals.p, 0, std::max<size_t>(s->n, 1) * 4, st));
        LAUNCH(c, k_pp_weighted_ncount, nblk(c->post.M, 128), 128, c->post.D, Q, c->key_b.as<uint32_t>(), c->post.M, c->post.vals.as<float>());
        LAUNCH(c, k_pp_interpolate<1>, nblk(nv, 128), 128, c->post.D, Q, s->verts.as<float>(), nv, c->post.vals.as<float>(), 1, c->post.out.as<float>());
        LAUNCH(c, k_pp_smoothstep, nblk(nv, 256), 256, nv, c->post.out.as<float>(), normalization, s->weights.as<float>());
        if (wnn_out) CK(cudaMemcpyAsync(wnn_out, c->post.out.p, (size_t)nv * 4, cudaMemcpyDefault, st));
        if (weights_out) CK(cudaMemcpyAsync(weights_out, s->weights.p, (size_t)nv * 4, cudaMemcpyDefault, st));
        CK(cudaStreamSynchronize(st));
        s->has_weights = 1;
        return SS_OK;
    });
}

// par_laplacian_smoothing_inplace (postprocessing.rs:17-53) on the surface's vertices.  weights: [nv] host or device; NULL
// selects the weights of ss_surface_compute_smoothing_weights_f32 if it ran on this surface, otherwise 1 for every vertex.
extern "C" int ss_surface_laplacian_smoothing_f32(ss_surface *s, uint32_t iterations, float beta, const float *weights) {
    int rc; ss_context *c = pp_context(s, false, &rc);
    if (!c) return rc;
    if (!s->nv || !iterations) return SS_OK;
    return ss_guard([&]() -> int {
        CK(cudaSetDevice(c->device));
        cudaStream_t st = c->stream;
        const uint32_t nv = (uint32_t)s->nv;
        pp_vertex_adjacency(c, s);
        const float *d_w = s->has_weights ? s->weights.as<float>() : nullptr;
        if (weights) {
            c->post.out.ensure((size_t)nv * 4);
            CK(cudaMemcpyAsync(c->post.out.p, weights, (size_t)nv * 4, cudaMemcpyDefault, st));
            d_w = c->post.out.as<float>();
        }
        c->post.tmpv.ensure((size_t)nv * 12);
        CK(cudaMemcpyAsync(c->post.tmpv.p, s->verts.p, (size_t)nv * 12, cudaMemcpyDeviceToDevice, st));   // vertex_buffer = vertices.clone()
        float *cur = s->verts.as<float>(), *buf = c->post.tmpv.as<float>();
        for (uint32_t it = 0; it < iterations; ++it) {
            std::swap(cur, buf);                                                                          // postprocessing.rs:31
            LAUNCH(c, k_pp_laplacian, nblk(nv, 256), 256, nv, cur, (const float *)buf, s->adj_row.as<uint32_t>(), s->adj_idx.as<uint32_t>(), d_w, beta);
        }
        if (cur != s->verts.as<float>()) CK(cudaMemcpyAsync(s->verts.p, cur, (size_t)nv * 12, cudaMemcpyDeviceToDevice, st));
        CK(cudaStreamSynchronize(st));
        return SS_OK;
    });
}

// Vertex normals at the surface's current (possibly smoothed) vertices, stored as the surface's normals:
// sph != 0: SphInterpolator::interpolate_normals (sph_interpolation.rs:82-133), else area-weighted triangle normals
// (mesh.rs:799-906).
extern "C" int ss_surface_compute_normals_f32(ss_surface *s, int sph) {
    int rc; ss_context *c = pp_context(s, sph != 0, &rc);
    if (!c) return rc;
    if (!s->nv) return SS_OK;
    return ss_guard([&]() -> int {
        CK(cudaSetDevice(c->device));
        cudaStream_t st = c->stream;
        const uint32_t nv = (uint32_t)s->nv;
        s->normals.ensure((size_t)nv * 12);
        if (sph) {
            LAUNCH(c, k_pp_sph_normals, nblk(nv, 128), 128, c->post.D, pp_query(c, s), s->verts.as<float>(), nv, s->normals.as<float>());
        } else {
            pp_vertex_triangles(c, s);
            LAUNCH(c, k_pp_area_normals, nblk(nv, 256), 256, nv, s->verts.as<float>(), s->tris.as<uint32_t>(), s->inc_row.as<uint32_t>(),
                   s->inc_idx.as<uint32_t>(), s->normals.as<float>());
        }
        CK(cudaStreamSynchronize(st));
        s->has_normals = 1;
        return SS_OK;
    });
}

// par_laplacian_smoothing_normals_inplace (postprocessing.rs:56-97) on the surface's normals.
extern "C" int ss_surface_smooth_normals_f32(ss_surface *s, uint32_t iterations) {
    int rc; ss_context *c = pp_context(s, false, &rc);
    if (!c) return rc;
    if (!s->has_normals) return ss_fail(SS_ERR_INVALID_PARAMETER, "the surface has no normals to smooth");
    if (!s->nv || !iterations) return SS_OK;
    return ss_guard([&]() -> int {
        CK(cudaSetDevice(c->device));
        cudaStream_t st = c->stream;
        const uint32_t nv = (uint32_t)s->nv;
        pp_vertex_adjacency(c, s);
        c->post.tmpv.ensure((size_t)nv * 12);
        float *a = s->normals.as<float>(), *b = c->post.tmpv.as<float>();
        for (uint32_t it = 0; it < iterations; ++it) {
            LAUNCH(c, k_pp_smooth_normals, nblk(nv, 256), 256, nv, (const float *)a, b, s->adj_row.as<uint32_t>(), s->adj_idx.as<uint32_t>());
            std::swap(a, b);
        }
        if (a != s->normals.as<float>()) CK(cudaMemcpyAsync(s->normals.p, a, (size_t)nv * 12, cudaMemcpyDeviceToDevice, st));
        CK(cudaStreamSynchronize(st));
        return SS_OK;
    });
}

// Wraps a caller-supplied triangle mesh (host or device pointers: verts nv x 3 f32, tris nt x 3 u32) in a surface so that the
// mesh-only entries above (ss_surface_laplacian_smoothing_f32 with explicit or unit weights, ss_surface_compute_normals_f32 with
// sph = 0, ss_surface_smooth_normals_f32, ss_surface_vertex_connectivity) serve the reference's free functions
// par_laplacian_smoothing_inplace / par_laplacian_smoothing_normals_inplace / par_vertex_normals / vertex_vertex_connectivity
// on any mesh.  There are no particles behind such a surface: the [bins] entries fail with SS_ERR_INVALID_PARAMETER.
extern "C" int ss_surface_from_mesh_f32(ss_context *c, const float *verts, uint64_t nv, const uint32_t *tris, uint64_t nt, ss_surface **out) {
    if (!c || !out || (nv && !verts) || (nt && !tris)) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL argument");
    *out = nullptr;
    if (nv >= 0x7fffffffull || nt * 6 >= 0x7fffffffull) return ss_fail(SS_ERR_INDEX_TOO_SMALL, "mesh too large for device post-processing");
    return with_new_surface(c, out, [&](ss_surface *s) -> int {
        cudaStream_t st = c->stream;
        s->owner = c; s->nv = nv; s->nt = nt; s->frame = 0;       // frame 0 never matches a reconstruction
        s->verts.ensure(std::max<uint64_t>(nv, 1) * 12); s->tris.ensure(std::max<uint64_t>(nt, 1) * 12);
        if (nv) CK(cudaMemcpyAsync(s->verts.p, verts, nv * 12, cudaMemcpyDefault, st));
        if (nt) CK(cudaMemcpyAsync(s->tris.p, tris, nt * 12, cudaMemcpyDefault, st));
        CK(cudaStreamSynchronize(st));
        return SS_OK;
    });
}

// Replaces the mesh of a surface (host or device arrays), e.g. after the host-side clean-up / decimation of SURVEY 8(f.4), and keeps
// the surface's link to its reconstruction: the SPH-based entries (smoothing weights, SPH normals, attribute interpolation) keep
// working on the new vertices.  Cached adjacency, weights and normals are dropped; the marching-cubes edge keys no longer apply.
extern "C" int ss_surface_replace_mesh_f32(ss_surface *s, const float *verts, uint64_t nv, const uint32_t *tris, uint64_t nt) {
    int rc; ss_context *c = pp_context(s, false, &rc);
    if (!c) return rc;
    if ((nv && !verts) || (nt && !tris)) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL argument");
    if (nv >= 0x7fffffffull || nt * 6 >= 0x7fffffffull) return ss_fail(SS_ERR_INDEX_TOO_SMALL, "mesh too large for device post-processing");
    return ss_guard([&]() -> int {
        CK(cudaSetDevice(c->device));
        cudaStream_t st = c->stream;
        s->verts.ensure(std::max<uint64_t>(nv, 1) * 12); s->tris.ensure(std::max<uint64_t>(nt, 1) * 12);
        if (nv) CK(cudaMemcpyAsync(s->verts.p, verts, nv * 12, cudaMemcpyDefault, st));
        if (nt) CK(cudaMemcpyAsync(s->tris.p, tris, nt * 12, cudaMemcpyDefault, st));
        CK(cudaStreamSynchronize(st));
        s->nv = nv; s->nt = nt;
        s->has_adj = s->has_inc = s->has_weights = s->has_normals = 0;
        s->vkeys.release();
        return SS_OK;
    });
}

// Replaces the surface's normals by caller-supplied ones ([nv * 3], host or device), e.g. to smooth an arbitrary normal field
// with ss_surface_smooth_normals_f32.
extern "C" int ss_surface_set_normals_f32(ss_surface *s, const float *normals) {
    int rc; ss_context *c = pp_context(s, false, &rc);
    if (!c) return rc;
    if (!normals && s->nv) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL argument");
    return ss_guard([&]() -> int {
        CK(cudaSetDevice(c->device));
        s->normals.ensure(std::max<uint64_t>(s->nv, 1) * 12);
        if (s->nv) CK(cudaMemcpyAsync(s->normals.p, normals, s->nv * 12, cudaMemcpyDefault, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        s->has_normals = 1;
        return SS_OK;
    });
}

// Vertex -> vertex connectivity of the mesh as CSR (TriMesh3d::vertex_vertex_connectivity, mesh.rs:290-306; neighbours in
// ascending order).  offsets: [nv + 1] u64, indices: [offsets[nv]] u32; pass indices = NULL to query the size first.
extern "C" int ss_surface_vertex_connectivity(ss_surface *s, uint64_t *offsets, uint32_t *indices, uint64_t *n_indices) {
    int rc; ss_context *c = pp_context(s, false, &rc);
    if (!c) return rc;
    if (!n_indices) return ss_fail(SS_ERR_INVALID_PARAMETER, "NULL argument");
    *n_indices = 0;
    if (!s->nv) { if (offsets) offsets[0] = 0; return SS_OK; }
    return ss_guard([&]() -> int {
        CK(cudaSetDevice(c->device));
        pp_vertex_adjacency(c, s);
        std::vector<uint32_t> row(s->nv + 1);
        CK(cudaMemcpy(row.data(), s->adj_row.p, (s->nv + 1) * 4, cudaMemcpyDeviceToHost));
        *n_indices = row[s->nv];
        if (offsets) for (uint64_t i = 0; i <= s->nv; ++i) offsets[i] = row[i];
        if (indices && row[s->nv]) CK(cudaMemcpy(indices, s->adj_idx.p, (size_t)row[s->nv] * 4, cudaMemcpyDeviceToHost));
        return SS_OK;
    });
}
#endif  // SS_POST_KERNELS_ONLY
