"""CPU oracle for the splashsurf reconstruct hot path -- TEST INFRASTRUCTURE ONLY.

Two checkers live here:

* ``liboracle.so`` (``splashsurf_oracle.c``): a plain-C restatement of the reference's f32/i64
  subdomain-grid pipeline with stage-level taps (densities, level-set tiles, vertex edge keys).
* ``reference()``: the reference's own prebuilt binary (pysplashsurf 0.14.0 wheel unpacked into
  ``oracle/_ref`` by ``oracle/build_ref.sh``), used to pin the restatement and as CPU baseline.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline / ``--impl reference`` legs
may import this package.  The product (``splashsurf_b200``) never does.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import sys

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None


class _Params(C.Structure):
    _fields_ = [
        ("particle_radius", C.c_float), ("rest_density", C.c_float), ("compact_support_radius", C.c_float),
        ("cube_size", C.c_float), ("iso_surface_threshold", C.c_float),
        ("has_particle_aabb", C.c_int32), ("aabb_min", C.c_float * 3), ("aabb_max", C.c_float * 3),
        ("enable_simd", C.c_int32), ("decomposition", C.c_int32),
        ("subdomain_num_cubes_per_dim", C.c_uint32), ("auto_disable", C.c_int32),
    ]


class _Grid(C.Structure):
    _fields_ = [("aabb_min", C.c_float * 3), ("aabb_max", C.c_float * 3), ("cell_size", C.c_float),
                ("np", C.c_int64 * 3), ("nc", C.c_int64 * 3)]


class _Result(C.Structure):
    _fields_ = [
        ("grid", _Grid), ("subdomain_grid", _Grid), ("used_decomposition", C.c_int32),
        ("n_filtered", C.c_uint64), ("inside_aabb", C.POINTER(C.c_uint8)), ("densities", C.POINTER(C.c_float)),
        ("nv", C.c_uint64), ("nt", C.c_uint64), ("vertices", C.POINTER(C.c_float)),
        ("triangles", C.POINTER(C.c_uint64)), ("vertex_keys", C.POINTER(C.c_int64)),
        ("n_subdomains", C.c_uint64), ("subdomain_flat", C.POINTER(C.c_int64)),
        ("subdomain_count", C.POINTER(C.c_uint64)), ("subdomain_sparse", C.POINTER(C.c_uint8)),
        ("max_particles", C.c_uint64), ("sparse_limit", C.c_uint64),
    ]


def build(force: bool = False) -> str:
    """Compile liboracle.so (gcc) and, when /root/reference is present, unpack oracle/_ref."""
    so = os.path.join(_HERE, "liboracle.so")
    src = os.path.join(_HERE, "splashsurf_oracle.c")
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "-B", "liboracle.so"], stdout=subprocess.DEVNULL)
    subprocess.call(["sh", os.path.join(_HERE, "build_ref.sh")])
    return so


def lib():
    global _LIB
    if _LIB is None:
        so = os.path.join(_HERE, "liboracle.so")
        if not os.path.exists(so):
            build()
        L = C.CDLL(so)
        L.so_reconstruct.restype = C.c_int
        L.so_reconstruct.argtypes = [C.c_void_p, C.c_uint64, C.POINTER(_Params), C.POINTER(C.POINTER(_Result)),
                                     C.c_int64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.so_free.argtypes = [C.POINTER(_Result)]
        L.so_levelset_tile.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint64, C.c_void_p, C.c_float,
                                       C.c_void_p, C.c_int64, C.c_void_p, C.c_float, C.c_float, C.c_int]
        L.so_kernel_scalar.restype = C.c_float
        L.so_kernel_scalar.argtypes = [C.c_float, C.c_float]
        L.so_kernel_avx.restype = C.c_float
        L.so_kernel_avx.argtypes = [C.c_float, C.c_float]
        L.so_sph_normals.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_float, C.c_float, C.c_void_p, C.c_uint64, C.c_void_p]
        L.so_num_threads.restype = C.c_int
        L.so_set_num_threads.argtypes = [C.c_int]
        _LIB = L
    return _LIB


def _grid_dict(g: _Grid) -> dict:
    return {"aabb_min": np.array(g.aabb_min, dtype=np.float32), "aabb_max": np.array(g.aabb_max, dtype=np.float32),
            "cell_size": np.float32(g.cell_size), "npoints": np.array(getattr(g, "np"), dtype=np.int64),
            "ncells": np.array(g.nc, dtype=np.int64)}


def absolute_params(particle_radius, smoothing_length, cube_size):
    """Front-end parameter mapping: pysplashsurf/src/reconstruction.rs:172-176 (f64 products, then f32)."""
    r = float(particle_radius)
    return np.float32(r), np.float32(2.0 * float(smoothing_length) * r), np.float32(float(cube_size) * r)


def reconstruct(particles, *, particle_radius, smoothing_length, cube_size, rest_density=1000.0,
                iso_surface_threshold=0.6, aabb_min=None, aabb_max=None, simd=True, subdomain_grid=True,
                subdomain_grid_auto_disable=True, subdomain_num_cubes_per_dim=64, multi_threading=True, tile_of_subdomain=None,
                want_neighbor_counts=False, want_neighbors=False, num_threads=None):
    """C-oracle counterpart of pysplashsurf.reconstruct_surface (same RELATIVE smoothing_length / cube_size).
    `tile_of_subdomain`: flat index of a tile whose level-set values are returned as d["tile"]: (S + 1)^3 on the subdomain path,
    65^3 on the global path (its grid cut into 64-cube tiles, as the device tiles it).
    `multi_threading` is accepted and ignored: the global path is restated with its sequential (deterministic) semantics."""
    L = lib()
    if num_threads is not None:
        L.so_set_num_threads(int(num_threads))
    xyz = np.ascontiguousarray(particles, dtype=np.float32).reshape(-1, 3)
    r, h, c = absolute_params(particle_radius, smoothing_length, cube_size)
    p = _Params()
    p.particle_radius, p.rest_density, p.compact_support_radius = float(r), float(np.float32(rest_density)), float(h)
    p.cube_size, p.iso_surface_threshold = float(c), float(np.float32(iso_surface_threshold))
    p.has_particle_aabb = int(aabb_min is not None and aabb_max is not None)
    if p.has_particle_aabb:
        p.aabb_min = (C.c_float * 3)(*[float(np.float32(v)) for v in aabb_min])
        p.aabb_max = (C.c_float * 3)(*[float(np.float32(v)) for v in aabb_max])
    p.enable_simd, p.decomposition = int(simd), int(subdomain_grid)
    p.subdomain_num_cubes_per_dim, p.auto_disable = int(subdomain_num_cubes_per_dim), int(subdomain_grid_auto_disable)
    S = int(subdomain_num_cubes_per_dim)
    # the subdomain path writes (S + 1)^3 floats, the global path the 65^3 points of a 64-cube tile of its grid (whatever S is):
    # room for both, shaped below by the path taken
    tmax = max(S, 64) + 1
    tile = np.zeros(tmax ** 3, dtype=np.float32) if tile_of_subdomain is not None else None
    ncnt = np.zeros(len(xyz), dtype=np.int64) if (want_neighbor_counts or want_neighbors) else None
    out = C.POINTER(_Result)()
    rc = L.so_reconstruct(xyz.ctypes.data, len(xyz), C.byref(p), C.byref(out),
                          -1 if tile_of_subdomain is None else int(tile_of_subdomain),
                          None if tile is None else tile.ctypes.data, None if ncnt is None else ncnt.ctypes.data, None, None)
    nbr = None
    if want_neighbors and rc == 0 and not p.has_particle_aabb:
        # second pass: fill the CSR lists with the offsets from the counts of the first pass
        L.so_free(out)
        off = np.concatenate([[0], np.cumsum(ncnt)]).astype(np.int64)
        idx = np.zeros(max(int(off[-1]), 1), dtype=np.int64)
        out = C.POINTER(_Result)()
        rc = L.so_reconstruct(xyz.ctypes.data, len(xyz), C.byref(p), C.byref(out), -1, None, ncnt.ctypes.data, off.ctypes.data, idx.ctypes.data)
        nbr = (off, idx[:int(off[-1])])
    try:
        res = out.contents
        d = {"rc": rc, "grid": _grid_dict(res.grid), "used_decomposition": bool(res.used_decomposition)}
        if rc != 0:
            return d
        n = res.n_filtered
        d["subdomain_grid"] = _grid_dict(res.subdomain_grid) if res.used_decomposition else None
        d["particle_densities"] = np.ctypeslib.as_array(res.densities, (n,)).copy() if n else np.zeros(0, np.float32)
        d["particle_inside_aabb"] = (np.ctypeslib.as_array(res.inside_aabb, (len(xyz),)).astype(bool).copy()
                                     if p.has_particle_aabb else None)
        nv, nt, ns = res.nv, res.nt, res.n_subdomains
        d["vertices"] = np.ctypeslib.as_array(res.vertices, (nv, 3)).copy() if nv else np.zeros((0, 3), np.float32)
        d["triangles"] = np.ctypeslib.as_array(res.triangles, (nt, 3)).copy() if nt else np.zeros((0, 3), np.uint64)
        d["vertex_keys"] = np.ctypeslib.as_array(res.vertex_keys, (nv, 4)).copy() if nv else np.zeros((0, 4), np.int64)
        d["subdomain_flat"] = np.ctypeslib.as_array(res.subdomain_flat, (ns,)).copy() if ns else np.zeros(0, np.int64)
        d["subdomain_count"] = np.ctypeslib.as_array(res.subdomain_count, (ns,)).copy() if ns else np.zeros(0, np.uint64)
        d["subdomain_sparse"] = np.ctypeslib.as_array(res.subdomain_sparse, (ns,)).astype(bool).copy() if ns else np.zeros(0, bool)
        d["max_particles"], d["sparse_limit"] = int(res.max_particles), int(res.sparse_limit)
        if tile is not None:
            tn = S + 1 if res.used_decomposition else 65
            tile = tile[:tn ** 3].reshape((tn,) * 3)
        d["tile"], d["neighbor_counts"], d["neighbors"] = tile, ncnt, nbr
        return d
    finally:
        L.so_free(out)


def levelset_tile(xyz, rho, *, global_min, cube_size, subdomain_ijk, subdomain_cubes, subdomain_min, h, rest_mass, mode):
    """One subdomain's level-set tile (mode 0: AVX2-FMA semantics, 1: scalar)."""
    L = lib()
    xyz = np.ascontiguousarray(xyz, dtype=np.float32)
    rho = np.ascontiguousarray(rho, dtype=np.float32)
    S = int(subdomain_cubes)
    phi = np.zeros((S + 1,) * 3, dtype=np.float32)
    gmin = np.ascontiguousarray(global_min, dtype=np.float32)
    smin = np.ascontiguousarray(subdomain_min, dtype=np.float32)
    sijk = np.ascontiguousarray(subdomain_ijk, dtype=np.int64)
    L.so_levelset_tile(phi.ctypes.data, xyz.ctypes.data, rho.ctypes.data, len(xyz), gmin.ctypes.data,
                       C.c_float(float(cube_size)), sijk.ctypes.data, S, smin.ctypes.data, C.c_float(float(h)),
                       C.c_float(float(rest_mass)), int(mode))
    return phi


def sph_rest_mass(particle_radius, rest_density=1000.0):
    """Sphere rest mass used by the pipeline's SPH interpolator (splashsurf/src/reconstruct.rs:1126-1129), f32."""
    r = np.float32(particle_radius)
    vol = np.float32(np.float32(4.0) * np.float32(np.pi / 3.0)) * np.float32(r * r * r)
    return np.float32(vol * np.float32(rest_density))


def sph_normals(particles, densities, points, *, compact_support_radius, particle_rest_mass):
    """SphInterpolator.interpolate_normals restated (summation order differs from the reference's R-tree order)."""
    L = lib()
    xyz = np.ascontiguousarray(particles, dtype=np.float32).reshape(-1, 3)
    rho = np.ascontiguousarray(densities, dtype=np.float32)
    pts = np.ascontiguousarray(points, dtype=np.float32).reshape(-1, 3)
    out = np.empty_like(pts)
    L.so_sph_normals(xyz.ctypes.data, rho.ctypes.data, len(xyz), C.c_float(float(np.float32(compact_support_radius))),
                     C.c_float(float(np.float32(particle_rest_mass))), pts.ctypes.data, len(pts), out.ctypes.data)
    return out


def num_threads() -> int:
    return int(lib().so_num_threads())


# ------------------------------------------------------------------ reference binary ----
def reference_available() -> bool:
    return os.path.exists(os.path.join(_HERE, "_ref", "pysplashsurf", "pysplashsurf.abi3.so"))


def reference():
    """Import the reference's own prebuilt pysplashsurf (oracle/_ref)."""
    if not reference_available():
        raise RuntimeError("oracle/_ref is missing: run `make -C oracle ref` where /root/reference exists")
    ref = os.path.join(_HERE, "_ref")
    if ref not in sys.path:
        sys.path.insert(0, ref)
    import pysplashsurf  # noqa: E402
    return pysplashsurf


# ------------------------------------------------------------------ canonical ordering ----
def edge_keys_from_positions(vertices, grid_min, cell_size):
    """Recover the MC grid edge (i, j, k, axis) that carries each vertex from its position (SURVEY.md 8c).

    Every marching-cubes vertex lies on exactly one grid edge: two coordinates are lattice values, the third is
    strictly between two lattice planes.  Done in float64 on the f32 inputs.
    """
    v = np.asarray(vertices, dtype=np.float64)
    q = (v - np.asarray(grid_min, dtype=np.float64)[None]) / float(cell_size)
    frac = np.abs(q - np.rint(q))
    axis = frac.argmax(1)
    ijk = np.rint(q).astype(np.int64)
    rows = np.arange(len(v))
    ijk[rows, axis] = np.floor(q[rows, axis]).astype(np.int64)
    return np.concatenate([ijk, axis[:, None].astype(np.int64)], axis=1)


def canonicalize(vertices, triangles, keys):
    """Sort vertices by edge key, remap triangles, rotate each to start at its min index, lexsort triangles."""
    keys = np.asarray(keys, dtype=np.int64)
    order = np.lexsort((keys[:, 3], keys[:, 2], keys[:, 1], keys[:, 0]))
    inv = np.empty(len(order), dtype=np.int64)
    inv[order] = np.arange(len(order))
    v = np.asarray(vertices)[order]
    k = keys[order]
    t = inv[np.asarray(triangles).astype(np.int64)]
    if len(t):
        m = t.argmin(1)
        t = np.stack([np.take_along_axis(t, ((m + s) % 3)[:, None], 1)[:, 0] for s in range(3)], axis=1)
        t = t[np.lexsort((t[:, 2], t[:, 1], t[:, 0]))]
    return v, t, k


def resolve_keys(vertices, grid_min, cell_size, known_keys, triangles=None, known_triangles=None, known_vertices=None):
    """Edge keys for a mesh whose keys are unknown (the reference binary's output), disambiguated with a
    trusted mesh (keys + triangles).

    With `known_vertices` (the trusted mesh's positions), a vertex whose f32 bits equal those of exactly one trusted vertex
    takes that vertex's key first.  Far from the origin a vertex close to a lattice point lies within the coordinates'
    rounding of it, so its position alone no longer tells its edge (two vertices near one lattice point come out swapped).

    A vertex with interpolation weight ~0 or ~1 sits on a lattice point, where `edge_keys_from_positions`
    cannot tell which of the six incident edges carries it (several such vertices usually share the point).
    Vertices whose inferred key is not in `known_keys` (or collides) are grouped by lattice point; every
    assignment of the free incident edges to the group is tried and the one under which most of the group's
    triangles also occur in `known_triangles` wins.  Unambiguous vertices are never touched.
    """
    import itertools
    keys = edge_keys_from_positions(vertices, grid_min, cell_size)
    known_keys = np.asarray(known_keys, dtype=np.int64)
    known = {tuple(k): i for i, k in enumerate(known_keys.tolist())}
    used = {}
    pending = []
    exact = set()
    if known_vertices is not None:
        by_bits = {}
        for j, b in enumerate(map(tuple, np.ascontiguousarray(known_vertices, dtype=np.float32).view(np.uint32).tolist())):
            by_bits.setdefault(b, []).append(j)
        for i, b in enumerate(map(tuple, np.ascontiguousarray(vertices, dtype=np.float32).view(np.uint32).tolist())):
            js = by_bits.get(b, [])
            k = tuple(known_keys[js[0]].tolist()) if len(js) == 1 else None
            if k is not None and k not in used:
                keys[i] = k; used[k] = i; exact.add(i)
    for i, k in enumerate(map(tuple, keys.tolist())):
        if i in exact:
            continue
        if k in known and k not in used:
            used[k] = i
        else:
            pending.append(i)
    if not pending:
        return keys
    v = np.asarray(vertices, dtype=np.float64)
    q = (v - np.asarray(grid_min, dtype=np.float64)[None]) / float(cell_size)
    # "on a lattice point": within 1e-3 cells, or within the f32 rounding of the coordinates where that is coarser
    near = max(1e-3, 4.0 * float(np.spacing(np.float32(np.abs(v).max()))) / float(cell_size)) if len(v) else 1e-3
    groups = {}
    for i in pending:
        groups.setdefault(tuple(np.rint(q[i]).astype(np.int64).tolist()), []).append(i)
    tri = None if triangles is None else np.asarray(triangles).astype(np.int64)
    ktri = None if known_triangles is None else np.asarray(known_triangles).astype(np.int64)

    def rot(t):
        m = min(range(3), key=lambda a: t[a])
        return (t[m], t[(m + 1) % 3], t[(m + 2) % 3])

    for P, members in groups.items():
        # a vertex already matched unambiguously may also sit at P with a swapped key: release those too
        cands = []
        for a in range(3):
            for off in (0, -1):
                k = list(P); k[a] += off
                cands.append((k[0], k[1], k[2], a))
        for k in cands:
            if k in used and used[k] not in members and used[k] not in exact:
                qi = q[used[k]]
                if np.abs(qi - np.rint(qi)).max() < near:
                    members.append(used.pop(k))
        free = [k for k in cands if k in known and k not in used]
        if len(free) < len(members):
            continue
        if tri is None or ktri is None or len(members) > 6:
            for i, k in zip(members, free):
                keys[i] = k; used[k] = i
            continue
        mset = set(members)
        tsel = tri[np.isin(tri, members).any(1)]
        kv = [known[k] for k in free]
        ksel = ktri[np.isin(ktri, kv).any(1)]
        kset = {rot(tuple(tuple(known_keys[a].tolist()) for a in t)) for t in ksel.tolist()}
        best, best_score = None, -1
        for perm in itertools.permutations(free, len(members)):
            assign = dict(zip(members, perm))
            score = 0
            for t in tsel.tolist():
                tk = rot(tuple(assign[a] if a in mset else tuple(keys[a].tolist()) for a in t))
                score += tk in kset
            if score > best_score:
                best, best_score = assign, score
        for i, k in best.items():
            keys[i] = k; used[k] = i
    return keys


def mesh_parity(vertices_a, triangles_a, keys_a, vertices_b, triangles_b, keys_b, subdomain_cubes=None):
    """Compare two meshes after canonical ordering.  Returns a dict of diagnostics."""
    va, ta, ka = canonicalize(vertices_a, triangles_a, keys_a)
    vb, tb, kb = canonicalize(vertices_b, triangles_b, keys_b)
    out = {"nv": (len(va), len(vb)), "nt": (len(ta), len(tb))}
    out["keys_equal"] = ka.shape == kb.shape and bool(np.array_equal(ka, kb))
    out["triangles_equal"] = ta.shape == tb.shape and bool(np.array_equal(ta, tb))
    if out["keys_equal"]:
        diff = np.abs(va.astype(np.float64) - vb.astype(np.float64))
        scale = np.maximum(np.abs(va), np.abs(vb)).astype(np.float64)
        out["max_abs"] = float(diff.max()) if len(diff) else 0.0
        out["max_rel"] = float((diff / np.maximum(scale, 1e-30)).max()) if len(diff) else 0.0
        neq = (va != vb).any(1)
        out["n_not_bitexact"] = int(neq.sum())
        if subdomain_cubes is not None and len(ka):
            S = int(subdomain_cubes)
            ax = ka[:, 3]
            onface = np.zeros(len(ka), dtype=bool)
            for d in range(3):
                onface |= (ax != d) & (ka[:, d] % S == 0)
            out["n_interior_not_bitexact"] = int((neq & ~onface).sum())
    return out
