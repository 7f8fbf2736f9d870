"""The level-set field's surface as a mesh (LevelSetField.mesh / ss_levelset_field_mesh_f32, DESIGN.md section 16) on the CPU executor
of the CUDA sources (also run with SS_EMUL_GUARD=1):

* with the defaults the mesh is the raw mesh of reconstruct_surface (simd=False for the standard level set) as a canonical mesh --
  vertex positions bit for bit per edge key, the same triangles -- in every mode, at S = 16 / 24 / 64, on sparse droplets, the
  clustered cloud and a jittered ball, and at R = 1, 6, 7, 8, 9, 17;
* a box at the field's cell gives the reconstruction's triangles whose cells lie in the box, bit for bit;
* at c/2, c/3, c/4, c, 1.7 c and 4 c the edge keys and triangles equal marching cubes on evaluate()'s lattice values (no brick or
  cell missing; at 4 c lattice bricks span several field groups), every vertex away from the field's cell is the f32 restatement
  a (1 - alpha) + b alpha of those values, no edge has more than two triangles and edges with one lie on the box faces;
* a lone particle 0.9 / 0.99 h from a brick's first point gets that brick listed and meshed;
* the clustered cloud reaches the 4096 slice and the selection walk; batches of 1 and 3 tiles give the same mesh;
* refusals, an empty box, n = 0, a stale handle and one context reused across a field, its meshes and a reconstruction.
The GPU-marked counterpart is tests/test_zzz_gpu_levelset_mesh.py."""
import ctypes as C

import numpy as np
import pytest

from levelset_field_harness import MODES, _ball, mode_kwargs
from test_anisotropic import KW, R, _cube
from test_averaged_surface import CASES
from test_emulated_pipeline import emu  # noqa: F401  (fixture: the package bound to the CPU executor)


def canonical(verts, tris, keys):
    """{edge key: position bytes} and the sorted triangles as edge-key triples rotated to start at their smallest key."""
    kk = [tuple(k) for k in np.asarray(keys, np.int64)]
    pos = {k: np.asarray(v, np.float32).tobytes() for k, v in zip(kk, verts)}
    assert len(pos) == len(kk), "two vertices on one edge"
    tri = []
    for t in np.asarray(tris, np.int64):
        e = [kk[int(i)] for i in t]
        r = e.index(min(e))
        tri.append(tuple(e[r:] + e[:r]))
    return pos, sorted(tri)


def assert_same_mesh(a, b, what=""):
    pa, ta = a
    pb, tb = b
    assert pa.keys() == pb.keys(), (what, len(pa), len(pb))
    bad = [k for k in pa if pa[k] != pb[k]]
    assert not bad, (what, len(bad), bad[:3])
    assert ta == tb, (what, len(ta), len(tb))


def mesh_canon(m):
    return canonical(m.mesh.vertices, m.mesh.triangles, m.vertex_edge_keys)


def rec_canon(rec):
    return canonical(rec.mesh.vertices, rec.mesh.triangles, rec.vertex_edge_keys)


def raw(ss, p, kw, mode):
    mk = mode_kwargs(ss, mode, p, kw)
    rec = ss.reconstruct_surface(p, simd=False, subdomain_grid_auto_disable=False, with_debug=True, **kw, **mk)
    f = ss.LevelSetField(p, **kw, **mk)
    return f, rec


def lattice_point(f, I, cs):
    """gmin + I * cs per axis in f32: (float)I * cs rounded, then + gmin rounded."""
    gmin = np.asarray(f.grid.aabb.min, np.float32)
    return (np.asarray(I, np.float32) * np.float32(cs)).astype(np.float32) + gmin


def check_restatement(f, m):
    """Every vertex: a (1 - alpha) + b alpha of evaluate()'s values at its edge's lattice points (bit for bit), whose inside flags
    differ; every edge has at most two triangles, and the edges with one lie on a face of the box."""
    keys = m.vertex_edge_keys
    if not len(keys):
        return 0
    cs = np.float32(m.cube_size)
    a_i = keys[:, :3]
    b_i = a_i.copy()
    b_i[np.arange(len(keys)), keys[:, 3]] += 1
    A, B = lattice_point(f, a_i, cs), lattice_point(f, b_i, cs)
    va, vb = f.evaluate(np.ascontiguousarray(A)), f.evaluate(np.ascontiguousarray(B))
    thr = np.float32(f.threshold)
    assert np.all((va > thr) != (vb > thr))
    with np.errstate(all="ignore"):
        alpha = ((thr - va) / (vb - va)).astype(np.float32)
        om = (np.float32(1) - alpha).astype(np.float32)
        pos = ((A * om[:, None]).astype(np.float32) + (B * alpha[:, None]).astype(np.float32)).astype(np.float32)
    assert np.array_equal(pos.view(np.uint32), m.mesh.vertices.view(np.uint32))
    assert_box_faces(m)
    return len(keys)


def assert_box_faces(m):
    """At most two triangles per edge; an edge with one has both vertices on one face of the box (the same extreme lattice plane on
    an axis neither vertex's edge runs along)."""
    tris = m.mesh.triangles.astype(np.int64)
    if not len(tris):
        return
    e = np.sort(np.concatenate([tris[:, [0, 1]], tris[:, [1, 2]], tris[:, [2, 0]]]), axis=1)
    ue, cnt = np.unique(e, axis=0, return_counts=True)
    assert cnt.max() <= 2
    one = ue[cnt == 1]
    keys = m.vertex_edge_keys
    ka, kb = keys[one[:, 0]], keys[one[:, 1]]
    on_face = np.zeros(len(one), bool)
    for d in range(3):
        for plane in (m.index_min[d], m.index_max[d]):
            on_face |= (ka[:, d] == plane) & (kb[:, d] == plane) & (ka[:, 3] != d) & (kb[:, 3] != d)
    assert on_face.all(), int((~on_face).sum())


def lattice_values(f, m):
    """evaluate() at every lattice point of the mesh's index range, as a dense (nx, ny, nz) array."""
    ax = [np.arange(m.index_min[d], m.index_max[d] + 1) for d in range(3)]
    I = np.stack(np.meshgrid(*ax, indexing="ij"), axis=-1).reshape(-1, 3)
    return f.evaluate(np.ascontiguousarray(lattice_point(f, I, m.cube_size))).reshape([len(a) for a in ax])


def mc_topology(ss, values, thr, lo):
    """Edge keys (global lattice indices: + lo) and triangles (rotated key triples, sorted) of the marching-cubes kernels of
    ss.marching_cubes on a dense array: the front end's tiling and edge padding, with the edge keys kept and the padded cells'
    triangles dropped as it drops them."""
    L = ss._LIB
    ncells = [n - 1 for n in values.shape]
    nt = [(c + 63) // 64 for c in ncells]
    padded = np.pad(values, [(0, t * 64 + 1 - n) for t, n in zip(nt, values.shape)], mode="edge")
    tiles, ijk = [], []
    for a in range(nt[0]):
        for b in range(nt[1]):
            for c_ in range(nt[2]):
                blk = padded[a * 64:a * 64 + 65, b * 64:b * 64 + 65, c_ * 64:c_ * 64 + 65]
                if blk.min() > thr or blk.max() < thr:
                    continue
                tiles.append(blk)
                ijk.append((a, b, c_))
    if not tiles:
        return set(), []
    tiles = np.ascontiguousarray(np.stack(tiles))
    ijk = np.ascontiguousarray(np.asarray(ijk, np.int32))
    ctx = ss.Context()
    s = C.c_void_p()
    try:
        assert L.ss_marching_cubes_tiles_f32(ctx._h, tiles.ctypes.data, len(tiles), ijk.ctypes.data, (C.c_float * 3)(0, 0, 0), C.c_float(1.0),
                                             C.c_float(float(thr)), C.byref(s)) == 0
        nv, ntri = L.ss_surface_num_vertices(s), L.ss_surface_num_triangles(s)
        keys, tris = np.empty((nv, 4), np.int64), np.empty((ntri, 3), np.uint32)
        if nv:
            L.ss_surface_copy_vertex_edge_keys(s, keys.ctypes.data)
        if ntri:
            L.ss_surface_copy_triangles_u32(s, tris.ctypes.data)
        L.ss_surface_free(s)
    finally:
        ctx.close()
    end = keys[:, :3].copy()
    end[np.arange(nv), keys[:, 3]] += 1
    bad = (end > np.asarray(values.shape) - 1).any(axis=1)
    tris = tris[~bad[tris].any(axis=1)]
    keys[:, :3] += np.asarray(lo, np.int64)
    _, tri = canonical(np.zeros((nv, 3), np.float32), tris, keys)
    return {tuple(keys[i]) for i in np.unique(tris)}, tri


def check_topology(ss, f, m):
    """The mesh's edge keys and triangles equal marching cubes on evaluate()'s values over the same lattice; False (skipped) where a
    value equals the threshold, which that front end refuses."""
    v = lattice_values(f, m)
    thr = np.float32(f.threshold)
    if np.any(v == thr):
        return False
    keys, tri = mc_topology(ss, v, thr, m.index_min)
    _, mtri = mesh_canon(m)
    assert {tuple(k) for k in m.vertex_edge_keys} == keys, (len(m.vertex_edge_keys), len(keys))
    assert mtri == tri, (len(mtri), len(tri))
    # the crossing edges of the lattice are exactly the mesh's vertices
    inside = v > thr
    n = 0
    for d in range(3):
        sl0, sl1 = [slice(None)] * 3, [slice(None)] * 3
        sl0[d], sl1[d] = slice(0, -1), slice(1, None)
        n += int(np.count_nonzero(inside[tuple(sl0)] != inside[tuple(sl1)]))
    assert n == len(m.vertex_edge_keys)
    return True


def spans_several_groups(f, m, S):
    """Whether some 8-point run of the lattice along x holds points of several field groups (subdomain of S cells, brick of 8 cells
    within it)."""
    c = np.float32(f.grid.cell_size)
    gmin = np.float32(f.grid.aabb.min[0])
    I = np.arange(m.index_min[0], m.index_max[0] + 1)
    x = lattice_point(f, np.stack([I, I, I], axis=1), m.cube_size)[:, 0]
    cell = np.clip(np.floor((x - gmin).astype(np.float32) / c), 0, f.grid.ncells_per_dim[0] - 1).astype(np.int64)
    g = (cell // S) * 1000 + (cell % S) // 8
    return any(len(np.unique(g[q:q + 8])) > 1 for q in range(0, len(g), 8))


# ------------------------------------------------------------------ defaults = the reconstruction ----
CLOUDS = dict({k: CASES[k][:2] for k in ("cube_S16", "splash_S24", "cube_S64", "droplets_sparse", "clustered_overflow")},
              ball=(lambda: _ball(0.1, 211), dict(KW, subdomain_num_cubes_per_dim=16)))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("name", list(CLOUDS))
def test_emulated_mesh_defaults_equal_reconstruction(emu, name, mode):  # noqa: F811
    gen, kw = CLOUDS[name]
    p = gen()
    f, rec = raw(emu, p, dict(kw), mode)
    m = f.mesh()
    assert len(m.mesh.triangles) > 0 and m.cube_size == np.float32(f.grid.cell_size)
    assert_same_mesh(mesh_canon(m), rec_canon(rec), (name, mode))
    assert m.paths["512"] > 0
    f.close()


@pytest.mark.parametrize("Rc", [1, 6, 7, 8, 9, 17])
@pytest.mark.parametrize("mode", MODES)
def test_emulated_mesh_cube_sizes_equal_reconstruction(emu, mode, Rc):  # noqa: F811
    p = _cube(6, 900 + Rc)
    kw = dict(particle_radius=R, smoothing_length=2.0, cube_size=4.0 / (Rc - 0.5), subdomain_num_cubes_per_dim=16)
    f, rec = raw(emu, p, kw, mode)
    assert int(np.ceil(np.float32(4 * R) / np.float32(f.grid.cell_size))) == Rc
    assert_same_mesh(mesh_canon(f.mesh()), rec_canon(rec), (mode, Rc))
    f.close()


# ------------------------------------------------------------------ a box at the field's cell ----
def box_triangles(rec, lo, hi):
    """The reconstruction's triangles whose cell (per axis the smallest point index of its vertices' edges) lies in [lo, hi)."""
    keys = rec.vertex_edge_keys
    tris = rec.mesh.triangles.astype(np.int64)
    cell = keys[tris][:, :, :3].min(axis=1)
    keep = np.all((cell >= lo) & (cell + 1 <= hi), axis=1)
    return canonical(rec.mesh.vertices, tris[keep], keys)


@pytest.mark.parametrize("mode", ["sph", "aniso", "avg", "corr_rad"])
def test_emulated_mesh_box_equals_reconstruction(emu, mode):  # noqa: F811
    gen, kw, _ = CASES["splash_S24"]
    p = gen()
    f, rec = raw(emu, p, dict(kw), mode)
    c = np.float32(f.grid.cell_size)
    gmin = np.asarray(f.grid.aabb.min, np.float64)
    n = np.asarray(f.grid.ncells_per_dim)
    boxes = [(np.array([3.3, 5.0, 7.7]), n * 0.6),                       # inside, across subdomain and brick faces
             (np.array([-4.0, 23.5, 10.0]), np.array([30.0, 49.0, 64.5])),  # across tile faces
             (np.array([-9.0, -9.0, -9.0]), n * 0.5),                    # partly outside the grid
             (n * 0.5, n + 7.0)]
    for blo, bhi in boxes:
        bmin = (gmin + blo * float(c)).astype(np.float32)
        bmax = (gmin + bhi * float(c)).astype(np.float32)
        m = f.mesh(aabb_min=bmin, aabb_max=bmax)
        lo = np.maximum(0, np.floor((bmin.astype(np.float64) - gmin) / float(c))).astype(np.int64)
        hi = np.minimum(n, np.ceil((bmax.astype(np.float64) - gmin) / float(c))).astype(np.int64)
        assert np.array_equal(m.index_min, lo) and np.array_equal(m.index_max, hi)
        pos, tri = mesh_canon(m)
        rpos, rtri = box_triangles(rec, lo, hi)
        assert tri == rtri, (mode, blo, len(tri), len(rtri))
        assert all(pos[k] == rpos[k] for k in pos)
        assert set(pos) == {k for t in tri for k in t}
    f.close()


# ------------------------------------------------------------------ other cube sizes ----
@pytest.mark.parametrize("mode", ["sph", "aniso", "avg", "corr", "rad"])
def test_emulated_mesh_other_cube_sizes(emu, mode):  # noqa: F811
    """At c/2, c/3, c/4 (misaligned boxes), c (a box), 1.7 c and 4 c (the whole grid): the topology equals marching cubes on evaluate()'s
    lattice values, so no brick or cell is missing, and every vertex equals its f32 restatement (away from the field's cell)."""
    gen, kw, _ = CASES["splash_S24"]
    p = gen()
    f, rec = raw(emu, p, dict(kw), mode)
    c = float(np.float32(f.grid.cell_size))
    gmin = np.asarray(f.grid.aabb.min, np.float64)
    q = np.quantile(rec.mesh.vertices, [0.3, 0.62], axis=0).astype(np.float32)      # a box across the surface, misaligned to the lattices
    checked, skipped = 0, 0
    for k in (0.5, 1.0 / 3.0, 0.25, 1.0, 1.7, 4.0):
        cs = np.float32(c * k)
        box = (q[0], q[1]) if k <= 1 else (None, None)
        m = f.mesh(cs, aabb_min=box[0], aabb_max=box[1])
        assert m.cube_size == cs and len(m.mesh.triangles) > 0
        if k != 1.0:
            check_restatement(f, m)
        else:
            assert_box_faces(m)
        if check_topology(emu, f, m):
            checked += 1
        else:
            skipped += 1
        if k == 4.0:
            assert spans_several_groups(f, m, kw["subdomain_num_cubes_per_dim"])
    print(mode, "topology checked", checked, "skipped (a value at the threshold)", skipped)
    assert checked >= 5
    f.close()


# ------------------------------------------------------------------ tiers, batches ----
def test_emulated_mesh_tiers_and_batches(emu):  # noqa: F811
    gen, kw, _ = CASES["clustered_overflow"]
    p = gen()
    f, rec = raw(emu, p, dict(kw), "sph")
    m = f.mesh()
    assert m.paths["4096"] > 0 and m.paths["select"] > 0, m.paths
    assert_same_mesh(mesh_canon(m), rec_canon(rec), "clustered")
    f.close()
    gen, kw, _ = CASES["splash_S24"]
    p = gen()
    f, rec = raw(emu, p, dict(kw), "avg")
    L = emu._LIB
    ref = f.mesh(np.float32(f.grid.cell_size) * np.float32(0.5))
    assert ref.batches >= 1
    try:
        for cap in (1, 3):
            L.ss_levelset_mesh_set_batch_tiles(cap)
            m = f.mesh(np.float32(f.grid.cell_size) * np.float32(0.5))
            assert m.batches > 1
            assert_same_mesh(mesh_canon(m), mesh_canon(ref), cap)
    finally:
        L.ss_levelset_mesh_set_batch_tiles(0)
    again = f.mesh(np.float32(f.grid.cell_size) * np.float32(0.5))
    assert np.array_equal(again.mesh.vertices.view(np.uint32), ref.mesh.vertices.view(np.uint32))
    assert np.array_equal(again.mesh.triangles, ref.mesh.triangles) and np.array_equal(again.vertex_edge_keys, ref.vertex_edge_keys)
    f.close()


def test_emulated_mesh_lone_particle(emu):  # noqa: F811
    """A lone particle 0.9 / 0.99 h from the first lattice point of a brick, the brick reaching away from it: the brick is listed, and
    with a threshold below the value at that point the brick is meshed, as marching cubes on the lattice values meshes it."""
    p = np.array([[0.0, 0.0, 0.0]], np.float32)
    kw = dict(particle_radius=R, smoothing_length=2.0, cube_size=0.5, subdomain_num_cubes_per_dim=16)
    h = 4.0 * R
    for frac in (0.9, 0.99):
        f = emu.LevelSetField(p, **kw)
        cs = np.float32(float(np.float32(f.grid.cell_size)) / 16)
        gmin = np.asarray(f.grid.aabb.min, np.float64)
        I = np.rint((frac * h / np.sqrt(3.0) - gmin) / float(cs)).astype(np.int64)
        P0 = lattice_point(f, I, cs)
        d = float(np.linalg.norm(P0.astype(np.float64)))
        assert frac - 0.01 < d / h < min(frac + 0.01, 0.9999), d / h
        v0 = float(f.evaluate(P0[None])[0])
        assert v0 > 0
        f.close()
        f = emu.LevelSetField(p, **kw, iso_surface_threshold=v0 / 2)
        box = ((P0 + np.float32(0.25) * cs).astype(np.float32), (P0 + np.float32(7.5) * cs).astype(np.float32))
        m = f.mesh(cs, aabb_min=box[0], aabb_max=box[1])
        assert np.array_equal(m.index_min, I) and np.array_equal(m.index_max, I + 8)
        assert m.paths["512"] >= 1
        assert len(m.mesh.triangles) > 0
        check_restatement(f, m)
        assert check_topology(emu, f, m)
        f.close()


# ------------------------------------------------------------------ edge cases ----
def test_emulated_mesh_refusals_and_reuse(emu):  # noqa: F811
    gen, kw, _ = CASES["cube_S16"]
    p = gen()
    ctx = emu.Context()
    f = emu.LevelSetField(p, **kw, context=ctx)
    L = emu._LIB
    nan = float("nan")
    for args in [dict(aabb_min=[0, 0, 0]), dict(aabb_max=[1, 1, 1])]:
        with pytest.raises(ValueError):
            f.mesh(**args)
    for cs, bmin, bmax in [(nan, None, None), (float("inf"), None, None), (0.0, [nan, 0, 0], [1, 1, 1]), (0.0, [0, 0, 0], [1, float("inf"), 1]),
                           (0.0, [1, 0, 0], [0, 1, 1])]:
        with pytest.raises(emu.SplashsurfError):
            f.mesh(cs or None, aabb_min=bmin, aabb_max=bmax)
    with pytest.raises(emu.SplashsurfError):
        f.mesh(np.float32(f.grid.cell_size) * np.float32(1e-6))             # lattice index above 2^20 - 1
    # through the C entry: one of the two box corners
    out = C.c_void_p()
    box = (C.c_float * 3)(0, 0, 0)
    assert L.ss_levelset_field_mesh_f32(f._s, box, None, C.c_float(0), C.byref(out)) == emu.SS_ERR_INVALID_PARAMETER
    assert L.ss_levelset_field_mesh_f32(f._s, None, None, C.c_float(nan), C.byref(out)) == emu.SS_ERR_INVALID_PARAMETER
    # a box outside the grid, a box without a cell: empty meshes
    far = np.asarray(f.grid.aabb.max, np.float32) + np.float32(100)
    assert len(f.mesh(aabb_min=far, aabb_max=far + 1).mesh.vertices) == 0
    g0 = np.asarray(f.grid.aabb.min, np.float32)
    assert len(f.mesh(aabb_min=g0, aabb_max=g0).mesh.triangles) == 0
    # the mesh owns its arrays; the field, its meshes and a reconstruction share the context
    m1 = f.mesh()
    v = f.evaluate(m1.mesh.vertices)
    assert np.all(np.isfinite(v))
    m2 = f.mesh()
    assert_same_mesh(mesh_canon(m1), mesh_canon(m2))
    emu.reconstruct_surface(p, context=ctx, **kw)
    with pytest.raises(emu.SplashsurfError):
        f.mesh()                                                            # stale handle
    f.close()
    # n = 0
    f0 = emu.LevelSetField(np.zeros((0, 3), np.float32), **kw, context=ctx)
    m0 = f0.mesh()
    assert len(m0.mesh.vertices) == 0 and len(m0.mesh.triangles) == 0
    f0.close()
    ctx.close()
