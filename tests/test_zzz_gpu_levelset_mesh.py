"""The level-set field's surface as a mesh (LevelSetField.mesh, DESIGN.md section 16) on the device: the cases of
tests/test_levelset_mesh.py on the H100 (tiers and batches printed), and on a 1 M-particle dam break in every mode the whole-grid mesh
equals the raw mesh of reconstruct_surface, and a region around the splash at cell / 4 has every vertex on a crossing edge by
evaluate(), 10 000 sampled vertices equal to the f32 restatement bit for bit, at most two triangles per edge, no non-manifold vertex,
and edges with one triangle only on the box faces."""
import numpy as np
import pytest

import test_levelset_mesh as T
from levelset_field_harness import MODES, mode_kwargs
from test_averaged_surface import CASES

pytestmark = pytest.mark.gpu


def packed(keys):
    k = np.asarray(keys, np.int64).astype(np.uint64)
    return (k[:, 0] << np.uint64(42)) | (k[:, 1] << np.uint64(22)) | (k[:, 2] << np.uint64(2)) | k[:, 3]


def canon_np(verts, tris, keys):
    """Vertices sorted by edge key (keys, position bits) and the triangles as key triples rotated to their smallest key, sorted."""
    pk = packed(keys)
    o = np.argsort(pk, kind="stable")
    assert len(np.unique(pk)) == len(pk)
    t = pk[np.asarray(tris, np.int64)]
    r = np.argmin(t, axis=1)
    t = np.stack([t[np.arange(len(t)), (r + q) % 3] for q in range(3)], axis=1)
    t = t[np.lexsort(t.T[::-1])] if len(t) else t
    return pk[o], np.asarray(verts, np.float32)[o].view(np.uint32), t


def assert_same_np(a, b, what=""):
    assert np.array_equal(a[0], b[0]), (what, len(a[0]), len(b[0]))
    assert np.array_equal(a[1], b[1]), (what, int(np.sum(np.any(a[1] != b[1], axis=1))))
    assert np.array_equal(a[2], b[2]), (what, len(a[2]), len(b[2]))


@pytest.mark.parametrize("name", ["cube_S16", "splash_S24", "cube_S64", "droplets_sparse"])
def test_cuda_mesh_defaults_equal_reconstruction(ss, name):
    gen, kw, _ = CASES[name]
    p = gen()
    for mode in MODES:
        f, rec = T.raw(ss, p, dict(kw), mode)
        m = f.mesh()
        print(name, mode, len(m.mesh.triangles), m.paths, m.batches)
        assert len(m.mesh.triangles) > 0
        T.assert_same_mesh(T.mesh_canon(m), T.rec_canon(rec), (name, mode))
        f.close()


def test_cuda_mesh_box_other_sizes_tiers_batches(ss):
    for mode in ("sph", "aniso", "avg", "corr_rad"):
        T.test_emulated_mesh_box_equals_reconstruction(ss, mode)
    for mode in ("sph", "aniso", "avg", "corr", "rad"):
        T.test_emulated_mesh_other_cube_sizes(ss, mode)
    T.test_emulated_mesh_tiers_and_batches(ss)
    T.test_emulated_mesh_lone_particle(ss)
    T.test_emulated_mesh_refusals_and_reuse(ss)


def test_cuda_mesh_dam_break(ss):
    from splashsurf_b200 import synthetic as syn
    x = syn.dam_break_scaled(1_000_000, 0.01, 3)
    kw = dict(particle_radius=0.01, smoothing_length=2.0, cube_size=0.5)
    ctx = ss.Context()
    try:
        for mode in MODES:
            mk = mode_kwargs(ss, mode, x, kw)
            rec = ss.reconstruct_surface(x, context=ctx, simd=False, subdomain_grid_auto_disable=False, with_debug=True, **kw, **mk)
            f = ss.LevelSetField(x, context=ctx, **kw, **mk)
            m = f.mesh()
            print(mode, "whole grid:", len(m.mesh.triangles), "triangles", m.paths, m.batches, "batches")
            assert_same_np(canon_np(m.mesh.vertices, m.mesh.triangles, m.vertex_edge_keys),
                           canon_np(rec.mesh.vertices, rec.mesh.triangles, rec.vertex_edge_keys), mode)
            # a region in the middle of the mesh (the 45 - 55 % quantiles of its vertices per axis) at cell / 4
            c = np.float32(f.grid.cell_size)
            v = rec.mesh.vertices
            q = np.quantile(v, [0.45, 0.55], axis=0)
            bmin, bmax = q[0].astype(np.float32), q[1].astype(np.float32)
            m4 = f.mesh(c / np.float32(4), aabb_min=bmin, aabb_max=bmax)
            print(mode, "cell/4 region:", len(m4.mesh.triangles), "triangles", m4.paths, m4.batches, "batches")
            assert len(m4.mesh.triangles) > 0
            keys = m4.vertex_edge_keys
            a_i = keys[:, :3]
            b_i = a_i.copy()
            b_i[np.arange(len(keys)), keys[:, 3]] += 1
            cs = np.float32(m4.cube_size)
            A, B = T.lattice_point(f, a_i, cs), T.lattice_point(f, b_i, cs)
            va, vb = f.evaluate(np.ascontiguousarray(A)), f.evaluate(np.ascontiguousarray(B))
            thr = np.float32(f.threshold)
            assert np.all((va > thr) != (vb > thr))
            sel = np.random.default_rng(5).choice(len(keys), min(10_000, len(keys)), replace=False)
            with np.errstate(all="ignore"):
                al = ((thr - va[sel]) / (vb[sel] - va[sel])).astype(np.float32)
                om = (np.float32(1) - al).astype(np.float32)
                pos = ((A[sel] * om[:, None]).astype(np.float32) + (B[sel] * al[:, None]).astype(np.float32)).astype(np.float32)
            assert np.array_equal(pos.view(np.uint32), m4.mesh.vertices[sel].view(np.uint32))
            tris = m4.mesh.triangles.astype(np.int64)
            e = np.sort(np.concatenate([tris[:, [0, 1]], tris[:, [1, 2]], tris[:, [2, 0]]]), axis=1)
            ue, cnt = np.unique(e, axis=0, return_counts=True)
            assert cnt.max() <= 2
            assert len(ss.find_non_manifold_vertices(m4.mesh)) == 0
            # edges with one triangle: both vertices on one box face
            one = ue[cnt == 1]
            lo, hi = m4.index_min, m4.index_max
            ka, kb = keys[one[:, 0]], keys[one[:, 1]]
            on_face = np.zeros(len(one), bool)
            for d in range(3):
                for plane in (lo[d], hi[d]):
                    on_face |= (ka[:, d] == plane) & (kb[:, d] == plane) & (ka[:, 3] != d) & (kb[:, 3] != d)
            assert on_face.all(), int((~on_face).sum())
            f.close()
    finally:
        ctx.close()
