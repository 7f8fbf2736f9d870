"""First crossings of the level-set field along rays and segments (LevelSetField.raycast, DESIGN.md section 15) on the device: the
device-versus-oracle cases of tests/test_levelset_raycast.py on the H100 with three times the rays (rounds and tiers printed),
host and CUDA-tensor rays give identical results, and on a 1 M-particle dam break 1 M camera rays and 1 M segments across the mesh
are consistent with evaluate(), inside() and the mesh in every mode."""
import numpy as np
import pytest

from levelset_field_harness import GRAD_MODES, MODES, _kw_abs, _same, mode_kwargs
from levelset_raycast_harness import camera_rays, check_raycast_vs_oracle, ray_sets
from test_anisotropic import KW, R, _clustered, _cube
from test_averaged_surface import CASES

pytestmark = pytest.mark.gpu

STEPS_REFINES = [(0.5, 24), (0.13, 1), (3.0, 64), (0.5, 0)]


def _rays(S, seed, scale):
    def of(f, p):
        return ray_sets(f.grid, _kw_abs(KW)[1], S, seed, scale, targets=p)
    return of


@pytest.mark.parametrize("name", ["splash_S24", "droplets_sparse"])
def test_cuda_raycast_equals_oracle(ss, name):
    gen, kw, _ = CASES[name]
    p = gen()
    for mode in MODES:
        res = check_raycast_vs_oracle(ss, p, kw, mode, _rays(kw["subdomain_num_cubes_per_dim"], 400, 3), STEPS_REFINES)
        print(name, mode, res)
        assert sum(r["status"][1] + r["status"][-1] for r in res) > 60, res


def test_cuda_raycast_cube_sizes_and_select(ss):
    for Rc in (1, 9):
        p = _cube(7, 900 + Rc)
        kw = dict(particle_radius=R, smoothing_length=2.0, cube_size=4.0 / (Rc - 0.5), subdomain_num_cubes_per_dim=16)
        for mode in ("sph", "avg"):
            print(Rc, mode, check_raycast_vs_oracle(ss, p, kw, mode, _rays(16, 410 + Rc, 2), [(0.5, 24), (3.0, 8)]))
    p = _clustered(507)

    def rays(f, _p):
        rng = np.random.default_rng(350)
        return (rng.uniform(0.1, 0.3, (200, 3)).astype(np.float32), rng.normal(size=(200, 3)).astype(np.float32),
                np.full(200, np.float32(0.2)))
    for mode in ("sph", "avg", "corr"):
        print("clustered", mode, check_raycast_vs_oracle(ss, p, dict(KW, subdomain_num_cubes_per_dim=16), mode, rays, [(0.5, 24)],
                                                         expect_tier="select"))


def test_cuda_raycast_host_and_device_rays_agree(ss):
    import torch
    p = _cube(12, 881)
    f = ss.LevelSetField(p, averaged_surface=ss.AveragedSurface(), **KW)
    try:
        o, d, tm = ray_sets(f.grid, _kw_abs(KW)[1], 16, 420, 20, targets=p)
        host = f.raycast(o, d, t_max=tm)
        dev = f.raycast(torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda(), t_max=torch.from_numpy(tm).cuda())
        assert dev.t.is_cuda and dev.status.dtype == torch.int8 and dev.rounds == host.rounds
        for a, b in ((host.t, dev.t), (host.positions, dev.positions), (host.values, dev.values), (host.gradients, dev.gradients)):
            assert _same(a, b.cpu().numpy())
        assert np.array_equal(host.status, dev.status.cpu().numpy())
        # the normals are those of normals() on the same side: numpy's and torch's norms may round differently
        hit = np.abs(host.status) == 1
        assert hit.sum() > 1000
        assert _same(host.normals[hit], f.normals(host.positions[hit]))
        assert _same(dev.normals.cpu().numpy()[hit], f.normals(dev.positions[torch.from_numpy(hit).cuda()]).cpu().numpy())
        one = f.raycast(torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda(), t_max=2.0, normals=False)
        assert one.normals is None and np.array_equal(one.status.cpu().numpy(), f.raycast(o, d, t_max=2.0, normals=False).status)
    finally:
        f.close()


def _segment_mesh_t(verts, tris, o, d):
    """Smallest t in [0, 1] of each segment o + t d against the triangles near it (float64 Moller-Trumbore); inf where none."""
    from scipy.spatial import cKDTree
    v = verts.astype(np.float64)
    a, b, c = v[tris[:, 0]], v[tris[:, 1]], v[tris[:, 2]]
    ctr = (a + b + c) / 3.0
    reach = float(np.max(np.linalg.norm(np.stack([a - ctr, b - ctr, c - ctr]), axis=2)))
    tree = cKDTree(ctr)
    out = np.full(len(o), np.inf)
    for i in range(len(o)):
        dd = d[i].astype(np.float64)
        mid = o[i].astype(np.float64) + 0.5 * dd
        near = np.asarray(tree.query_ball_point(mid, 0.5 * np.linalg.norm(dd) + reach), np.int64)
        if not len(near):
            continue
        e1, e2 = b[near] - a[near], c[near] - a[near]
        pv = np.cross(dd, e2)
        det = np.einsum("ij,ij->i", e1, pv)
        ok = np.abs(det) > 1e-30
        inv = np.where(ok, 1.0 / np.where(ok, det, 1.0), 0.0)
        tv = o[i].astype(np.float64) - a[near]
        u = np.einsum("ij,ij->i", tv, pv) * inv
        qv = np.cross(tv, e1)
        w = (qv @ dd) * inv
        t = np.einsum("ij,ij->i", e2, qv) * inv
        sel = ok & (u >= 0) & (w >= 0) & (u + w <= 1) & (t >= 0) & (t <= 1)
        if sel.any():
            out[i] = t[sel].min()
    return out


def test_cuda_raycast_dam_break(ss):
    """1 M-particle dam break, every mode: 1 M camera rays and 1 M segments from mesh vertices moved by up to 2 cells.  Values equal
    evaluate(positions) bit for bit, every hit's inside flag is opposite to its origin's, normals are finite where the gradient is
    not 0, entering camera hits face the ray, and 2000 segments agree with the raw mesh within sqrt(3) cells plus the bracket."""
    import torch
    from splashsurf_b200 import synthetic as syn
    x = syn.dam_break_scaled(1_000_000, 0.01, 3)
    kw = dict(particle_radius=0.01, smoothing_length=2.0, cube_size=0.5)
    ctx = ss.Context()
    try:
        for mode in MODES:
            mk = mode_kwargs(ss, mode, x, kw)
            g = ss.reconstruct_surface(x, context=ctx, simd=False, subdomain_grid_auto_disable=False, **kw, **mk)
            verts, tris = np.asarray(g.mesh.vertices), np.asarray(g.mesh.triangles).astype(np.int64)
            f = ss.LevelSetField(x, context=ctx, **kw, **mk)
            c = float(f.grid.cell_size)
            grad = mode in GRAD_MODES
            rng = np.random.default_rng(430)
            co, cd, _ = camera_rays(f.grid, 1000, 431)
            sel = rng.integers(0, len(verts), 1_000_000)
            so = (verts[sel] + rng.uniform(-1, 1, (len(sel), 3)) * c).astype(np.float32)
            u = rng.normal(size=(len(sel), 3))
            sd = (u / np.linalg.norm(u, axis=1, keepdims=True) * rng.uniform(0.05, 2.0, (len(sel), 1)) * c).astype(np.float32)
            for what, o, d, tm in (("camera", co, cd, None), ("segments", so, sd, 1.0)):
                od, dd = torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda()
                torch.cuda.synchronize()
                hits = f.raycast(od, dd, t_max=tm, normals=grad)
                paths = f.paths
                st = hits.status.cpu().numpy()
                hit = np.abs(st) == 1
                pos = hits.positions[torch.from_numpy(hit).cuda()]
                assert _same(hits.values.cpu().numpy()[hit], f.evaluate(pos).cpu().numpy()), (mode, what)
                assert np.array_equal(f.inside(pos).cpu().numpy(), ~f.inside(od[torch.from_numpy(hit).cuda()]).cpu().numpy()), (mode, what)
                share = None
                if grad:
                    gr, nr = hits.gradients.cpu().numpy()[hit], hits.normals.cpu().numpy()[hit]
                    nz = np.any(gr != 0, axis=1)
                    assert np.isfinite(nr[nz]).all(), (mode, what)
                    enter = (st[hit] == 1) & nz
                    share = float(np.mean(np.einsum("ij,ij->i", nr[enter], d[hit][enter]) < 0)) if enter.any() else None
                    # measured on the H100 (700 W): every entering hit of both workloads faces the ray, in every mode with a gradient
                    assert share is not None and share >= 0.99, (mode, what, share)
                print(mode, what, "hits", int(hit.sum()), "of", len(o), "rounds", hits.rounds, "paths", paths,
                      "entering hits facing the ray", share)
            # 2000 segments against the raw mesh
            k = 2000
            hits = f.raycast(so[:k], sd[:k], t_max=1.0, step=0.5 * c, refine=24, normals=False)
            tmesh = _segment_mesh_t(verts, tris, so[:k], sd[:k])
            both = (np.abs(hits.status) == 1) & np.isfinite(tmesh)
            nd = np.linalg.norm(sd[:k].astype(np.float64), axis=1)
            diff = np.abs(hits.t.astype(np.float64)[both] - tmesh[both]) * nd[both]
            tol = np.sqrt(3.0) * c + 0.5 * c * 2.0 ** -24
            print(mode, "segments hitting field and mesh", int(both.sum()), "largest |t_field - t_mesh| in cells", float(diff.max()) / c)
            assert both.sum() > 200 and np.all(diff <= tol), (mode, float(diff.max()) / c)
            f.close()
    finally:
        ctx.close()
