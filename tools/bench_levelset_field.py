#!/usr/bin/env python3
"""Times the level-set field at arbitrary points (LevelSetField, DESIGN.md §13) on one GPU, for every level set: standard, anisotropic,
averaged, corrected, and both with per-particle radii uniform in [0.8, 1.2] r.  Per mode: the create time (decomposition, densities,
anisotropy, binning; host clock around the synchronous call), and the query rate for three point sets held on the device:
  * tiles: every grid point of a block of whole 64-cube tiles around the busiest subdomain (dense sampling);
  * uniform: `--points` points uniform in the grid's box;
  * near_mesh: the vertices of the mode's mesh, each moved by up to one cell (sphere tracing, whitewater classification).
Each query is timed over `--steps` calls after `--warmup` (CUDA events around the call, which ends in a device synchronise).  Beside
them, the same mode's level-set stage of reconstruct_surface and the grid points it evaluated, for ns per grid point.  The card name,
power limit and SM clock are read at the start and at the end.  Prints one JSON line; writes nothing.

With `--gradient` the corrected modes are left out (they have no gradient, DESIGN.md §13.1) and every query is also timed as a
gradient query (LevelSetField.gradient, §13.1) on the same points, the two alternating call by call.

    python tools/bench_levelset_field.py                         # cfg-4: the 50 M-particle dam break
    python tools/bench_levelset_field.py --particles 1000000 --points 1000000
    python tools/bench_levelset_field.py --gradient              # value and gradient queries side by side
    python tools/bench_levelset_field.py --hessian               # value, gradient, Hessian and curvature queries side by side

With `--hessian` (implies `--gradient`) the Hessian (LevelSetField.hessian, §13.2) and curvature (LevelSetField.curvature) queries
are timed as well, the four alternating call by call.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"unknown ({e})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--particles", type=int, default=50_000_400, help="dam break with cfg-4 proportions (default: cfg-4 itself)")
    ap.add_argument("--points", type=int, default=10_000_000)
    ap.add_argument("--tiles", type=int, default=2, help="tiles per axis of the dense block")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--modes", default="standard,anisotropic,averaged,averaged_corrected,averaged_radii,averaged_corrected_radii")
    ap.add_argument("--gradient", action="store_true", help="also time the gradient query (modes with a gradient only)")
    ap.add_argument("--hessian", action="store_true", help="also time the gradient, Hessian and curvature queries (modes with a Hessian only)")
    a = ap.parse_args()
    a.gradient = a.gradient or a.hessian
    import numpy as np
    import torch
    import splashsurf_b200 as ss
    from splashsurf_b200 import synthetic as syn
    card_before = card()
    x = syn.dam_break_50m() if a.particles == 50_000_400 else syn.dam_break_scaled(a.particles, 0.01, 3)
    kw = dict(particle_radius=0.01, smoothing_length=2.0, cube_size=0.5)
    radii = (np.random.default_rng(4).uniform(0.8, 1.2, len(x)) * 0.01).astype(np.float32)
    corr = ss.JacobianCorrection()
    modes = {"standard": {}, "anisotropic": dict(anisotropy=ss.Anisotropy()), "averaged": dict(averaged_surface=ss.AveragedSurface()),
             "averaged_corrected": dict(averaged_surface=ss.AveragedSurface(correction=corr)),
             "averaged_radii": dict(averaged_surface=ss.AveragedSurface(), particle_radii=radii),
             "averaged_corrected_radii": dict(averaged_surface=ss.AveragedSurface(correction=corr), particle_radii=radii)}
    out = {"tool": "bench_levelset_field", "particles": len(x), "workload": "dam break, r = 0.01, -l 2, -c 0.5", "card_before": card_before,
           "steps": a.steps, "warmup": a.warmup, "runs": []}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for mode in a.modes.split(","):
        if a.gradient and "corrected" in mode:
            continue
        mk = modes[mode]
        # the same mode's reconstruction: level-set stage time, grid points it evaluated, and the mesh for the near-mesh points
        # (on a context of its own, closed before the field is built: the reconstruction keeps tile buffers of a third of the memory)
        rctx = ss.Context(0)
        rec = ss.reconstruct_surface(x, context=rctx, with_debug=True, subdomain_grid_auto_disable=False, **kw, **mk)
        tiles = int(len(rec.subdomains["flat"]))
        nsd = rec.subdomain_grid.ncells_per_dim
        busiest = int(rec.subdomains["flat"][np.argmax(rec.subdomains["count"])])
        corner = np.array([busiest // (nsd[1] * nsd[2]), (busiest // nsd[2]) % nsd[1], busiest % nsd[2]], np.int64)
        S = 64
        ls_points = tiles * (S + 1) ** 3
        c = np.float32(rec.grid.cell_size)
        lo = np.asarray(rec.grid.aabb.min, np.float32)
        verts = rec.mesh.vertices
        ls_ms = float(rec.timings["levelset"])
        rng = np.random.default_rng(5)
        near = (verts + rng.uniform(-1, 1, verts.shape).astype(np.float32) * c).astype(np.float32)
        del rec
        rctx.close()
        # the field's query scratch grows with the largest point set and stays with its context: one context per mode
        ctx = ss.Context(0)
        t0 = time.perf_counter()
        f = ss.LevelSetField(x, context=ctx, **kw, **mk)
        create_ms = (time.perf_counter() - t0) * 1e3
        n = a.tiles * S
        first = np.clip(corner - a.tiles // 2, 0, np.maximum(np.asarray(nsd) - a.tiles, 0)) * S
        idx = np.stack(np.meshgrid(*[np.arange(n, dtype=np.int64)] * 3, indexing="ij"), -1).reshape(-1, 3) + first
        sets = {"tiles": (lo + idx.astype(np.float32) * c).astype(np.float32),
                "uniform": rng.uniform(f.grid.aabb.min, f.grid.aabb.max, (a.points, 3)).astype(np.float32),
                "near_mesh": near}
        run = {"mode": mode, "create_ms": round(create_ms, 2), "threshold": f.threshold, "levelset_stage_ms": round(ls_ms, 3),
               "levelset_grid_points": ls_points, "levelset_ns_per_grid_point": ls_ms * 1e6 / max(ls_points, 1), "queries": {}}
        for name, pts in sets.items():
            dev = torch.from_numpy(pts).cuda()
            torch.cuda.synchronize()
            extra = {"gradient": f.gradient} if a.gradient else {}
            if a.hessian:
                extra.update(hessian=f.hessian, curvature=f.curvature)
            for _ in range(a.warmup):
                v = f.evaluate(dev)
                for call in extra.values():
                    call(dev)
            ms, xms = [], {k: [] for k in extra}
            for _ in range(a.steps):
                ev0.record()
                v = f.evaluate(dev)
                ev1.record()
                torch.cuda.synchronize()
                ms.append(ev0.elapsed_time(ev1))
                for k, call in extra.items():
                    ev0.record()
                    r = call(dev)
                    ev1.record()
                    torch.cuda.synchronize()
                    xms[k].append(ev0.elapsed_time(ev1))
                    if k == "gradient":
                        gv, g = r
                    elif k == "hessian":
                        hv, hg = r[0], r[1]
                    del r
            best = min(ms)
            q = {"points": len(pts), "ms": [round(t, 3) for t in ms], "ns_per_point": best * 1e6 / max(len(pts), 1),
                 "inside_fraction": float((v > f.threshold).sum()) / max(len(pts), 1), "paths": f.paths}
            for k, t in xms.items():
                q[f"{k}_ms"] = [round(x, 3) for x in t]
                q[f"{k}_ns_per_point"] = min(t) * 1e6 / max(len(pts), 1)
            if a.gradient:
                q.update(values_equal=bool(torch.equal(gv, v)), zero_gradient_fraction=float((g == 0).all(1).float().mean()))
            if a.hessian:
                q.update(hessian_values_equal=bool(torch.equal(hv, v)), hessian_gradients_equal=bool(torch.equal(hg, g)))
                del hv, hg
            if a.gradient:
                del gv, g
            run["queries"][name] = q
            del dev, v
        f.close()
        ctx.close()
        out["runs"].append(run)
        sys.stderr.write(f"{mode}: create {create_ms:.1f} ms, " + ", ".join(f"{k} {q['ns_per_point']:.2f} ns/pt" + "".join(
            f" ({x} {q[x + '_ns_per_point']:.2f})" for x in ("gradient", "hessian", "curvature") if x + "_ns_per_point" in q)
            for k, q in run["queries"].items()) + "\n")
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
