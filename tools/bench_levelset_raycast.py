#!/usr/bin/env python3
"""Times the first-crossing ray cast of the level-set field (LevelSetField.raycast, DESIGN.md §15) on one GPU, for every level set:
standard, anisotropic, averaged, corrected, and both with per-particle radii uniform in [0.8, 1.2] r.  Two workloads per mode, rays
held on the device:
  * camera: a `--width` x `--height` pinhole camera outside the grid's box looking at its centre (ray-marched previews, visibility);
  * segments: `--segments` segments from the mode's mesh vertices, each moved by up to one cell, of length up to 2 cells (continuous
    collision of particles against the liquid).
Each call is timed with CUDA events around it, best of `--steps` after `--warmup` calls (the call ends in a device synchronise).
Per workload: ms, rays per second, rounds, the tiers of the last call, the hit fraction.  The card name, power limit and SM clock
are read at the start and at the end.  Prints one JSON line; with `--image FILE.ppm` also writes a normal-shaded picture of the
first mode's camera workload.

    python tools/bench_levelset_raycast.py                           # cfg-4: the 50 M-particle dam break
    python tools/bench_levelset_raycast.py --particles 1000000 --segments 1000000 --modes standard
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"unknown ({e})"


def camera(grid, width, height, np):
    """Pinhole camera at 1.2 box diagonals from the centre, looking at it, 40 degrees vertical field of view."""
    lo, hi = np.asarray(grid.aabb.min, np.float64), np.asarray(grid.aabb.max, np.float64)
    ctr, diag = 0.5 * (lo + hi), float(np.linalg.norm(hi - lo))
    eye = ctr + 1.2 * diag * np.array([0.55, 0.45, 0.7]) / np.linalg.norm([0.55, 0.45, 0.7])
    fwd = (ctr - eye) / np.linalg.norm(ctr - eye)
    right = np.cross(fwd, [0.0, 1.0, 0.0])
    right /= np.linalg.norm(right)
    up = np.cross(right, fwd)
    s = np.tan(np.radians(20.0))
    v, u = np.meshgrid((np.arange(height) + 0.5) / height * 2 - 1, (np.arange(width) + 0.5) / width * 2 - 1, indexing="ij")
    d = fwd + (u.reshape(-1, 1) * s * width / height) * right - (v.reshape(-1, 1) * s) * up
    return np.repeat(eye[None].astype(np.float32), len(d), 0), d.astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--particles", type=int, default=50_000_400, help="dam break with cfg-4 proportions (default: cfg-4 itself)")
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--segments", type=int, default=10_000_000)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--refine", type=int, default=24)
    ap.add_argument("--modes", default="standard,anisotropic,averaged,averaged_corrected,averaged_radii,averaged_corrected_radii")
    ap.add_argument("--image", default=None, help="write the first mode's camera hits, normal-shaded, as a binary PPM")
    a = ap.parse_args()
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
    out = {"tool": "bench_levelset_raycast", "particles": len(x), "workload": "dam break, r = 0.01, -l 2, -c 0.5", "card_before": card_before,
           "steps": a.steps, "warmup": a.warmup, "refine": a.refine, "runs": []}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    image_done = False
    for mode in a.modes.split(","):
        mk = modes[mode]
        # the mode's raw mesh for the segments, on a context of its own closed before the field is built
        rctx = ss.Context(0)
        rec = ss.reconstruct_surface(x, context=rctx, subdomain_grid_auto_disable=False, **kw, **mk)
        verts = rec.mesh.vertices
        del rec
        rctx.close()
        ctx = ss.Context(0)
        f = ss.LevelSetField(x, context=ctx, **kw, **mk)
        c = float(f.grid.cell_size)
        rng = np.random.default_rng(5)
        sel = rng.integers(0, len(verts), a.segments)
        so = (verts[sel] + rng.uniform(-1, 1, (a.segments, 3)).astype(np.float32) * np.float32(c)).astype(np.float32)
        u = rng.normal(size=(a.segments, 3))
        sd = (u / np.linalg.norm(u, axis=1, keepdims=True) * rng.uniform(0.05, 2.0, (a.segments, 1)) * c).astype(np.float32)
        del verts, sel, u
        co, cd = camera(f.grid, a.width, a.height, np)
        normals = "corrected" not in mode
        run = {"mode": mode, "threshold": f.threshold, "cell_size": c, "workloads": {}}
        for name, o, d, tm in (("camera", co, cd, None), ("segments", so, sd, 1.0)):
            od, dd = torch.from_numpy(o).cuda(), torch.from_numpy(d).cuda()
            torch.cuda.synchronize()
            for _ in range(a.warmup):
                hits = f.raycast(od, dd, t_max=tm, refine=a.refine, normals=normals)
            ms = []
            for _ in range(a.steps):
                del hits
                ev0.record()
                hits = f.raycast(od, dd, t_max=tm, refine=a.refine, normals=normals)
                ev1.record()
                torch.cuda.synchronize()
                ms.append(ev0.elapsed_time(ev1))
            st = hits.status
            best = min(ms)
            run["workloads"][name] = {"rays": len(o), "ms": [round(t, 3) for t in ms], "rays_per_s": len(o) / (best * 1e-3),
                                      "rounds": hits.rounds, "paths": f.paths,
                                      "hit_fraction": float((st.abs() == 1).float().mean()), "enter": int((st == 1).sum()),
                                      "leave": int((st == -1).sum()), "sample_limit": int((st == 2).sum())}
            if name == "camera" and a.image and normals and not image_done:
                n = hits.normals.cpu().numpy().reshape(a.height, a.width, 3)
                light = np.array([0.4, 0.8, 0.45]) / np.linalg.norm([0.4, 0.8, 0.45])
                shade = np.clip(np.nan_to_num(n @ light, nan=0.0), 0, 1) * 0.8 + 0.2
                hit = (hits.status.cpu().numpy().reshape(a.height, a.width) != 0) & np.isfinite(n).all(2)
                img = np.where(hit[..., None], (shade[..., None] * np.array([120, 170, 255])), np.array([24, 24, 28])).astype(np.uint8)
                with open(a.image, "wb") as fh:
                    fh.write(f"P6 {a.width} {a.height} 255\n".encode() + img.tobytes())
                image_done = True
            del hits, od, dd
        f.close()
        ctx.close()
        out["runs"].append(run)
        sys.stderr.write(f"{mode}: " + ", ".join(f"{k} {w['ms'][0] if len(w['ms']) == 1 else min(w['ms']):.2f} ms ({w['rays_per_s'] / 1e6:.1f} M rays/s, "
                                                 f"{w['rounds']} rounds, hits {w['hit_fraction']:.3f})" for k, w in run["workloads"].items()) + "\n")
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
