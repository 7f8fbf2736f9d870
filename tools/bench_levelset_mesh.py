#!/usr/bin/env python3
"""Times LevelSetField.mesh (DESIGN.md §16) on one GPU for every level set: standard, anisotropic, averaged, corrected, and both with
per-particle radii uniform in [0.8, 1.2] r.  Cases per mode:
  * grid: the whole grid at the field's cell (the reconstruction's raw mesh), beside the level-set + marching-cubes stage time of the
    same mode's reconstruct_surface (simd off for the standard level set);
  * splash / 2 and splash / 4: a region in the middle of the mesh (the 45 - 55 % quantiles of its vertices per axis) at cell / 2 and
    cell / 4.
Each call is timed with CUDA events around it, best of `--steps` after `--warmup` calls (the call ends in a device synchronise).
Per case: ms, triangles, the listed bricks per tier of the last call, batches, and the peak device memory of one more call (the
largest drop of the free memory, sampled every 0.2 ms from another thread, result included); for the regions also the route without
mesh(): evaluate() on the same lattice as a CUDA tensor plus marching_cubes on the values (host arrays), timed the same way.  The card name, power limit and SM
clock are read at the start and at the end.  Prints one JSON line.

    python tools/bench_levelset_mesh.py                              # cfg-4: the 50 M-particle dam break
    python tools/bench_levelset_mesh.py --particles 1000000 --modes standard
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader", "-i", "0"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"unknown ({e})"


def peak_bytes(torch, fn):
    """The largest drop of the free device memory while fn() runs."""
    free0 = torch.cuda.mem_get_info()[0]
    low = [free0]
    done = threading.Event()

    def sample():
        while not done.is_set():
            low[0] = min(low[0], torch.cuda.mem_get_info()[0])
            time.sleep(0.0002)
    t = threading.Thread(target=sample)
    t.start()
    try:
        r = fn()
    finally:
        done.set()
        t.join()
    return free0 - low[0], r


def evaluate_mc(torch, ss, f, m, cs, ev0, ev1, steps, max_points=200_000_000):
    """The route without mesh(): evaluate() on the same lattice built as a CUDA tensor, then marching_cubes on the values; best of
    `steps` after one warm-up, None where the lattice has more than max_points points, the error where the front end refuses."""
    ax = [torch.arange(int(m.index_min[d]), int(m.index_max[d]) + 1, device="cuda") for d in range(3)]
    if ax[0].numel() * ax[1].numel() * ax[2].numel() > max_points:
        return None
    gmin = torch.tensor(f.grid.aabb.min, dtype=torch.float32, device="cuda")

    def run():
        I = torch.stack(torch.meshgrid(*ax, indexing="ij"), dim=-1).reshape(-1, 3)
        pts = (I.to(torch.float32) * float(cs)) + gmin
        v = f.evaluate(pts).reshape(len(ax[0]), len(ax[1]), len(ax[2])).cpu().numpy()
        return ss.marching_cubes(v, iso_surface_threshold=f.threshold, cube_size=float(cs), translation=pts[0].cpu().numpy())
    try:
        run()
        ms = []
        for _ in range(steps):
            torch.cuda.synchronize()
            ev0.record()
            run()
            ev1.record()
            torch.cuda.synchronize()
            ms.append(ev0.elapsed_time(ev1))
        return min(ms)
    except ss.SplashsurfError as e:
        return f"refused: {e}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--particles", type=int, default=50_000_400, help="dam break with cfg-4 proportions (default: cfg-4 itself)")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--modes", default="standard,anisotropic,averaged,averaged_corrected,averaged_radii,averaged_corrected_radii")
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
    out = {"tool": "bench_levelset_mesh", "particles": len(x), "workload": "dam break, r = 0.01, -l 2, -c 0.5", "card_before": card_before,
           "steps": a.steps, "warmup": a.warmup, "runs": []}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for mode in a.modes.split(","):
        mk = modes[mode]
        rctx = ss.Context(0)
        rec = ss.reconstruct_surface(x, context=rctx, simd=False, subdomain_grid_auto_disable=False, **kw, **mk)
        t = rec.timings
        stage_ms = float(t.get("levelset", 0.0)) + float(t.get("marching_cubes", 0.0))
        q = np.quantile(rec.mesh.vertices, [0.45, 0.55], axis=0).astype(np.float32)
        del rec
        rctx.close()
        ctx = ss.Context(0)
        f = ss.LevelSetField(x, context=ctx, **kw, **mk)
        c = np.float32(f.grid.cell_size)
        run = {"mode": mode, "cell_size": float(c), "levelset_plus_mc_stage_ms": stage_ms, "cases": {}}
        for name, cs, box in (("grid", None, {}), ("splash/2", c / np.float32(2), dict(aabb_min=q[0], aabb_max=q[1])),
                              ("splash/4", c / np.float32(4), dict(aabb_min=q[0], aabb_max=q[1]))):
            m = None
            for _ in range(a.warmup):
                m = f.mesh(cs, **box)
            ms = []
            for _ in range(a.steps):
                m = None
                torch.cuda.synchronize()
                ev0.record()
                m = f.mesh(cs, **box)
                ev1.record()
                torch.cuda.synchronize()
                ms.append(ev0.elapsed_time(ev1))
            m = None
            peak, m = peak_bytes(torch, lambda: f.mesh(cs, **box))
            run["cases"][name] = {"ms": [round(v, 3) for v in ms], "best_ms": min(ms), "triangles": len(m.mesh.triangles),
                                  "paths": m.paths, "batches": m.batches, "index_min": m.index_min.tolist(), "index_max": m.index_max.tolist(),
                                  "peak_device_bytes": int(peak)}
            if name != "grid":
                run["cases"][name]["evaluate_marching_cubes_ms"] = evaluate_mc(torch, ss, f, m, cs, ev0, ev1, a.steps)
            del m
        f.close()
        ctx.close()
        out["runs"].append(run)
        sys.stderr.write(f"{mode}: stage {stage_ms:.1f} ms; " + ", ".join(f"{k} {w['best_ms']:.1f} ms ({w['triangles']} tris, {w['paths']}, "
                                                                         f"{w['batches']} batches, {w['peak_device_bytes'] / 1e9:.2f} GB)"
                                                                         for k, w in run["cases"].items()) + "\n")
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
