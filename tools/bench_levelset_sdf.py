#!/usr/bin/env python3
"""Times the narrow-band signed distance grid (LevelSetField.signed_distance, DESIGN.md §14) on one GPU, for every level set:
standard (simd off), anisotropic, averaged, corrected, and averaged with per-particle radii uniform in [0.8, 1.2] r.  Per mode the
raw mesh of reconstruct_surface is copied to the device, then the call (device mesh in, device arrays out) is timed with CUDA events
around it (it ends in a device synchronise), best of `--steps` after `--warmup`.  Reported: ms, ns per listed grid point, listed and
candidate bricks, (brick, triangle) pairs and passes, the tier counts, and the device memory the call held at its peak, measured in
one more call by sampling the free device memory.  The card name, power limit and SM clock are read at the start and at the
end.  Prints one JSON line; writes nothing.

    python tools/bench_levelset_sdf.py                            # cfg-4: the 50 M-particle dam break, band 3
    python tools/bench_levelset_sdf.py --particles 10000000 --modes standard,anisotropic
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def peak_device_bytes(call):
    """Runs call() while a thread samples the device's free memory (cudaMemGetInfo) every 0.2 ms; returns (result, the largest drop
    of free memory below its value before the call).  The library allocates outside torch's allocator, so this is what it held at
    its peak, up to what happened between two samples."""
    import threading
    import time
    import torch
    torch.cuda.synchronize()
    torch.cuda.empty_cache()                       # the result's tensors count too
    free0 = torch.cuda.mem_get_info()[0]
    low = [free0]
    done = threading.Event()

    def sample():
        while not done.is_set():
            low[0] = min(low[0], torch.cuda.mem_get_info()[0])
            time.sleep(0.0002)
    th = threading.Thread(target=sample)
    th.start()
    try:
        out = call()
        torch.cuda.synchronize()
    finally:
        done.set()
        th.join()
    return out, free0 - low[0]


def main():
    from bench_levelset_field import card
    ap = argparse.ArgumentParser()
    ap.add_argument("--particles", type=int, default=50_000_400, help="dam break with cfg-4 proportions (default: cfg-4 itself)")
    ap.add_argument("--band", type=int, default=3)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    # anisotropic: its cfg-4 mesh has 522 M triangles and the call runs out of device memory (DESIGN.md §14); pass it explicitly
    ap.add_argument("--modes", default="standard,averaged,averaged_corrected,averaged_radii")
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
             "averaged_radii": dict(averaged_surface=ss.AveragedSurface(), particle_radii=radii)}
    out = {"tool": "bench_levelset_sdf", "particles": len(x), "workload": "dam break, r = 0.01, -l 2, -c 0.5", "band": a.band,
           "card_before": card_before, "steps": a.steps, "warmup": a.warmup, "runs": []}
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for mode in a.modes.split(","):
        mk = modes[mode]
        rctx = ss.Context(0)
        rec = ss.reconstruct_surface(x, context=rctx, simd=False, subdomain_grid_auto_disable=False, **kw, **mk)
        verts = torch.from_numpy(rec.mesh.vertices).cuda()
        tris = torch.from_numpy(rec.mesh.triangles.astype(np.int32)).cuda()
        del rec
        rctx.close()
        ctx = ss.Context(0)
        f = ss.LevelSetField(x, context=ctx, **kw, **mk)
        torch.cuda.synchronize()
        free_gb = torch.cuda.mem_get_info()[0] / 2 ** 30
        sys.stderr.write(f"{mode}: {len(tris)} triangles, {free_gb:.1f} GB free before the call\n")
        for _ in range(a.warmup):
            g = f.signed_distance((verts, tris), band=a.band)
            del g
        ms = []
        for _ in range(a.steps):
            ev0.record()
            g = f.signed_distance((verts, tris), band=a.band)
            ev1.record()
            torch.cuda.synchronize()
            ms.append(ev0.elapsed_time(ev1))
        del g
        g, peak = peak_device_bytes(lambda: f.signed_distance((verts, tris), band=a.band))
        nl = int(g.brick_coords.shape[0])
        ncand = g.paths["shared"] + g.paths["global"]
        run = {"mode": mode, "vertices": int(len(verts)), "triangles": int(len(tris)), "ms": [round(t, 3) for t in ms],
               "best_ms": round(min(ms), 3), "listed_bricks": nl, "listed_points": nl * 512,
               "ns_per_listed_point": min(ms) * 1e6 / max(nl * 512, 1), "candidate_bricks": ncand, "pairs": g.passes["pairs"],
               "passes": g.passes["passes"], "tiers": g.paths, "grid_bricks": int(np.prod(g.brick_inside.shape)),
               "peak_device_mb_measured": round(peak / 2 ** 20, 1), "free_gb_before": round(free_gb, 1)}
        out["runs"].append(run)
        sys.stderr.write(f"{mode}: {min(ms):.2f} ms, {nl} listed / {ncand} candidate bricks, {g.passes}, tiers {g.paths}, "
                         f"peak {peak / 2 ** 20:.0f} MB\n")
        del g
        f.close()
        ctx.close()
        del verts, tris
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
