#!/usr/bin/env python3
"""Times the averaged-position surface (DESIGN.md §12), plain and with the Jacobian correction (§12.1), each also with per-particle radii
uniform in [0.8, 1.2] r (§12.2), beside the standard reconstruction on the same cloud and the same context, one GPU: device-resident
steps through splashsurf_b200.distributed.Runner (what bench.py times), the modes alternated `--rounds` times (`--modes` picks some).
Per mode and round: mean device ms per step over `--steps` timed steps after `--warmup` untimed ones, the stage times of the last step
(CUDA events) and the mesh size.  The card name and its power limit are read at the start and at the end.  Prints one JSON line;
writes nothing.

    python tools/bench_averaged.py                          # cfg-4: the 50 M-particle dam break
    python tools/bench_averaged.py --particles 10000000 --steps 3
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--particles", type=int, default=50_000_400, help="dam break with cfg-4 proportions (default: cfg-4 itself)")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--modes", default="plain,averaged,averaged_corrected,averaged_radii,averaged_corrected_radii")
    a = ap.parse_args()
    import numpy as np
    import torch
    import splashsurf_b200 as ss
    from splashsurf_b200 import distributed as ssd
    from splashsurf_b200 import synthetic as syn
    card_before = card()
    x = syn.dam_break_50m() if a.particles == 50_000_400 else syn.dam_break_scaled(a.particles, 0.01, 3)
    ctx = ss.Context(0)
    params = ss.make_params(particle_radius=0.01, smoothing_length=2.0, cube_size=0.5)
    corr = ss.AveragedSurface(correction=ss.JacobianCorrection())
    runners = {"plain": ssd.Runner(ctx, params, 1, 0, 0), "averaged": ssd.Runner(ctx, params, 1, 0, 0, averaged_surface=ss.AveragedSurface()),
               "averaged_corrected": ssd.Runner(ctx, params, 1, 0, 0, averaged_surface=corr),
               "averaged_radii": ssd.Runner(ctx, params, 1, 0, 0, averaged_surface=ss.AveragedSurface()),
               "averaged_corrected_radii": ssd.Runner(ctx, params, 1, 0, 0, averaged_surface=corr)}
    runners = {m: runners[m] for m in a.modes.split(",")}
    dev = torch.from_numpy(x).cuda()
    radii = torch.from_numpy((np.random.default_rng(4).uniform(0.8, 1.2, len(x)) * 0.01).astype(np.float32)).cuda()
    for m in ("averaged_radii", "averaged_corrected_radii"):
        if m in runners:
            runners[m].particle_radii = radii
    torch.cuda.synchronize()
    out = {"tool": "bench_averaged", "particles": len(x), "workload": "dam break, r = 0.01, -l 2, -c 0.5", "card_before": card_before,
           "steps": a.steps, "warmup": a.warmup, "runs": []}
    for rnd in range(a.rounds):
        for mode, runner in runners.items():
            for _ in range(a.warmup):
                runner.step(dev, copy_out=False)
            ms = []
            for _ in range(a.steps):
                res = runner.step(dev, copy_out=False)
                ms.append(res["device_ms"])
            out["runs"].append({"mode": mode, "round": rnd + 1, "ms_per_step": sum(ms) / len(ms), "ms_steps": [round(v, 2) for v in ms],
                                "mparticles_per_s": len(x) / (sum(ms) / len(ms) * 1e-3) / 1e6,
                                "stage_ms_last_step": {k: round(v, 3) for k, v in res["timings"].items() if isinstance(v, float)},
                                "vertices": int(res["nv"]), "triangles": int(res["nt"])})
            sys.stderr.write(f"{mode} round {rnd + 1}: {out['runs'][-1]['ms_per_step']:.1f} ms/step\n")
    out["card_after"] = card()
    ctx.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
