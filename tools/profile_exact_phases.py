#!/usr/bin/env python3
"""Phase breakdown of the exact level-set pass (k_exact_warp, 512-candidate tier) on the bench.py workload (cfg-4, the 50 M-particle
dam break, with bench.RECON_KW) through splashsurf_b200.distributed.Runner: `--warmup` untimed steps, then one step with the
instrumented kernel (Context.set_exact_phases), which sums clock64() cycles per warp and phase over every warp of its launches
(exact pass and fix-up pass of every tile batch).  The phases: run lookup, wait for the bulk copies, staging of the sort keys and
remainder splits, sort, per-sub-box list compaction, fold, stores.  The instrumented step is slower than a plain one and its
stage times are not reported.  Writes OUT/exact_phases.json with the card's name, power limit and maximum SM clock read before
and after.  Needs a CUDA device; there is no fallback.

    python tools/profile_exact_phases.py --out profiles/exact_phases
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--particles", type=int, default=50_000_400, help="target particle count of the dam break (default: cfg-4)")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", required=True, help="output directory (created)")
    ap.add_argument("--label", default="", help="free-form name of the build, stored in the JSON")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("profile_exact_phases.py needs a CUDA device")
    import bench
    import splashsurf_b200 as ss
    from splashsurf_b200 import distributed as ssd
    from profile_step import card
    card_before = card()
    x, desc = bench.make_cloud(a.particles)
    ctx = ss.Context(0)
    runner = ssd.Runner(ctx, ss.make_params(**bench.RECON_KW), 1, 0, 0)
    dev = torch.from_numpy(x).cuda()
    torch.cuda.synchronize()
    for _ in range(a.warmup):
        runner.step(dev, copy_out=False)
    torch.cuda.synchronize()
    ctx.set_exact_phases(True)
    runner.step(dev, copy_out=False)
    torch.cuda.synchronize()
    ph = ctx.exact_phases()
    ctx.set_exact_phases(False)
    ctx.close()
    bricks = ph.pop("bricks")
    total = sum(ph.values())
    phases = {k: {"warp_cycles": v, "share": round(v / total, 4) if total else 0.0,
                  "cycles_per_brick": round(v / bricks, 1) if bricks else 0.0} for k, v in ph.items()}
    out = {"tool": "profile_exact_phases", "label": a.label, "workload": desc, "particles": len(x), "recon_kw": bench.RECON_KW,
           "warmup": a.warmup, "card_before": card_before, "card_after": card(), "source_hash": ss.build.source_hash(),
           "bricks_timed": bricks, "warp_cycles_total": total,
           "cycles_per_brick": round(total / bricks, 1) if bricks else 0.0, "phases": phases}
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "exact_phases.json"), "w") as f:
        json.dump(out, f, indent=1)
    for k, v in phases.items():
        sys.stderr.write(f"{k:12s} {100 * v['share']:5.1f} %  {v['cycles_per_brick']:10.1f} cycles per brick\n")
    print(json.dumps({k: out[k] for k in ("label", "card_before", "bricks_timed", "cycles_per_brick")}))


if __name__ == "__main__":
    main()
