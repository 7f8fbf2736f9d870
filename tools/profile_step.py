#!/usr/bin/env python3
"""Per-kernel breakdown of one reconstruction step on the GPU: the bench.py workload (cfg-4, the 50 M-particle dam break, with
bench.RECON_KW) through splashsurf_b200.distributed.Runner, `--warmup` untimed steps, then one step under torch.profiler with CUDA
activities.  Writes OUT/profile_step.json: per kernel name the total device time, the number of launches and the share of the
step's kernel time; the stage times of the profiled step (CUDA events, `timings`), its brick counters, the work counters of one
extra instrumented step (levelset_cert_evals, levelset_pairs), and the card's name, power limit and maximum SM clock read before and
after.  Needs a CUDA device; there is no fallback.

    python tools/profile_step.py --out profiles/step
    python tools/profile_step.py --particles 10000000 --out /tmp/prof
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card() -> str:
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                          capture_output=True, text=True, timeout=30, check=True).stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--particles", type=int, default=50_000_400, help="target particle count of the dam break (default: cfg-4)")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", required=True, help="output directory (created)")
    a = ap.parse_args()
    import torch
    from torch.profiler import ProfilerActivity, profile
    if not torch.cuda.is_available():
        raise SystemExit("profile_step.py needs a CUDA device")
    import bench
    import splashsurf_b200 as ss
    from splashsurf_b200 import distributed as ssd
    card_before = card()
    x, desc = bench.make_cloud(a.particles)
    ctx = ss.Context(0)
    runner = ssd.Runner(ctx, ss.make_params(**bench.RECON_KW), 1, 0, 0)
    dev = torch.from_numpy(x).cuda()
    torch.cuda.synchronize()
    for _ in range(a.warmup):
        runner.step(dev, copy_out=False)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        res = runner.step(dev, copy_out=False)
        torch.cuda.synchronize()
    kernels = {}
    for ev in prof.events():
        if ev.device_type != torch.autograd.DeviceType.CUDA:
            continue
        k = kernels.setdefault(ev.name, {"device_ms": 0.0, "launches": 0})
        k["device_ms"] += ev.time_range.elapsed_us() / 1e3
        k["launches"] += 1
    total = sum(k["device_ms"] for k in kernels.values())
    for k in kernels.values():
        k["share"] = k["device_ms"] / total if total > 0 else 0.0
        k["device_ms"] = round(k["device_ms"], 4)
    kernels = dict(sorted(kernels.items(), key=lambda kv: -kv[1]["device_ms"]))
    tm = res["timings"]
    ctx.set_count_pairs(True)
    tc = runner.step(dev, copy_out=False)["timings"]
    ctx.set_count_pairs(False)
    out = {"tool": "profile_step", "workload": desc, "particles": len(x), "recon_kw": bench.RECON_KW, "warmup": a.warmup,
           "card_before": card_before, "card_after": card(), "device_ms_step": res["device_ms"], "kernel_ms_total": round(total, 4),
           "timings": {k: round(v, 4) for k, v in tm.items() if isinstance(v, float) and not k.startswith("bricks_")},
           "bricks": {k: int(v) for k, v in tm.items() if k.startswith("bricks_")},
           "levelset_cert_evals": float(tc.get("levelset_cert_evals", 0.0)), "levelset_pairs": float(tc["levelset_pairs"]),
           "kernels": kernels}
    os.makedirs(a.out, exist_ok=True)
    with open(os.path.join(a.out, "profile_step.json"), "w") as f:
        json.dump(out, f, indent=1)
    ctx.close()
    for name, k in list(kernels.items())[:25]:
        sys.stderr.write(f"{k['device_ms']:10.3f} ms {k['launches']:6d} x {100 * k['share']:5.1f} %  {name[:110]}\n")
    print(json.dumps({k: out[k] for k in ("card_before", "device_ms_step", "kernel_ms_total", "timings")}))


if __name__ == "__main__":
    main()
