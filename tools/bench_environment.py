"""Cost of environment lighting (Context.set_environment), alternating in one process. Two arms, three settings each:
    settings  sky (no map: the reference's gradient sky), sky_map (scenes.sky_environment(1024, 512), 8 MB),
              random_4k (a 4096 x 2048 random map, 128 MB: larger than L2)
    draw      the fast draw of the 46-sphere scene, 1280 x 720 x 4 spp, into a device buffer (auto variant)
    rays      trace_rays over a 2048 x 1024 equirectangular panorama from the camera's origin, spp 4
Each round runs every (arm, setting) `--steps` times; the time of a call is tpt_last_kernel_ms (CUDA events around its
kernels) and its rays the call's own count; the summary gives Mray/s of the median call with the card name, power limit
and max SM clock read in the same run.
    python tools/bench_environment.py [--steps 50] [--rounds 3] [--warmup 5]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

W, H, SPP = 1280, 720, 4
PW, PH = 2048, 1024


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    return q or "unknown"


def panorama_rays(origin):
    """One ray per texel centre of a PW x PH lat-long panorama, in the map's own mapping (row 0 at the zenith)."""
    u, v = np.meshgrid(np.arange(PW) + 0.5, np.arange(PH) + 0.5)
    phi, theta = u / PW * 2 * np.pi - np.pi, v / PH * np.pi
    d = np.stack([np.sin(theta) * np.sin(phi), np.cos(theta), -np.sin(theta) * np.cos(phi)], -1).reshape(-1, 3)
    return np.concatenate([np.broadcast_to(origin, d.shape), d], 1).astype(np.float32)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    import torch
    import toypathtracer_b200 as tpt
    from toypathtracer_b200 import scenes

    dev = torch.device("cuda", 0)
    ctx = tpt.Context(0)
    sph, mats, cam, em = scenes.reference_scene(W, H)
    ctx.set_scene(sph, mats, cam, em)
    ctx.set_spp(SPP)
    img = torch.zeros((H, W, 4), dtype=torch.float32, device=dev)
    rays = torch.from_numpy(panorama_rays(cam["origin"][0].astype(np.float64))).to(dev)
    out = torch.empty((len(rays), 4), dtype=torch.float32, device=dev)
    maps = {"sky": None, "sky_map": scenes.sky_environment(1024, 512),
            "random_4k": torch.rand((2048, 4096, 4), generator=torch.Generator().manual_seed(3)).to(dev)}

    def call(arm):
        if arm == "draw":
            n = ctx.draw(0, 1, W, H, img, flags=0, mode=tpt.MODE_FAST)
        else:
            _, n = ctx.trace_rays(rays, spp=SPP, out=out)
        return n, ctx.last_kernel_ms()

    times = {(a, s): [] for a in ("draw", "rays") for s in maps}
    counts = {}
    for r in range(args.rounds):
        for s, m in maps.items():
            ctx.set_environment(m)
            for a in ("draw", "rays"):
                for i in range(args.warmup + args.steps):
                    n, ms = call(a)
                    if i >= args.warmup:
                        times[(a, s)].append(ms)
                        counts[(a, s)] = n
    res = {"card": card(), "workload": {"draw": f"46-sphere scene {W}x{H}x{SPP}spp fast draw (auto variant)",
                                        "rays": f"trace_rays over a {PW}x{PH} equirect panorama, spp {SPP}"},
           "results": {}}
    for (a, s), t in times.items():
        med = statistics.median(t)
        res["results"][f"{a}/{s}"] = {"median_ms": round(med, 4), "min_ms": round(min(t), 4), "max_ms": round(max(t), 4),
                                      "rays": counts[(a, s)], "mray_s": round(counts[(a, s)] / med / 1e3, 1)}
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
