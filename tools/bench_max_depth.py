"""Cost and effect of the fast mode's "max_depth" option, alternating in one process. Cases, on the 46-sphere scene:
    draw/default        the fast draw, 1280 x 720 x 4 spp, into a device buffer, default options (what bench.py's `value` runs)
    draw/kform0         the same draw with "fast_kform" 0: the instance a draw with max_depth other than 10 runs, capped at 10
    draw/depthN         the draw with max_depth N, N in 1, 3, 16, 64, 256
    medS/depthN         the draw with a scattering medium (sigma_s S in 4 and 16, g 0.6, no absorption) in the glass sphere
                        (id 7), max_depth N in 10, 64, 256; with it, the mean of trace_rays (spp 16) over the camera rays
                        whose first hit is sphere 7 (the sphere-7 pixel mean)
Each round runs every case `--steps` times; the time of a call is tpt_last_kernel_ms (CUDA events around its kernels)
and its rays the call's own count; the summary gives the median call's ms and Mray/s with the card name, power limit and
max SM clock read in the same run.
    python tools/bench_max_depth.py [--steps 100] [--rounds 1] [--warmup 5]"""
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
GLASS = 7


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    return q or "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=1)
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
    rays_all = scenes.camera_rays(cam, W, H)
    (_a, _n, ids), _ = ctx.trace_aovs(rays_all)
    rays7 = torch.from_numpy(rays_all[ids == GLASS]).to(dev)
    out = torch.empty((len(rays7), 4), dtype=torch.float32, device=dev)

    def medium(s):
        m = np.zeros((len(sph), 5), np.float32)
        m[GLASS] = (0.0, 0.0, 0.0, s, 0.6)
        return m

    # case -> (media, fast_kform, max_depth)
    cases = {"draw/default": (None, 2, 10), "draw/kform0": (None, 0, 10)}
    for n in (1, 3, 16, 64, 256):
        cases[f"draw/depth{n}"] = (None, 2, n)
    for s in (4, 16):
        for n in (10, 64, 256):
            cases[f"med{s}/depth{n}"] = (medium(float(s)), 2, n)

    times = {c: [] for c in cases}
    counts, kernels, means = {}, {}, {}
    for r in range(args.rounds):
        for c, (media, kform, n) in cases.items():
            ctx.set_media(media)
            ctx.set_option("fast_kform", kform)
            ctx.set_option("max_depth", n)
            for i in range(args.warmup + args.steps):
                rays = ctx.draw(0, 1, W, H, img, flags=0, mode=tpt.MODE_FAST)
                if i >= args.warmup:
                    times[c].append(ctx.last_kernel_ms())
                    counts[c] = rays
            kernels[c] = ctx.last_kernels()
            if media is not None and r == 0:
                acc = np.zeros(3)
                for f in range(4):
                    ctx.trace_rays(rays7, spp=16, frame=f, out=out)
                    acc += out[:, :3].double().mean(0).cpu().numpy()
                means[c] = [round(float(v), 5) for v in acc / 4]
    res = {"card": card(), "workload": f"46-sphere scene {W}x{H}x{SPP}spp fast draw (auto variant), medians of "
                                       f"{args.steps * args.rounds} calls; sphere7_mean: trace_rays spp 16 x 4 frames over "
                                       f"the {len(rays7)} camera rays whose first hit is sphere {GLASS}",
           "results": {}}
    for c, t in times.items():
        med = statistics.median(t)
        res["results"][c] = {"median_ms": round(med, 4), "min_ms": round(min(t), 4), "max_ms": round(max(t), 4),
                             "rays": counts[c], "mray_s": round(counts[c] / med / 1e3, 1), "kernels": kernels[c]}
        if c in means:
            res["results"][c]["sphere7_mean"] = means[c]
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
