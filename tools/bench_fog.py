"""Cost of fog between the spheres (Context.set_fog), alternating in one process. Cases, on the 46-sphere scene:
    draw/default       the fast draw, 1280 x 720 x 4 spp, into a device buffer, default options (what bench.py's `value` runs)
    draw/kform0        the same draw without fog with "fast_kform" 0: the instance a draw with fog runs
    draw/thin          the draw with a thin fog around the camera and both lights, B = {(0, 0, -1.5), 6}, sigma_a 0.01,
                       sigma_s 0.05, g 0.3
    draw/dense         the draw with a dense fog in the same ball, sigma_a 0.05, sigma_s 0.4, g 0.3
    draw/dense_nolight the dense fog with light sampling off
Each round runs every case `--steps` times; the time of a call is tpt_last_kernel_ms (CUDA events around its kernels)
and its rays the call's own count; the summary gives Mray/s of the median call with the card name, power limit and max
SM clock read in the same run.
    python tools/bench_fog.py [--steps 50] [--rounds 3] [--warmup 5]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

W, H, SPP = 1280, 720, 4
BALL = dict(centre=(0.0, 0.0, -1.5), radius=6.0)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    return q or "unknown"


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
    thin = dict(BALL, sigma_a=0.01, sigma_s=0.05, g=0.3)
    dense = dict(BALL, sigma_a=0.05, sigma_s=0.4, g=0.3)

    # case -> (fog, fast_kform, light_sampling)
    cases = {"draw/default": (None, 2, 1), "draw/kform0": (None, 0, 1), "draw/thin": (thin, 2, 1),
             "draw/dense": (dense, 2, 1), "draw/dense_nolight": (dense, 2, 0)}
    times = {c: [] for c in cases}
    counts, kernels = {}, {}
    for r in range(args.rounds):
        for c, (fog, kform, ls) in cases.items():
            if fog is None:
                ctx.set_fog(None)
            else:
                ctx.set_fog(**fog)
            ctx.set_option("fast_kform", kform)
            ctx.set_option("light_sampling", ls)
            ctx.set_scene(sph, mats, cam, em)      # light sampling is packed with the scene
            for i in range(args.warmup + args.steps):
                n = ctx.draw(0, 1, W, H, img, flags=0, mode=tpt.MODE_FAST)
                ms = ctx.last_kernel_ms()
                if i >= args.warmup:
                    times[c].append(ms)
                    counts[c] = n
            kernels[c] = ctx.last_kernels()
    res = {"card": card(), "workload": f"46-sphere scene {W}x{H}x{SPP}spp fast draw (auto variant)", "results": {}}
    for c, t in times.items():
        med = statistics.median(t)
        res["results"][c] = {"median_ms": round(med, 4), "min_ms": round(min(t), 4), "max_ms": round(max(t), 4),
                             "rays": counts[c], "mray_s": round(counts[c] / med / 1e3, 1), "kernels": kernels[c]}
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
