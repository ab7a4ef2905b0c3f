"""Cost of sphere albedo textures (Context.set_textures), alternating in one process. Cases:
    draw/textured      the fast draw of the 46-sphere scene, 1280 x 720 x 4 spp, into a device buffer (auto variant), every
                       sphere textured (8 layers of 512 x 256, random, 32 MB)
    draw/kform0        the same draw untextured with "fast_kform" 0: the instance the textured draw runs, with the flag off
    draw/default       the same draw untextured with the default options (what bench.py's `value` runs)
    rays/textured      trace_rays over the 1280 x 720 camera rays of the same scene, spp 4, textured
    rays/default       the same untextured, default options
Each round runs every case `--steps` times; the time of a call is tpt_last_kernel_ms (CUDA events around its kernels)
and its rays the call's own count; the summary gives Mray/s of the median call with the card name, power limit and max
SM clock read in the same run.
    python tools/bench_textures.py [--steps 50] [--rounds 3] [--warmup 5]"""
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
TW, TH, TL = 512, 256, 8


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
    rays = torch.from_numpy(scenes.camera_rays(cam, W, H)).to(dev)
    out = torch.empty((len(rays), 4), dtype=torch.float32, device=dev)
    tex = torch.rand((TL, TH, TW, 4), generator=torch.Generator().manual_seed(3)).to(dev)
    layers = np.arange(len(sph), dtype=np.int32) % TL

    # case -> (textured, fast_kform, arm)
    cases = {"draw/textured": (True, 2, "draw"), "draw/kform0": (False, 0, "draw"), "draw/default": (False, 2, "draw"),
             "rays/textured": (True, 2, "rays"), "rays/default": (False, 2, "rays")}

    def call(arm):
        if arm == "draw":
            n = ctx.draw(0, 1, W, H, img, flags=0, mode=tpt.MODE_FAST)
        else:
            _, n = ctx.trace_rays(rays, spp=SPP, out=out)
        return n, ctx.last_kernel_ms()

    times = {c: [] for c in cases}
    counts, kernels = {}, {}
    for r in range(args.rounds):
        for c, (textured, kform, arm) in cases.items():
            ctx.set_textures(tex if textured else None, layers)
            ctx.set_option("fast_kform", kform)
            for i in range(args.warmup + args.steps):
                n, ms = call(arm)
                if i >= args.warmup:
                    times[c].append(ms)
                    counts[c] = n
            kernels[c] = ctx.last_kernels()
    res = {"card": card(), "workload": {"draw": f"46-sphere scene {W}x{H}x{SPP}spp fast draw (auto variant)",
                                        "rays": f"trace_rays over the {W}x{H} camera rays, spp {SPP}",
                                        "textures": f"{TL} layers of {TW}x{TH}, every sphere textured"},
           "results": {}}
    for c, t in times.items():
        med = statistics.median(t)
        res["results"][c] = {"median_ms": round(med, 4), "min_ms": round(min(t), 4), "max_ms": round(max(t), 4),
                             "rays": counts[c], "mray_s": round(counts[c] / med / 1e3, 1), "kernels": kernels[c]}
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
