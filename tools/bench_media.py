"""Cost of media inside glass spheres (Context.set_media), alternating in one process. Cases, on the 46-sphere scene:
    draw/default       the fast draw, 1280 x 720 x 4 spp, into a device buffer, default options (what bench.py's `value` runs)
    draw/kform0        the same draw without media with "fast_kform" 0: the instance a draw with media runs
    draw/absorbing     the draw with an absorbing medium (sigma_a (0.6, 0.3, 0.1), sigma_s 0) in the glass sphere (id 7)
    draw/scattering    the draw with a scattering medium (sigma_a (0.6, 0.3, 0.1), sigma_s 4, g 0.6) in sphere 7
    rays7/kform0       trace_rays, spp 4, over the camera rays whose first hit is sphere 7, without media, "fast_kform" 0
    rays7/scattering   the same rays with the scattering medium
Each round runs every case `--steps` times; the time of a call is tpt_last_kernel_ms (CUDA events around its kernels)
and its rays the call's own count; the summary gives Mray/s of the median call with the card name, power limit and max
SM clock read in the same run.
    python tools/bench_media.py [--steps 50] [--rounds 3] [--warmup 5]"""
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
    rays_all = scenes.camera_rays(cam, W, H)
    ctx.set_option("fast_kform", 0)
    (_a, _n, ids), _ = ctx.trace_aovs(rays_all)
    rays7 = torch.from_numpy(rays_all[ids == GLASS]).to(dev)
    out = torch.empty((len(rays7), 4), dtype=torch.float32, device=dev)
    absorbing = np.zeros((len(sph), 5), np.float32)
    absorbing[GLASS] = (0.6, 0.3, 0.1, 0.0, 0.0)
    scattering = absorbing.copy()
    scattering[GLASS, 3:] = (4.0, 0.6)

    # case -> (media, fast_kform, arm)
    cases = {"draw/default": (None, 2, "draw"), "draw/kform0": (None, 0, "draw"), "draw/absorbing": (absorbing, 2, "draw"),
             "draw/scattering": (scattering, 2, "draw"), "rays7/kform0": (None, 0, "rays"),
             "rays7/scattering": (scattering, 2, "rays")}

    def call(arm):
        if arm == "draw":
            n = ctx.draw(0, 1, W, H, img, flags=0, mode=tpt.MODE_FAST)
        else:
            _, n = ctx.trace_rays(rays7, spp=SPP, out=out)
        return n, ctx.last_kernel_ms()

    times = {c: [] for c in cases}
    counts, kernels = {}, {}
    for r in range(args.rounds):
        for c, (media, kform, arm) in cases.items():
            ctx.set_media(media)
            ctx.set_option("fast_kform", kform)
            for i in range(args.warmup + args.steps):
                n, ms = call(arm)
                if i >= args.warmup:
                    times[c].append(ms)
                    counts[c] = n
            kernels[c] = ctx.last_kernels()
    res = {"card": card(), "workload": {"draw": f"46-sphere scene {W}x{H}x{SPP}spp fast draw (auto variant)",
                                        "rays7": f"trace_rays, spp {SPP}, over the {len(rays7)} camera rays whose first "
                                                 f"hit is sphere {GLASS}"},
           "results": {}}
    for c, t in times.items():
        med = statistics.median(t)
        res["results"][c] = {"median_ms": round(med, 4), "min_ms": round(min(t), 4), "max_ms": round(max(t), 4),
                             "rays": counts[c], "mray_s": round(counts[c] / med / 1e3, 1), "kernels": kernels[c]}
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
