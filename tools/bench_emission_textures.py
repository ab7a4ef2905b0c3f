"""Cost of sphere emission textures (Context.set_emission_textures), alternating in one process. Cases:
    draw/default       the fast draw of the 46-sphere scene, 1280 x 720 x 4 spp, into a device buffer (auto variant),
                       untextured with the default options (what bench.py's `value` runs)
    draw/kform0        the same draw untextured with "fast_kform" 0: the instance the textured draws run, flags off
    draw/albedo        the same draw with albedo textures on every sphere (8 layers of 512 x 256, random, 32 MB)
    draw/emission      the same draw with emission textures on every emitter (8 layers of 512 x 256, random)
    draw/both          both sets at once
    irr/plain          trace_irradiance, spp 4, at the primary hits of the 1280 x 720 camera rays (trace_aovs), facing
                       the camera, each with its sphere's id
    irr/emission       the same with the emission textures set
Each round runs every case `--steps` times; the time of a call is tpt_last_kernel_ms (CUDA events around its kernels)
and its rays the call's own count; the summary gives the median call and its Mray/s with the card name, power limit
and max SM clock read in the same run.
    python tools/bench_emission_textures.py [--steps 50] [--rounds 3] [--warmup 5]"""
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
    gen = torch.Generator().manual_seed(3)
    alb = torch.rand((TL, TH, TW, 4), generator=gen).to(dev)
    emi = (2.0 * torch.rand((TL, TH, TW, 4), generator=gen)).to(dev)
    every = np.arange(len(sph), dtype=np.int32) % TL
    emitters = np.full(len(sph), -1, np.int32)
    lit = np.nonzero((mats["emissive"] != 0).any(1))[0]
    emitters[lit] = np.arange(len(lit)) % TL

    # the primary hits of the camera rays, facing the camera, on their spheres
    (_a, nrm, ids), _ = ctx.trace_aovs(rays)
    hit = ids >= 0
    r, nrm, ids = rays[hit], nrm[hit], ids[hit].contiguous()
    p = r[:, :3] + r[:, 3:] / r[:, 3:].norm(dim=1, keepdim=True) * nrm[:, 3:4]
    n = torch.where(((nrm[:, :3] * r[:, 3:]).sum(1, keepdim=True) > 0), -nrm[:, :3], nrm[:, :3])
    points = torch.cat([p, n], 1).contiguous()
    out = torch.empty((len(points), 4), dtype=torch.float32, device=dev)

    # case -> (albedo textures, emission textures, fast_kform, arm)
    cases = {"draw/default": (False, False, 2, "draw"), "draw/kform0": (False, False, 0, "draw"),
             "draw/albedo": (True, False, 2, "draw"), "draw/emission": (False, True, 2, "draw"),
             "draw/both": (True, True, 2, "draw"),
             "irr/plain": (False, False, 2, "irr"), "irr/emission": (False, True, 2, "irr")}

    def call(arm):
        if arm == "draw":
            k = ctx.draw(0, 1, W, H, img, flags=0, mode=tpt.MODE_FAST)
        else:
            _, k = ctx.trace_irradiance(points, ids, spp=SPP, out=out)
        return k, ctx.last_kernel_ms()

    times = {c: [] for c in cases}
    counts, kernels = {}, {}
    for _r in range(args.rounds):
        for c, (albedo, emission, kform, arm) in cases.items():
            ctx.set_textures(alb if albedo else None, every)
            ctx.set_emission_textures(emi if emission else None, emitters)
            ctx.set_option("fast_kform", kform)
            for i in range(args.warmup + args.steps):
                k, ms = call(arm)
                if i >= args.warmup:
                    times[c].append(ms)
                    counts[c] = k
            kernels[c] = ctx.last_kernels()
    res = {"card": card(), "workload": {"draw": f"46-sphere scene {W}x{H}x{SPP}spp fast draw (auto variant)",
                                        "irr": f"trace_irradiance at {len(points)} primary hits, spp {SPP}",
                                        "textures": f"{TL} layers of {TW}x{TH}; albedo on every sphere, emission on "
                                                    f"the {len(lit)} emitters"},
           "results": {}}
    for c, t in times.items():
        med = statistics.median(t)
        res["results"][c] = {"median_ms": round(med, 4), "min_ms": round(min(t), 4), "max_ms": round(max(t), 4),
                             "rays": counts[c], "mray_s": round(counts[c] / med / 1e3, 1), "kernels": kernels[c]}
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
