"""What "emission_texture_sampling" costs and what it buys, the option on and off alternating in one process, under a
hot-spot lamp: every emitter of the 46-sphere scene carries one 64 x 32 emission layer that is dark (0.05) except for a
2 x 2 patch of bright texels on its lower half.
    draw        the fast draw, 1280 x 720 x 4 spp, into a device buffer (auto variant)
    irradiance  trace_irradiance at 10^6 points on the ground around the scene (normal +y), spp 4
    quality     relative L2 against a high-spp reference (option on, streams disjoint from the arms') after equal GPU
                time: the frames (draw) or samples (irradiance) each setting fits into the time of --frames sampled calls
    set_emit    tpt_set_emission_textures time for 8 layers of 512 x 256 on 46 spheres, host and device texels (no
                option needed: run the script on two builds to compare them; a build without the option reports set_emit
                only)
Call time is tpt_last_kernel_ms (CUDA events around the call's kernels); the card name, power limit and max SM clock are
read in the same run.
    python tools/bench_emission_texture_sampling.py [--steps 30] [--rounds 3] [--warmup 3] [--frames 16] [--ref 512]"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

W, H, SPP = 1280, 720, 4
NPTS = 1_000_000


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    return q or "unknown"


def hot_spot_layer(w=64, h=32):
    t = np.full((1, h, w, 3), 0.05, np.float32)
    t[0, 22:24, 31:33] = (400.0, 320.0, 240.0)
    return t


def rel_l2(a, b):
    a, b = np.asarray(a, np.float64)[..., :3], np.asarray(b, np.float64)[..., :3]
    return float(np.sqrt(((a - b) ** 2).sum() / (b ** 2).sum()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--ref", type=int, default=512, help="reference: this many 4-spp frames / irradiance calls")
    args = ap.parse_args()
    import torch
    import toypathtracer_b200 as tpt
    from toypathtracer_b200 import scenes

    dev = torch.device("cuda", 0)
    ctx = tpt.Context(0)
    res = {"card": card(), "results": {}}
    sph, mats, cam, em = scenes.reference_scene(W, H)
    ctx.set_scene(sph, mats, cam, em)

    # set_emission_textures: 8 layers of 512 x 256, host and device texels (median of 3)
    big = np.random.default_rng(1).uniform(0, 2, (8, 256, 512, 4)).astype(np.float32)
    layers = (np.arange(len(sph)) % 8).astype(np.int32)
    for where, arg in (("host", big), ("device", torch.from_numpy(big).to(dev))):
        t = []
        for _ in range(3):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ctx.set_emission_textures(arg, layers)
            t.append((time.perf_counter() - t0) * 1e3)
        res["results"][f"set_emit/8x512x256/{where}"] = {"median_ms": round(statistics.median(t), 2)}
    ctx.set_emission_textures(None)
    try:
        ctx.set_option("emission_texture_sampling", 0)
    except tpt.TptError:
        print(json.dumps(res, indent=1))
        return

    emitters = (mats["emissive"] != 0).any(1)
    ctx.set_emission_textures(hot_spot_layer(), np.where(emitters, 0, -1).astype(np.int32))
    ctx.set_spp(SPP)
    img = torch.zeros((H, W, 4), dtype=torch.float32, device=dev)
    rng = np.random.default_rng(2)
    p = np.stack([rng.uniform(-4, 4, NPTS), np.zeros(NPTS), rng.uniform(-4, 2, NPTS)], 1)
    pts = torch.from_numpy(np.concatenate([p, np.broadcast_to([0.0, 1.0, 0.0], (NPTS, 3))], 1).astype(np.float32)).to(dev)
    out = torch.empty((NPTS, 4), dtype=torch.float32, device=dev)

    def call(arm, spp=SPP, frame=0):
        if arm == "draw":
            n = ctx.draw(frame, 1, W, H, img, flags=0, mode=tpt.MODE_FAST)
        else:
            _, n = ctx.trace_irradiance(pts, spp=spp, frame=frame, out=out)
        return n, ctx.last_kernel_ms()

    times, counts = {}, {}
    for _r in range(args.rounds):
        for on in (0, 1):
            ctx.set_option("emission_texture_sampling", on)
            for a in ("draw", "irradiance"):
                for i in range(args.warmup + args.steps):
                    n, ms = call(a)
                    if i >= args.warmup:
                        times.setdefault((a, on), []).append(ms)
                        counts[(a, on)] = n
    per = {}
    for (a, on), t in times.items():
        med = statistics.median(t)
        per[(a, on)] = med
        res["results"][f"{a}/{'on' if on else 'off'}"] = {"median_ms": round(med, 4), "min_ms": round(min(t), 4),
                                                          "max_ms": round(max(t), 4), "rays": counts[(a, on)],
                                                          "mray_s": round(counts[(a, on)] / med / 1e3, 1)}

    # quality at equal GPU time; the reference takes frames 10^6 + f, disjoint from the arms' frames 0 ..
    ctx.set_option("emission_texture_sampling", 1)
    q = {}
    for a in ("draw", "irradiance"):
        acc = None
        for f in range(args.ref):
            call(a, frame=1_000_000 + f)
            cur = (img if a == "draw" else out).double()
            acc = cur.clone() if acc is None else acc + cur
        ref = (acc / args.ref).cpu().numpy()
        budget = args.frames * per[(a, 1)]
        q[a] = {}
        for on in (0, 1):
            ctx.set_option("emission_texture_sampling", on)
            nf = max(1, int(round(budget / per[(a, on)])))
            if a == "draw":
                buf = torch.zeros((H, W, 4), dtype=torch.float32, device=dev)
                ctx.draw(0, nf, W, H, buf, flags=tpt.kFlagProgressive, mode=tpt.MODE_FAST)
                est = buf.cpu().numpy()
            else:
                _, _n = ctx.trace_irradiance(pts, spp=SPP * nf, frame=0, out=out)
                est = out.cpu().numpy()
            q[a]["on" if on else "off"] = {"calls": nf, "ms": round(ctx.last_kernel_ms(), 3), "rel_l2": round(rel_l2(est, ref), 5)}
        ctx.set_option("emission_texture_sampling", 1)
    res["results"]["quality_equal_time"] = q
    res["config"] = {"steps": args.steps, "rounds": args.rounds, "warmup": args.warmup, "frames": args.frames, "ref": args.ref}
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
