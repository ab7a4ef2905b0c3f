"""What "environment_sampling" costs and what it buys, sampling on and off alternating in one process, under a sun map:
scenes.sky_environment(2048, 1024) plus a 0.53 degree disc 30 degrees above the horizon that gives most of the horizontal
irradiance (built here, as the tests build theirs).
    draw        the fast draw of the 46-sphere scene, 1280 x 720 x 4 spp, into a device buffer (auto variant)
    irradiance  trace_irradiance at 10^6 points (the camera's origin, normals spread over the upper hemisphere), spp 4
    quality     relative L2 of the draw against a high-spp reference (sampling on, --ref-frames frames of 4 spp) after
                equal GPU time: the frames each setting fits into the time of --frames sampled frames
    set_env     tpt_set_environment time for 1024 x 512 and 4096 x 2048 maps, host and device (no option needed: run
                the script on two builds to compare them; a build without the option reports set_env only)
Call time is tpt_last_kernel_ms (CUDA events around the call's kernels); the card name, power limit and max SM clock are
read in the same run.
    python tools/bench_environment_sampling.py [--steps 30] [--rounds 3] [--warmup 3] [--frames 16] [--ref-frames 1024]"""
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


def sun_map(scenes, w=2048, h=1024):
    m = scenes.sky_environment(w, h)[..., :3].astype(np.float64)
    elev, rad = np.radians(30.0), np.radians(0.53) / 2
    s = np.array([0.3 * np.cos(elev), np.sin(elev), -np.sqrt(0.91) * np.cos(elev)])
    s /= np.linalg.norm(s)
    theta, phi = np.arccos(s[1]), np.arctan2(s[0], -s[2])
    j0, i0 = int(theta / np.pi * h), int((phi + np.pi) / (2 * np.pi) * w)
    sub = (np.arange(8) + 0.5) / 8
    radiance = 4.0 / (np.pi * rad ** 2 * s[1])          # 4 units of irradiance on a horizontal receiver
    for j in range(j0 - 4, j0 + 5):
        for i in range(i0 - 6, i0 + 7):
            uu, vv = np.meshgrid(i + sub, j + sub)
            ph, th = uu / w * 2 * np.pi - np.pi, vv / h * np.pi
            d = np.stack([np.sin(th) * np.sin(ph), np.cos(th), -np.sin(th) * np.cos(ph)], -1).reshape(-1, 3)
            m[j % h, i % w] += radiance * float((d @ s > np.cos(rad)).mean())
    return m.astype(np.float32)


def rel_l2(a, b):
    a, b = np.asarray(a, np.float64)[..., :3], np.asarray(b, np.float64)[..., :3]
    return float(np.sqrt(((a - b) ** 2).sum() / (b ** 2).sum()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--ref-frames", type=int, default=1024)
    args = ap.parse_args()
    import torch
    import toypathtracer_b200 as tpt
    from toypathtracer_b200 import scenes

    dev = torch.device("cuda", 0)
    ctx = tpt.Context(0)
    res = {"card": card(), "results": {}}

    # set_environment: host and device maps (median of 3)
    for (mw, mh) in ((1024, 512), (4096, 2048)):
        m = np.random.default_rng(1).uniform(0, 2, (mh, mw, 4)).astype(np.float32)
        for where, arg in (("host", m), ("device", torch.from_numpy(m).to(dev))):
            t = []
            for _ in range(3):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                ctx.set_environment(arg)
                t.append((time.perf_counter() - t0) * 1e3)
            res["results"][f"set_env/{mw}x{mh}/{where}"] = {"median_ms": round(statistics.median(t), 2)}
    ctx.set_environment(None)
    try:
        ctx.set_option("environment_sampling", 0)
    except tpt.TptError:
        print(json.dumps(res, indent=1))
        return

    sph, mats, cam, em = scenes.reference_scene(W, H)
    ctx.set_scene(sph, mats, cam, em)
    ctx.set_spp(SPP)
    ctx.set_environment(sun_map(scenes))
    img = torch.zeros((H, W, 4), dtype=torch.float32, device=dev)
    rng = np.random.default_rng(2)
    nrm = rng.normal(size=(NPTS, 3))
    nrm[:, 1] = np.abs(nrm[:, 1])
    nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    pts = torch.from_numpy(np.concatenate([np.broadcast_to(cam["origin"][0], (NPTS, 3)), nrm], 1).astype(np.float32)).to(dev)
    out = torch.empty((NPTS, 4), dtype=torch.float32, device=dev)

    def call(arm):
        if arm == "draw":
            n = ctx.draw(0, 1, W, H, img, flags=0, mode=tpt.MODE_FAST)
        else:
            _, n = ctx.trace_irradiance(pts, spp=SPP, out=out)
        return n, ctx.last_kernel_ms()

    times, counts = {}, {}
    for _r in range(args.rounds):
        for on in (0, 1):
            ctx.set_option("environment_sampling", on)
            for a in ("draw", "irradiance"):
                for i in range(args.warmup + args.steps):
                    n, ms = call(a)
                    if i >= args.warmup:
                        times.setdefault((a, on), []).append(ms)
                        counts[(a, on)] = n
    for (a, on), t in times.items():
        med = statistics.median(t)
        res["results"][f"{a}/{'on' if on else 'off'}"] = {"median_ms": round(med, 4), "min_ms": round(min(t), 4),
                                                          "max_ms": round(max(t), 4), "rays": counts[(a, on)],
                                                          "mray_s": round(counts[(a, on)] / med / 1e3, 1)}

    # quality at equal GPU time
    def frames(n):
        # frames [0, n) in one call: the progressive blend from frame 0 is their mean
        buf = torch.zeros((H, W, 4), dtype=torch.float32, device=dev)
        ctx.draw(0, n, W, H, buf, flags=tpt.kFlagProgressive, mode=tpt.MODE_FAST)
        return buf.cpu().numpy(), ctx.last_kernel_ms()

    ctx.set_option("environment_sampling", 1)
    acc = torch.zeros((H, W, 4), dtype=torch.float64, device=dev)
    ref_ms = 0.0
    for f in range(args.ref_frames):          # streams of frames 10^6 + f: disjoint from the arms' frames 0 ..
        ctx.draw(1_000_000 + f, 1, W, H, img, flags=0, mode=tpt.MODE_FAST)
        ref_ms += ctx.last_kernel_ms()
        acc += img.double()
    ref = (acc / args.ref_frames).cpu().numpy()
    per = {on: statistics.median(times[("draw", on)]) for on in (0, 1)}
    budget = args.frames * per[1]
    q = {}
    for on in (0, 1):
        ctx.set_option("environment_sampling", on)
        nf = max(1, int(round(budget / per[on])))
        img_on, ms = frames(nf)
        q["on" if on else "off"] = {"frames": nf, "ms": round(ms, 3), "rel_l2": round(rel_l2(img_on, ref), 5)}
    res["results"]["quality"] = {"reference": f"sampling on, {args.ref_frames} x {SPP} spp ({ref_ms:.1f} ms)", **q}
    res["workload"] = {"draw": f"46-sphere scene {W}x{H}x{SPP}spp fast draw (auto variant) under the sun map",
                       "irradiance": f"trace_irradiance at {NPTS} points, spp {SPP}"}
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
