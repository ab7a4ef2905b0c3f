"""Kernel time of Context.trace_samples against the mean calls it extends, alternating in one process: the 46-sphere scene,
1280x720 camera_rays (one ray per pixel) at spp 4 into device buffers, and the points of the rays' primary hits (found once
with trace_aovs, with their sphere ids) for the irradiance arms. Arms:
    trace_rays, samples_rays (sums only), samples_rays_sq4 (sums and squares), trace_irradiance, samples_points (with
    squares), samples_list (rays, a shuffled list over half the inputs, with squares).
Each round runs every arm `--steps` times; the time of a call is tpt_last_kernel_ms (CUDA events around its kernels on the
launching stream), and the summary gives the median over all steps with the card name, power limit and max SM clock read
in the same run.
    python tools/bench_trace_samples.py [--steps 100] [--rounds 5] [--warmup 10]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

W, H, SPP = 1280, 720, 4


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    return q or "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    import torch
    import toypathtracer_b200 as tpt

    dev = torch.device("cuda", 0)
    ctx = tpt.Context(0)
    sph, mats, cam, em = tpt.reference_scene(W, H)
    ctx.set_scene(sph, mats, cam, em)
    stream = torch.cuda.Stream(dev)
    torch.cuda.set_stream(stream)
    rays = torch.from_numpy(tpt.camera_rays(cam, W, H, per_pixel=1, seed=0)).to(dev)
    n = len(rays)
    (_, nrm, ids), _ = ctx.trace_aovs(rays)
    hit = ids >= 0
    points = torch.cat([rays[hit, :3] + nrm[hit, 3:] * rays[hit, 3:], nrm[hit, :3]], 1).contiguous()
    point_ids = ids[hit].contiguous()
    half = torch.randperm(n, generator=torch.Generator().manual_seed(1))[: n // 2].to(torch.int32).to(dev)
    out = torch.empty((n, 4), dtype=torch.float32, device=dev)
    eout = torch.empty((len(points), 4), dtype=torch.float32, device=dev)
    s4, q4 = torch.zeros((n, 4), device=dev), torch.zeros((n, 4), device=dev)
    sp, qp = torch.zeros((len(points), 4), device=dev), torch.zeros((len(points), 4), device=dev)
    sl, ql = torch.zeros((len(half), 4), device=dev), torch.zeros((len(half), 4), device=dev)
    sc = stream.cuda_stream
    calls = {
        "trace_rays": lambda f: ctx.trace_rays(rays, spp=SPP, frame=f, out=out, stream=sc, want_rays=False),
        "samples_rays": lambda f: ctx.trace_samples(rays, None, False, None, SPP, f, s4, stream=sc, want_rays=False),
        "samples_rays_sq4": lambda f: ctx.trace_samples(rays, None, False, None, SPP, f, s4, q4, stream=sc, want_rays=False),
        "trace_irradiance": lambda f: ctx.trace_irradiance(points, point_ids, spp=SPP, frame=f, out=eout, stream=sc,
                                                           want_rays=False),
        "samples_points": lambda f: ctx.trace_samples(points, point_ids, True, None, SPP, f, sp, qp, stream=sc,
                                                      want_rays=False),
        "samples_list": lambda f: ctx.trace_samples(rays, None, False, half, SPP, f, sl, ql, stream=sc, want_rays=False),
    }
    for f in range(args.warmup):
        for call in calls.values():
            call(f)
    ms = {k: [] for k in calls}
    for r in range(args.rounds):
        for name, call in calls.items():
            got = []
            for s in range(args.steps):
                call(args.warmup + s)
                got.append(ctx.last_kernel_ms())
            ms[name] += got
            print(json.dumps({"round": r, "call": name, "median_ms": statistics.median(got)}), flush=True)
    med = {k: statistics.median(v) for k, v in ms.items()}
    print(json.dumps({"card": card(), "size": f"{W}x{H}", "spp": SPP, "points": len(points), "list": len(half),
                      "median_ms": med,
                      "ratios": {"samples_rays/trace_rays": med["samples_rays"] / med["trace_rays"],
                                 "samples_rays_sq4/trace_rays": med["samples_rays_sq4"] / med["trace_rays"],
                                 "samples_points/trace_irradiance": med["samples_points"] / med["trace_irradiance"],
                                 "samples_list/samples_rays_sq4": med["samples_list"] / med["samples_rays_sq4"]}}))


if __name__ == "__main__":
    main()
