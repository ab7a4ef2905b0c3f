"""Throughput of Context.trace_rays and Context.trace_irradiance against the fast draw of the same image, alternating in one
process: the 46-sphere scene at 1280x720, camera_rays with one ray per pixel at spp 4 (the draw: one 4-spp frame, flags 0;
the irradiance arm: E at the rays' primary hits, found once with trace_aovs, with their sphere ids) into device buffers,
CUDA events around each call on the launching stream, L2 flushed (256 MiB fill) between steps outside the events, as
tools/bench_light_sampling.py times. Rounds alternate the calls so that clock and neighbour drift hit both alike. Prints one
JSON line per round and a summary with the card name and power limit read in the same run.
    python tools/bench_trace_rays.py [--steps 200] [--rounds 5] [--warmup 10]
Mray/s counts every traced ray (path and shadow rays), as bench.py does; an irradiance point is not a ray, so that arm
counts one ray fewer per sample than a camera ray that reaches the same point."""
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
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    import torch
    import toypathtracer_b200 as tpt

    dev = torch.device("cuda", 0)
    ctx = tpt.Context(0)
    sph, mats, cam, em = tpt.reference_scene(W, H)
    ctx.set_scene(sph, mats, cam, em)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    stream = torch.cuda.Stream(dev)
    torch.cuda.set_stream(stream)
    image = torch.zeros((H, W, 4), dtype=torch.float32, device=dev)
    rays = torch.from_numpy(tpt.camera_rays(cam, W, H, per_pixel=1, seed=0)).to(dev)
    out = torch.empty((W * H, 4), dtype=torch.float32, device=dev)
    (_, nrm, ids), _ = ctx.trace_aovs(rays)
    hit = ids >= 0
    points = torch.cat([rays[hit, :3] + nrm[hit, 3:] * rays[hit, 3:], nrm[hit, :3]], 1).contiguous()
    point_ids = ids[hit].contiguous()
    eout = torch.empty((len(points), 4), dtype=torch.float32, device=dev)
    calls = {
        "draw": lambda f: ctx.draw(f, 1, W, H, image, flags=0, mode=tpt.MODE_FAST, stream=stream.cuda_stream, want_rays=False),
        "trace_rays": lambda f: ctx.trace_rays(rays, spp=SPP, frame=f, out=out, stream=stream.cuda_stream, want_rays=False),
        "irradiance": lambda f: ctx.trace_irradiance(points, point_ids, spp=SPP, frame=f, out=eout, stream=stream.cuda_stream,
                                                     want_rays=False),
    }
    for f in range(args.warmup):
        for call in calls.values():
            call(f)
    rates = {k: [] for k in calls}
    for r in range(args.rounds):
        for name, call in calls.items():
            ctx.read_ray_count(stream.cuda_stream)         # reset the accumulated counter
            torch.cuda.synchronize(dev)
            evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
            for s in range(args.steps):
                flush.fill_(s & 0xFF)
                evs[s][0].record(stream)
                call(args.warmup + s)
                evs[s][1].record(stream)
            torch.cuda.synchronize(dev)
            ms = sum(a.elapsed_time(b) for a, b in evs)
            n = ctx.read_ray_count(stream.cuda_stream)
            rates[name].append(n / (ms * 1e-3) / 1e6)
            print(json.dumps({"round": r, "call": name, "Mray_per_s": rates[name][-1], "ms_per_step": ms / args.steps,
                              "rays_per_step": n / args.steps, "steps": args.steps}), flush=True)
    print(json.dumps({"card": card(), "median_Mray_per_s": {k: statistics.median(v) for k, v in rates.items()},
                      "trace_rays_over_draw": statistics.median(rates["trace_rays"]) / statistics.median(rates["draw"]),
                      "irradiance_points": len(points)}),
          flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
