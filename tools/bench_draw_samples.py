"""Throughput of Context.draw_samples over every pixel against the fast draw of the same image, alternating in one
process: the 46-sphere scene at 1280x720 (--width/--height: 3840x2160 runs pick_queue's 8-CTA instance), spp 4, device
buffers — the draw (one 4-spp frame, flags 0), draw_samples with sums only, and draw_samples with sums and second
moments. CUDA events around each call on the launching stream, L2
flushed (256 MiB fill) between steps outside the events, as tools/bench_trace_rays.py times. Rounds alternate the three
so that clock and neighbour drift hit all alike. Prints one JSON line per round and a summary with the card name and
power limit read in the same run.
    python tools/bench_draw_samples.py [--steps 200] [--rounds 5] [--warmup 10] [--width 1280 --height 720]
Mray/s counts every traced ray (path and shadow rays), as bench.py does."""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SPP = 4


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True).stdout.strip()
    return q or "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--width", type=int, default=1280)
    ap.add_argument("--height", type=int, default=720)
    args = ap.parse_args()
    W, H = args.width, args.height
    import torch
    import toypathtracer_b200 as tpt

    dev = torch.device("cuda", 0)
    ctx = tpt.Context(0)
    sph, mats, cam, em = tpt.reference_scene(W, H)
    ctx.set_scene(sph, mats, cam, em)
    ctx.set_spp(SPP)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    stream = torch.cuda.Stream(dev)
    torch.cuda.set_stream(stream)
    image = torch.zeros((H, W, 4), dtype=torch.float32, device=dev)
    sum4 = torch.zeros((W * H, 4), dtype=torch.float32, device=dev)
    sq4 = torch.zeros((W * H, 4), dtype=torch.float32, device=dev)
    s = stream.cuda_stream
    calls = {
        "draw": lambda f: ctx.draw(f, 1, W, H, image, flags=0, mode=tpt.MODE_FAST, stream=s, want_rays=False),
        "samples": lambda f: ctx.draw_samples(f, W, H, None, SPP, sum4, None, stream=s, want_rays=False),
        "samples_moments": lambda f: ctx.draw_samples(f, W, H, None, SPP, sum4, sq4, stream=s, want_rays=False),
    }
    for f in range(args.warmup):
        for call in calls.values():
            call(f)
    rates = {k: [] for k in calls}
    ms_step = {k: [] for k in calls}
    for r in range(args.rounds):
        for name, call in calls.items():
            ctx.read_ray_count(s)                          # reset the accumulated counter
            torch.cuda.synchronize(dev)
            evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
            for k in range(args.steps):
                flush.fill_(k & 0xFF)
                evs[k][0].record(stream)
                call(args.warmup + k)
                evs[k][1].record(stream)
            torch.cuda.synchronize(dev)
            ms = sum(a.elapsed_time(b) for a, b in evs)
            n = ctx.read_ray_count(s)
            rates[name].append(n / (ms * 1e-3) / 1e6)
            ms_step[name].append(ms / args.steps)
            print(json.dumps({"round": r, "call": name, "Mray_per_s": rates[name][-1], "ms_per_step": ms / args.steps,
                              "rays_per_step": n / args.steps, "steps": args.steps}), flush=True)
    med = {k: statistics.median(v) for k, v in rates.items()}
    print(json.dumps({"card": card(), "size": [W, H], "median_Mray_per_s": med,
                      "median_ms_per_step": {k: statistics.median(v) for k, v in ms_step.items()},
                      "samples_over_draw": med["samples"] / med["draw"],
                      "moments_over_draw": med["samples_moments"] / med["draw"]}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
