"""Kernel time of Context.draw_aovs against the fast draw of the same image, alternating in one process: the 46-sphere
scene at 1280x720, spp 4, one frame, flags 0, device buffers (albedo, normal and ids for the AOV pass). Each step is timed
with the call's own tpt_last_kernel_ms (CUDA events around its kernels on the launching stream), L2 flushed (256 MiB fill)
between steps, as tools/bench_trace_rays.py does. Rounds alternate the two so that clock and neighbour drift hit both
alike. Prints one JSON line per round and a summary with the card name and power limit read in the same run.
    python tools/bench_aovs.py [--steps 200] [--rounds 5] [--warmup 10]"""
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
    ctx.set_spp(SPP)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    stream = torch.cuda.Stream(dev)
    torch.cuda.set_stream(stream)
    image = torch.zeros((H, W, 4), dtype=torch.float32, device=dev)
    albedo = torch.zeros((H, W, 4), dtype=torch.float32, device=dev)
    normal = torch.zeros((H, W, 4), dtype=torch.float32, device=dev)
    ids = torch.zeros((H, W), dtype=torch.int32, device=dev)
    calls = {
        "draw": lambda f: ctx.draw(f, 1, W, H, image, flags=0, mode=tpt.MODE_FAST, stream=stream.cuda_stream, want_rays=False),
        "draw_aovs": lambda f: ctx.draw_aovs(f, 1, W, H, albedo, normal, ids, flags=0, stream=stream.cuda_stream, want_rays=False),
    }
    for f in range(args.warmup):
        for call in calls.values():
            call(f)
    ms = {k: [] for k in calls}
    for r in range(args.rounds):
        for name, call in calls.items():
            ctx.read_ray_count(stream.cuda_stream)         # reset the accumulated counter
            step_ms = []
            for s in range(args.steps):
                flush.fill_(s & 0xFF)
                call(args.warmup + s)
                step_ms.append(ctx.last_kernel_ms())       # synchronises on the call's end event
            n = ctx.read_ray_count(stream.cuda_stream)
            ms[name].append(statistics.median(step_ms))
            print(json.dumps({"round": r, "call": name, "median_kernel_ms": ms[name][-1], "rays_per_step": n / args.steps,
                              "Mray_per_s": n / args.steps / (ms[name][-1] * 1e-3) / 1e6, "steps": args.steps}), flush=True)
    med = {k: statistics.median(v) for k, v in ms.items()}
    print(json.dumps({"card": card(), "median_kernel_ms": med, "aovs_over_draw": med["draw_aovs"] / med["draw"]}), flush=True)
    ctx.close()


if __name__ == "__main__":
    main()
