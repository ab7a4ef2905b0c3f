"""Throughput with the light_sampling option on and off, timed like bench.py's 1-GPU leg: the 46-sphere scene at
1280x720, one 4-spp frame (flags 0) per step into a device image, CUDA events around each draw on the launching
stream, L2 flushed (256 MiB fill) between steps outside the events. Prints one JSON line per (mode, light_sampling).
    python tools/bench_light_sampling.py [--steps 500] [--warmup 10]
Mray/s counts every traced ray (path and shadow rays), as bench.py does."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

W, H = 1280, 720


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=500)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    import torch
    import toypathtracer_b200 as tpt

    dev = torch.device("cuda", 0)
    ctx = tpt.Context(0)
    sph, mats, cam, em = tpt.reference_scene(W, H)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    stream = torch.cuda.Stream(dev)
    torch.cuda.set_stream(stream)
    image = torch.zeros((H, W, 4), dtype=torch.float32, device=dev)
    for mode_name, mode in (("fast", tpt.MODE_FAST), ("exact", tpt.MODE_EXACT)):
        for ls in (1, 0):
            ctx.set_option("light_sampling", ls)
            ctx.set_scene(sph, mats, cam, em)              # the option is a scene flag
            for s in range(args.warmup):
                ctx.draw(s, 1, W, H, image, flags=0, mode=mode, stream=stream.cuda_stream, want_rays=False)
            ctx.read_ray_count(stream.cuda_stream)         # reset the accumulated counter
            torch.cuda.synchronize(dev)
            evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
            for s in range(args.steps):
                flush.fill_(s & 0xFF)
                evs[s][0].record(stream)
                ctx.draw(args.warmup + s, 1, W, H, image, flags=0, mode=mode, stream=stream.cuda_stream, want_rays=False)
                evs[s][1].record(stream)
            torch.cuda.synchronize(dev)
            ms = sum(a.elapsed_time(b) for a, b in evs)
            rays = ctx.read_ray_count(stream.cuda_stream)
            print(json.dumps({"mode": mode_name, "light_sampling": ls, "Mray_per_s": rays / (ms * 1e-3) / 1e6,
                              "ms_per_frame": ms / args.steps, "rays_per_frame": rays / args.steps, "steps": args.steps}),
                  flush=True)
    ctx.set_option("light_sampling", 1)
    ctx.close()


if __name__ == "__main__":
    main()
