"""A/B timing of the slab queue's pass-1 operand source in one process: "fast_kform" 2 (pair array in the kernel
parameter for scenes of <= 64 padded spheres, sweep form 4) against "fast_kform" 3 (the same pair array in shared memory,
form 2), in alternating rounds on the bench workload (46 spheres, 1280x720, 4 spp, device buffer, L2 flushed between
draws, CUDA events). Also: the 8-CTA instances (variant 9), 3840x2160 x 16 spp and the 4096-sphere scene (which never
takes form 4). Prints one JSON line per (case, form, round) and the card it ran on.
    python tools/ab_sweep_const.py [rounds=6] [draws=100]"""
import json, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import toypathtracer_b200 as tpt

rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 6
draws = int(sys.argv[2]) if len(sys.argv) > 2 else 100
q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                   capture_output=True, text=True).stdout.strip()
print(json.dumps({"gpu": q}), flush=True)

ctx = tpt.Context(0)
stream = torch.cuda.Stream(); torch.cuda.set_stream(stream); sh = stream.cuda_stream
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")


def timed(w, h, nf, variant, kform, n, flags):
    ctx.set_option("fast_variant", variant); ctx.set_option("fast_kform", kform)
    img = torch.zeros((h, w, 4), dtype=torch.float32, device="cuda")
    for r in range(2):
        ctx.draw(r * nf, nf, w, h, img, flags=flags, mode=1, stream=sh, want_rays=False)
    ctx.read_ray_count(sh)
    ms = []
    for r in range(n):
        flush.fill_(r & 0xFF)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        ctx.draw((2 + r) * nf, nf, w, h, img, flags=flags, mode=1, stream=sh, want_rays=False)
        e1.record(stream)
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    rays = ctx.read_ray_count(sh)
    return sum(ms) / n, rays / sum(ms) / 1e3


cases = [("720p x4spp", 1280, 720, 1, 3, 0, draws, tpt.reference_scene),
         ("720p x4spp 8-CTA", 1280, 720, 1, 9, 0, draws, tpt.reference_scene),
         ("4K x16spp", 3840, 2160, 4, 3, 2, max(draws // 20, 3), tpt.reference_scene),
         ("4096 spheres 720p x4spp", 1280, 720, 1, 3, 0, max(draws // 10, 3), tpt.stress_scene)]
for case, w, h, nf, variant, flags, n, scene in cases:
    ctx.set_scene(*scene(w, h))
    for rnd in range(rounds):
        for kform in ((2, 3) if rnd % 2 == 0 else (3, 2)):
            ms, mray = timed(w, h, nf, variant, kform, n, flags)
            print(json.dumps({"case": case, "fast_kform": kform, "round": rnd, "ms": round(ms, 4), "mray_s": round(mray, 1)}), flush=True)
