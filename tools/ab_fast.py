"""A/B timing of one build of the fast kernel (TPT_LIB_PATH selects the library): 1280x720 x 4 spp per frame, device
buffer, L2 flushed between draws, CUDA events, for the variants given (-1 = the automatic choice), plus 4K x 16 spp.
Scenes: the 46-sphere reference scene, or the 4096-sphere stress scene.
    TPT_LIB_PATH=... python tools/ab_fast.py <label> [variants=3] [reps=200] [frames=1] [--scene stress] [--kform 2] [--no-4k]"""
import argparse, json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import toypathtracer_b200 as tpt

ap = argparse.ArgumentParser()
ap.add_argument("label")
ap.add_argument("variants", nargs="?", default="3")
ap.add_argument("reps", nargs="?", type=int, default=200)
ap.add_argument("frames", nargs="?", default="1")
ap.add_argument("--scene", choices=("reference", "stress"), default="reference")
ap.add_argument("--kform", type=int, default=2, help="the fast_kform option")
ap.add_argument("--no-4k", action="store_true")
args = ap.parse_args()
variants = [int(v) for v in args.variants.split(",")]
ctx = tpt.Context(0)
stream = torch.cuda.Stream(); torch.cuda.set_stream(stream); sh = stream.cuda_stream
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")


def scene(w, h):
    if args.scene == "stress":
        s = tpt.stress_scene(w, h, count=4096)
        return s[0], s[1], s[2], None
    return tpt.reference_scene(w, h)


def run(case, w, h, nf, variant, reps, flags=0):
    ctx.set_scene(*scene(w, h))
    ctx.set_option("fast_variant", variant); ctx.set_option("fast_kform", args.kform)
    img = torch.zeros((h, w, 4), dtype=torch.float32, device="cuda")
    for r in range(3):
        ctx.draw(r * nf, nf, w, h, img, flags=flags, mode=1, stream=sh, want_rays=False)
    ctx.read_ray_count(sh)
    ms = []
    for r in range(reps):
        flush.fill_(r & 0xFF)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        ctx.draw((3 + r) * nf, nf, w, h, img, flags=flags, mode=1, stream=sh, want_rays=False)
        e1.record(stream)
        torch.cuda.synchronize()
        ms.append(e0.elapsed_time(e1))
    rays = ctx.read_ray_count(sh)
    tot = sum(ms)
    print(json.dumps({"build": label, "scene": args.scene, "kform": args.kform, "case": case, "variant": variant,
                      "ms": tot / reps, "ms_min": min(ms), "mray_s": rays / tot / 1e3}), flush=True)


label = args.label
frames = [int(v) for v in args.frames.split(",")]
for v in variants:
    for nf in frames:
        run("720p x%dspp" % (4 * nf), 1280, 720, nf, v, max(args.reps // nf, 3), flags=0 if nf == 1 else 2)
if not args.no_4k:
    run("4K x16spp", 3840, 2160, 4, variants[0], max(args.reps // 20, 3), flags=2)
