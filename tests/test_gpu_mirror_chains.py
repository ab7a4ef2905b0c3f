"""Every trace kernel instance against the float64 mirror-chain oracle of tests/mirror_chain.py, through the depth cap:
caller rays ray by ray (value, alpha, exact ray count) at every padded sphere-count tail, past 64 KB of blob and at the
largest stageable scene, for every sweep form the scene allows, with light sampling on and off, in short launches and in
launches long enough for the 8-CTA instances; images of a degenerate camera (one chain per draw) in every fast variant,
exact-mode lane form and reference-GPU mode; draw_samples' pixel lists. Every check asserts, through
Context.last_kernels(), which instance ran, and the union over the module must equal mirror_chain.COVERAGE: every trace kernel the
library ships is tied to an exact multi-bounce answer, or its exclusion is stated."""
import numpy as np
import pytest
import torch

import furnace as F
import mirror_chain as mc
import test_sweep_oracle as so
from conftest import bits_differ
from test_gpu_rays import _scaled
from test_gpu_sweep_oracle import BELOW

pytestmark = pytest.mark.gpu

COUNTS = [1, 2, 3] + BELOW + [65, 68, 127, 1300, "max"]
LAYOUTS = ("compact", "spread")
SLAB_PIX = 64                       # tpt_fast.cu kSlabPix
LONG_SLABS_PER_WARP = 48            # pick_queue: launches with at least this many slabs per warp take the 8-CTA instance

DRIVEN = {k for k, v in mc.COVERAGE.items() if not v.startswith("excluded")}


# ---- which instance the launchers pick (a restatement of tpt_fast.cu's pick rules, to check them) ---------------------
def _a16(x):
    return (x + 15) // 16 * 16


def _blob(count, n_lights):
    simd = (count + 3) // 4 * 4
    geom = _a16(simd * 16) + _a16(simd * 4) + _a16(max(n_lights, 1) * 32)
    total = geom + 2 * _a16((count + 1) * 16) + _a16((count + 1) * 4)
    return simd, (total if total <= 64 * 1024 else geom), total


def _smem(staged, pairs=0, buffers=0):
    return ((staged + 127) & ~127) + pairs + buffers if pairs + buffers else staged


def queue_kform(count, n_lights, kopt, gate):
    simd, staged, _ = _blob(count, n_lights)
    fit = _smem(staged, simd * 16, 24 * 2048) <= 200 * 1024
    if kopt == 0:
        return 0
    if gate:
        return 1 if kopt == 1 or not fit else 2
    return 3 if kopt >= 2 and fit else 0


def queue_instance(src, count, n_lights, kopt, gate, ls, variant=3, long=False, moments=False):
    simd, staged, total = _blob(count, n_lights)
    kf = queue_kform(count, n_lights, kopt, gate)
    if kf == 2 and kopt == 2 and simd <= 64 and src != "samples" and not (src == "queue" and variant == 4):
        kf = 4
    big = _smem(staged, simd * 16 if kf in (2, 3) else 0, 4 * 2048) > 36 * 1024 or staged != total
    eight = variant == 9 or (variant == 3 and long)
    if big:
        shape = (768, 1)
    elif kf in (2, 4) and eight:
        shape = (128, 8)
    elif src == "queue" and variant == 4:
        shape = (128, 7)
    else:
        shape = (128, 6)
    tail = f", {str(moments).lower()}" if src == "samples" else ""
    return f"k_fast_{src}{'' if ls else '_nolight'}<{shape[0]}, {shape[1]}, {kf}{tail}>"


def group_kform(count, kopt, gate):
    return 0 if not (gate and kopt) else (1 if kopt == 1 or (count + 3) // 4 * 4 > 1024 else 2)


def image_instances(mode, a, count, n_lights, kopt, gate, ls):
    """The trace kernel a draw launches: mode fast (a = variant), exact (a = exact_lanes), refgpu / refgpu_native."""
    if mode == "exact":
        lanes = 65 if a == 0 else a
        return {1: "k_trace_exact_flat<1>", 2: "k_trace_exact<1>", 8: "k_trace_exact<8>", 9: "k_trace_exact_flat<8>",
                32: "k_trace_exact<32>", 64: "k_trace_exact_split<1, 0, 1>", 65: "k_trace_exact_split<2, 0, 1>",
                66: "k_trace_exact_split<3, 0, 1>", 67: "k_trace_exact_split<4, 0, 1>", 70: "k_trace_exact_cluster",
                71: "k_trace_exact_split<2, 0, 2>"}[lanes]
    if mode == "refgpu":
        return "k_refgpu<true, RgSetupPlain<true>>"
    if mode == "refgpu_native":
        k2 = gate and kopt >= 2 and (count + 3) // 4 * 4 <= 1024
        return "k_refgpu<false, RgSetupK2>" if k2 else "k_refgpu<false, RgSetupPlain<false>>"
    v = a
    if v in (3, 4, 9):
        return queue_instance("queue", count, n_lights, kopt, gate, ls, variant=v)
    if v == 8:
        _, staged, total = _blob(count, n_lights)
        return f"k_fast_group{'' if ls else '_nolight'}<6, {group_kform(count, kopt, gate)}, {str(staged == total).lower()}>"
    if v == 5:
        return f"k_fast_tileq<6, {group_kform(count, kopt, gate)}>"
    return {0: "k_fast_mega", 1: "k_fast_persistent<2>", 2: "k_fast_persistent<3>", 6: "k_fast_wave<3>",
            7: "k_fast_wave<4>"}[v]


def ran(ctx, want, seen):
    got = ctx.last_kernels()
    seen.update(got)
    assert got == [want], (got, want)


# ---- scenes and their oracle, and the instances launched, once per module ---------------------------------------------
@pytest.fixture(scope="module")
def scenes():
    """scene(count, layout) -> (spheres, materials, light ids, well-conditioned rays, their oracle results), computed
    once per module (mirror_chain.oracle_scene: the same rays test_mirror_chain_oracle checks the oracle on)."""
    cache = {}

    def scene(count, layout):
        if (count, layout) not in cache:
            s, m, em, rays, res = mc.oracle_scene(count, layout)
            well = res["well"]
            cache[(count, layout)] = (s, m, em, rays[well], mc.subset(res, well))
        return cache[(count, layout)]
    return scene


@pytest.fixture(scope="module")
def seen():
    """The trace kernel instances the module's checks launched (test_coverage_is_complete compares them with the table)."""
    return set()


@pytest.fixture
def mctx(gpu_ctx):
    yield gpu_ctx
    for k, v in (("fast_kform", 2), ("mitsuba_compare", 0), ("light_sampling", 1), ("fast_variant", -1),
                 ("exact_lanes", 0)):
        gpu_ctx.set_option(k, v)
    gpu_ctx.set_spp(4)


def _num_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


# ---- 1. caller rays ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("count", COUNTS, ids=[str(c) for c in COUNTS])
def test_caller_rays(mctx, scenes, seen, count, layout):
    """Every well-conditioned ray at spp 2, raw and with rescaled directions, under every fast_kform and with light
    sampling on and off, then the same rays repeated into a launch of >= 48 slabs per warp at spp 64 (the 8-CTA
    instance where the scene runs forms 2 or 4): values within the oracle's tolerance, alpha 0, exact ray counts."""
    s, m, em, rays, res = scenes(count, layout)
    n = len(s)
    gate = so.gate_passes(s)
    assert len(rays) >= 20 and (res["seg_cpu"] >= 2).any()
    mctx.set_option("mitsuba_compare", 0)
    # >= 48 slabs of 64 rays per warp on every SM: n * spp >= 48 * SMs * 32 * 64
    rep_ = -(-LONG_SLABS_PER_WARP * _num_sms() * 32 * SLAB_PIX // 64 // len(rays)) + 1
    long_rays = torch.from_numpy(np.tile(rays, (rep_, 1))).cuda()
    for kopt in (0, 1, 2, 3):
        mctx.set_option("fast_kform", kopt)
        for ls in (1, 0):
            mctx.set_option("light_sampling", ls)
            mctx.set_scene(s, m, mc.point_camera(mc.CAMERA_O, (0, 0, -1))[0], em)
            for scaled in (False, True):
                r = _scaled(rays, 5 + kopt) if scaled else rays
                out, traced = mctx.trace_rays(torch.from_numpy(r).cuda(), spp=2, frame=kopt)
                ran(mctx, queue_instance("rays", n, len(em), kopt, gate and kopt != 0, ls), seen)
                out = out.cpu().numpy()
                err = np.abs(out[:, :3] - res["v_cpu"]).max(1)
                tol = res["tol_cpu"] + 4 * 2.0 ** -23 * np.abs(res["v_cpu"]).max(1)
                bad = err > tol
                assert not bad.any(), (count, layout, kopt, ls, scaled, int(bad.sum()), np.nonzero(bad)[0][:5],
                                       res["seg_cpu"][bad][:5], (err / tol)[bad][:5])
                assert (out[:, 3] == 0).all()
                assert traced == 2 * int(res["seg_cpu"].sum()), (count, layout, kopt, ls, traced, 2 * int(res["seg_cpu"].sum()))
            out, traced = mctx.trace_rays(long_rays, spp=64, frame=9)
            ran(mctx, queue_instance("rays", n, len(em), kopt, gate and kopt != 0, ls, long=True), seen)
            out = out.cpu().numpy().reshape(rep_, len(rays), 4)
            v, tol = res["v_cpu"], res["tol_cpu"] + 70 * 2.0 ** -23 * np.abs(res["v_cpu"]).max(1)
            assert (np.abs(out[..., :3] - v).max(2) <= tol).all(), (count, layout, kopt, ls, "long")
            assert (out[..., 3] == 0).all()
            assert traced == 64 * rep_ * int(res["seg_cpu"].sum()), (count, layout, kopt, ls, "long", traced)


# ---- 2. images of a degenerate camera ------------------------------------------------------------------------------
IMAGE_COUNTS = [1, 2, 3, 46, 64, 65, 127, "1000L", 1300]
FAST = [("fast", v) for v in range(10)]
EXACT = [("exact", a) for a in (0, 1, 2, 8, 9, 32, 64, 65, 66, 67, 70, 71)]
REFGPU = [("refgpu", 0), ("refgpu_native", 0)]
MODE_NUM = {"exact": 0, "fast": 1, "refgpu": 2, "refgpu_native": 3}
# w, h, spp, frame0, frames, flags, buffer, rows (row0, numRows, rowStep, packed)
SHAPES = [(7, 5, 2, 0, 1, 0, "device", None),
          (13, 3, 1, 3, 2, 2, "pageable", None),                # weighted prev
          (9, 6, 2, 1, 2, 2, "pinned", (1, 3, 2, 0)),           # row shard
          (11, 4, 1, 0, 1, 0, "device", (1, 2, 1, 1))]          # packed band


def _chain_cameras(s, m, rays, res, mitsuba, rule):
    """Degenerate cameras for well-conditioned chains of every segment count present: [(camera, oracle of its ray)]."""
    out = []
    for L in range(1, mc.CAP[rule] + 1):
        idx = np.nonzero(res[f"seg_{rule}"] == L)[0]
        for i in idx[:2]:
            cam, ray = mc.point_camera(rays[i, :3], rays[i, 3:])
            r = mc.chains(ray[None], s, m, mitsuba=mitsuba)
            if r["well"][0] and r[f"seg_{rule}"][0] == L:
                out.append((cam, mc.subset(r, 0)))
                break
    return out


def _buffer(kind, arr):
    if kind == "device":
        return torch.from_numpy(arr.copy()).cuda()
    if kind == "pinned":
        t = torch.empty(arr.shape, dtype=torch.float32, pin_memory=True)
        t.numpy()[...] = arr
        return t
    return arr.copy()


def _to_numpy(kind, buf):
    if kind == "device":
        torch.cuda.synchronize()
        return buf.cpu().numpy()
    return buf.numpy().copy() if kind == "pinned" else buf


def draw_chain(ctx, mode, a, cam, orc, shape, frames=None, seed=0):
    w, h, spp, f0, n, flags, bkind, rows = shape
    n = frames or n
    rule = "gpu" if mode.startswith("refgpu") else "cpu"
    ctx.set_camera(cam)
    ctx.set_spp(spp)
    row0, nrows, step, packed = rows if rows is not None else (0, h, 1, 0)
    ys = np.arange(row0, row0 + nrows * step, step)
    bh = nrows if packed else h
    prev = np.random.default_rng(seed).uniform(0, 1, (bh, w, 4)).astype(np.float32)
    buf = _buffer(bkind, prev)
    total = ctx.draw(f0, n, w, h, buf, flags=flags, mode=MODE_NUM[mode], rows=rows)
    got = _to_numpy(bkind, buf)
    drawn = np.arange(nrows) if packed else ys
    v = orc[f"v_{rule}"]
    exp, tol = F.furnace_expect(prev[drawn, :, :3], v, f0, n, flags, spp)
    W, _ = F.frame_weights(f0, n, flags)
    tol = tol + (1 - W) * orc[f"tol_{rule}"] + 2.0 ** -22 * np.abs(exp)
    err = np.abs(got[drawn, :, :3] - exp)
    fails = []
    if (err > tol).any():
        fails.append(f"{mode}{a} {shape}: worst {float((err / tol).max()):.3g} x tol, got {got[drawn][0, 0, :3]}, want {exp[0, 0]}")
    want = nrows * w * spp * n * int(orc[f"seg_{rule}"])
    if total != want:
        fails.append(f"{mode}{a} {shape}: rays {total} != {want}")
    untouched = np.setdiff1d(np.arange(bh), drawn)
    if untouched.size and bits_differ(got[untouched], prev[untouched]).any():
        fails.append(f"{mode}{a} {shape}: rows outside the draw changed")
    return fails


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("count", IMAGE_COUNTS, ids=[str(c) for c in IMAGE_COUNTS])
def test_images(mctx, scenes, seen, count, layout):
    """One chain per draw, chains of every segment count present in the scene, in every mode; each draw's pixels are
    prev * W + v * (1 - W), its ray count pixels x spp x frames x segments."""
    s, m, em, rays, res = scenes(count, layout)
    n = len(s)
    gate = so.gate_passes(s)
    fails = []
    for mitsuba in (0, 1):
        mctx.set_option("mitsuba_compare", mitsuba)
        cams = {rule: _chain_cameras(s, m, rays, res, bool(mitsuba), rule) for rule in ("cpu", "gpu")}
        want = 2 if n == 1 else 8
        assert len(cams["cpu"]) >= want and len(cams["gpu"]) >= want, (count, layout, len(cams["cpu"]), len(cams["gpu"]))
        if 2 <= n < 1000:
            assert max(int(o["seg_cpu"]) for _, o in cams["cpu"]) == mc.CAP["cpu"]
        modes = [(md, a, k, ls) for md, a in FAST for k in (0, 1, 2, 3) for ls in (1, 0)]
        modes += [(md, a, 2, 1) for md, a in EXACT] + [("exact", 0, 2, 0)]
        modes += [(md, a, k, ls) for md, a in REFGPU for k in (0, 2) for ls in (1, 0)]
        for j, (md, a, kopt, ls) in enumerate(modes):
            if md == "fast" and a not in (3, 4, 5, 8, 9) and kopt != 2:
                continue                          # variants 0-2, 6, 7 have one sweep of their own
            mctx.set_option("fast_kform", kopt)
            mctx.set_option("light_sampling", ls)
            if md == "fast":
                mctx.set_option("fast_variant", a)
            elif md == "exact":
                mctx.set_option("exact_lanes", a)
            cam0 = cams["gpu" if md.startswith("refgpu") else "cpu"]
            mctx.set_scene(s, m, cam0[0][0], em)
            for i, (cam, orc) in enumerate(cam0 if not mitsuba else cam0[::4]):
                shape = SHAPES[(i + j) % len(SHAPES)]
                fails += draw_chain(mctx, md, a, cam, orc, shape, seed=i + j)
                want = image_instances(md, a, n, len(em), kopt, gate and kopt != 0, ls)
                got = mctx.last_kernels()
                seen.update(got)
                if got != [want]:
                    fails.append(f"{md}{a} kform{kopt} ls{ls}: ran {got}, expected {want}")
    # 257 frames once (the fast mode's 256-frame launch split), on the longest chain
    mctx.set_option("mitsuba_compare", 0)
    mctx.set_option("fast_variant", 3); mctx.set_option("fast_kform", 2); mctx.set_option("light_sampling", 1)
    cam, orc = _chain_cameras(s, m, rays, res, False, "cpu")[-1]
    mctx.set_scene(s, m, cam, em)
    fails += draw_chain(mctx, "fast", 3, cam, orc, (5, 3, 1, 0, 257, 2, "device", None), seed=99)
    assert not fails, "\n".join([f"{count} {layout}"] + fails[:20])


# ---- 3. pixel lists ------------------------------------------------------------------------------------------------
SAMPLE_COUNTS = [3, 46, 127, 1300]


@pytest.mark.parametrize("layout", LAYOUTS)
@pytest.mark.parametrize("count", SAMPLE_COUNTS)
def test_pixel_lists(mctx, scenes, seen, count, layout):
    """draw_samples with the degenerate camera: sums spp v, squares spp v^2, exact ray counts, short and long lists."""
    s, m, em, rays, res = scenes(count, layout)
    gate = so.gate_passes(s)
    cam, orc = _chain_cameras(s, m, rays, res, False, "cpu")[-1]
    v, tv = orc["v_cpu"], orc["tol_cpu"]
    w, h = 37, 5
    for kopt in (0, 1, 2, 3):
        mctx.set_option("fast_kform", kopt)
        for ls in (1, 0):
            mctx.set_option("light_sampling", ls)
            mctx.set_scene(s, m, cam, em)
            for moments in (False, True):
                for long in ((False, True) if count < 1300 and kopt >= 2 and gate else (False,)):
                    if long:
                        W = 512
                        H = -(-LONG_SLABS_PER_WARP * _num_sms() * 32 * SLAB_PIX // 16 // W) + 1
                        pixels, spp = None, 16
                        npx = W * H
                    else:
                        W, H, spp = w, h, 3
                        pixels = np.random.default_rng(count).integers(0, W * H, 150).astype(np.int32)
                        npx = len(pixels)
                    sq = torch.zeros((npx, 4), dtype=torch.float32, device="cuda") if moments else None
                    s4 = torch.zeros((npx, 4), dtype=torch.float32, device="cuda")
                    pix = None if pixels is None else torch.from_numpy(pixels).cuda()
                    (s4, sq), traced = mctx.draw_samples(2, W, H, pix, spp, s4, sq)
                    ran(mctx, queue_instance("samples", len(s), len(em), kopt, gate and kopt != 0, ls, long=long,
                                             moments=moments), seen)
                    got = s4.cpu().numpy()
                    tol = spp * tv + spp * spp * 2.0 ** -23 * np.abs(v).max()
                    assert (np.abs(got[:, :3] - spp * v).max(1) <= tol).all(), (count, layout, kopt, ls, moments, long)
                    assert (got[:, 3] == spp).all()
                    if moments:
                        g2 = sq.cpu().numpy()
                        tol2 = 2 * spp * np.abs(v).max() * tv + spp * spp * 2.0 ** -22 * (v * v).max()
                        assert (np.abs(g2[:, :3] - spp * v * v).max(1) <= tol2).all()
                    assert traced == npx * spp * int(orc["seg_cpu"])


# ---- 4. coverage ---------------------------------------------------------------------------------------------------
def test_coverage_is_complete(request, seen):
    """The union of the instances the module's checks launched equals the driven part of the table: an instance the
    pick rules no longer reach, or one nobody ties to an answer, fails here. The union is only complete when every test
    of the module was selected and ran before this one; otherwise the check is skipped, not failed."""
    mine = [it for it in request.session.items if getattr(it, "module", None) is request.module]
    total = 2 * (len(COUNTS) + len(IMAGE_COUNTS) + len(SAMPLE_COUNTS)) + 1
    if len(mine) != total or mine[-1] is not request.node:
        pytest.skip(f"needs all {total} tests of the module, this one last ({len(mine)} selected)")
    missing = sorted(DRIVEN - seen)
    extra = sorted(seen - DRIVEN)
    assert not missing and not extra, (missing, extra)
