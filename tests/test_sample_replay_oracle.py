"""CPU checks of the sample replay (tests/sample_replay.py), no GPU:
1. streams: fmix32 / pixel_seed / XorShift32 against a plain-integer restatement;
2. means: over many streams the replay's pixel means agree with the furnace closed forms B1 (light sampling on and off),
   B2, B3, B4 (cpu rule) and B5 within 5 se, independently of any kernel;
3. mirror chains: on mirror_chain's all-mirror scenes the replay's values, ray counts and verdicts agree with
   mirror_chain.chains, the replay being at most more conservative;
4. float32 emulation: path_step with every op rounded to float32 and every MUFU result perturbed within its assumed bound
   takes the replay's path (hit ids, draws, ray count) and lands within tolerance on every well-conditioned sample;
5. the replay decides enough: per scene a floor on the well fraction, and module-wide floors on well samples with each
   feature (depth cap, shadow ray reaching or missing its light, Fresnel reflection and refraction; total internal
   reflection has none, see FLAG_FLOOR; metal absorbed, terminal sky after >= 3 vertices, rough metal). The counts are
   printed."""
import numpy as np
import pytest

import furnace as F
import mirror_chain as mc
import sample_replay as sr

M32 = 0xFFFFFFFF


def _fmix_int(h):
    h ^= h >> 16; h = (h * 0x85EBCA6B) & M32; h ^= h >> 13; h = (h * 0xC2B2AE35) & M32; h ^= h >> 16
    return h


def test_streams_match_plain_integers():
    rng = np.random.default_rng(0)
    idx = np.concatenate([rng.integers(0, 2 ** 32, 200, dtype=np.uint64), [0, 1, 2 ** 32 - 1]]).astype(np.uint64)
    for frame in (0, 1, 77, 2 ** 31 + 5):
        got = sr.pixel_seed(idx, frame)
        want = [(_fmix_int((int(i) * 0x9E3779B9 + _fmix_int((frame + 0x7F4A7C15) & M32)) & M32) | 1) for i in idx]
        assert got.tolist() == want
    x = got.copy()
    for _ in range(5):
        x = sr.xorshift32(x)
        want = [(lambda v: (lambda v: (v ^ (v << 15)) & M32)((lambda v: v ^ (v >> 17))((v ^ (v << 13)) & M32)))(int(w))
                for w in want]
        assert x.tolist() == want
    assert sr.u01(np.array([0xFF000000, 0xFFFFFFFF, 0x00000001], np.uint32)).tolist() == [0.0, 1 - 2.0 ** -24, 2.0 ** -24]
    # list calls seed by input index: entry k of [5, 2] is input 5's or 2's stream
    assert sr.ray_seeds(np.array([5, 2]), 3, 1, 9).tolist() == [sr.pixel_seed(16, 9).item(), sr.pixel_seed(7, 9).item()]


# ---- 2. closed forms ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["b1_ls", "b1_nols", "b2", "b3_r06", "b4", "b5"])
def test_means_match_closed_forms(name):
    s, m, cam, em, w, h, e, bins, mitsuba, ls = F.b_case(name)
    sc = sr.Scene(s, m, em, mitsuba=mitsuba, ls=ls)
    y, x = np.divmod(np.arange(w * h), w)
    batches = []
    B, spp = 8, 6
    for b in range(B):
        acc = np.zeros((w * h, 3))
        for k in range(spp):
            r = sr.replay(sc, sr.draw_seeds(x, y, w, B * spp, b * spp + k, 1), camera=(cam, w, h, x, y))
            acc += r["v"]
        batches.append((acc / spp).reshape(h, w, 3))
    rep = F.check_bins(np.stack(batches), e, bins)
    print(name, [(int(b), np.round(mn, 5).tolist(), np.round(se, 6).tolist()) for b, mn, _, se in rep])


# ---- 3. mirror chains ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("count,layout", [(3, "spread"), (46, "compact"), (46, "spread"), (127, "compact")])
def test_agrees_with_mirror_chains(count, layout):
    s, m, em = mc.corridor(count, layout)
    rays = mc.candidate_rays(s, 800, seed=5 + count)
    ch = mc.chains(rays, s, m)
    for ls in (True, False):
        res = sr.replay(sr.Scene(s, m, em, ls=ls), sr.ray_seeds(np.arange(len(rays)), 1, 0, 0), rays=rays)
        assert not (res["well"] & ~ch["well"]).any(), "the replay may only be the more conservative"
        w = res["well"]
        assert w.mean() > 0.5 * ch["well"].mean()
        assert (res["rays"][w] == ch["seg_cpu"][w]).all()
        assert (res["draws"] == 0).all()                       # roughness 0: no draw at all
        assert (np.abs(res["v"][w] - ch["v_cpu"][w]).max(1) <= np.minimum(res["tol"][w], ch["tol_cpu"][w]) + 1e-12).all()


# ---- 4. float32 emulation, 5. floors -----------------------------------------------------------------------------------
EMU = [(3, "compact"), (40, "compact"), (40, "spread"), (120, "compact"), (300, "compact")]
WELL_FLOOR = {(3, "compact"): 0.3, (40, "compact"): 0.15, (40, "spread"): 0.1, (120, "compact"): 0.12,
              (300, "compact"): 0.08}
# about half of what the replay decides here (cap 949, shadow hit 645, occluded 173, reflect 34, refract 101, absorbed
# 126, sky after 3 vertices 2410, rough metal 521 well samples). Total internal reflection has no floor: inside a sphere
# the incidence angle never changes, so a ray that reflects totally once does so until the depth cap, and the verdict's
# error bound, which grows geometrically with each grazing internal bounce, calls none of those paths well conditioned.
# The emulation still checks that the replay and float32 take the same branches there.
FLAG_FLOOR = {"cap": 400, "shadow_hit": 300, "shadow_occluded": 80, "fresnel_reflect": 15, "fresnel_refract": 50,
              "metal_absorbed": 60, "sky_after_3": 1000, "rough_metal": 250}
_counts = {}


def _compare(res, e):
    L = max(res["trail"].shape[1], e["trail"].shape[1])
    a = np.full((len(res["v"]), L), -3); a[:, :res["trail"].shape[1]] = res["trail"]
    b = np.full((len(res["v"]), L), -3); b[:, :e["trail"].shape[1]] = e["trail"]
    return ((a != b) & (a != -4)).any(1) | (e["rays"] != res["rays"]) | (e["draws"] != res["draws"])


@pytest.mark.parametrize("count,layout", EMU)
def test_emulated_float32_stays_within_the_verdict(count, layout):
    s, m, em = sr.mixed_corridor(count, layout)
    rays = np.concatenate([sr.candidate_rays(s, 1500, seed=count), sr.inside_glass_rays(s, m, 300, seed=count)])
    x, y = np.divmod(np.arange(24 * 16), 24)[::-1]
    pts, self_ = sr.surface_points(s, m, em, 300, seed=count)
    for ls in (True, False):
        sc = sr.Scene(s, m, em, ls=ls)
        starts = [dict(rays=rays, state=sr.ray_seeds(np.arange(len(rays)), 1, 0, 1)),
                  dict(camera=(sr.lens_camera(), 24, 16, x, y), state=sr.draw_seeds(x, y, 24, 1, 0, 2)),
                  dict(points=pts, point_ids=self_, point_self=self_, state=sr.ray_seeds(np.arange(len(pts)), 1, 0, 3))]
        for j, kw in enumerate(starts):
            res = sr.replay(sc, **kw)
            for seed in range(3):
                e = sr.replay(sc, A=sr.Emulated(seed * 7 + j), **kw)
                div = _compare(res, e) & res["well"]
                err = np.abs(e["v"] - res["v"]).max(1)
                over = res["well"] & ~div & (err > res["tol"])
                assert not div.any() and not over.any(), (ls, j, seed, [sr.describe(res, i) for i in np.nonzero(div | over)[0][:4]])
            if j == 0 and ls:
                wf = float(res["well"].mean())
                print(f"{count} {layout}: well fraction {wf:.3f}, flags {sr.flag_counts(res)}")
                assert wf >= WELL_FLOOR[(count, layout)]
            c = _counts.setdefault("all", {})
            for k, v in sr.flag_counts(res).items():
                c[k] = c.get(k, 0) + v


def test_feature_floors():
    """Module-wide: every feature appears on enough well-conditioned samples (needs the emulation tests first)."""
    if "all" not in _counts:
        pytest.skip("needs test_emulated_float32_stays_within_the_verdict")
    print("well samples per feature:", _counts["all"])
    low = {k: (_counts["all"][k], f) for k, f in FLAG_FLOOR.items() if _counts["all"][k] < f}
    assert not low, low
