"""The mirror-chain oracle of tests/mirror_chain.py checked before it judges any kernel: against a 60-digit decimal tracer
of the same float32 inputs, against a float32 emulation of the fast path with perturbed approximate operations on every
chain the GPU file relies on (this is what shows its well-conditioned verdict is conservative), against the CPU restatements of the reference's two estimators (the cpu rule: 11 segments
with a terminal emission; the gpu rule: 10 without), its coverage table against the kernels the library ships, and the
share of chains it decides, per scene (the thresholds the GPU file relies on)."""
import decimal
import os
import re
import shutil
import subprocess
import zlib

import numpy as np
import pytest

import furnace as F
import mirror_chain as mc
import test_sweep_oracle as so
from test_gpu_mirror_chains import COUNTS, IMAGE_COUNTS, SAMPLE_COUNTS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "toypathtracer_b200", "libtpt_b200.so")


# ---- 1. against high-precision arithmetic --------------------------------------------------------------------------
def decimal_chain(ray, sph, mats, mitsuba=False):
    """The ideal chain of one float32 ray in 60-digit decimal: exact roots, the normal (pos - s) * invRadius with the
    float32 invRadius, exact reflect and normalize. Returns (ids, value under the cpu rule, value under the gpu rule)."""
    Dc = lambda x: decimal.Decimal(float(x))
    centres, r2 = so.scene_arrays(sph)
    inv = sph["invRadius"]
    alb, emis = mats["albedo"], mats["emissive"]
    tmin, tmax = Dc(so.T_MIN), Dc(so.T_MAX)
    with decimal.localcontext() as lc:
        lc.prec = 60
        o = [Dc(v) for v in ray[:3]]
        d = [Dc(v) for v in ray[3:]]
        nd = sum(x * x for x in d).sqrt()
        d = [x / nd for x in d]
        T, col, ids = [Dc(1)] * 3, [Dc(0)] * 3, []
        v_gpu = None

        def sky(dy):
            if mitsuba:
                return [Dc(c) for c in F.MITSUBA_SKY]
            t = (dy + 1) / 2
            return [((1 - t) + t * Dc(c)) * Dc(0.3) for c in (0.5, 0.7, 1.0)]

        for k in range(11):
            best, bid = None, -1
            for j in range(len(r2)):
                co = [Dc(centres[j, i]) - o[i] for i in range(3)]
                nb = sum(co[i] * d[i] for i in range(3))
                disc = nb * nb - (sum(x * x for x in co) - Dc(r2[j]))
                if disc > 0:
                    sq = disc.sqrt()
                    t = nb - sq if nb - sq > tmin else nb + sq
                    if tmin < t < tmax and (best is None or t < best):
                        best, bid = t, j
            ids.append(bid)
            if bid < 0:
                col = [c + tt * s for c, tt, s in zip(col, T, sky(d[1]))]
                if v_gpu is None:
                    v_gpu = col
                break
            E = [Dc(e) for e in emis[bid]]
            if k == 10:
                col = [c + tt * e for c, tt, e in zip(col, T, E)]
                break
            pos = [o[i] + best * d[i] for i in range(3)]
            n = [(pos[i] - Dc(centres[bid, i])) * Dc(inv[bid]) for i in range(3)]
            dn = sum(d[i] * n[i] for i in range(3))
            refl = [d[i] - 2 * dn * n[i] for i in range(3)]
            rl = sum(x * x for x in refl).sqrt()
            out = [x / rl for x in refl]
            col = [c + tt * e for c, tt, e in zip(col, T, E)]
            if sum(out[i] * n[i] for i in range(3)) <= 0:
                v_gpu = v_gpu or col
                break
            T = [tt * Dc(a) for tt, a in zip(T, alb[bid])]
            if k == 9 and v_gpu is None:
                v_gpu = col
            o, d = pos, out
        return ids, np.array([float(c) for c in col]), np.array([float(c) for c in v_gpu])


def test_oracle_matches_decimal_tracer():
    """~200 well-conditioned chains of every length (the cap included) on three scenes: the same id sequence, and the
    decimal values within the oracle's tolerance under both rules."""
    checked, at_cap = 0, 0
    for count, layout, per_len in ((3, "compact", 8), (20, "spread", 7), (68, "compact", 6)):
        s, m, _ = mc.corridor(count, layout)
        rays = mc.candidate_rays(s, 1200, seed=3 + count)
        res = mc.chains(rays, s, m)
        for i in mc.pick_chains(res, per_len, rng_seed=count):
            ids, v_cpu, v_gpu = decimal_chain(rays[i], s, m)
            L = int(res["seg_cpu"][i])
            assert ids == list(res["ids"][i, :L]), (count, layout, i, ids, res["ids"][i])
            assert np.abs(v_cpu - res["v_cpu"][i]).max() <= res["tol_cpu"][i], (count, i, v_cpu, res["v_cpu"][i])
            assert np.abs(v_gpu - res["v_gpu"][i]).max() <= res["tol_gpu"][i], (count, i, v_gpu, res["v_gpu"][i])
            checked += 1
            at_cap += bool(res["cap"][i])
    assert checked >= 150 and at_cap >= 10, (checked, at_cap)


# ---- 2. bounds against a float32 emulation of the fast path ----------------------------------------------------------
# The fast kernels' arithmetic in float32, held in float64 arrays: every operation rounds its float64 result once to
# float32 (an FMA's product of two float32 values is exact in float64, so a*b + c rounds once, up to a double rounding the
# bounds do not depend on), and every approximate operation — rsqrt.approx in normalize, sqrt.approx in the sweep —
# returns its exact value times (1 + delta), delta drawn uniformly within the PTX ISA's documented bound (2^-22.9).
APPROX_REL = 2.0 ** -22.9


def _r(x):
    return np.asarray(x, np.float64).astype(np.float32).astype(np.float64)


def _fma(a, b, c):
    return _r(a * b + c)


def _dot(a, b):
    """dot(a, b) = a.x b.x + a.y b.y + a.z b.z as the compiler contracts it: fma(z, z', fma(y, y', x x'))."""
    return _fma(a[..., 2], b[..., 2], _fma(a[..., 1], b[..., 1], _r(a[..., 0] * b[..., 0])))


def _approx(x, rng):
    return _r(x * (1.0 + rng.uniform(-APPROX_REL, APPROX_REL, np.shape(x))))


def _normalize(v, rng):
    """M<false>::normalize: v * rsqrtf(dot(v, v))."""
    return _r(v * _approx(1.0 / np.sqrt(_dot(v, v)), rng)[..., None])


def _sweep(o, d, S, R2, K, form, rng, chunk=1 << 21):
    """Nearest hit of rays o, d [n, 3] against spheres S [m, 3], r^2 R2 [m] (form "reference": co = s - o, nb = co.d,
    -c = R - co.co; form "expanded": nb = s.d - o.d, c = K + o.o - 2 s.o with K = fl32(|s|^2 - r^2)), pass 1's rejection
    (discr < 0, or the centre behind with the origin outside, by sign bits), then pass 2 in ascending id order with
    t = nb - sqrt(discr), nb + sqrt(discr) when that is <= tMin, accepted when tMin < t < best. Returns ids (-1 sky), t."""
    n = len(o)
    ids, best = np.full(n, -1), np.full(n, so.T_MAX)
    step = max(1, chunk // max(len(R2), 1))
    for a in range(0, n, step):
        oo_, dd = o[a:a + step, None, :], d[a:a + step, None, :]
        if form == "reference":
            co = _r(S[None] - oo_)
            nb = _fma(co[..., 0], dd[..., 0], _fma(co[..., 1], dd[..., 1], _r(co[..., 2] * dd[..., 2])))
            negc = _fma(-co[..., 0], co[..., 0], _fma(-co[..., 1], co[..., 1], _fma(-co[..., 2], co[..., 2], R2[None])))
            c = -negc
        else:
            # FastHitterK: nod = -fma(ox, dx, fma(oy, dy, oz dz)), oo = fma(ox, ox, fma(oy, oy, oz oz))
            nod = -_fma(oo_[..., 0], dd[..., 0], _fma(oo_[..., 1], dd[..., 1], _r(oo_[..., 2] * dd[..., 2])))
            oo = _fma(oo_[..., 0], oo_[..., 0], _fma(oo_[..., 1], oo_[..., 1], _r(oo_[..., 2] * oo_[..., 2])))
            nb = _fma(S[None, :, 0], dd[..., 0], _fma(S[None, :, 1], dd[..., 1], _fma(S[None, :, 2], dd[..., 2], nod)))
            c = _fma(S[None, :, 0], -2 * oo_[..., 0], _fma(S[None, :, 1], -2 * oo_[..., 1],
                                                             _fma(S[None, :, 2], -2 * oo_[..., 2], _r(K[None] + oo))))
        discr = _fma(nb, nb, -c)
        rej = np.signbit(discr) | (np.signbit(nb) & ~np.signbit(c))
        ok = ~rej & (discr > 0)
        sq = _approx(np.sqrt(np.where(ok, discr, 0.0)), rng)
        t = _r(nb - sq)
        t = np.where(t <= so.T_MIN, _r(nb + sq), t)
        t = np.where(ok & (t > so.T_MIN) & (t < so.T_MAX), t, np.inf)
        w = np.argmin(t, 1)                   # the first minimum: strict '<' in ascending id order
        tw = t[np.arange(len(t)), w]
        hit = np.isfinite(tw)
        ids[a:a + step] = np.where(hit, w, -1)
        best[a:a + step] = np.where(hit, tw, so.T_MAX)
    return ids, best


def emulate_chains(rays, sph, mats, form, rng, mitsuba=False):
    """path_step's Metal branch (roughness 0) in emulated float32 for caller rays (normalised on load): per ray the
    hit ids [n, 11] (-2 past the end), and the value and segment count under the cpu rule (11 segments, terminal
    emission) and the gpu rule (10 segments, none). Form "reference" includes form 0's padded spheres (centre 10000^3,
    r^2 = 0, ids >= count): a hit on one is a wrong id."""
    count = len(sph)
    centres, r2 = so.scene_arrays(sph)
    S, R2 = centres.astype(np.float64), r2.astype(np.float64)
    simd = (count + 3) // 4 * 4
    if form == "reference" and simd != count:
        S = np.concatenate([S, np.full((simd - count, 3), so.PAD)])
        R2 = np.concatenate([R2, np.zeros(simd - count)])
    K = _r((S * S).sum(1) - R2)
    inv = sph["invRadius"].astype(np.float64)
    alb, emis = mats["albedo"].astype(np.float64), mats["emissive"].astype(np.float64)
    sky_c = _r(np.array([0.5, 0.7, 1.0]))
    n = len(rays)
    o = rays[:, :3].astype(np.float64)
    d = _normalize(rays[:, 3:].astype(np.float64), rng)
    thr, col = np.ones((n, 3)), np.zeros((n, 3))
    out = dict(ids=np.full((n, 11), -2), seg_cpu=np.zeros(n, int), seg_gpu=np.zeros(n, int), v_cpu=np.zeros((n, 3)),
               v_gpu=np.zeros((n, 3)))
    alive = np.ones(n, bool)
    for k in range(11):
        idx = np.nonzero(alive)[0]
        if not len(idx):
            break
        hid, t = _sweep(o[idx], d[idx], S, R2, K, form, rng)
        out["ids"][idx, k] = hid
        mi = idx[hid < 0]
        if len(mi):
            if mitsuba:
                sk = np.broadcast_to(_r(F.MITSUBA_SKY), (len(mi), 3))
            else:
                tt = _r(0.5 * _r(d[mi, 1] + 1.0))[:, None]
                sk = _r(_fma(tt, sky_c, _r(1.0 - tt)) * _r(0.3))
            v = _fma(thr[mi], sk, col[mi])
            out["v_cpu"][mi], out["seg_cpu"][mi] = v, k + 1
            if k < 10:
                out["v_gpu"][mi], out["seg_gpu"][mi] = v, k + 1
            alive[mi] = False
        hi, hid, t = idx[hid >= 0], hid[hid >= 0], t[hid >= 0]
        if not len(hi):
            continue
        if (hid >= count).any():              # a padded sphere: no material the oracle knows; its id already differs
            hid = np.minimum(hid, count - 1)
        E = emis[hid]
        if k == 10:
            out["v_cpu"][hi], out["seg_cpu"][hi] = _fma(thr[hi], E, col[hi]), 11
            alive[hi] = False
            break
        pos = _fma(d[hi], t[:, None], o[hi])
        nrm = _r(_r(pos - S[hid]) * inv[hid][:, None])
        dn2 = _r(2.0 * _dot(d[hi], nrm))
        refl = _fma(-dn2[:, None], nrm, d[hi])
        out_d = _normalize(refl, rng)
        up = _dot(out_d, nrm) > 0
        col[hi] = _fma(thr[hi], E, col[hi])
        ended = hi[~up]                       # the reflection points into the surface: Metal ends the path
        for rule in ("cpu", "gpu"):
            out[f"v_{rule}"][ended], out[f"seg_{rule}"][ended] = col[ended], k + 1
        alive[ended] = False
        go, hg = up, hi[up]
        if k == 9:
            out["v_gpu"][hg], out["seg_gpu"][hg] = col[hg], 10
        thr[hg] = _r(thr[hg] * alb[hid[go]])
        o[hg], d[hg] = pos[go], out_d[go]
    return out


EMULATED = sorted({(c, l) for c in COUNTS + IMAGE_COUNTS + SAMPLE_COUNTS for l in ("compact", "spread")}, key=str)


@pytest.mark.parametrize("count,layout", EMULATED, ids=[f"{c}-{l}" for c, l in EMULATED])
def test_oracle_bounds_hold_for_emulated_float32(count, layout):
    """Every chain the oracle calls well conditioned, in every scene the GPU file runs (1300 spheres, the largest
    stageable scene and chains at the cap included), three times with fresh perturbations of the approximate operations
    and in every sweep form the scene can run (both forms where it passes the expanded-form gate, else the reference
    form): the emulated float32 path hits the oracle's spheres in order, traces its segment counts, and its values lie
    within the oracle's tolerance under both rules."""
    s, m, _, rays, res = mc.oracle_scene(count, layout)
    well = res["well"]
    r, ora = rays[well], mc.subset(res, well)
    assert len(r) >= 20
    rng = np.random.default_rng(zlib.crc32(f"{count}-{layout}".encode()))
    forms = ("reference", "expanded") if so.gate_passes(s) else ("reference",)
    for form in forms:
        for draw in range(3):
            em = emulate_chains(r, s, m, form, rng)
            for rule in ("cpu", "gpu"):
                assert (em[f"seg_{rule}"] == ora[f"seg_{rule}"]).all(), (form, draw, rule)
                err = np.abs(em[f"v_{rule}"] - ora[f"v_{rule}"]).max(1)
                bad = err > ora[f"tol_{rule}"]
                assert not bad.any(), (form, draw, rule, int(bad.sum()), (err / ora[f"tol_{rule}"])[bad][:5])
            L = ora["seg_cpu"]
            mask = np.arange(11)[None] < L[:, None]
            assert (np.where(mask, em["ids"], -2) == np.where(mask, ora["ids"], -2)).all(), (form, draw)
    print(f"{count} {layout}: {len(r)} chains ({int(ora['cap'].sum())} at the cap) x {3 * len(forms)} emulated runs")


# ---- 3. the reference's semantics, through the CPU restatements ------------------------------------------------------
@pytest.fixture(scope="module")
def restatements(oracle):
    from oracle import nolight
    if not (os.path.exists(nolight.pyoracle.ORC_SO) and os.path.exists(nolight.pyoracle.RGO_SO)):
        nolight.build()
    return {("orc", 1): oracle.orc_render, ("rgo", 1): oracle.rgo_render,
            ("orc", 0): nolight.pyoracle.orc_render, ("rgo", 0): nolight.pyoracle.rgo_render}


@pytest.mark.parametrize("mitsuba", [0, 1])
@pytest.mark.parametrize("ls", [1, 0])
@pytest.mark.parametrize("which", ["orc", "rgo"])
def test_restatements_follow_the_chain_rules(restatements, which, ls, mitsuba):
    """A degenerate camera (every sample of every pixel the same ray) on chains of 1 segment, chains that reach the sky
    after k bounces and chains that reach the cap: the CPU path's restatement gives prev W + v (1 - W) with the cpu
    rule's v and w h spp segments rays per frame; the GPU shader's does so with the gpu rule (at most 10 segments, no
    terminal emission), which differs from the cpu rule's value on every chain that reaches the cap."""
    fn = restatements[(which, ls)]
    rule = "cpu" if which == "orc" else "gpu"
    s, m, _ = mc.corridor(46, "compact")
    rays = mc.candidate_rays(s, 1500, seed=5)
    res = mc.chains(rays, s, m, mitsuba=bool(mitsuba))
    w, h, spp = 3, 2, 2
    lengths, capped = set(), 0
    for L in range(1, 12):
        idx = np.nonzero(res["well"] & (res["seg_cpu"] == L))[0][:2]
        if L == 11:                          # chains whose 11th segment hits a sphere (the cap) and ones that miss
            idx = np.concatenate([np.nonzero(res["well"] & res["cap"])[0][:3], np.nonzero(res["well"] & (res["seg_cpu"] == L) & ~res["cap"])[0][:1]])
        for i in idx:
            cam, ray = mc.point_camera(rays[i, :3], rays[i, 3:])
            r = mc.chains(ray[None], s, m, mitsuba=bool(mitsuba))
            if not r["well"][0]:
                continue
            v, tol_v, seg = r[f"v_{rule}"][0], r[f"tol_{rule}"][0], int(r[f"seg_{rule}"][0])
            for f0, n, flags in ((0, 1, 0), (2, 3, 2)):
                prev = np.random.default_rng(i + f0).uniform(0, 1, (h, w, 4)).astype(np.float32)
                out = fn(s, m, cam, w, h, f0, n, flags=flags, spp=spp, mitsuba=bool(mitsuba), buf=prev.copy())
                buf, rays_pf = out[0], out[1]
                exp, tol = F.furnace_expect(prev[..., :3], v, f0, n, flags, spp)
                W, _ = F.frame_weights(f0, n, flags)
                tol = tol + (1 - W) * tol_v + 2.0 ** -22 * np.abs(exp)
                err = np.abs(buf[..., :3] - exp)
                assert (err <= tol).all(), (which, ls, mitsuba, L, float((err / tol).max()))
                assert rays_pf == [w * h * spp * seg] * n, (which, ls, L, rays_pf, seg)
            lengths.add(seg)
            if r["cap"][0]:
                capped += 1
                assert int(r["seg_gpu"][0]) == 10 and int(r["seg_cpu"][0]) == 11
                assert np.abs(r["v_cpu"][0] - r["v_gpu"][0]).max() > 50 * (r["tol_cpu"][0] + r["tol_gpu"][0])
    assert capped >= 1 and len(lengths) >= 9, (which, sorted(lengths), capped)
    print(f"{which} ls={ls} mitsuba={mitsuba}: segment counts {sorted(lengths)}, {capped} chains at the cap "
          f"({'11 segments, terminal emission' if rule == 'cpu' else '10 segments, no terminal emission'})")


# ---- 4. the coverage table against the binary -----------------------------------------------------------------------
def test_kernel_signature_decodes_the_mangling():
    import toypathtracer_b200 as tpt
    assert tpt.kernel_signature("_ZN3tpt12k_fast_queueILi128ELi6ELi4EEEvNS_10DrawParamsEPKh") == "k_fast_queue<128, 6, 4>"
    assert tpt.kernel_signature("_ZN3tpt14k_fast_samplesILi768ELi1ELi3ELb1EEEvNS_10DrawParamsE") == "k_fast_samples<768, 1, 3, true>"
    assert (tpt.kernel_signature("_ZN3tpt8k_refgpuILb1ENS_12RgSetupPlainILb1EEEEEvNS_10DrawParamsEPKh")
            == "k_refgpu<true, RgSetupPlain<true>>")
    assert tpt.kernel_signature("_ZN3tpt8k_refgpuILb0ENS_9RgSetupK2EEEvNS_10DrawParamsE") == "k_refgpu<false, RgSetupK2>"
    assert tpt.kernel_signature("_ZN3tpt11k_fast_megaENS_10DrawParamsEPKhNS_15SceneBlobLayoutEiij") == "k_fast_mega"
    assert tpt.kernel_signature("k_plain") == "k_plain"


@pytest.mark.skipif(shutil.which("cuobjdump") is None or not os.path.exists(LIB), reason="needs cuobjdump and the built library")
def test_coverage_table_lists_every_kernel_of_the_library():
    """Every __global__ function in libtpt_b200.so is in the coverage table (driven by a named GPU check, or excluded
    with a reason), and the table names nothing the library lacks."""
    import toypathtracer_b200 as tpt
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    shipped = {tpt.kernel_signature(n) for n in re.findall(r"Function : (\S+)", sass)}
    assert len(shipped) > 100
    assert shipped == set(mc.COVERAGE), (sorted(shipped - set(mc.COVERAGE)), sorted(set(mc.COVERAGE) - shipped))
    for name, why in mc.COVERAGE.items():
        assert why.startswith("excluded: ") or why in ("test_caller_rays", "test_images", "test_pixel_lists"), name


# ---- 5. what the oracle decides, per scene ---------------------------------------------------------------------------
SENSITIVITY = [(1, "compact"), (2, "compact"), (3, "spread"), (46, "compact"), (46, "spread"), (64, "compact"),
               (127, "spread"), (1300, "compact"), (1300, "spread")]


@pytest.mark.parametrize("count,layout", SENSITIVITY, ids=[f"{c}-{l}" for c, l in SENSITIVITY])
def test_oracle_decides_enough_chains(count, layout):
    """The well-conditioned share of the candidate rays, and the chains at the cap, with the candidate counts the GPU
    file uses: enough of every segment count for its per-length picks."""
    s, m, _ = mc.corridor(count, layout)
    rays = mc.candidate_rays(s, 1500 if count <= 1300 else 400, seed=17 + count)
    res = mc.chains(rays, s, m)
    w = res["well"]
    hist = np.bincount(res["seg_cpu"][w], minlength=12)[1:]
    print(f"{count} {layout}: well-conditioned {w.mean():.3f} of {len(rays)}, at the cap {int((w & res['cap']).sum())}, "
          f"segments 1..11: {hist.tolist()}")
    assert w.mean() > (0.3 if count >= 1000 else 0.6), w.mean()
    if count >= 2:
        assert (hist[:10] > 0).all() or count >= 1000, hist
        assert (w & res["cap"]).sum() >= (0 if count >= 1000 else 5)
