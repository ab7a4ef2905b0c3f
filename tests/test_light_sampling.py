"""DO_LIGHT_SAMPLING 0 (Config.h:24) as a runtime switch, without a GPU: the restatements with the switch off
(oracle/nolight.mk) against the reference compiled with it off (oracle/_ref/libtoyref_nolight.so,
libtoyref_small_mitsuba_nolight.so; stored results in tests/golden/ref_checks_nolight.json), the host build of the
integrator with kSceneNoLightSampling, and the SASS of the no-light-sampling fast kernels."""
import ctypes
import functools
import hashlib
import json
import os
import re
import shutil
import subprocess
import sys

import numpy as np
import pytest

from conftest import bits_differ
from test_host_sim import sim_render
from test_oracle import GOLD, golden_scene, image_digest, ref_scene_golden

K_SCENE_NO_LIGHT_SAMPLING = 2     # tpt_types.h SceneFlags
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="session")
def oracle_nl():
    """oracle/pyoracle.py's functions with DO_LIGHT_SAMPLING 0 (oracle/nolight.py)."""
    from oracle import nolight
    if not (os.path.exists(nolight.pyoracle.ORC_SO) and os.path.exists(nolight.pyoracle.RGO_SO)):
        nolight.build()
    return nolight.pyoracle


@functools.lru_cache(maxsize=None)
def nolight_checks():
    """What the reference compiled with DO_LIGHT_SAMPLING 0 produced (tests/golden/make_golden_refchecks_nolight.py)."""
    return json.load(open(os.path.join(GOLD, "ref_checks_nolight.json")))


def nolight_scene_golden(key):
    """The variant's GetSceneDesc export: byte for byte the stock build's (stored in ref_checks.json), which is checked."""
    arrays = ref_scene_golden(key.replace("nolight_", "").replace("_nolight", ""))
    s = nolight_checks()["scenes"][key]
    sha = lambda a: hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()
    assert [sha(a) for a in arrays[:3]] == [s["spheres"], s["materials"], s["camera"]], key
    assert list(arrays[3]) == s["emissives"], key
    return arrays


def assert_matches_nolight_render(key, buf, rays):
    """Per-frame ray counts and pixels (padded-sphere pixels excluded) equal the DO_LIGHT_SAMPLING 0 reference's `key`."""
    g = nolight_checks()["renders"][key]
    assert list(rays) == g["rays"], key
    assert image_digest(buf, g["pads"]) == g["digest"], key


@pytest.fixture(scope="session")
def host_sim_flags(tmp_path_factory):
    """tests/host_sim/exact_sim_flags.cpp: the host build of the integrator with settable scene flags."""
    so = str(tmp_path_factory.mktemp("host_sim_flags") / "exact_sim_flags.so")
    subprocess.run(["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-mfma", "-fPIC", "-shared", "-o", so,
                    os.path.join(ROOT, "tests", "host_sim", "exact_sim_flags.cpp"), "-lpthread", "-lm"], check=True)
    return {"exact_sim": ctypes.CDLL(so)}


@pytest.mark.parametrize("variant,mitsuba", [("nolight", False), ("small_mitsuba_nolight", True)])
def test_restatement_equals_reference_without_light_sampling(oracle, oracle_nl, variant, mitsuba):
    live = oracle.have_ref_variant(variant)
    for (w, h) in [(200, 120), (320, 180)]:
        sph, mats, cam, em = nolight_scene_golden(f"{variant}_{w}x{h}")
        for flags in (0, 2):
            obuf, orays, pads = oracle_nl.orc_render(sph, mats, cam, w, h, 0, 3, flags=flags, mitsuba=mitsuba)
            assert_matches_nolight_render(f"{variant}_{w}x{h}_f0_n3_flags{flags}", obuf, orays)
            if live:
                rbuf, rrays = oracle.ref_render(w, h, 0, 3, flags=flags, variant=variant)
                assert orays == rrays
                assert not bits_differ(obuf, rbuf, pads).any()


def test_restatement_without_light_sampling_720p(oracle_nl):
    sph, mats, cam, em = nolight_scene_golden("nolight_1280x720")
    obuf, orays, pads = oracle_nl.orc_render(sph, mats, cam, 1280, 720, 0, 3, flags=0)
    assert_matches_nolight_render("nolight_1280x720_f0_n3_flags0", obuf, orays)


@pytest.mark.parametrize("variant,stock", [("nolight", ""), ("small_mitsuba_nolight", "small_mitsuba")])
def test_nolight_scene_export_equals_stock(oracle, variant, stock):
    """UpdateTest still builds the emissive list: GetSceneDesc exports the same bytes with the switch off."""
    for (w, h) in [(200, 120), (320, 180)]:
        a = nolight_scene_golden(f"{variant}_{w}x{h}")       # asserts the stored hashes equal the stock export's
        b = ref_scene_golden(f"{stock + '_' if stock else ''}{w}x{h}")
        assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))
        if oracle.have_ref_variant(variant):
            live = oracle.ref_scene(w, h, variant=variant)
            assert all(x.tobytes() == y.tobytes() for x, y in zip(live, a))


def _small_scenes():
    import toypathtracer_b200 as tpt
    cam = tpt.make_camera((0, 1, 4), (0, 0, 0), (0, 1, 0), 45, 2.0, 0.05, 4)
    for n, lights in ((3, ()), (4, (1,)), (7, (0, 1, 2, 4, 6))):
        s = np.zeros(n, tpt.SPHERE_DTYPE); m = np.zeros(n, tpt.MATERIAL_DTYPE)
        for i in range(n):
            s[i] = ((i - n / 2, 0, 0), 0.45, 0)
            m[i] = (i % 3, (0.7, 0.6, 0.5), (4, 4, 4) if i in lights else (0, 0, 0), 0.1, 1.5)
        yield s, m, cam


@pytest.mark.parametrize("form", ["nested", "flat", "split"])
def test_integrator_without_light_sampling_matches_restatement(host_sim_flags, oracle_nl, form):
    """tpt_integrator.cuh (host build) with kSceneNoLightSampling: bit-identical to the restatement with the switch off
    on the golden scene, the 203-sphere runtime scene (padded spheres) and scenes with 0, 1 and 5 lights."""
    import toypathtracer_b200 as tpt
    kw = dict(flat=form == "flat", split=form == "split")
    host_sim_flags["exact_sim"].sim_set_scene_flags(K_SCENE_NO_LIGHT_SAMPLING)
    try:
        sph, mats, cam, em = golden_scene()
        obuf, orays, pads = oracle_nl.orc_render(sph, mats, cam, 192, 108, 0, 3, flags=2)
        buf, rays = sim_render(host_sim_flags, sph, mats, cam, 192, 108, 0, 3, 2, **kw)
        assert rays == orays and not bits_differ(buf, obuf, pads).any()
        s2, m2, c2, e2 = tpt.stress_scene(160, 90, count=203)
        obuf, orays, pads = oracle_nl.orc_render(s2, m2, c2, 160, 90, 3, 2, flags=2)
        buf, rays = sim_render(host_sim_flags, s2, m2, c2, 160, 90, 3, 2, 2, **kw)
        assert rays == orays and not bits_differ(buf, obuf, pads).any()
        for s3, m3, c3 in _small_scenes():
            obuf, orays, pads = oracle_nl.orc_render(s3, m3, c3, 64, 32, 0, 2, flags=2, spp=3)
            buf, rays = sim_render(host_sim_flags, s3, m3, c3, 64, 32, 0, 2, 2, spp=3, **kw)
            assert rays == orays and not bits_differ(buf, obuf, pads).any()
    finally:
        host_sim_flags["exact_sim"].sim_set_scene_flags(0)


def test_refgpu_oracle_without_light_sampling_is_the_same_estimator_statistically(oracle, oracle_nl):
    """Mirror of test_oracle.test_refgpu_oracle_is_the_same_estimator_statistically with both switches off."""
    sph, mats, cam, em = golden_scene()
    w, h, nf = 160, 90, 64
    a, ra, _ = oracle_nl.orc_render(sph, mats, cam, w, h, 0, nf, flags=2)
    c = a.copy()
    oracle_nl.orc_render(sph, mats, cam, w, h, nf, nf, flags=2, buf=c)
    a2 = 2.0 * c[..., :3].astype(np.float64) - a[..., :3]
    b, rb = oracle_nl.rgo_render(sph, mats, cam, w, h, 0, nf, flags=2)
    assert (b[..., 3] == 1).all()
    rl2 = lambda x, y: float(np.sqrt(((x.astype(np.float64) - y) ** 2).sum() / (y.astype(np.float64) ** 2).sum()))
    floor = rl2(a2, a[..., :3])
    assert rl2(b[..., :3], a[..., :3]) < 1.15 * floor
    assert 0.985 < sum(rb) / sum(ra) <= 1.0005
    ma, mb = a[..., :3].reshape(-1, 3).mean(0), b[..., :3].reshape(-1, 3).mean(0)
    assert (np.abs(ma - mb) < 0.01 * ma).all(), (ma, mb)
    # and it is a different image from the light-sampled one: no shadow rays at all
    _, rls, _ = oracle.orc_render(sph, mats, cam, w, h, 0, 2, flags=2)
    assert sum(ra[:2]) < 0.6 * sum(rls)


def _res_usage(lib, demangle):
    """{demangled kernel name: (registers, stack bytes)} from cuobjdump -res-usage."""
    out = subprocess.run(["cuobjdump", "-res-usage", lib], capture_output=True, text=True, check=True).stdout
    res, cur = {}, None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            cur = demangle(m.group(1))
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+)", line)
        if m and cur:
            res[cur] = (int(m.group(1)), int(m.group(2)))
    return res


LIB = os.path.join(ROOT, "toypathtracer_b200", "libtpt_b200.so")


@pytest.mark.skipif(shutil.which("cuobjdump") is None or not os.path.exists(LIB), reason="needs cuobjdump and the built library")
def test_nolight_fast_kernels_sass():
    """The no-light-sampling twins of the queue / group kernels exist for every instance the launcher can pick, stage the
    scene with TMA (UBLKCP), do not spill and use no more registers than their light-sampling twins."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import sass_counts
    rows = {name: cnt for name, n, cnt in sass_counts.kernel_counts(LIB)}
    res = _res_usage(LIB, sass_counts.demangle)
    twins = [n for n in rows if n.startswith("k_fast_queue_nolight<") or n.startswith("k_fast_group_nolight<")]
    for inst in ["k_fast_queue_nolight<128, 6, %d>" % k for k in range(4)] + ["k_fast_queue_nolight<128, 8, 2>"] + \
                ["k_fast_queue_nolight<768, 1, %d>" % k for k in range(4)] + \
                ["k_fast_group_nolight<6, %d, %d>" % (k, a) for k in range(3) for a in (0, 1)]:
        assert inst in twins, inst
    for name in twins:
        assert rows[name]["UBLKCP"] > 0, name
        twin = name.replace("_nolight", "")
        assert twin in rows, twin
        reg, stack = res[name]
        assert stack == 0, name
        assert reg <= res[twin][0], (name, reg, res[twin][0])
