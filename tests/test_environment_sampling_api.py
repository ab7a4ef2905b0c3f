"""The "environment_sampling" option without a GPU: the library accepts it and the header documents it; the table
builder (toypathtracer_b200/csrc/tpt_env_tables.h, built with g++ into a small library by a fixture here) against a
float64 numpy model of the pinned weights and of the alias sampler on the 2^-24 grid of the draws; and the compiled
kernel set: the sampling code sits in the slab queue's reference-form 6-CTA and 768-thread light-sampling instances
and nowhere else.

The numpy model (env_weights_model, realised_model, sample_cells) is shared with tests/test_gpu_environment_sampling.py."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

from test_irradiance_api import _NoLib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ONE = 1 << 24


# ---- float64 model of tpt_env_tables.h ------------------------------------------------------------------------------
def env_weights_model(rgb):
    """w(i, j) = sin(theta_j) * max over the 3 x 3 neighbourhood (columns wrap, rows clamp) of mean(R, G, B)."""
    H, W = rgb.shape[:2]
    m = rgb[..., :3].astype(np.float64).sum(-1) / 3.0
    r = np.maximum(np.maximum(np.roll(m, 1, axis=1), m), np.roll(m, -1, axis=1))
    up = r[np.maximum(np.arange(H) - 1, 0)]
    dn = r[np.minimum(np.arange(H) + 1, H - 1)]
    mx = np.maximum(np.maximum(up, r), dn)
    return np.sin((np.arange(H) + 0.5) * np.pi / H)[:, None] * mx


def index_counts(n):
    """How many of the 2^24 values k draw index i = (k * n) >> 24."""
    i = np.arange(n + 1, dtype=np.int64)
    lo = (i * ONE + n - 1) // n
    return np.diff(lo)


def realised_model(prob, alias):
    """The probability each entry of an alias table (float32 prob, int alias) is drawn with: index (k n) >> 24, kept
    when the 24-bit test draw m / 2^24 < prob, else its alias. Exact: integer numerators over 2^48."""
    n = len(prob)
    cnt = index_counts(n)
    keep = np.clip(np.ceil(prob.astype(np.float64) * ONE), 0, ONE).astype(np.int64)
    num = np.bincount(np.arange(n), cnt * keep, minlength=n) + np.bincount(alias, cnt * (ONE - keep), minlength=n)
    return num.astype(np.float64) / float(ONE) / float(ONE)


def split_tables(W, H, rows, cols):
    r = np.frombuffer(rows, dtype=[("p", "<f4"), ("a", "<i4")])
    c = np.frombuffer(cols, dtype=[("p", "<f4"), ("a", "<i4")]).reshape(H, W)
    return r["p"].copy(), r["a"].copy(), c["p"].copy(), c["a"].copy()


def sample_cells(k1, u2, k3, u4, W, H, rp, ra, cp, ca):
    """The sampler's cell choice from its first four draws (k: 24-bit integers, u: RandomFloat01 values), vectorised."""
    j = (k1.astype(np.uint64) * np.uint64(H)) >> np.uint64(24)
    j = j.astype(np.int64)
    j = np.where(u2 < rp[j], j, ra[j])
    i = ((k3.astype(np.uint64) * np.uint64(W)) >> np.uint64(24)).astype(np.int64)
    i = np.where(u4 < cp[j, i], i, ca[j, i])
    return i, j


# ---- the g++ build of the builder -----------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def tables_lib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp("env_tables") / "env_tables_check.so")
    src = os.path.join(ROOT, "tests", "host_sim", "env_tables_check.cpp")
    subprocess.run(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-o", out, src], check=True)
    L = ctypes.CDLL(out)
    L.env_tables_check.argtypes = [ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    L.env_tables_check.restype = ctypes.c_int
    L.env_slot_size.argtypes = [ctypes.c_int, ctypes.c_int]
    L.env_slot_size.restype = ctypes.c_longlong
    return L


def build_tables(L, img):
    H, W = img.shape[:2]
    tex = np.zeros((H, W, 4), np.float32)
    tex[..., :img.shape[2]] = img
    tex[..., 3] = -7.0                         # alpha is overwritten only when the map is sampleable
    rows = bytearray(8 * H)
    cols = bytearray(8 * W * H)
    w = np.zeros((H, W), np.float64)
    rb = (ctypes.c_char * len(rows)).from_buffer(rows)
    cb = (ctypes.c_char * len(cols)).from_buffer(cols)
    ok = L.env_tables_check(tex.ctypes.data, W, H, ctypes.addressof(rb), ctypes.addressof(cb), w.ctypes.data)
    return ok, tex, bytes(rows), bytes(cols), w


def _maps():
    rng = np.random.default_rng(11)
    rand = rng.exponential(1.0, (19, 37, 3)).astype(np.float32)
    rand[rng.random((19, 37)) < 0.3] = 0.0
    one_hot = np.zeros((16, 32, 3), np.float32)
    one_hot[5, 31] = (3.0, 0.0, 1.0)                          # on the wrapping column
    pole = np.full((24, 48, 3), 1e-3, np.float32)
    pole[0] = 50.0
    pole[-1] = 20.0
    sun = np.full((64, 128, 3), 0.2, np.float32)
    sun[20, 40] = 4.0e4
    return {
        "random": rand,
        "one_hot": one_hot,
        "single_row": rng.random((1, 29, 3)).astype(np.float32),
        "single_column": rng.random((23, 1, 3)).astype(np.float32),
        "1x1": np.array([[[0.5, 1.0, 2.0]]], np.float32),
        "pole_heavy": pole,
        "sun": sun,
        "wide": rng.random((3, 4099, 3)).astype(np.float32),
    }


MAPS = _maps()


@pytest.mark.parametrize("name", sorted(MAPS))
def test_tables_match_the_float64_model(tables_lib, name):
    img = MAPS[name]
    H, W = img.shape[:2]
    ok, tex, rows, cols, w = build_tables(tables_lib, img)
    assert ok == 1
    # weights per the pinned formula
    wm = env_weights_model(img)
    np.testing.assert_allclose(w, wm, rtol=1e-15, atol=0)
    rp, ra, cp, ca = split_tables(W, H, rows, cols)
    assert ((ra >= 0) & (ra < H)).all() and ((ca >= 0) & (ca < W)).all()
    assert ((rp >= 0) & (rp <= 1)).all() and ((cp >= 0) & (cp <= 1)).all()
    # the alpha channel holds exactly the probability the stored tables realise
    prow = realised_model(rp, ra)
    P = np.zeros((H, W))
    for j in range(H):
        P[j] = prow[j] * realised_model(cp[j], ca[j])
    assert np.array_equal(tex[..., 3], P.astype(np.float32)), "alpha is not the realised cell probability"
    # ... which sums to one within float rounding and follows the weights up to the 2^-24 index grid
    assert abs(float(tex[..., 3].astype(np.float64).sum()) - 1.0) < 1e-6
    target = wm / wm.sum()
    assert np.abs(P - target).sum() <= 2.0 * (H + W + 2) / ONE + 1e-9
    # zero-weight cells (and rows) are never drawn: zero probability, never an alias, never kept
    rowW = wm.sum(1)
    assert ((prow == 0) == (rowW == 0)).all()
    assert ((P == 0) == (wm == 0)).all()
    assert (rowW[ra] > 0).all() or (rowW == 0).sum() == 0
    for j in np.nonzero(rowW > 0)[0]:
        z = wm[j] == 0
        assert (cp[j][z] == 0).all() and (wm[j][ca[j]] > 0).all()
    assert (rp[rowW == 0] == 0).all() and (rowW[ra] > 0).all()


def test_tables_of_an_all_black_map_are_not_built(tables_lib):
    ok, tex, rows, cols, w = build_tables(tables_lib, np.zeros((8, 16, 3), np.float32))
    assert ok == 0 and (w == 0).all()
    assert (tex[..., 3] == -7.0).all()


def test_sampler_model_draws_cells_with_the_realised_probability(tables_lib):
    """sample_cells (the GPU test's model of the kernel's cell choice) draws cells with the alpha channel's
    probabilities: 2^22 draws from a numpy XorShift-free uniform source, chi-square over the cells."""
    img = MAPS["random"]
    H, W = img.shape[:2]
    ok, tex, rows, cols, w = build_tables(tables_lib, img)
    rp, ra, cp, ca = split_tables(W, H, rows, cols)
    rng = np.random.default_rng(5)
    n = 1 << 22
    k1, k3 = rng.integers(0, ONE, n), rng.integers(0, ONE, n)
    u2, u4 = (rng.integers(0, ONE, n) / ONE).astype(np.float32), (rng.integers(0, ONE, n) / ONE).astype(np.float32)
    i, j = sample_cells(k1, u2, k3, u4, W, H, rp, ra, cp, ca)
    got = np.bincount(j * W + i, minlength=W * H).astype(np.float64)
    P = tex[..., 3].astype(np.float64).ravel()
    assert got[P == 0].sum() == 0
    m = P > 0
    chi2 = float((((got - n * P) ** 2)[m] / (n * P[m])).sum())
    dof = int(m.sum()) - 1
    assert chi2 < dof + 6 * np.sqrt(2 * dof), (chi2, dof)
    assert np.array_equal(index_counts(H), np.bincount(((np.arange(ONE, dtype=np.uint64) * np.uint64(H)) >> np.uint64(24)).astype(np.int64)))


def test_slot_size(tables_lib):
    for W, H in [(1, 1), (37, 19), (4096, 2048)]:
        assert tables_lib.env_slot_size(W, H) == 24 * W * H + 8 * H


# ---- option and header -----------------------------------------------------------------------------------------------
def test_context_set_option_passes_the_key(libs):
    class Rec(_NoLib):
        def __init__(self):
            self.calls = []

        def tpt_set_option(self, h, key, value):
            self.calls.append((key, value))
            return 0

    ctx = libs.Context.__new__(libs.Context)
    ctx._L, ctx._h, ctx.device, ctx.spp = Rec(), ctypes.c_void_p(), 0, 4
    ctx.set_option("environment_sampling", 1)
    assert ctx._L.calls and ctx._L.calls[-1][1] == 1
    assert ctx._L.calls[-1][0] in (b"environment_sampling", "environment_sampling")


def test_header_documents_the_option():
    hdr = open(os.path.join(ROOT, "include", "tpt_b200.h")).read()
    m = re.search(r'"environment_sampling" \(default 0[^)]*\)', hdr)
    assert m, "include/tpt_b200.h does not document \"environment_sampling\""
    assert "not light-sampled" not in hdr
    env = hdr[hdr.index("Environment lighting for the fast mode"):hdr.index("int tpt_set_environment")]
    assert "environment_sampling" in env


# ---- where the sampling code is compiled ----------------------------------------------------------------------------
SAMPLING_INSTANCES = {f"k_fast_{k}<{t}, {m}, 0{mo}>"
                      for k, mos in (("queue", [""]), ("rays", [""]), ("samples", [", false", ", true"]))
                      for t, m in ((128, 6), (768, 1)) for mo in mos}


def _sass_by_kernel(lib):
    out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout
    parts = re.split(r"\n\s+Function : (\S+)\n", out)
    names = parts[1::2]
    dm = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout.split("\n")
    return {re.sub(r"^void tpt::|\(.*$", "", d): body for d, body in zip(dm, parts[2::2])}


@pytest.fixture(scope="module")
def sass(libs):
    if not os.path.exists(libs.LIB_PATH):
        pytest.skip("library not built")
    return _sass_by_kernel(libs.LIB_PATH)


def test_sampling_code_is_in_the_sampling_instances_only(sass):
    """The environment sampler's 64-bit read-only table loads (alias entries {prob, alias}) appear exactly in the
    reference-form light-sampling slab-queue instances at 6 CTAs and 768 threads."""
    have = {k for k in sass if k.startswith("k_fast_")}
    expect = {k for k in have if k in SAMPLING_INSTANCES}
    assert len(expect) == 8, sorted(expect)
    signed = {k for k, body in sass.items() if re.search(r"LDG\.E\.64\.CONSTANT", body)}
    assert signed == expect, (sorted(signed - expect), sorted(expect - signed))


def test_sampling_instances_keep_the_kernel_rules(sass):
    """No jump table on the path kind, no generic loads, and the bulk copy, in the sampling instances."""
    for k in SAMPLING_INSTANCES & set(sass):
        body = sass[k]
        assert "UBLKCP" in body, k
    for k in ("k_fast_queue<128, 6, 0>", "k_fast_queue<128, 6, 2>"):
        assert len(re.findall(r"\bBRX\b", sass[k])) == 0, k
        assert len(re.findall(r"\bLD\.E\b", sass[k])) == 0, k
    for k in SAMPLING_INSTANCES & set(sass):
        if k.startswith("k_fast_samples"):
            assert len(re.findall(r"REDG\.E\.ADD\.F32x4", sass[k])) in (1, 2), k
