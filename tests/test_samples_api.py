"""tpt_draw_samples without a GPU: the library exports it, its moments instances cost one more reduction, and the
adaptive stopping rule picks the pixels its documentation says. The binding's signature and the wrapper's refusals are
checked with the other caller-buffer calls in test_aovs_api.py."""
import ctypes
import os
import shutil
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports(libs):
    assert hasattr(ctypes.CDLL(libs.LIB_PATH), "tpt_draw_samples")


@pytest.mark.skipif(shutil.which("cuobjdump") is None, reason="needs cuobjdump")
def test_moments_cost_one_more_reduction(libs):
    """The plain instances add a finished path with one red.global.add.v4.f32, the moments instances with two."""
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import sass_counts
    k = {name: cnt for name, _, cnt in sass_counts.kernel_counts(libs.LIB_PATH)}
    inst = [n for n in k if n.startswith("k_fast_samples")]
    assert len(inst) == 36, inst
    for n in inst:
        assert k[n]["REDG.F32x4"] == (2 if n.endswith(", 1>") else 1), n
        assert k[n]["UBLKCP"] >= 1 and k[n]["tensor"] == 0, n
    for n in ("k_fast_samples<128, 6, 2, 0>", "k_fast_samples<128, 8, 2, 1>", "k_fast_samples<768, 1, 3, 1>"):
        assert k[n]["LDS.128"] >= 128 and k[n]["FFMA"] >= 600, n


def test_adaptive_pixels_rule(libs):
    """Four pixels with 4 samples: a constant one (se 0), a noisy dark one, a noisy bright one below the bound, and one
    already at max_spp."""
    samples = {0: [[0.5, 0.5, 0.5]] * 4,
               1: [[0.0] * 3, [0.2] * 3, [0.0] * 3, [0.2] * 3],      # mean 0.1, se 0.0577 > 0.1 * 0.15
               2: [[9.9] * 3, [10.1] * 3, [9.9] * 3, [10.1] * 3],     # mean 10, se 0.0577 < 0.1 * 10.05
               3: [[0.0] * 3, [0.2] * 3, [0.0] * 3, [0.2] * 3]}
    s = torch.zeros((4, 4), dtype=torch.float64)
    q = torch.zeros((4, 4), dtype=torch.float64)
    for i, v in samples.items():
        v = torch.tensor(v, dtype=torch.float64)
        s[i, :3], s[i, 3], q[i, :3] = v.sum(0), len(v), (v * v).sum(0)
    s[3] *= 16; q[3] *= 16                                            # 64 samples: at max_spp
    idx = libs.adaptive_pixels(s, q, 0.1, 64)
    assert idx.dtype == torch.int32 and idx.tolist() == [1]
    assert libs.adaptive_pixels(s, q, 0.001, 64).tolist() == [1, 2]
    assert libs.adaptive_pixels(s, q, 0.001, 65).tolist() == [1, 2, 3]
    # one sample says nothing about the variance: such pixels are always picked
    one = torch.tensor([[0.5, 0.5, 0.5, 1.0]], dtype=torch.float64)
    assert libs.adaptive_pixels(one, one * one, 10.0, 64).tolist() == [0]
    # as a 2 x 2 image every pixel neighbours pixel 1, but pixel 3 already has max_spp
    assert libs.adaptive_pixels(s, q, 0.1, 64, (2, 2)).tolist() == [0, 1, 2]
    img_s = s[[0, 0, 0, 0, 0, 0, 0, 0, 1]].clone()        # 3 x 3, the noisy pixel in a corner: its 2 x 2 block grows
    img_q = q[[0, 0, 0, 0, 0, 0, 0, 0, 1]].clone()
    assert libs.adaptive_pixels(img_s, img_q, 0.1, 64, (3, 3)).tolist() == [4, 5, 7, 8]
