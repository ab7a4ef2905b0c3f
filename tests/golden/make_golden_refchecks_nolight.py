"""Generates tests/golden/ref_checks_nolight.json: what the reference compiled with DO_LIGHT_SAMPLING 0
(oracle/_ref/libtoyref_nolight.so, libtoyref_small_mitsuba_nolight.so, built by oracle/nolight.mk where the reference
sources are present) produced, so that the comparisons with it run everywhere. Run where the reference has been built:

    make -C oracle -f nolight.mk all && python tests/golden/make_golden_refchecks_nolight.py

  scenes   sha256 of each array of the variant's GetSceneDesc export (the switch does not change the export: the tests
           check these against the stock build's stored export in ref_checks.json)
  renders  per-frame ray counts and image_digest() of the backbuffer after UpdateTest + DrawTest per frame, the same
           record as ref_checks.json's; every render is also checked against the restatement with the switch off
"""
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from oracle import pyoracle  # noqa: E402
from oracle.nolight import pyoracle as nolight  # noqa: E402
from test_oracle import image_digest  # noqa: E402

VARIANTS = {"nolight": False, "small_mitsuba_nolight": True}      # variant -> DO_MITSUBA_COMPARE


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def main():
    for v in VARIANTS:
        assert pyoracle.have_ref_variant(v), "build the reference variants first: make -C oracle -f nolight.mk all"
    scenes, renders = {}, {}

    def scene(key, w, h, variant):
        s = pyoracle.ref_scene(w, h, variant=variant)
        scenes[key] = {"spheres": sha(s[0]), "materials": sha(s[1]), "camera": sha(s[2]), "emissives": [int(e) for e in s[3]]}
        return s

    def render(key, s, w, h, f0, n, flags, variant):
        sph, mats, cam, em = s
        rbuf, rrays = pyoracle.ref_render(w, h, f0, n, flags=flags, variant=variant)
        obuf, orays, pads = nolight.orc_render(sph, mats, cam, w, h, f0, n, flags=flags, mitsuba=VARIANTS[variant])
        assert orays == rrays and image_digest(obuf, pads) == image_digest(rbuf, pads), key
        renders[key] = {"rays": rrays, "pads": [list(p) for p in pads], "digest": image_digest(rbuf, pads)}

    for v in VARIANTS:
        for (w, h) in [(200, 120), (320, 180)]:
            s = scene(f"{v}_{w}x{h}", w, h, v)
            for flags in (0, 2):
                render(f"{v}_{w}x{h}_f0_n3_flags{flags}", s, w, h, 0, 3, flags, v)
    render("nolight_1280x720_f0_n3_flags0", scene("nolight_1280x720", 1280, 720, "nolight"), 1280, 720, 0, 3, 0, "nolight")
    json.dump({"scenes": scenes, "renders": renders}, open(os.path.join(HERE, "ref_checks_nolight.json"), "w"), indent=1)
    print(len(scenes), "scenes,", len(renders), "renders")


if __name__ == "__main__":
    main()
