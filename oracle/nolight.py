"""TEST INFRASTRUCTURE — the oracles with DO_LIGHT_SAMPLING 0 (Config.h:24), built by oracle/nolight.mk.

`oracle.nolight.pyoracle` is a second instance of oracle/pyoracle.py whose library paths point at the _nolight builds,
so it offers the same functions with the same signatures:
    orc_render   the CPU restatement with the switch off          (_ref/liboracle_nolight.so)
    rgo_render   the GPU shader's restatement with the switch off  (_ref/librefgpu_nolight.so)
    ref_render / ref_scene(variant="nolight" | "small_mitsuba_nolight")  the reference compiled with the switch off
"""
import importlib.util
import os
import subprocess

from oracle import pyoracle as _stock

_DIR = os.path.dirname(os.path.abspath(__file__))


def build(quiet: bool = True):
    subprocess.run(["make", "-C", _DIR, "-f", "nolight.mk", "all"], check=True,
                   stdout=subprocess.DEVNULL if quiet else None, stderr=subprocess.STDOUT if quiet else None)


_spec = importlib.util.spec_from_file_location("oracle._pyoracle_nolight", _stock.__file__)
pyoracle = importlib.util.module_from_spec(_spec)
_spec.loader.exec_module(pyoracle)
pyoracle.ORC_SO = os.path.join(_DIR, "_ref", "liboracle_nolight.so")
pyoracle.RGO_SO = os.path.join(_DIR, "_ref", "librefgpu_nolight.so")
pyoracle.build = build
