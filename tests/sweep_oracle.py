"""Loaders of the two sweep-view CHECKER libraries (test infrastructure; never imported by the product package).

  load_overlaps_ref() -> oracle/_ref/libsweep_overlaps_ref.so   the reference's own GenerateCameraOverlaps.cpp
  load_equirect_ref() -> oracle/_ref/libsweep_equirect_ref.so   the reference's own GenerateEquirect.cpp

Both are built by oracle/sweepview.mk (oracle/ref_bridge_sweepview.cpp) and exported through capi.SweepView.  None is
returned when a library has not been built.
"""
import os

from facebook360_dep_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref")

_cache = {}


def _load(name):
    if name not in _cache:
        path = os.path.join(REF_DIR, name)
        _cache[name] = capi.SweepView(path) if os.path.exists(path) else None
    return _cache[name]


def load_overlaps_ref():
    return _load("libsweep_overlaps_ref.so")


def load_equirect_ref():
    return _load("libsweep_equirect_ref.so")
