"""Loader of the canopy checker (test infrastructure; never imported by the product package).

``load()`` compiles tests/canopy_oracle.cpp — the CPU restatement of include/derp_canopy.h, built on the rephotography
checker — with the depth oracle's flags (oracle/Makefile: -O3 -funroll-loops -ffp-contract=off) into a temporary
directory, once per process, and returns its ``capi.Canopy`` binding.  Nothing is written in the tree.
"""
import atexit
import os
import shutil
import subprocess
import tempfile

from facebook360_dep_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "canopy_oracle.cpp")
_cache = {}


def load():
    if "lib" not in _cache:
        tmp = tempfile.mkdtemp(prefix="canopy_oracle_")
        atexit.register(shutil.rmtree, tmp, True)
        out = os.path.join(tmp, "libcanopy_oracle.so")
        subprocess.check_call([os.environ.get("CXX", "g++"), "-std=c++17", "-O3", "-funroll-loops", "-ffp-contract=off",
                               "-fPIC", "-Wall", "-Wextra", "-Wno-unused-parameter", "-pthread", "-shared",
                               "-Wl,-Bsymbolic", "-Wl,--exclude-libs,ALL", "-o", out, SRC])
        _cache["lib"] = capi.Canopy(out)
    return _cache["lib"]
