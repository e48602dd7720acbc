"""Loaders of the two equirect-mesh CHECKER libraries of include/derp_eqrmesh.h (test infrastructure; never imported by the
product package), both built by oracle/eqrmesh.mk and bound through capi.EqrMesh:

  load_oracle() -> oracle/libeqrmesh_oracle.so        the CPU restatement (oracle/eqrmesh_oracle.cpp)
  load_ref()    -> oracle/_ref/libeqrmesh_ref.so      the reference's own MeshUtil.h / MeshSimplifier.cpp
                                                      (oracle/ref_bridge_eqrmesh.cpp); None when it has not been built
"""
import os

from facebook360_dep_b200 import capi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_LIB = os.path.join(ROOT, "oracle", "libeqrmesh_oracle.so")
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libeqrmesh_ref.so")

_cache = {}


def load_oracle():
    if "oracle" not in _cache:
        _cache["oracle"] = capi.EqrMesh(ORACLE_LIB)
    return _cache["oracle"]


def load_ref():
    if "ref" not in _cache:
        _cache["ref"] = capi.EqrMesh(REF_LIB) if os.path.exists(REF_LIB) else None
    return _cache["ref"]
