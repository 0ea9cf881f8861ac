"""Serial C checker of the hole-filling rule (fill_oracle.c) -- TEST INFRASTRUCTURE ONLY.

Only tests/ load it; the product (igneous_b200/) never imports it.  `build()` compiles
libfill_oracle.so next to the source with the host C compiler (called by __graft_entry__.build()).
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libfill_oracle.so")
_LIB = None


def build(force=False):
  src = os.path.join(_HERE, "fill_oracle.c")
  if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
    cc = os.environ.get("CC", "gcc")
    subprocess.check_call([cc, "-O2", "-fPIC", "-std=c11", "-Wall", "-Wextra", "-shared", "-o", _SO, src])
  return _SO


def lib():
  global _LIB
  if _LIB is None:
    _LIB = ctypes.CDLL(build())
    _LIB.orc_fill_holes.restype = ctypes.c_int
  return _LIB


def _u64(X):
  X = np.asarray(X)
  if X.ndim == 2:
    X = X[:, :, None]
  return np.asfortranarray(X.astype(np.uint64))


def _p(a):
  return ctypes.c_void_p(a.ctypes.data)


def dilate(X):
  """fastmorph.dilate(X, mode=multilabel, background_only=True) by the rule (mesh.py:211-218)."""
  X = np.asarray(X)
  a = _u64(X)
  out = np.empty_like(a, order="F")
  u = ctypes.c_uint64
  lib().orc_dilate_multilabel(_p(a), u(a.shape[0]), u(a.shape[1]), u(a.shape[2]), _p(out))
  return out.astype(X.dtype).reshape(X.shape, order="F")


def fill_holes(X0, fix_borders=False, p=0):
  """(filled, holes) of fastmorph.fill_holes_v2(X0, fix_borders, merge_threshold = 1 - p/100)."""
  X0 = np.asarray(X0)
  a = _u64(X0)
  filled = np.empty_like(a, order="F")
  holes = np.empty_like(a, order="F")
  u = ctypes.c_uint64
  rc = lib().orc_fill_holes(_p(a), u(a.shape[0]), u(a.shape[1]), u(a.shape[2]), ctypes.c_int(int(bool(fix_borders))),
                            ctypes.c_int(int(p)), _p(filled), _p(holes))
  if rc != 0:
    raise MemoryError("orc_fill_holes: allocation failed")
  return (filled.astype(X0.dtype).reshape(X0.shape, order="F"), holes.astype(X0.dtype).reshape(X0.shape, order="F"))


def fill_level(X, level):
  """MeshTask(fill_holes=level) on a renumbered block (mesh.py:211-228): (filled, holes)."""
  X0 = dilate(X) if level >= 3 else np.asarray(X)
  return fill_holes(X0, fix_borders=level >= 2, p=max(0, level - 3))
