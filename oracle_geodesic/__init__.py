"""Serial C checker of the geodesic rule of DESIGN.md §5e (geodesic_oracle.c) -- TEST INFRASTRUCTURE ONLY.

Only tests/ load it; the product (igneous_b200/) never imports it.  `build()` compiles
libgeodesic_oracle.so next to the source with the host C compiler (called by __graft_entry__.build()).
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libgeodesic_oracle.so")
_LIB = None


class NoParent(ValueError):
  """a reached voxel has no predecessor under the parent rule"""


def build(force=False):
  src = os.path.join(_HERE, "geodesic_oracle.c")
  if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
    cc = os.environ.get("CC", "gcc")
    subprocess.check_call([cc, "-O2", "-fPIC", "-std=c11", "-Wall", "-Wextra", "-ffp-contract=off", "-shared",
                           "-o", _SO, src, "-lm"])
  return _SO


def lib():
  global _LIB
  if _LIB is None:
    _LIB = ctypes.CDLL(build())
    _LIB.orc_geodesic.restype = ctypes.c_int
  return _LIB


def _p(a):
  return ctypes.c_void_p(a.ctypes.data) if a is not None else None


def geodesic(labels, sources, connectivity=26, anisotropy=(1, 1, 1), weights=None, parents=False):
  """dist (float32), or (dist, parents uint32) of a 1-, 2- or 3-D label array (axes beyond its own have
  extent 1); sources are linear F-order indices; weights None = euclidean edge lengths."""
  labels = np.asarray(labels)
  shape = labels.shape + (1,) * (3 - labels.ndim)
  lab = np.asfortranarray(labels.reshape(shape).astype(np.uint64))
  src = np.ascontiguousarray(np.atleast_1d(sources), dtype=np.uint64)
  a = (ctypes.c_float * 3)(*[float(v) for v in anisotropy])
  w = None if weights is None else np.asfortranarray(np.asarray(weights, dtype=np.float32).reshape(shape))
  dist = np.empty(shape, np.float32, order="F")
  par = np.empty(shape, np.uint32, order="F") if parents else None
  u = ctypes.c_uint64
  rc = lib().orc_geodesic(_p(lab), u(shape[0]), u(shape[1]), u(shape[2]), ctypes.c_int(connectivity), a, _p(w),
                          _p(src), u(src.size), _p(dist), _p(par))
  if rc == 1:
    raise MemoryError("orc_geodesic: allocation failed")
  if rc == 3:
    raise ValueError("orc_geodesic: a source outside the volume or on label 0")
  if rc == 2:
    raise NoParent("orc_geodesic: a reached voxel has no parent under the rule")
  dist = dist.reshape(labels.shape, order="F")
  return (dist, par.reshape(labels.shape, order="F")) if parents else dist
