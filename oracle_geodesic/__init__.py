"""Serial C checkers of the geodesic rule of DESIGN.md §5e (geodesic_oracle.c) and of the TEASAR path loop of
§5f (teasar_oracle.c) -- TEST INFRASTRUCTURE ONLY.

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
  srcs = [os.path.join(_HERE, s) for s in ("geodesic_oracle.c", "teasar_oracle.c")]
  if force or not os.path.exists(_SO) or any(os.path.getmtime(_SO) < os.path.getmtime(s) for s in srcs):
    cc = os.environ.get("CC", "gcc")
    subprocess.check_call([cc, "-O2", "-fPIC", "-std=c11", "-Wall", "-Wextra", "-ffp-contract=off", "-shared",
                           "-o", _SO] + srcs + ["-lm"])
  return _SO


def lib():
  global _LIB
  if _LIB is None:
    _LIB = ctypes.CDLL(build())
    _LIB.orc_geodesic.restype = ctypes.c_int
    _LIB.orc_teasar.restype = ctypes.c_int
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


NONE = 0xFFFFFFFF


def teasar(objects, k, anisotropy, dbf, daf, pdrf, roots, parents=None, before=(), after=(), scale=10.0, const=10.0,
           max_paths=None):
  """The path loop of DESIGN.md §5f on given fields: uint32 next (F order, NONE outside the skeleton, the voxel
  itself at a root).  objects: 3-D u32 ids 1..k; roots: k + 1 linear indices (entry 0 unused); parents None
  means fix_branching; before / after: linear indices in the order given."""
  shape = objects.shape
  F = lambda a, dt: np.asfortranarray(np.asarray(a, dtype=dt).reshape(shape, order="F"))
  obj = F(objects, np.uint32)
  fields = [F(v, np.float32) for v in (dbf, daf, pdrf)]
  par = None if parents is None else F(parents, np.uint32)
  arr = lambda v: np.ascontiguousarray(np.asarray(v, dtype=np.uint64).reshape(-1))
  r, b, a_ = arr(roots), arr(before), arr(after)
  an = (ctypes.c_float * 3)(*[float(v) for v in anisotropy])
  nxt = np.empty(shape, np.uint32, order="F")
  bad = ctypes.c_uint64(0)
  u = ctypes.c_uint64
  mp = (1 << 64) - 1 if max_paths is None else int(max_paths)
  rc = lib().orc_teasar(_p(obj), u(shape[0]), u(shape[1]), u(shape[2]), u(k), an, *[_p(v) for v in fields], _p(par),
                        _p(r), _p(b), u(b.size), _p(a_), u(a_.size), ctypes.c_float(scale), ctypes.c_float(const),
                        u(mp), _p(nxt), ctypes.byref(bad))
  if rc == 1:
    raise MemoryError("orc_teasar: allocation failed")
  if rc == 2:
    raise NoParent("orc_teasar: the path voxel at linear index %d has no next voxel" % (bad.value - 1))
  if rc == 3:
    raise ValueError("orc_teasar: a root lies off its object")
  return nxt
