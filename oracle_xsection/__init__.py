"""Serial C checker of the cross-sectional area rule of DESIGN.md §5i (xsection_oracle.c) -- TEST
INFRASTRUCTURE ONLY.

Only tests/ and tools/ load it; the product (igneous_b200/) never imports it.  `build()` compiles
libxsection_oracle.so next to the source with the host C compiler (called by __graft_entry__.build()).
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libxsection_oracle.so")
_LIB = None


def build(force=False):
  src = os.path.join(_HERE, "xsection_oracle.c")
  if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
    cc = os.environ.get("CC", "gcc")
    subprocess.check_call([cc, "-O2", "-fPIC", "-std=c11", "-Wall", "-Wextra", "-ffp-contract=off", "-shared",
                           "-o", _SO, src, "-lm"])
  return _SO


def lib():
  global _LIB
  if _LIB is None:
    _LIB = ctypes.CDLL(build())
    _LIB.orc_xs_normals.restype = ctypes.c_int
    _LIB.orc_xs_sections.restype = ctypes.c_int
  return _LIB


def _p(a):
  return ctypes.c_void_p(a.ctypes.data)


def normals(voxels, edges, anisotropy, window):
  """float64 (V, 3) normal of every vertex: voxels int64 (V, 3), edges (E, 2) indices into them"""
  vox = np.ascontiguousarray(np.asarray(voxels, np.int64).reshape(-1, 3))
  e = np.ascontiguousarray(np.asarray(edges).reshape(-1, 2), dtype=np.uint32)
  a = np.ascontiguousarray(anisotropy, np.float64)
  out = np.zeros((len(vox), 3), np.float64)
  rc = lib().orc_xs_normals(ctypes.c_uint64(len(vox)), _p(vox), ctypes.c_uint64(len(e)), _p(e), _p(a),
                            ctypes.c_uint64(int(window)), _p(out))
  if rc == 1:
    raise MemoryError("orc_xs_normals: allocation failed")
  if rc:
    raise ValueError("orc_xs_normals: an edge index outside the vertices")
  return out


def sections(labels, voxels, point_labels, normals, anisotropy):
  """(float32 area, uint8 contacts, voxels visited) per point: labels a 3-D array, voxels int64 (P, 3),
  point_labels (P,) the label each point measures (in the array's values), normals float64 (P, 3)"""
  lab = np.asarray(labels)
  vol = np.asfortranarray(lab.view({1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}[lab.dtype.itemsize])
                          .astype(np.uint64))
  sx, sy, sz = vol.shape
  vox = np.asarray(voxels, np.int64).reshape(-1, 3)
  lin = np.ascontiguousarray(vox[:, 0] + sx * (vox[:, 1] + sy * vox[:, 2]), dtype=np.uint64)
  pl = np.ascontiguousarray(point_labels, np.uint64)
  nn = np.ascontiguousarray(np.asarray(normals, np.float64).reshape(-1, 3))
  a = np.ascontiguousarray(anisotropy, np.float64)
  area, contacts = np.zeros(len(lin), np.float32), np.zeros(len(lin), np.uint8)
  visited = ctypes.c_uint64(0)
  rc = lib().orc_xs_sections(_p(vol), ctypes.c_uint64(sx), ctypes.c_uint64(sy), ctypes.c_uint64(sz),
                             ctypes.c_uint64(len(lin)), _p(lin), _p(pl), _p(nn), _p(a), _p(area), _p(contacts),
                             ctypes.byref(visited))
  if rc == 1:
    raise MemoryError("orc_xs_sections: allocation failed")
  if rc:
    raise ValueError("orc_xs_sections: a point outside the volume")
  return area, contacts, int(visited.value)
