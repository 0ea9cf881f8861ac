"""Serial C checker of the skeleton merge and postprocess rule of DESIGN.md §5h (merge_oracle.c) -- TEST
INFRASTRUCTURE ONLY.

Only tests/ and tools/ load it; the product (igneous_b200/) never imports it.  `build()` compiles
libmerge_oracle.so next to the source with the host C compiler (called by __graft_entry__.build()).
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libmerge_oracle.so")
_LIB = None


def build(force=False):
  src = os.path.join(_HERE, "merge_oracle.c")
  if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
    cc = os.environ.get("CC", "gcc")
    subprocess.check_call([cc, "-O2", "-fPIC", "-std=c11", "-Wall", "-Wextra", "-ffp-contract=off", "-shared",
                           "-o", _SO, src, "-lm"])
  return _SO


def lib():
  global _LIB
  if _LIB is None:
    _LIB = ctypes.CDLL(build())
    _LIB.orc_skeleton_merge.restype = ctypes.c_int
    _LIB.orc_skeleton_merge_capacity.restype = ctypes.c_uint64
    _LIB.orc_skeleton_merge_capacity.argtypes = [ctypes.c_uint64] * 3
  return _LIB


def _p(a):
  return ctypes.c_void_p(a.ctypes.data)


def merge(packed, dust_threshold=4000, tick_threshold=6000, max_cable_length=None, vertex_types=True):
  """(bytes buffer, uint64 table (L, 4) of (label row, byte offset, nv, ne)) of a packed batch, as
  igneous_b200.kimimaro.pack_fragments makes it; ValueError on the input the device refuses"""
  P = {k: np.ascontiguousarray(v) for k, v in packed.items()}
  L = P["label_frag"].size - 1
  cap = lib().orc_skeleton_merge_capacity(L, P["radius"].size, P["edges"].shape[0])
  buf = np.zeros(max(int(cap), 8), np.uint8)
  table = np.zeros((L, 4), np.uint64)
  nb = ctypes.c_uint64(0)
  mc = float("inf") if max_cable_length is None else float(max_cable_length)
  rc = lib().orc_skeleton_merge(
    ctypes.c_uint64(L), _p(P["label_frag"]), _p(P["frag_vert"]), _p(P["frag_edge"]), _p(P["frag_box"]),
    _p(P["vertices"]), _p(P["radius"]), _p(P["vertex_types"]), _p(P["edges"]), ctypes.c_double(dust_threshold),
    ctypes.c_double(tick_threshold), ctypes.c_double(mc), ctypes.c_int(int(bool(vertex_types))), _p(buf),
    ctypes.c_uint64(buf.size), _p(table), ctypes.byref(nb))
  if rc == 1:
    raise MemoryError("orc_skeleton_merge: allocation failed")
  if rc == 2:
    raise ValueError("orc_skeleton_merge: an edge index outside its fragment")
  if rc == 3:
    raise ValueError("orc_skeleton_merge: a non-finite vertex")
  if rc:
    raise ValueError("orc_skeleton_merge: status %d" % rc)
  return buf[:int(nb.value)], table
