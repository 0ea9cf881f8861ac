"""Drop-in for `kimimaro.skeletonize`: TEASAR skeletons of every object of a chunk at once, on H100.

Reference call site (seung-lab/igneous):
  igneous/tasks/skeleton.py:54, :312   SkeletonTask -> kimimaro.skeletonize(all_labels, teasar_params, ...)

The rule is DESIGN.md §5f (kimimaro parity is unpinned offline).  Objects are the 26-connected parts of
each label; each gets the fields of `teasar.fields`, then every object traces its k-th path in the same
round: the target is the valid voxel farthest from the root, the path runs to the skeleton built so far,
and every path voxel invalidates a box of half-extents floor((scale * DBF + const) / anisotropy) around it.
Objects, fields, the loop and the compaction of the skeleton run in libigneous_b200
(igneous_b200/csrc/geodesic.cu); the host splits the compacted skeleton by label.  There is no CPU
fallback.
"""
import ctypes
import time

import numpy as np

from . import _shim
from .teasar import device_fields

__all__ = ["skeletonize", "Skeleton", "DEFAULT_TEASAR_PARAMS"]

# seconds per phase of the last call, each ending where the host already waits for the device (diagnostic)
last_phase_seconds = {}

_UNSIGNED = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}

# kimimaro's defaults as recalled (unpinned); soma_* are read only to refuse soma mode
DEFAULT_TEASAR_PARAMS = {
  "scale": 10, "const": 10, "pdrf_scale": 100000, "pdrf_exponent": 4, "soma_acceptance_threshold": 3500,
  "soma_detection_threshold": 750, "soma_invalidation_const": 300, "soma_invalidation_scale": 2, "max_paths": None,
}


class Skeleton:
  """One label's skeleton: vertices (N, 3) float32 in physical units, edges (E, 2) uint32, radii (N,)
  float32, vertex_types (N,) uint8 and the label as id."""

  def __init__(self, vertices, edges, radii, vertex_types, id):
    self.vertices, self.edges, self.radii, self.vertex_types, self.id = vertices, edges, radii, vertex_types, id

  def empty(self):
    return self.vertices.shape[0] == 0

  def __repr__(self):
    return "Skeleton(id=%r, vertices=%d, edges=%d)" % (self.id, self.vertices.shape[0], self.edges.shape[0])


def _targets(points, arr, what):
  """linear F-order indices of voxels (x, y, z) of the caller's array; ValueError on background"""
  pts = np.asarray(points, dtype=np.int64).reshape(-1, 3) if len(points) else np.zeros((0, 3), np.int64)
  if pts.size and (pts.min() < 0 or np.any(pts >= np.array(arr.shape))):
    raise ValueError("kimimaro.skeletonize: a target of %s lies outside the volume of shape %r" % (what, arr.shape))
  for p in pts:
    if arr[tuple(p)] == 0:
      raise ValueError("kimimaro.skeletonize: the target %r of %s lies on background" % (tuple(int(c) for c in p),
                                                                                          what))
  return np.ascontiguousarray(np.ravel_multi_index(tuple(pts.T), arr.shape, order="F"), dtype=np.uint64)


def skeletonize(all_labels, teasar_params=DEFAULT_TEASAR_PARAMS, object_ids=None, anisotropy=(1, 1, 1),
                dust_threshold=1000, progress=False, fix_branching=True, in_place=False, fix_borders=True,
                parallel=1, parallel_chunk_size=100, extra_targets_before=[], extra_targets_after=[],
                fill_holes=False, fix_avocados=False, voxel_graph=None, ctx=None):
  """{label: Skeleton} of every label of a 3-D array with an object of at least dust_threshold voxels.
  `progress`, `parallel`, `parallel_chunk_size` and `in_place` are accepted and ignored.  fill_holes,
  fix_avocados, voxel_graph and soma mode (an object whose largest DBF exceeds soma_detection_threshold)
  raise NotImplementedError.  last_phase_seconds holds the host-clock time of each phase of the last call."""
  if fill_holes or fix_avocados or voxel_graph is not None:
    raise NotImplementedError("igneous_b200 kimimaro.skeletonize: fill_holes, fix_avocados and voxel_graph are "
                              "not supported")
  arr = np.asarray(all_labels)
  if arr.ndim != 3:
    raise ValueError("kimimaro.skeletonize: expected a 3-D label array, got shape %r" % (arr.shape,))
  if not (arr.dtype == np.bool_ or arr.dtype.kind in "iu"):
    raise NotImplementedError("igneous_b200 kimimaro.skeletonize: label dtype %s is not supported" % arr.dtype)
  p = dict(DEFAULT_TEASAR_PARAMS)
  p.update(teasar_params or {})
  scale, const = float(p["scale"]), float(p["const"])
  if not (np.isfinite(scale) and scale >= 0 and np.isfinite(const) and const >= 0):
    raise ValueError("kimimaro.skeletonize: scale %r and const %r must be finite and >= 0" % (p["scale"], p["const"]))
  if int(p["pdrf_exponent"]) != p["pdrf_exponent"]:
    raise NotImplementedError("igneous_b200 kimimaro.skeletonize: pdrf_exponent must be a whole number")
  max_paths = (1 << 64) - 1 if p["max_paths"] is None else int(p["max_paths"])
  a = tuple(float(v) for v in anisotropy)
  if len(a) != 3 or not all(np.isfinite(v) and v > 0 for v in a):
    raise ValueError("kimimaro.skeletonize: anisotropy %r must be three positive finite values" % (anisotropy,))
  # the kernels take an F-order volume; linear indices below are F-order indices of the caller's axes
  vol = np.asfortranarray(arr.view(_UNSIGNED[arr.dtype.itemsize]))
  n = vol.size
  before = _targets(extra_targets_before, arr, "extra_targets_before")
  after = _targets(extra_targets_after, arr, "extra_targets_after")
  if n == 0:
    return {}
  ctx = ctx or _shim.default_context()
  lib, h, ptr = ctx.lib, ctx.handle, _shim.ptr
  ca = (ctypes.c_float * 3)(*a)
  bufs = []

  def alloc(nbytes):
    bufs.append(ctx.alloc(max(int(nbytes), 8)))
    return bufs[-1]

  try:
    last_phase_seconds.clear()
    t0 = time.perf_counter()

    def phase(name):
      nonlocal t0
      t = time.perf_counter()
      last_phase_seconds[name] = t - t0
      t0 = t

    raw = alloc(vol.nbytes)
    ctx.h2d(raw, vol)
    lab = alloc(n * 4)
    k = ctypes.c_uint64(0)
    _shim.check(lib.ign_renumber_dev(h, ptr(raw), _shim.dtype_code(vol.dtype), n, ptr(lab), None, 0,
                                     ctypes.byref(k)))
    K = int(k.value)
    if K and object_ids is not None:
      # the original label of each renumbered one: renumber again into a table of K entries
      uniq = alloc(K * 8)
      _shim.check(lib.ign_renumber_dev(h, ptr(raw), _shim.dtype_code(vol.dtype), n, ptr(lab), ptr(uniq), K,
                                       ctypes.byref(k)))
      orig = np.empty(K, np.uint64)
      ctx.d2h(orig, uniq)
      ctx.sync()
      wanted = np.asarray(list(object_ids)).astype(arr.dtype).view(_UNSIGNED[arr.dtype.itemsize]).astype(np.uint64)
      drop = np.ascontiguousarray(np.nonzero(~np.isin(orig, wanted))[0] + 1, dtype=np.uint64)
      if drop.size:
        _shim.check(lib.ign_remap_dev(h, ptr(lab), _shim.IGN_U32, n, ptr(drop), ptr(np.zeros_like(drop)),
                                      drop.size, 1))
    obj = alloc(n * 4)
    m = ctypes.c_uint64(0)
    _shim.check(lib.ign_teasar_objects_dev(h, ptr(lab), *vol.shape, K, 26, int(dust_threshold), ptr(obj),
                                           ctypes.byref(m)))
    M = int(m.value)
    phase("upload_objects")
    if M == 0:
      return {}
    if fix_borders:
      # kimimaro's order: the caller's before-targets, then the border targets
      cap = 2 * (vol.shape[1] * vol.shape[2] + vol.shape[0] * vol.shape[2] + vol.shape[0] * vol.shape[1])
      d_border, nb = alloc(cap * 8), ctypes.c_uint64(0)
      _shim.check(lib.ign_teasar_border_targets_dev(h, ptr(obj), *vol.shape, M, ca, ptr(d_border), cap,
                                                    ctypes.byref(nb)))
      border = np.empty(int(nb.value), np.uint64)
      if border.size:
        ctx.d2h(border, d_border, border.nbytes)
        ctx.sync()
      before = np.concatenate([before, border])
      phase("border_targets")
    d_before, d_after = alloc(before.nbytes), alloc(after.nbytes)
    if before.size:
      ctx.h2d(d_before, before)
    if after.size:
      ctx.h2d(d_after, after)
    d = device_fields(ctx, obj, M, vol.shape, ca, p["pdrf_scale"], p["pdrf_exponent"], alloc,
                      before=(d_before, before.size), parents=not fix_branching)
    roots, dbf_max = np.empty(M + 1, np.uint64), np.empty(M + 1, np.float32)
    ctx.d2h(roots, d["roots"])
    ctx.d2h(dbf_max, d["dbf_max"])
    ctx.sync()
    phase("fields")
    soma = np.nonzero(dbf_max[1:] > float(p["soma_detection_threshold"]))[0]
    if soma.size:
      o = int(soma[0]) + 1
      label = arr.reshape(-1, order="F")[int(roots[o])]
      raise NotImplementedError("igneous_b200 kimimaro.skeletonize: label %d has an object whose largest distance "
                                "to the boundary, %g, exceeds soma_detection_threshold %g; soma mode is not "
                                "supported" % (int(label), float(dbf_max[o]), float(p["soma_detection_threshold"])))
    skel, nxt, rad = alloc(n * 4), alloc(n * 4), alloc(n * 4)
    count = ctypes.c_uint64(0)
    _shim.check(lib.ign_teasar_paths_dev(
      h, ptr(obj), *vol.shape, M, ca, ptr(d["dbf"]), ptr(d["daf"]), ptr(d["pdrf"]),
      ptr(d["dist"]) if fix_branching else None, None if fix_branching else ptr(d["parents"]), ptr(d["roots"]),
      ptr(d_before), before.size, ptr(d_after), after.size, scale, const, max_paths, ptr(skel), ptr(nxt), ptr(rad),
      ctypes.byref(count)))
    c = int(count.value)
    index, following, radii = np.empty(c, np.uint32), np.empty(c, np.uint32), np.empty(c, np.float32)
    if c:
      ctx.d2h(index, skel, c * 4)
      ctx.d2h(following, nxt, c * 4)
      ctx.d2h(radii, rad, c * 4)
      ctx.sync()
    phase("loop")
  finally:
    for b in bufs:
      b.free()
  out = _assemble(arr, index, following, radii, a)
  phase("assembly")
  return out


def _assemble(arr, index, following, radii, anisotropy):
  """split the compacted skeleton (ascending F-order indices, next voxel, radius) by label"""
  labels = arr.reshape(-1, order="F")[index]
  order = np.argsort(labels, kind="stable")  # within a label the indices stay ascending
  rank = np.empty(order.size, np.int64)
  rank[order] = np.arange(order.size)
  starts = np.concatenate([[0], np.flatnonzero(np.diff(labels[order])) + 1, [order.size]])
  group = np.repeat(np.arange(starts.size - 1), np.diff(starts))  # label group of each sorted position
  # edges (v, next(v)) as positions within the label, smaller first, sorted per label
  tree = following != index
  e0, e1 = rank[tree], rank[np.searchsorted(index, following[tree])]
  g = group[e0]
  lo, hi = np.minimum(e0, e1) - starts[g], np.maximum(e0, e1) - starts[g]
  eo = np.lexsort((hi, lo, g))
  edges = np.stack([lo[eo], hi[eo]], axis=1).astype(np.uint32)
  ecut = np.searchsorted(g[eo], np.arange(starts.size))
  coords = np.stack(np.unravel_index(index[order].astype(np.int64), arr.shape, order="F"), axis=1)
  vertices = coords.astype(np.float32) * np.asarray(anisotropy, dtype=np.float32)
  rad = radii[order].astype(np.float32)
  out = {}
  for j in range(starts.size - 1):
    a, b = starts[j], starts[j + 1]
    label = int(labels[order[a]])
    out[label] = Skeleton(vertices[a:b], np.ascontiguousarray(edges[ecut[j]:ecut[j + 1]]), rad[a:b],
                          np.zeros(b - a, np.uint8), label)
  return out
