"""The fields TEASAR reads, for every label of a chunk at once, on H100.

Reference call site (seung-lab/igneous):
  igneous/tasks/skeleton.py:54, :312   SkeletonTask -> kimimaro.skeletonize, which per object computes a
                                       distance-to-boundary field, a root, a distance-from-root field,
                                       a penalty field and the shortest-path parents under it

fields() runs those steps for all labels in the same launches and keeps every array on the device in
between (DESIGN.md §5e; kimimaro parity is unpinned offline).  It stops at the parents: path
extraction, the rolling-ball invalidation and SkeletonTask are not here.  There is no CPU fallback.
"""
import ctypes

import numpy as np

from . import _shim

__all__ = ["fields"]

_UNSIGNED = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}
CONNECTIVITY = 26


def fields(labels, anisotropy=(1, 1, 1), pdrf_scale=100000, pdrf_exponent=4, dbf=None, ctx=None):
  """For a 3-D label array (the labels are the objects; 0 is background), a dict of
    labels   the labels renumbered 1..K by first appearance in F order (uint32, F order)
    mapping  {original label: renumbered label}
    roots    (K, 3) voxel of each renumbered label's root, row l - 1 for label l
    dbf      float32 distance to the boundary: edt(labels, anisotropy, black_border=True) unless given
    daf      float32 26-connected geodesic distance from the label's root
    pdrf     float32 pdrf_scale * (1 - dbf / (1.01 max dbf))^pdrf_exponent + daf / max daf, the maxima
             per label, every operation rounded to float32 (pdrf_exponent a whole number from 1 to 64)
    parents  uint32 parents (F-order index + 1, 0 at the roots and on background) of the shortest paths
             from the roots where entering a voxel costs its pdrf
  The root of a label is the voxel farthest (26-connected, ties to the lowest F-order index) from the
  label's first voxel in F order; parts of a label that its first voxel does not reach keep daf = +inf,
  pdrf = 0 and parents = 0.
  Raises IgneousB200Error, for the whole chunk and every label of it, when the parent rule finds a reached
  voxel without a predecessor of lower (distance, index) under the penalty field (DESIGN.md §5e: float32
  addition stalled on a stretch entered from a higher index); the message names such a voxel by its
  F-order index, and `labels` at that index is the object to leave out or to solve on its own."""
  arr = np.asarray(labels)
  if arr.ndim != 3:
    raise ValueError("teasar.fields: expected a 3-D label array, got shape %r" % (arr.shape,))
  if not (arr.dtype == np.bool_ or arr.dtype.kind in "iu"):
    raise NotImplementedError("igneous_b200 teasar.fields: label dtype %s is not supported" % arr.dtype)
  if int(pdrf_exponent) != pdrf_exponent:
    raise NotImplementedError("igneous_b200 teasar.fields: pdrf_exponent must be a whole number")
  vol = np.asfortranarray(arr.view(_UNSIGNED[arr.dtype.itemsize]))
  n = vol.size
  out = {"labels": np.zeros(vol.shape, np.uint32, order="F"), "mapping": {}, "roots": np.zeros((0, 3), np.int64)}
  for name, dt in (("dbf", np.float32), ("daf", np.float32), ("pdrf", np.float32), ("parents", np.uint32)):
    out[name] = np.zeros(vol.shape, dt, order="F")
  if n == 0:
    return out
  ctx = ctx or _shim.default_context()
  lib, h, ptr = ctx.lib, ctx.handle, _shim.ptr
  a = (ctypes.c_float * 3)(*[float(v) for v in anisotropy])
  bufs = []

  def alloc(nbytes):
    bufs.append(ctx.alloc(nbytes))
    return bufs[-1]

  try:
    raw = alloc(vol.nbytes)
    ctx.h2d(raw, vol)
    lab, uniq = alloc(n * 4), alloc(n * 8)
    k = ctypes.c_uint64(0)
    _shim.check(lib.ign_renumber_dev(h, ptr(raw), _shim.dtype_code(vol.dtype), n, ptr(lab), ptr(uniq), n,
                                     ctypes.byref(k)))
    K = int(k.value)
    ctx.d2h(out["labels"], lab)
    orig = np.empty(K, np.uint64)
    if K:
      ctx.d2h(orig, uniq)
    ctx.sync()
    out["mapping"] = {int(u): i + 1 for i, u in enumerate(orig)}
    if (out["labels"] == 0).any():
      out["mapping"][0] = 0
    if K == 0:
      return out
    d = device_fields(ctx, lab, K, vol.shape, a, pdrf_scale, pdrf_exponent, alloc, dbf=dbf)
    d_dbf, d_daf, d_pdrf, d_par, roots = d["dbf"], d["daf"], d["pdrf"], d["parents"], d["roots"]
    root_index = np.empty(K + 1, np.uint64)
    ctx.d2h(root_index, roots)
    for name, buf in (("dbf", d_dbf), ("daf", d_daf), ("pdrf", d_pdrf), ("parents", d_par)):
      ctx.d2h(out[name], buf)
    ctx.sync()
    out["roots"] = np.stack(np.unravel_index(root_index[1:].astype(np.int64), vol.shape, order="F"), axis=1)
    return out
  finally:
    for b in bufs:
      b.free()


def device_fields(ctx, lab, K, shape, a, pdrf_scale, pdrf_exponent, alloc, dbf=None, before=None, parents=True):
  """The chain of fields() on device buffers: `lab` a device u32 volume of `shape` (F order) with labels
  1..K, `a` the ctypes anisotropy, `alloc(nbytes)` a device allocator whose buffers the caller frees.
  dbf: a host array to upload instead of the edt.  before: (device u64 buffer, count) of target voxels;
  the last one on each label replaces its root.  parents=False leaves the parents out (the distance
  under the penalty field is still computed).  Returns device buffers {dbf, daf, pdrf, dist, parents
  (or None), roots, dbf_max}; roots and dbf_max have K + 1 entries, entry 0 unused."""
  lib, h, ptr = ctx.lib, ctx.handle, _shim.ptr
  n = int(np.prod(shape))
  U32 = _shim.IGN_U32
  d_dbf, d_daf, d_pdrf, d_dist = (alloc(n * 4) for _ in range(4))
  d_par = alloc(n * 4) if parents else None
  index, roots, dbf_max, daf_max = alloc((K + 1) * 8), alloc((K + 1) * 8), alloc((K + 1) * 4), alloc((K + 1) * 4)
  if dbf is None:
    _shim.check(lib.ign_edt_dev(h, ptr(lab), U32, *shape, a, 1, 0, ptr(d_dbf)))
  else:
    dbf = np.asfortranarray(dbf, dtype=np.float32)
    if dbf.shape != tuple(shape):
      raise ValueError("teasar.fields: dbf of shape %r for labels of shape %r" % (dbf.shape, tuple(shape)))
    ctx.h2d(d_dbf, dbf)

  def argmax(field, values):
    _shim.check(lib.ign_label_argmax_dev(h, ptr(lab), U32, n, ptr(field), K, ptr(index), ptr(values)))

  def geodesic(sources, weights, dist, parents):
    # entry 0 of an argmax index belongs to label 0: the K sources start one entry in
    _shim.check(lib.ign_geodesic_dev(h, ptr(lab), U32, *shape, CONNECTIVITY, a, weights, sources.offset(8), K,
                                     ptr(dist), parents))

  # the first voxel of every label: the argmax of an all-zero field goes to the lowest index
  ctx.memset(d_daf, 0, n * 4)
  argmax(d_daf, daf_max)
  geodesic(index, None, d_pdrf, None)  # distance from the first voxel, parked in the pdrf buffer
  argmax(d_pdrf, daf_max)
  ctx.d2d(roots, index, (K + 1) * 8)
  if before is not None and before[1]:
    _shim.check(lib.ign_teasar_last_target_dev(h, ptr(lab), n, K, ptr(before[0]), before[1], ptr(roots)))
  geodesic(roots, None, d_daf, None)
  argmax(d_dbf, dbf_max)
  argmax(d_daf, daf_max)
  _shim.check(lib.ign_teasar_pdrf_dev(h, ptr(lab), U32, n, ptr(d_dbf), ptr(d_daf), ptr(dbf_max), ptr(daf_max), K,
                                      float(pdrf_scale), int(pdrf_exponent), ptr(d_pdrf)))
  geodesic(roots, ptr(d_pdrf), d_dist, ptr(d_par) if parents else None)
  return {"dbf": d_dbf, "daf": d_daf, "pdrf": d_pdrf, "dist": d_dist, "parents": d_par, "roots": roots,
          "dbf_max": dbf_max}
