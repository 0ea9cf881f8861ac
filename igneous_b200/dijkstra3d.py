"""Drop-in for the `dijkstra3d` wheel's distance and parent fields, running on H100, for every label of
a chunk in one call.

Reference call site (seung-lab/igneous):
  igneous/tasks/skeleton.py:54, :312   SkeletonTask -> kimimaro.skeletonize, whose TEASAR reads, per
                                       object, dijkstra3d.euclidean_distance_field (root and
                                       distance-from-root) and dijkstra3d.parental_field (paths)

The rule is DESIGN.md §5e (parity with the wheel is unpinned offline).  Voxels are joined when they are
neighbours under `connectivity` and carry the same non-zero label; every step of a path is one float32
addition; the result is the least value over all paths from a source of the voxel's label, +inf on
label 0 and where no source reaches, and it equals a heap Dijkstra with the same additions bit for
bit.  The solver runs in libigneous_b200 (ign_geodesic, igneous_b200/csrc/geodesic.cu); there is no CPU
fallback.

Beyond the wheel's one-object calls, `source` may name one voxel per label ({label: voxel}) or a list of
voxels, `source_indices=` takes a 1-D integer array of linear indices in the array's memory order
instead, and the weighted calls take `labels=`: all objects of the array are solved in the same
launches.

Parents are uint32: the linear index + 1, in the array's own memory order, of the voxel's predecessor;
0 for a source, an unreached voxel and label 0.  path_from_parents walks them.
"""
import ctypes

import numpy as np

from . import _shim

__all__ = ["euclidean_distance_field", "distance_field", "parental_field", "path_from_parents"]

_UNSIGNED = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}
_CONNECTIVITY = {1: {6: 6, 18: 6, 26: 6, 4: 6, 8: 6}, 2: {4: 6, 8: 18}, 3: {6: 6, 18: 18, 26: 26}}


def _labels(data, what):
  arr = np.asarray(data)
  if arr.ndim not in (1, 2, 3):
    raise ValueError("%s: expected a 1-, 2- or 3-D array, got shape %r" % (what, arr.shape))
  if arr.dtype == np.bool_ or arr.dtype.kind in "iu":
    return arr.view(_UNSIGNED[arr.dtype.itemsize])  # only equality matters
  raise NotImplementedError("igneous_b200 %s: label dtype %s is not supported (bool or integer labels)"
                            % (what, arr.dtype))


def _source_indices(source, indices, arr, rev):
  """linear indices, in arr's memory order, of the voxels `source` names in the caller's label array arr,
  or `indices` as given"""
  if (source is None) == (indices is None):
    raise ValueError("give the sources as `source` (voxels) or as `source_indices` (linear indices), not both")
  if indices is not None:
    idx = np.asarray(indices)
    if idx.ndim != 1 or (idx.size and idx.dtype.kind not in "iu") or (idx.size and int(idx.min()) < 0):
      raise ValueError("source_indices must be a 1-D array of non-negative integers")
    return np.ascontiguousarray(idx, dtype=np.uint64)
  if isinstance(source, dict):
    for label, v in source.items():
      v = tuple(int(c) for c in np.atleast_1d(v))
      if len(v) != arr.ndim or any(c < 0 or c >= n for c, n in zip(v, arr.shape)) or arr[v] != label:
        raise ValueError("source %r does not lie on label %r" % (v, label))
    source = list(source.values())
  src = np.asarray(source)
  if src.size and (src.dtype.kind not in "iu" or src.ndim > 2 or (src.ndim == 2 and src.shape[1] != arr.ndim)
                   or (src.ndim == 1 and arr.ndim > 1 and src.size != arr.ndim)):
    raise ValueError("source must be a voxel, a list of voxels or {label: voxel} of a %d-D array" % arr.ndim)
  src = src.reshape(-1, arr.ndim).astype(np.int64)
  if src.size and (src.min() < 0 or np.any(src >= np.array(arr.shape))):
    raise ValueError("a source lies outside the array of shape %r" % (arr.shape,))
  return np.ascontiguousarray(np.ravel_multi_index(tuple(src.T), arr.shape, order="C" if rev else "F"),
                              dtype=np.uint64)


def _solve(labels, source, indices, connectivity, anisotropy, weights, parents, ctx, what):
  arr = _labels(labels, what)
  try:
    conn = _CONNECTIVITY[arr.ndim][connectivity]
  except KeyError:
    raise ValueError("%s: connectivity %r is not one of %s for a %d-D array"
                     % (what, connectivity, sorted(_CONNECTIVITY[arr.ndim]), arr.ndim))
  if weights is not None:
    weights = np.asarray(weights)
    if weights.shape != arr.shape:
      raise ValueError("%s: weights of shape %r for labels of shape %r" % (what, weights.shape, arr.shape))
  # the kernels take an F-order volume: a C-order array is passed as its transpose, whose axes (and
  # anisotropy) run in reverse and whose F-order linear index is the array's own C-order index
  rev = arr.ndim > 1 and arr.flags.c_contiguous and not arr.flags.f_contiguous
  if arr.size == 0:
    return np.zeros(arr.shape, np.float32), (np.zeros(arr.shape, np.uint32) if parents else None)
  src = _source_indices(source, indices, np.asarray(labels), rev)
  vol = arr.T if rev else np.asfortranarray(arr)
  a = np.atleast_1d(np.asarray(anisotropy, dtype=np.float64))
  if a.shape == (3,) and arr.ndim < 3:
    a = a[:arr.ndim]  # the wheel's (x, y, z) default on an array with fewer axes: the array's own
  if a.shape not in ((1,), (arr.ndim,)):
    raise ValueError("%s: anisotropy %r does not have one value per array axis (%d)" % (what, anisotropy, arr.ndim))
  a = tuple(float(v) for v in np.broadcast_to(a, (arr.ndim,)))
  if not all(np.isfinite(v) and v > 0 for v in a):
    raise ValueError("%s: anisotropy %r must be positive and finite" % (what, anisotropy))
  a = (a[::-1] if rev else a) + (1.0,) * (3 - arr.ndim)
  w = None
  if weights is not None:
    w = np.asarray(weights.T if rev else weights, dtype=np.float32, order="F")
  shape = vol.shape + (1,) * (3 - vol.ndim)
  dist = np.empty(vol.shape, np.float32, order="F")
  par = np.empty(vol.shape, np.uint32, order="F") if parents else None
  ctx = ctx or _shim.default_context()
  _shim.check(ctx.lib.ign_geodesic(ctx.handle, _shim.ptr(vol), _shim.dtype_code(vol.dtype), *shape, conn,
                                   (ctypes.c_float * 3)(*a), _shim.ptr(w) if w is not None else None,
                                   _shim.ptr(src), src.size, _shim.ptr(dist),
                                   _shim.ptr(par) if parents else None))
  if rev:
    dist, par = dist.T, (par.T if parents else None)
  return dist, par


def _no_free_space(free_space_radius):
  if free_space_radius != 0:
    raise NotImplementedError("igneous_b200 dijkstra3d: free_space_radius other than 0 is not supported")


def euclidean_distance_field(field, source=None, anisotropy=(1, 1, 1), connectivity=26, free_space_radius=0,
                             source_indices=None, ctx=None):
  """float32 geodesic distance from `source` through `field`, a mask or a label array: each step costs
  the anisotropic Euclidean length of the step, rounded to float32.  `source`: a voxel, a list of
  voxels or {label: voxel}; or `source_indices`: linear indices in the array's memory order.  With one
  source per label every object of the array gets its own field in the same call."""
  _no_free_space(free_space_radius)
  return _solve(field, source, source_indices, connectivity, anisotropy, None, False, ctx,
                "euclidean_distance_field")[0]


def _weighted(field, source, indices, connectivity, labels, parents, ctx, what):
  field = np.asarray(field)
  if labels is None:
    labels = np.ones(field.shape, np.uint8, order="C" if field.flags.c_contiguous and not field.flags.f_contiguous
                     else "F")
  return _solve(labels, source, indices, connectivity, 1.0, field, parents, ctx, what)


def distance_field(field, source=None, connectivity=26, labels=None, source_indices=None, ctx=None):
  """float32 least cost from `source` where entering voxel q costs field[q] (finite and >= 0; the
  source's own value is not paid).  Without `labels` the whole array is one object."""
  return _weighted(field, source, source_indices, connectivity, labels, False, ctx, "distance_field")[0]


def parental_field(field, source=None, connectivity=26, labels=None, source_indices=None, ctx=None):
  """uint32 parents of the shortest paths of distance_field (see the module text).  Raises
  IgneousB200Error when a reached voxel has no predecessor of lower (distance, index): a stretch where
  float32 addition stalls, entered from a higher index.  The message names such a voxel; the refusal is of
  the whole call, every label of it."""
  return _weighted(field, source, source_indices, connectivity, labels, True, ctx, "parental_field")[1]


def path_from_parents(parents, target):
  """(n, ndim) array of the voxels from the source to `target`, following `parents`."""
  parents = np.asarray(parents)
  order = "C" if parents.flags.c_contiguous and not parents.flags.f_contiguous else "F"
  i = int(np.ravel_multi_index(tuple(int(c) for c in np.atleast_1d(target)), parents.shape, order=order))
  flat = parents.reshape(-1, order=order)
  path = [i]
  while flat[i]:
    i = int(flat[i]) - 1
    path.append(i)
    if len(path) > flat.size:
      raise ValueError("path_from_parents: the parents hold a cycle")
  return np.stack(np.unravel_index(np.array(path[::-1]), parents.shape, order=order), axis=1)
