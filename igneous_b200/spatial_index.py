"""Drop-in for the `find_objects` helper of the spatial index task, running on H100.

Reference call site (seung-lab/igneous):
  igneous/tasks/spatial_index.py:10-20,56   find_objects(img) -> scipy.ndimage.find_objects

The per-label bounding boxes come from one read of the volume in libigneous_b200
(ign_find_objects, igneous_b200/csrc/stats.cu); there is no CPU fallback.
"""
import ctypes

import numpy as np

from . import _shim

__all__ = ["find_objects", "bounding_boxes"]

_EMPTY = 0xFFFFFFFF


def _volume(labels):
  """3-D label array -> (F-contiguous array, reversed) where `reversed` means the array is the
  transpose of the caller's C-order input, so its axes come back in reverse order."""
  arr = np.asarray(labels)
  if arr.ndim != 3:
    raise ValueError("find_objects: expected a 3-D array, got shape %r" % (arr.shape,))
  if arr.dtype == np.bool_:
    arr = arr.view(np.uint8)
  _shim.require_unsigned(arr.dtype, "find_objects")
  if arr.dtype.kind != "u":
    raise NotImplementedError("igneous_b200 find_objects: dtype %s is not an unsigned integer" % arr.dtype)
  if arr.flags.c_contiguous and not arr.flags.f_contiguous:
    return arr.T, True
  return np.asfortranarray(arr), False


def bounding_boxes(labels, max_label=0, ctx=None):
  """(N, 6) int64 array: row l - 1 is (min, min, min, max, max, max) of label l over the three
  axes of `labels`, maxima exclusive (slice stops); row of a label without voxels is all -1.
  N is `max_label`, or the largest label when it is 0 (labels above max_label are ignored)."""
  vol, rev = _volume(labels)
  n = int(max_label)
  if n < 0:
    raise ValueError("find_objects: max_label %d is negative" % n)
  if n >= 1 << 32:  # refused before the (N, 6) result is allocated
    raise NotImplementedError("igneous_b200 find_objects: max_label %d is 2^32 or more; renumber the labels first "
                              "(fastremap.renumber)" % n)
  if vol.size == 0:
    return np.full((n, 6), -1, dtype=np.int64)
  code = _shim.dtype_code(vol.dtype)
  sx, sy, sz = vol.shape
  ctx = ctx or _shim.default_context()
  if n == 0:
    found = ctypes.c_uint64(0)
    _shim.check(ctx.lib.ign_find_objects(ctx.handle, _shim.ptr(vol), code, sx, sy, sz, ctypes.byref(found), None))
    n = int(found.value)
  out = np.full((n, 6), -1, dtype=np.int64)
  if n == 0:
    return out
  N = n
  boxes = np.empty((N, 6), dtype=np.uint32)
  nn = ctypes.c_uint64(N)
  _shim.check(ctx.lib.ign_find_objects(ctx.handle, _shim.ptr(vol), code, sx, sy, sz, ctypes.byref(nn),
                                       _shim.ptr(boxes)))
  present = boxes[:, 0] != _EMPTY
  out[present, :3] = boxes[present, :3]
  out[present, 3:] = boxes[present, 3:].astype(np.int64) + 1
  if rev:
    out = out[:, [2, 1, 0, 5, 4, 3]]
  return out


def find_objects(labels, max_label=0, ctx=None):
  """scipy.ndimage.find_objects(labels, max_label) for 3-D unsigned labels below 2^32: a list
  with one entry per label 1..N, a tuple of slices in array-axis order or None for a label
  without voxels.  C- and F-order inputs give the same answer.  A largest label of 2^32 or more
  raises NotImplementedError (renumber the labels first)."""
  boxes = bounding_boxes(labels, max_label, ctx)
  return [None if b[0] < 0 else (slice(b[0], b[3]), slice(b[1], b[4]), slice(b[2], b[5]))
          for b in boxes.tolist()]
