"""Drop-in for the `cc3d` (connected-components-3d) calls on the igneous hot
path, running on H100.

Reference call sites (seung-lab/igneous):
  igneous/tasks/image/ccl.py:169-172  cc3d.dust(labels, threshold=, connectivity=6, in_place=True)
  igneous/tasks/image/ccl.py:173      cc3d.connected_components(labels, connectivity=6, out_dtype=np.uint64)
  igneous/tasks/image/ccl.py:235-238  ... return_N=True
Only 6-connectivity is implemented (the only one igneous's CCL uses).
Output ids are 1..N in order of each component's first voxel in Fortran
raster order of the array as given; 0 stays background.
"""
import ctypes

import numpy as np

from . import _shim

__all__ = ["connected_components", "dust", "ccl_task"]

_OUT_OK = (np.dtype(np.uint16), np.dtype(np.uint32), np.dtype(np.uint64))


def _volume(labels):
  labels = np.asarray(labels)
  if labels.ndim == 2:
    labels = labels[:, :, np.newaxis]
  if labels.ndim == 1:
    labels = labels[:, np.newaxis, np.newaxis]
  if labels.ndim != 3:
    raise ValueError("cc3d: expected a 1-, 2- or 3-D array, got ndim=%d" % labels.ndim)
  return np.asfortranarray(labels)


def _require_6(connectivity):
  if connectivity != 6:
    raise NotImplementedError(
      "igneous_b200.cc3d implements connectivity=6 only (got %r)" % (connectivity,))


def connected_components(labels, connectivity=6, out_dtype=None, return_N=False, ctx=None):
  _require_6(connectivity)
  shape_in = np.asarray(labels).shape
  arr = _volume(labels)
  if arr.dtype == np.bool_:
    arr = arr.view(np.uint8)
  out_dtype = np.dtype(np.uint32 if out_dtype is None else out_dtype)
  if out_dtype not in _OUT_OK:
    raise NotImplementedError("cc3d out_dtype must be uint16/uint32/uint64, got %s" % out_dtype)
  out = np.zeros(arr.shape, dtype=out_dtype, order="F")
  n = ctypes.c_uint64(0)
  if arr.size:
    ctx = ctx or _shim.default_context()
    sx, sy, sz = arr.shape
    _shim.check(ctx.lib.ign_ccl6(ctx.handle, _shim.ptr(arr), _shim.dtype_code(arr.dtype), sx, sy, sz,
                                 _shim.ptr(out), _shim.dtype_code(out_dtype), ctypes.byref(n)))
  out = out.reshape(shape_in, order="F")
  return (out, int(n.value)) if return_N else out


def dust(img, threshold, connectivity=6, in_place=False, ctx=None):
  """Zero every 6-connected component with fewer than `threshold` voxels."""
  _require_6(connectivity)
  src = np.asarray(img)
  if threshold is None or threshold <= 0 or src.size == 0:
    return src if in_place else src.copy(order="F")
  arr = _volume(src)
  work = arr.view(np.uint8) if arr.dtype == np.bool_ else arr
  if work is src or np.shares_memory(work, src):
    work = work.copy(order="F") if not in_place else work
  ctx = ctx or _shim.default_context()
  sx, sy, sz = work.shape
  _shim.check(ctx.lib.ign_dust(ctx.handle, _shim.ptr(work), _shim.dtype_code(work.dtype), sx, sy, sz, int(threshold)))
  res = work.view(src.dtype).reshape(src.shape, order="F")
  if in_place:
    if not np.shares_memory(res, src):
      src[...] = res  # caller's array was not Fortran contiguous
    return img if isinstance(img, np.ndarray) else src
  return res


def ccl_task(image, shape, threshold_gte=None, threshold_lte=None, dust_threshold=0,
             label_offset=0, ctx=None):
  """The fused body shared by CCLFacesTask / CCLEquivalancesTask / RelabelCCLTask
  (igneous/tasks/image/ccl.py:165-175, 228-240, 331-344): threshold_image ->
  blackout_non_face_rails(shape) -> dust -> 6-connected CCL -> += label_offset
  with the background re-zeroed, in one pass over HBM.  Returns (uint64 labels, N)."""
  arr = _volume(image)
  if arr.dtype == np.bool_:
    arr = arr.view(np.uint8)
  if threshold_gte is not None or threshold_lte is not None:
    _shim.require_unsigned(arr.dtype, "thresholded CCL")
    if arr.dtype == np.uint64:
      for t in (threshold_gte, threshold_lte):
        # the kernel receives the threshold as a double and compares integer bounds derived from it
        if isinstance(t, (int, np.integer)) and float(int(t)) != int(t):
          raise NotImplementedError("igneous_b200.cc3d.ccl_task: uint64 threshold %d is not exactly "
                                    "representable as a double" % int(t))
  ctx = ctx or _shim.default_context()
  sx, sy, sz = arr.shape
  out = np.zeros(arr.shape, dtype=np.uint64, order="F")
  n = ctypes.c_uint64(0)
  if arr.size:
    _shim.check(ctx.lib.ign_ccl_task(
      ctx.handle, _shim.ptr(arr), _shim.dtype_code(arr.dtype), sx, sy, sz,
      threshold_gte is not None, float(threshold_gte) if threshold_gte is not None else 0.0,
      threshold_lte is not None, float(threshold_lte) if threshold_lte is not None else 0.0,
      int(shape[0]), int(shape[1]), int(shape[2]), int(dust_threshold or 0), int(label_offset),
      _shim.ptr(out), ctypes.byref(n)))
  return out, int(n.value)
