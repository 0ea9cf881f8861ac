"""Drop-in for the `edt` wheel's multi-label anisotropic Euclidean distance transform, running on H100.

Reference call site (seung-lab/igneous):
  igneous/tasks/skeleton.py:54, :312   SkeletonTask -> kimimaro.skeletonize, whose distance-to-boundary
                                       field is edt.edt(labels, anisotropy, black_border)

The rule is DESIGN.md §5d (parity with the wheel is unpinned offline): edtsq[p] = 0 where the label is
0, else the least sum_i (anisotropy[i] * (p_i - q_i))^2 over voxels q of another label, the one-voxel
shell around the array counting as label 0 with black_border; +inf where there is no such q.  edt is
its float32 sqrt.  Labels are compared for equality only.  The transform runs in libigneous_b200
(ign_edt, igneous_b200/csrc/edt.cu); there is no CPU fallback.
"""
import ctypes

import numpy as np

from . import _shim

__all__ = ["edt", "edtsq"]

_UNSIGNED = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}


def _labels(data):
  arr = np.asarray(data)
  if arr.ndim not in (1, 2, 3):
    raise ValueError("edt: expected a 1-, 2- or 3-D array, got shape %r" % (arr.shape,))
  if arr.dtype == np.bool_ or arr.dtype.kind in "iu":
    return arr.view(_UNSIGNED[arr.dtype.itemsize])  # only equality matters
  raise NotImplementedError("igneous_b200 edt: label dtype %s is not supported (bool or integer labels)" % arr.dtype)


def _anisotropy(anisotropy, ndim):
  if anisotropy is None:
    return (1.0,) * ndim
  a = np.atleast_1d(np.asarray(anisotropy, dtype=np.float64))
  if a.shape == (1,):
    a = np.repeat(a, ndim)
  if a.shape != (ndim,):
    raise ValueError("edt: anisotropy %r does not have one value per array axis (%d)" % (anisotropy, ndim))
  if not np.all(np.isfinite(a) & (a > 0)):
    raise ValueError("edt: anisotropy %r must be positive and finite" % (anisotropy,))
  return tuple(float(v) for v in a)


def _run(data, anisotropy, black_border, order, voxel_graph, squared, ctx):
  if voxel_graph is not None:
    raise NotImplementedError("igneous_b200 edt: voxel_graph is not supported")
  if order not in ("K", "C", "F", "A"):
    raise ValueError("edt: order must be 'K', 'C', 'F' or 'A', got %r" % (order,))
  arr = _labels(data)
  a = _anisotropy(anisotropy, arr.ndim)
  if arr.size == 0:
    return np.zeros(arr.shape, dtype=np.float32)
  # the kernels take an F-order volume: a C-order array is passed as its transpose, whose axes
  # (and anisotropy) run in reverse; the result is transposed back
  rev = arr.ndim > 1 and arr.flags.c_contiguous and not arr.flags.f_contiguous
  vol = arr.T if rev else np.asfortranarray(arr)
  a = a[::-1] if rev else a
  shape = vol.shape + (1,) * (3 - vol.ndim)
  aniso = (ctypes.c_float * 3)(*(a + (float("inf"),) * (3 - vol.ndim)))  # +inf: an axis the array lacks
  out = np.empty(vol.shape, dtype=np.float32, order="F")
  ctx = ctx or _shim.default_context()
  _shim.check(ctx.lib.ign_edt(ctx.handle, _shim.ptr(vol), _shim.dtype_code(vol.dtype), *shape, aniso,
                              bool(black_border), squared, _shim.ptr(out)))
  return out.T if rev else out


def edtsq(data, anisotropy=None, black_border=False, order="K", parallel=1, voxel_graph=None, ctx=None):
  """Squared multi-label anisotropic Euclidean distance transform of a 1-, 2- or 3-D label array:
  float32 of the input's shape (0 on label 0, +inf where no other label nor black border exists).
  `anisotropy` has one value per array axis (default 1.0); `order` and `parallel` are accepted and
  ignored (the axes are the array's axes whatever its memory order)."""
  return _run(data, anisotropy, black_border, order, voxel_graph, True, ctx)


def edt(data, anisotropy=None, black_border=False, order="K", parallel=1, voxel_graph=None, ctx=None):
  """sqrt of edtsq, correctly rounded in float32 (edt == np.sqrt(edtsq) bit for bit)."""
  return _run(data, anisotropy, black_border, order, voxel_graph, False, ctx)
