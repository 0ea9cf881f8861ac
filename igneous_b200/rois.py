"""The device half of compute_rois (DESIGN.md §5k): a slab of a layer thresholded on the GPU, then the
bounding boxes of the 26-connected components of the result that have at least dust_threshold voxels.
Only the boxes come back to the host."""
import math

import numpy as np

from . import _shim
from .storage import DeviceCutout


def _float32_threshold(t):
  """float32 t' with v > t == v > t' for every float32 v, under numpy's rules: a Python scalar (weakly
  typed) is rounded to float32 first; a numpy scalar of a wider type makes numpy compare in that type, and
  then t' is the largest float32 not above t"""
  with np.errstate(over="ignore"):
    t32 = np.float32(t)
  strong = isinstance(t, np.generic) and np.result_type(np.float32, t) != np.float32
  if strong and not np.isnan(t32) and float(t32) > float(t):
    t32 = np.nextafter(t32, np.float32(-np.inf))
  return t32


def threshold_dev(cutout, t):
  """np.greater(channel 0 of a DeviceCutout, t) as a u8 (0 / 1) DeviceCutout [x, y, z, 1], as numpy
  computes it: an unsigned integer layer compares exactly with floor(t) (every voxel is greater than a
  negative t, none than NaN or +inf), a float32 layer as _float32_threshold describes.  Signed integer
  layers raise NotImplementedError: the kernel compares unsigned."""
  ctx = cutout.ctx
  dt = np.dtype(cutout.dtype)
  _shim.require_unsigned(dt, "threshold")
  X, Y, Z = cutout.shape[:3]
  out = DeviceCutout.empty((X, Y, Z, 1), np.uint8, ctx)
  n = X * Y * Z
  if n == 0:
    return out
  if dt.kind == "f":
    bits = int(_float32_threshold(t).view(np.uint32))
  else:
    tf = float(t)
    if math.isnan(tf) or tf == math.inf:
      ctx.memset(out.buf, 0, n)
      return out
    bits = -1 if tf == -math.inf else math.floor(t)
    if bits < 0:
      ctx.memset(out.buf, 1, n)
      return out
    bits = min(bits, 2 ** 64 - 1)
  _shim.check(ctx.lib.ign_threshold_dev(ctx.handle, cutout.ptr, _shim.dtype_code(dt), n, bits, out.ptr))
  return out


def component_boxes_dev(mask, dust_threshold):
  """The 26-connected components of the non-zero voxels of a u8 DeviceCutout [x, y, z, 1] with at least
  dust_threshold voxels -> uint32 array (N, 7) of {voxel count, min x, min y, min z, max x, max y, max z}
  (maxima inclusive), in the order of each component's first voxel in F order (cc3d's numbering)."""
  ctx = mask.ctx
  X, Y, Z = mask.shape[:3]
  n = np.zeros(1, dtype=np.uint64)
  # room for the densest 26-connected layout (host pages never written are never touched); a slab of
  # 2^32 - 1 voxels or more is refused by the call before it writes, so it gets none
  cap = (X + 1) // 2 * ((Y + 1) // 2) * ((Z + 1) // 2) if X * Y * Z < 2 ** 32 - 1 else 0
  rows = np.empty((cap, 7), dtype=np.uint32)
  _shim.check(ctx.lib.ign_label_parts_dev(ctx.handle, mask.ptr, _shim.IGN_U8, X, Y, Z, 26, max(int(dust_threshold), 0),
                                          None, _shim.ptr(rows), cap, _shim.ptr(n)))
  return rows[:int(n[0])].copy()


def channel0(cutout):
  """channel 0 of a DeviceCutout, as a view of the same device memory"""
  return DeviceCutout(cutout.buf, tuple(cutout.shape[:3]) + (1,), cutout.dtype, cutout.ctx)
