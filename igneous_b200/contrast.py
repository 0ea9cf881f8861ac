"""Luminance histograms, contrast stretch, CLAHE and quantization on H100.

Reference call sites (seung-lab/igneous):
  igneous/tasks/image/image.py:374-376  np.bincount(img2d) accumulated into `levels` (LuminanceLevelsTask)
  igneous/tasks/image/image.py:257-280  per-slice stretch, np.round, np.clip, astype (ContrastNormalizationTask)
  igneous/tasks/image/image.py:285-314  find_section_clamping_values
  igneous/tasks/image/image.py:185,202  cv2.createCLAHE(clipLimit, tileGridSize).apply(img) (CLAHETask)
  igneous/tasks/image/image.py:158-159  (image * 255.0).astype(np.uint8) (QuantizeTask)

The rules are those of DESIGN.md §5b.  Everything but find_section_clamping_values (a
host-side scan of one histogram per slice) runs in libigneous_b200; there is no CPU
fallback.
"""
import numpy as np

from . import _shim

__all__ = ["histogram", "find_section_clamping_values", "stretch", "quantize", "clahe", "createCLAHE"]

_LEVEL_DTYPES = (np.dtype(np.uint8), np.dtype(np.uint16))


def _levels_dtype(dtype, what):
  dt = np.dtype(dtype)
  if dt not in _LEVEL_DTYPES:
    raise NotImplementedError("igneous_b200 %s: dtype %s is not supported (uint8 / uint16 only)" % (what, dt))
  return dt


def histogram(arr, ctx=None):
  """Exact per-value counts of a uint8 / uint16 array: uint64 array of 256 / 65,536 bins
  (np.bincount(arr.ravel(), minlength=2**bits))."""
  arr = np.asarray(arr)
  dt = _levels_dtype(arr.dtype, "histogram")
  hist = np.zeros(1 << (8 * dt.itemsize), dtype=np.uint64)
  if arr.size:
    flat = np.ascontiguousarray(arr.ravel(order="K"))
    ctx = ctx or _shim.default_context()
    _shim.check(ctx.lib.ign_histogram(ctx.handle, _shim.ptr(flat), _shim.dtype_code(dt), flat.size, _shim.ptr(hist)))
  return hist


def find_section_clamping_values(levels, lower_fract, upper_fract):
  """(lower, upper): the last bin whose cdf fraction is at most lower_fract / upper_fract, with
  bin 0 left out of the counts (image.py:285-314; note the caller passes 1 - upper_clip_fraction).
  (0, 0) when every count outside bin 0 is zero."""
  cdf = np.asarray(levels, dtype=np.uint64).copy()
  if cdf.size == 0:
    return 0, 0
  cdf[0] = 0
  cdf = np.cumsum(cdf, dtype=np.uint64)
  total = float(cdf[-1])
  if total == 0:
    return 0, 0
  frac = cdf.astype(np.float64) / total

  def last_at_or_below(f):
    above = np.flatnonzero(frac > float(f))
    first = int(above[0]) if above.size else cdf.size
    return max(first - 1, 0)

  return last_at_or_below(lower_fract), last_at_or_below(upper_fract)


def stretch(image, levels_per_z, lower_clip, upper_clip, minval=None, maxval=None, out_dtype=None, ctx=None):
  """ContrastNormalizationTask's per-slice stretch of an (x, y, z[, c]) uint8 / uint16 image.
  levels_per_z[z] is slice z's histogram; lower_clip / upper_clip are the clip fractions (upper
  as the task takes it, i.e. the fraction cut from the top).  Returns an array of out_dtype
  (default: the input's dtype) with the input's shape."""
  image = np.asarray(image)
  dt = _levels_dtype(image.dtype, "stretch")
  out_dtype = np.dtype(out_dtype if out_dtype is not None else dt)
  if out_dtype not in (np.dtype(np.uint8), np.dtype(np.uint16), np.dtype(np.uint32), np.dtype(np.float32)):
    raise NotImplementedError("igneous_b200 stretch: output dtype %s is not supported" % out_dtype)
  arr = np.asfortranarray(image if image.ndim != 2 else image[:, :, np.newaxis])
  if arr.ndim not in (3, 4):
    raise ValueError("stretch expects a 2-, 3- or 4-D array, got shape %r" % (image.shape,))
  sx, sy, sz = arr.shape[:3]
  sc = arr.shape[3] if arr.ndim == 4 else 1
  if len(levels_per_z) != sz:
    raise ValueError("stretch: %d histograms for %d slices" % (len(levels_per_z), sz))
  maxval_t = float(2 ** (8 * dt.itemsize) - 1)
  lo = 0.0 if minval is None else float(minval)
  hi = maxval_t if maxval is None else float(maxval)
  if out_dtype.kind == "u":
    # the clip runs in float32, so the bounds are checked as float32 values: a uint32 maxval above
    # 4294967040 rounds to 2^32, which the cast to uint32 cannot hold
    top = float(np.iinfo(out_dtype).max)
    lo32, hi32 = float(np.float32(lo)), float(np.float32(hi))
    if not (0.0 <= lo32 <= top and 0.0 <= hi32 <= top):
      raise ValueError("stretch: clip range [%r, %r] (in float32 [%r, %r]) outside %s's [0, %d]"
                       % (lo, hi, lo32, hi32, out_dtype, top))
  if lo > hi:
    raise ValueError("stretch: minval %r > maxval %r" % (lo, hi))
  bounds = [find_section_clamping_values(lv, lower_clip, 1 - upper_clip) for lv in levels_per_z]
  lower = np.array([b[0] for b in bounds], dtype=np.uint32)
  upper = np.array([b[1] for b in bounds], dtype=np.uint32)
  out = np.empty(arr.shape, dtype=out_dtype, order="F")
  if arr.size:
    ctx = ctx or _shim.default_context()
    _shim.check(ctx.lib.ign_contrast_stretch(
      ctx.handle, _shim.ptr(arr), _shim.dtype_code(dt), sx, sy, sz, sc, _shim.ptr(lower), _shim.ptr(upper), lo, hi,
      _shim.ptr(out), _shim.dtype_code(out_dtype)))
  return out.reshape(image.shape, order="F")


def quantize(image, ctx=None):
  """QuantizeTask's rule on channel 0 of a float32 (x, y, z[, c]) image: uint8 (x, y, z, 1) with
  trunc(v * 255), saturated to [0, 255], NaN -> 0."""
  image = np.asarray(image)
  if image.dtype != np.float32:
    raise NotImplementedError("igneous_b200 quantize: dtype %s is not float32" % image.dtype)
  if image.ndim == 3:
    image = image[..., np.newaxis]
  if image.ndim != 4:
    raise ValueError("quantize expects a 3- or 4-D array, got shape %r" % (image.shape,))
  chan = np.asfortranarray(image[..., 0])
  out = np.empty(chan.shape + (1,), dtype=np.uint8, order="F")
  if chan.size:
    ctx = ctx or _shim.default_context()
    _shim.check(ctx.lib.ign_quantize(ctx.handle, _shim.ptr(chan), chan.size, _shim.ptr(out)))
  return out


def clahe(stack, clip_limit=40.0, tile_grid_size=(8, 8), ctx=None):
  """cv2.createCLAHE(clip_limit, tile_grid_size).apply on every z-slice of an (x, y[, z]) uint8 /
  uint16 stack, all slices in one call.  Axis 0 is OpenCV's rows, so tile_grid_size[0] tiles go
  across axis 1 and tile_grid_size[1] across axis 0."""
  stack = np.asarray(stack)
  if stack.dtype not in _LEVEL_DTYPES:
    raise NotImplementedError("igneous_b200 clahe: dtype %s is not supported (uint8 / uint16 only)" % stack.dtype)
  arr = np.asfortranarray(stack if stack.ndim != 2 else stack[:, :, np.newaxis])
  if arr.ndim != 3:
    raise ValueError("clahe expects a 2- or 3-D array, got shape %r" % (stack.shape,))
  gx, gy = (int(v) for v in tile_grid_size)
  if gx < 1 or gy < 1:
    raise ValueError("clahe: tile_grid_size %r" % (tile_grid_size,))
  out = np.empty(arr.shape, dtype=arr.dtype, order="F")
  if arr.size:
    ctx = ctx or _shim.default_context()
    _shim.check(ctx.lib.ign_clahe(ctx.handle, _shim.ptr(arr), _shim.dtype_code(arr.dtype), *arr.shape,
                                  float(clip_limit), gx, gy, _shim.ptr(out)))
  return out.reshape(stack.shape, order="F")


class CLAHE:
  """What cv2.createCLAHE returns, for the calls CLAHETask makes."""

  def __init__(self, clipLimit=40.0, tileGridSize=(8, 8)):
    self.clipLimit = float(clipLimit)
    self.tileGridSize = tuple(int(v) for v in tileGridSize)

  def apply(self, src, dst=None):
    src = np.asarray(src)
    if src.ndim != 2:
      raise ValueError("CLAHE.apply expects a 2-D image, got shape %r" % (src.shape,))
    return clahe(src, self.clipLimit, self.tileGridSize)

  def getClipLimit(self):
    return self.clipLimit

  def getTilesGridSize(self):
    return self.tileGridSize


def createCLAHE(clipLimit=40.0, tileGridSize=(8, 8)):
  """Drop-in for cv2.createCLAHE (igneous/tasks/image/image.py:185)."""
  return CLAHE(clipLimit, tileGridSize)
