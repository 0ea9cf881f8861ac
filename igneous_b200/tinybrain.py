"""Drop-in for the `tinybrain` calls on the igneous hot path, running on H100.

Reference call sites (seung-lab/igneous):
  igneous/tasks/image/image.py:46-55  downsample_method_to_fn binds
      tinybrain.downsample_with_averaging / downsample_segmentation (+sparse)
  igneous/tasks/image/image.py:91     mips = fn(image, factors[0], num_mips=num_mips)

Same names, argument meaning and return convention (a list of `num_mips`
Fortran-ordered arrays with the input's number of dimensions).  Everything is
computed by libigneous_b200 on the GPU; there is no CPU fallback.
"""
import numpy as np

from . import _shim

__all__ = ["downsample_segmentation", "downsample_with_averaging", "downsample_with_min_pooling",
           "downsample_with_max_pooling", "downsample_with_striding"]

# upstream render rule for integer averaging; parity unpinned offline
# (SURVEY.md 8(c)), so it stays a runtime knob.
DEFAULT_ROUNDING = _shim.ROUND_FLOOR


def _is_221(factor):
  f = tuple(int(v) for v in factor)
  return f[:3] == (2, 2, 1) and all(v == 1 for v in f[3:])


def _out_shapes(shape, num_mips):
  shapes = []
  sx, sy = shape[0], shape[1]
  for _ in range(num_mips):
    sx, sy = (sx + 1) // 2, (sy + 1) // 2
    shapes.append((sx, sy) + tuple(shape[2:]))
  return shapes


def _pool(img, factor, num_mips, mode, flag, ctx):
  num_mips = int(num_mips)
  if num_mips < 1:
    return []
  img = np.asarray(img)
  ndim = img.ndim
  arr, sx, sy, nz = _shim.as_fortran_volume(img)
  code = _shim.dtype_code(arr.dtype)
  if not mode:
    _shim.require_unsigned(arr.dtype, "averaging")
  if not mode and code == _shim.IGN_U64:
    raise NotImplementedError("igneous_b200 averaging: uint64 images are not supported")
  ctx = ctx or _shim.default_context()
  shapes = _out_shapes(arr.shape, num_mips)
  outs = [np.empty(s, dtype=arr.dtype, order="F") for s in shapes]
  if arr.size:
    fn = ctx.lib.ign_pool_mode_2x2x1 if mode else ctx.lib.ign_pool_avg_2x2x1
    _shim.check(fn(ctx.handle, _shim.ptr(arr), code, sx, sy, nz, num_mips, int(flag),
                   _shim.void_pp([o.ctypes.data for o in outs])))
  if ndim == 2:
    outs = [o[:, :, 0] for o in outs]
  return outs


def downsample_segmentation(img, factor, num_mips=1, sparse=False, ctx=None):
  """2x2x1 mode pooling pyramid (COUNTLESS 2-D, recursive per mip); other factors of
  1 or 2 per axis (2x2x2 ...) use the generic block-mode kernel."""
  if not _is_221(factor):
    return _select(img, factor, num_mips, _OP_MODE_SPARSE if sparse else _OP_MODE, ctx)
  return _pool(img, factor, num_mips, True, bool(sparse), ctx)


def downsample_with_averaging(img, factor, num_mips=1, sparse=False, ctx=None,
                              rounding=None):
  """2x2x1 average pooling pyramid (exact sums in groups of four mips); other factors
  of 1 or 2 per axis (2x2x2 ...) use the generic block-average kernel, recursively."""
  rounding = DEFAULT_ROUNDING if rounding is None else rounding
  if sparse or not _is_221(factor):
    if np.asarray(img).dtype == np.uint64:
      raise NotImplementedError("igneous_b200 averaging: uint64 images are not supported")
    # sparse=True: mean of the non-zero samples (generic kernel for every factor)
    return _select(img, factor, num_mips, (_OP_AVG_SPARSE if sparse else _OP_AVG) + int(rounding), ctx)
  return _pool(img, factor, num_mips, False, rounding, ctx)


# ign_pool_select ops
_OP_MIN, _OP_MAX, _OP_STRIDE, _OP_MODE, _OP_MODE_SPARSE, _OP_AVG, _OP_AVG_SPARSE = 0, 1, 2, 3, 4, 5, 8


def _select(img, factor, num_mips, op, ctx):
  f = tuple(int(v) for v in factor)
  if len(f) < 3 or any(v not in (1, 2) for v in f[:3]) or any(v != 1 for v in f[3:]):
    raise NotImplementedError("igneous_b200 pooling: factors must be 1 or 2 per axis, got %r" % (factor,))
  num_mips = int(num_mips)
  img = np.asarray(img)
  if op not in (_OP_STRIDE, _OP_MODE):  # min / max / averages / sparse modes order or add values
    _shim.require_unsigned(img.dtype, "min / max / average / sparse pooling")
  if num_mips < 1:
    return []
  arr = np.asfortranarray(img)
  if arr.ndim == 2:
    arr = arr[:, :, np.newaxis]
  chans = [arr] if arr.ndim == 3 else [arr[..., c] for c in range(arr.shape[3])]
  ctx = ctx or _shim.default_context()
  per_chan = []
  for ch in chans:
    ch = np.asfortranarray(ch)
    sx, sy, sz = ch.shape
    outs, shp = [], (sx, sy, sz)
    for _ in range(num_mips):
      shp = tuple((s + ff - 1) // ff for s, ff in zip(shp, f[:3]))
      outs.append(np.empty(shp, dtype=ch.dtype, order="F"))
    if ch.size:
      _shim.check(ctx.lib.ign_pool_select(ctx.handle, _shim.ptr(ch), _shim.dtype_code(ch.dtype), sx, sy, sz, *f[:3],
                                          num_mips, op, _shim.void_pp([o.ctypes.data for o in outs])))
    per_chan.append(outs)
  if img.ndim == 4:
    return [np.asfortranarray(np.stack([pc[m] for pc in per_chan], axis=3)) for m in range(num_mips)]
  res = per_chan[0]
  return [o[:, :, 0] for o in res] if img.ndim == 2 else res


def downsample_dev(cutout, method, factor, num_mips, sparse=False, rounding=None, ctx=None):
  """The pyramid of a device cutout ([x,y,z,c] F-order, storage.DeviceCutout) as a list of `num_mips`
  device cutouts, computed where the cutout is.  method: "mode", "average", "min", "max" or
  "striding"; the same kernels, rules and refusals as the host functions above."""
  from .storage import DeviceCutout
  num_mips = int(num_mips)
  if num_mips < 1:
    return []
  ctx = ctx or _shim.default_context()
  dt = np.dtype(cutout.dtype)
  rounding = DEFAULT_ROUNDING if rounding is None else rounding
  sx, sy, sz, nc = cutout.shape
  if method == "average" and dt == np.uint64:
    raise NotImplementedError("igneous_b200 averaging: uint64 images are not supported")
  if _is_221(factor) and (method == "mode" or (method == "average" and not sparse)):
    if method == "average":
      _shim.require_unsigned(dt, "averaging")
    outs = [DeviceCutout.empty(s + (nc,), dt, ctx) for s in _out_shapes((sx, sy, sz), num_mips)]
    if cutout.size:
      fn = ctx.lib.ign_pool_mode_2x2x1_dev if method == "mode" else ctx.lib.ign_pool_avg_2x2x1_dev
      _shim.check(fn(ctx.handle, cutout.ptr, _shim.dtype_code(dt), sx, sy, sz * nc, num_mips,
                     int(sparse) if method == "mode" else int(rounding), _shim.void_pp([o.buf.ptr for o in outs])))
    return outs
  op = {"min": _OP_MIN, "max": _OP_MAX, "striding": _OP_STRIDE,
        "mode": _OP_MODE_SPARSE if sparse else _OP_MODE,
        "average": (_OP_AVG_SPARSE if sparse else _OP_AVG) + int(rounding)}[method]
  f = tuple(int(v) for v in factor)
  if len(f) < 3 or any(v not in (1, 2) for v in f[:3]) or any(v != 1 for v in f[3:]):
    raise NotImplementedError("igneous_b200 pooling: factors must be 1 or 2 per axis, got %r" % (factor,))
  if op not in (_OP_STRIDE, _OP_MODE):
    _shim.require_unsigned(dt, "min / max / average / sparse pooling")
  shapes, shp = [], (sx, sy, sz)
  for _ in range(num_mips):
    shp = tuple((s + ff - 1) // ff for s, ff in zip(shp, f[:3]))
    shapes.append(shp)
  outs = [DeviceCutout.empty(s + (nc,), dt, ctx) for s in shapes]
  if cutout.size:
    for c in range(nc):  # one channel per call, as the host path does
      ins = cutout.buf.ptr + c * sx * sy * sz * dt.itemsize
      chans = [o.buf.ptr + c * int(np.prod(s)) * dt.itemsize for o, s in zip(outs, shapes)]
      _shim.check(ctx.lib.ign_pool_select_dev(ctx.handle, ins, _shim.dtype_code(dt), sx, sy, sz, *f[:3], num_mips,
                                              op, _shim.void_pp(chans)))
  return outs


def downsample_with_min_pooling(img, factor, num_mips=1, ctx=None):
  return _select(img, factor, num_mips, _OP_MIN, ctx)


def downsample_with_max_pooling(img, factor, num_mips=1, ctx=None):
  return _select(img, factor, num_mips, _OP_MAX, ctx)


def downsample_with_striding(img, factor, num_mips=1, ctx=None):
  return _select(img, factor, num_mips, _OP_STRIDE, ctx)
