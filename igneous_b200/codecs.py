"""Chunk codecs of the Precomputed format on H100 (SURVEY.md 8(f) row 1).

`compressed_segmentation` is what CloudVolume applies on the host either side of the hot path
when a segmentation layer asks for it (igneous/task_creation/common.py:215-236 set_encoding,
igneous/tasks/image/image.py:95-100 uploads, ccl.py:346-356); here the chunk is encoded /
decoded where the labels already are.  Byte-identical to the CPU restatement in oracle/ (whose
encoder layout is itself parity-unpinned: no upstream vector exists offline).

crackle and compresso are NOT implemented: both are un-vendored third-party formats whose
specifications are not in the reference checkout.
"""
import ctypes as c

import numpy as np

from . import _shim

__all__ = ["cseg_encode", "cseg_decode"]


def _chunk(labels):
  arr = np.asarray(labels)
  if arr.ndim == 3:
    arr = arr[..., np.newaxis]
  if arr.ndim != 4:
    raise ValueError("compressed_segmentation chunks are [x, y, z] or [x, y, z, channel] arrays")
  if arr.dtype not in (np.uint32, np.uint64):
    raise NotImplementedError("compressed_segmentation holds uint32 / uint64 labels, got %s" % arr.dtype)
  return np.asfortranarray(arr)


def cseg_encode(labels, block_size=(8, 8, 8), ctx=None):
  """labels [x,y,z(,c)] uint32 / uint64 -> the chunk file as bytes."""
  arr = _chunk(labels)
  ctx = ctx or _shim.default_context()
  sx, sy, sz, sc = arr.shape
  bx, by, bz = (int(v) for v in block_size)
  args = [ctx.handle, _shim.ptr(arr), c.c_int(_shim.dtype_code(arr.dtype)), c.c_uint64(sx), c.c_uint64(sy),
          c.c_uint64(sz), c.c_uint64(sc), c.c_uint32(bx), c.c_uint32(by), c.c_uint32(bz)]
  n = c.c_uint64(0)
  gx, gy, gz = -(-sx // bx), -(-sy // by), -(-sz // bz)
  # worst case: every voxel its own table entry
  cap = sc * (1 + 2 * gx * gy * gz + (arr.dtype.itemsize // 4 + 1) * gx * gy * gz * bx * by * bz)
  cap = int(min(cap, 1 << 26))
  out = np.empty(cap, dtype=np.uint32)
  _shim.check(ctx.lib.ign_cseg_encode(*args, _shim.ptr(out), c.c_uint64(cap), c.byref(n)))
  if n.value > cap:  # does not happen for 24-bit addressable chunks; kept for safety
    out = np.empty(int(n.value), dtype=np.uint32)
    _shim.check(ctx.lib.ign_cseg_encode(*args, _shim.ptr(out), c.c_uint64(n.value), c.byref(n)))
  return out[:int(n.value)].tobytes()


def cseg_decode(data, shape, dtype, block_size=(8, 8, 8), ctx=None):
  """chunk file bytes -> labels [x,y,z,c] (Fortran order)."""
  dtype = np.dtype(dtype)
  if dtype not in (np.uint32, np.uint64):
    raise NotImplementedError("compressed_segmentation holds uint32 / uint64 labels, got %s" % dtype)
  words = np.frombuffer(data, dtype=np.uint32)
  shape = tuple(int(v) for v in shape)
  if len(shape) == 3:
    shape = shape + (1,)
  ctx = ctx or _shim.default_context()
  out = np.empty(shape, dtype=dtype, order="F")
  bx, by, bz = (int(v) for v in block_size)
  _shim.check(ctx.lib.ign_cseg_decode(
    ctx.handle, _shim.ptr(np.ascontiguousarray(words)), c.c_uint64(len(words)), c.c_int(_shim.dtype_code(dtype)),
    c.c_uint64(shape[0]), c.c_uint64(shape[1]), c.c_uint64(shape[2]), c.c_uint64(shape[3]), c.c_uint32(bx),
    c.c_uint32(by), c.c_uint32(bz), _shim.ptr(out)))
  return out
