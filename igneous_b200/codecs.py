"""Chunk codecs of the Precomputed format on H100 (SURVEY.md 8(f) row 1).

`compressed_segmentation` is what CloudVolume applies on the host either side of the hot path
when a segmentation layer asks for it (igneous/task_creation/common.py:215-236 set_encoding,
igneous/tasks/image/image.py:95-100 uploads, ccl.py:346-356); here the chunk is encoded /
decoded where the labels already are.  Byte-identical to the CPU restatement in oracle/ (whose
encoder layout is itself parity-unpinned: no upstream vector exists offline).

`jpeg` is the encoding of uint8 image layers (igneous_cli/cli.py:64, `jpeg_quality` in
set_encoding).  A chunk [x, y, z(, 1)] is one grayscale JPEG of width sx and height sy*sz; the
encoder writes libjpeg's default stream byte for byte, the decoder reproduces libjpeg's islow
decode (oracle_jpeg/ restates both; tests/golden/jpeg_libjpeg.npz pins them to libjpeg-turbo).
Chunks are encoded / decoded a batch per call.

crackle and compresso are NOT implemented: both are un-vendored third-party formats whose
specifications are not in the reference checkout.
"""
import ctypes as c

import numpy as np

from . import _shim

__all__ = ["cseg_encode", "cseg_decode", "jpeg_encode", "jpeg_decode", "jpeg_encode_batch", "jpeg_decode_batch",
           "cseg_encode_batch_dev", "cseg_decode_batch_dev", "jpeg_encode_batch_dev", "jpeg_decode_batch_dev"]


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
  args = [ctx.handle, _shim.ptr(arr), _shim.dtype_code(arr.dtype), sx, sy, sz, sc, bx, by, bz]
  n = c.c_uint64(0)
  # the worst case, capped at the longest stream the format allows: per channel its offset word and at
  # most 0xFFFFFF + 1024 words (the encoder refuses longer channels before it looks at the capacity)
  cap = min(cseg_capacity_words([(sx, sy, sz)], sc, arr.dtype, block_size), sc * (0xFFFFFF + 1024 + 1))
  out = np.empty(cap, dtype=np.uint32)
  _shim.check(ctx.lib.ign_cseg_encode(*args, _shim.ptr(out), cap, c.byref(n)))
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
  _shim.check(ctx.lib.ign_cseg_decode(ctx.handle, _shim.ptr(np.ascontiguousarray(words)), len(words),
                                      _shim.dtype_code(dtype), shape[0], shape[1], shape[2], shape[3], bx, by, bz,
                                      _shim.ptr(out)))
  return out


JPEG_MAX_SIDE = 65535


def _jpeg_shape(shape):
  shape = tuple(int(v) for v in shape)
  if len(shape) == 4:
    if shape[3] != 1:
      raise NotImplementedError("jpeg chunks hold one channel, got %d" % shape[3])
    shape = shape[:3]
  if len(shape) != 3 or min(shape) < 1:
    raise ValueError("jpeg chunks are non-empty [x, y, z] or [x, y, z, 1] arrays, got shape %r" % (shape,))
  if shape[0] > JPEG_MAX_SIDE or shape[1] * shape[2] > JPEG_MAX_SIDE:
    raise ValueError("a jpeg chunk is an image of sx by sy*sz pixels, at most %d per side; got %r"
                     % (JPEG_MAX_SIDE, shape))
  return shape


def _jpeg_chunk(chunk):
  arr = np.asarray(chunk)
  if arr.dtype != np.uint8:
    raise NotImplementedError("jpeg holds uint8 images, got %s" % arr.dtype)
  shape = _jpeg_shape(arr.shape)
  return np.asfortranarray(arr[..., 0] if arr.ndim == 4 else arr), shape


def _restart(restart_interval):
  """None: one block row per chunk (-1 at the C ABI); 0: no restart markers; n: every n blocks."""
  if restart_interval is None:
    return -1
  ri = int(restart_interval)
  if not 0 <= ri <= 65535:
    raise ValueError("restart_interval must be in 0..65535 blocks, got %d" % ri)
  return ri


def jpeg_encode_batch(chunks, quality=85, restart_interval=None, ctx=None):
  """uint8 chunks [x,y,z(,1)] -> list of jpeg files (bytes), one call for the batch.
  restart_interval: None = a restart marker after every block row (so the GPU decoder can give
  each row its own thread), 0 = none, n = every n 8x8 blocks."""
  quality = int(quality)
  if not 1 <= quality <= 100:
    raise ValueError("jpeg quality must be in 1..100, got %d" % quality)
  ri = _restart(restart_interval)
  arrs, shapes = zip(*[_jpeg_chunk(ch) for ch in chunks]) if len(chunks) else ((), ())
  n = len(arrs)
  packed = np.concatenate([a.reshape(-1, order="F") for a in arrs]) if n else np.zeros(1, np.uint8)
  shp = np.ascontiguousarray(np.array(shapes, dtype=np.uint32).reshape(n, 3)) if n else np.zeros((1, 3), np.uint32)
  ctx = ctx or _shim.default_context()
  offsets = np.zeros(n + 1, dtype=np.uint64)
  need = c.c_uint64(0)
  args = [ctx.handle, _shim.ptr(packed), n, _shim.ptr(shp), quality, ri]
  # a first guess that holds smooth image data; the call reports the size when it does not
  cap = max(4096, packed.size // 2 + 1024 * n)
  out = np.empty(cap, dtype=np.uint8)
  _shim.check(ctx.lib.ign_jpeg_encode(*args, _shim.ptr(out), cap, _shim.ptr(offsets), c.byref(need)))
  if need.value > cap:
    out = np.empty(int(need.value), dtype=np.uint8)
    _shim.check(ctx.lib.ign_jpeg_encode(*args, _shim.ptr(out), need.value, _shim.ptr(offsets), c.byref(need)))
  return [out[int(offsets[i]):int(offsets[i + 1])].tobytes() for i in range(n)]


def jpeg_encode(chunk, quality=85, restart_interval=None, ctx=None):
  """uint8 chunk [x,y,z(,1)] -> the jpeg file as bytes."""
  return jpeg_encode_batch([chunk], quality, restart_interval, ctx)[0]


def jpeg_decode_batch(datas, shapes, ctx=None):
  """jpeg files + their chunk shapes [x,y,z] or [x,y,z,1] -> list of uint8 chunks (Fortran order,
  in the shapes given), one call for the batch."""
  if len(datas) != len(shapes):
    raise ValueError("%d streams but %d shapes" % (len(datas), len(shapes)))
  n = len(datas)
  if n == 0:
    return []
  given = [tuple(int(v) for v in s) for s in shapes]
  shp = np.ascontiguousarray(np.array([_jpeg_shape(s) for s in given], dtype=np.uint32).reshape(n, 3))
  lens = np.array([len(d) for d in datas], dtype=np.uint64)
  offsets = np.zeros(n + 1, dtype=np.uint64)
  np.cumsum(lens, out=offsets[1:])
  packed = np.frombuffer(b"".join(bytes(d) for d in datas), dtype=np.uint8)
  if packed.size == 0:
    packed = np.zeros(1, np.uint8)
  vox = shp.astype(np.uint64).prod(axis=1)
  out = np.empty(max(int(vox.sum()), 1), dtype=np.uint8)
  ctx = ctx or _shim.default_context()
  _shim.check(ctx.lib.ign_jpeg_decode(ctx.handle, _shim.ptr(np.ascontiguousarray(packed)), _shim.ptr(offsets), n,
                                      _shim.ptr(shp), _shim.ptr(out)))
  res, at = [], 0
  for s, v in zip(given, vox):
    res.append(out[at:at + int(v)].reshape(s, order="F"))
    at += int(v)
  return res


def jpeg_decode(data, shape, ctx=None):
  """jpeg file bytes -> uint8 chunk of `shape` ([x,y,z] or [x,y,z,1], Fortran order)."""
  return jpeg_decode_batch([data], [shape], ctx)[0]


# ------------------------------------------------------------------ device batches
# The storage layer's read and write paths: chunks packed back to back in device memory (chunk i an
# F-order [sx, sy, sz, sc] array, shapes an n x 3 uint32 host array), one call per batch.

def cseg_capacity_words(shapes, sc, dtype, block_size):
  """words that the compressed_segmentation files of these chunks can need at most: per channel the
  offset word, two header words per block and (label words + one index word) per block voxel"""
  bx, by, bz = (int(v) for v in block_size)
  per = np.dtype(dtype).itemsize // 4 + 1
  total = 0
  for sx, sy, sz in np.asarray(shapes, dtype=np.int64).reshape(-1, 3):
    g = (-(-int(sx) // bx)) * (-(-int(sy) // by)) * (-(-int(sz) // bz))
    total += int(sc) * (1 + 2 * g + per * g * bx * by * bz)
  return total


def cseg_encode_batch_dev(chunks, dtype, shapes, sc, block_size=(8, 8, 8), ctx=None):
  """device chunks -> list of compressed_segmentation files (bytes): one batched encode, one D2H"""
  ctx = ctx or _shim.default_context()
  dtype = np.dtype(dtype)
  shapes = np.ascontiguousarray(np.asarray(shapes, dtype=np.uint32).reshape(-1, 3))
  n = shapes.shape[0]
  if n == 0:
    return []
  cap = cseg_capacity_words(shapes, sc, dtype, block_size)
  out = ctx.alloc(cap * 4)
  d_off = ctx.alloc((n + 1) * 8)
  nw = c.c_uint64(0)
  bx, by, bz = (int(v) for v in block_size)
  _shim.check(ctx.lib.ign_cseg_encode_batch_dev(ctx.handle, _shim.ptr(chunks), _shim.dtype_code(dtype), n,
                                                _shim.ptr(shapes), int(sc), bx, by, bz, _shim.ptr(out), cap,
                                                _shim.ptr(d_off), c.byref(nw)))
  words = np.empty(max(int(nw.value), 1), dtype=np.uint32)
  offs = np.empty(n + 1, dtype=np.uint64)
  ctx.d2h(words, out, int(nw.value) * 4)
  ctx.d2h(offs, d_off)
  ctx.sync()
  return [words[int(offs[i]):int(offs[i + 1])].tobytes() for i in range(n)]


def cseg_decode_batch_dev(streams, byte_offsets, dtype, shapes, sc, block_size, out, ctx=None):
  """compressed_segmentation files packed in device memory (stream i at byte_offsets[i] ..
  byte_offsets[i+1], host) -> the packed chunks in `out` (device)"""
  ctx = ctx or _shim.default_context()
  byte_offsets = np.asarray(byte_offsets, dtype=np.int64)
  if np.any(byte_offsets % 4):
    bad = int(np.nonzero(byte_offsets % 4)[0][0])
    raise ValueError("compressed_segmentation stream %d does not start or end on a 4-byte word" % max(bad - 1, 0))
  shapes = np.ascontiguousarray(np.asarray(shapes, dtype=np.uint32).reshape(-1, 3))
  woff = np.ascontiguousarray(byte_offsets // 4, dtype=np.uint64)
  bx, by, bz = (int(v) for v in block_size)
  _shim.check(ctx.lib.ign_cseg_decode_batch_dev(ctx.handle, _shim.ptr(streams), _shim.ptr(woff), shapes.shape[0],
                                                _shim.dtype_code(dtype), _shim.ptr(shapes), int(sc), bx, by, bz,
                                                _shim.ptr(out)))


def jpeg_encode_batch_dev(chunks, shapes, quality=85, ctx=None):
  """uint8 device chunks (one channel) -> list of jpeg files: one batched encode, one D2H"""
  ctx = ctx or _shim.default_context()
  quality = int(quality)
  if not 1 <= quality <= 100:
    raise ValueError("jpeg quality must be in 1..100, got %d" % quality)
  shapes = np.ascontiguousarray(np.array([_jpeg_shape(s) for s in np.asarray(shapes).reshape(-1, 3)],
                                         dtype=np.uint32).reshape(-1, 3))
  n = shapes.shape[0]
  if n == 0:
    return []
  px = int(shapes.astype(np.int64).prod(axis=1).sum())
  offsets = np.zeros(n + 1, dtype=np.uint64)
  need = c.c_uint64(0)
  args = [ctx.handle, _shim.ptr(chunks), n, _shim.ptr(shapes), quality, _restart(None)]
  cap = max(4096, px // 2 + 1024 * n)  # as jpeg_encode_batch: a first guess, the call reports the size
  out = ctx.alloc(cap)
  _shim.check(ctx.lib.ign_jpeg_encode_dev(*args, _shim.ptr(out), cap, _shim.ptr(offsets), c.byref(need)))
  if need.value > cap:
    cap = int(need.value)
    out = ctx.alloc(cap)
    _shim.check(ctx.lib.ign_jpeg_encode_dev(*args, _shim.ptr(out), cap, _shim.ptr(offsets), c.byref(need)))
  host = np.empty(max(int(need.value), 1), dtype=np.uint8)
  ctx.d2h(host, out, int(need.value))
  ctx.sync()
  return [host[int(offsets[i]):int(offsets[i + 1])].tobytes() for i in range(n)]


def jpeg_decode_batch_dev(streams, byte_offsets, shapes, out, ctx=None):
  """jpeg files packed in device memory (stream i at byte_offsets[i] .. byte_offsets[i+1], host) ->
  the packed uint8 chunks in `out` (device)"""
  ctx = ctx or _shim.default_context()
  shapes = np.ascontiguousarray(np.array([_jpeg_shape(s) for s in np.asarray(shapes).reshape(-1, 3)],
                                         dtype=np.uint32).reshape(-1, 3))
  offs = np.ascontiguousarray(np.asarray(byte_offsets, dtype=np.uint64))
  _shim.check(ctx.lib.ign_jpeg_decode_dev(ctx.handle, _shim.ptr(streams), _shim.ptr(offs), shapes.shape[0],
                                          _shim.ptr(shapes), _shim.ptr(out)))
