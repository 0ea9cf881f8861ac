"""Serial C restatement of the grayscale JPEG chunk codec (jpeg_oracle.c) -- TEST INFRASTRUCTURE ONLY.

Only tests/ load it; the product (igneous_b200/) never imports it.  `build()` compiles
libjpeg_oracle.so next to the source with the host C compiler (called by __graft_entry__.build()).

A chunk [x, y, z] of uint8 is the image of width sx and height sy*sz (Fortran order is the raster).
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libjpeg_oracle.so")
_LIB = None

OK, MALFORMED, UNSUPPORTED, SHAPE = 0, -2, -3, -4


def build(force=False):
  src = os.path.join(_HERE, "jpeg_oracle.c")
  if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
    cc = os.environ.get("CC", "gcc")
    subprocess.check_call([cc, "-O2", "-fPIC", "-std=c11", "-Wall", "-Wextra", "-shared", "-o", _SO, src])
  return _SO


def lib():
  global _LIB
  if _LIB is None:
    _LIB = ctypes.CDLL(build())
    _LIB.orc_jpeg_encode.restype = ctypes.c_size_t
    _LIB.orc_jpeg_decode.restype = ctypes.c_int
  return _LIB


def _image(chunk):
  a = np.asarray(chunk)
  if a.ndim == 4:
    if a.shape[3] != 1:
      raise ValueError("one channel only")
    a = a[..., 0]
  if a.ndim == 2:
    a = a[:, :, None]
  if a.dtype != np.uint8 or a.ndim != 3:
    raise ValueError("uint8 [x, y, z] chunks only")
  return np.asfortranarray(a)


def row_interval(sx):
  """The restart interval igneous_b200 writes by default: one block row."""
  return (int(sx) + 7) // 8


def encode(chunk, quality=85, restart_interval=None):
  a = _image(chunk)
  sx, sy, sz = a.shape
  ri = row_interval(sx) if restart_interval is None else int(restart_interval)
  u = ctypes.c_uint32
  args = (ctypes.c_void_p(a.ctypes.data), u(sx), u(sy * sz), ctypes.c_int(int(quality)), u(ri))
  n = lib().orc_jpeg_encode(*args, None, ctypes.c_size_t(0))
  out = np.empty(n, np.uint8)
  lib().orc_jpeg_encode(*args, ctypes.c_void_p(out.ctypes.data), ctypes.c_size_t(n))
  return out.tobytes()


def decode_status(data, shape):
  """-> (status, chunk [x, y, z] Fortran order or None)"""
  sx, sy, sz = (int(v) for v in shape[:3])
  buf = np.frombuffer(bytes(data), np.uint8)
  out = np.empty((sx, sy, sz), np.uint8, order="F")
  rc = lib().orc_jpeg_decode(ctypes.c_void_p(buf.ctypes.data), ctypes.c_size_t(len(buf)), ctypes.c_uint32(sx),
                             ctypes.c_uint32(sy * sz), ctypes.c_void_p(out.ctypes.data))
  return rc, (out if rc == OK else None)


def decode(data, shape):
  rc, out = decode_status(data, shape)
  if rc != OK:
    raise ValueError("orc_jpeg_decode: status %d" % rc)
  return out
