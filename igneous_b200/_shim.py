"""ctypes binding of libigneous_b200.so (the C ABI in include/igneous_b200.h).

This module is the only place Python touches the native library.  There is no
CPU fallback: if the library is missing, or no CUDA device is visible, every
compute call raises.

The header is the only statement of the ABI: load() reads its prototypes and sets
argtypes / restype on every declared function, so callers pass Python ints and
floats and ctypes converts (and type-checks) them.  Pointers are c_void_p, which
takes None, ints, c_void_p values (ptr()), ctypes arrays and byref(...).
"""
import ctypes
import os
import re
import threading

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(os.path.dirname(_HERE), "include", "igneous_b200.h")
_LIB_ENV = "IGNEOUS_B200_LIB"
_DEV_ENV = "IGNEOUS_B200_DEVICE"

IGN_U8, IGN_U16, IGN_U32, IGN_U64, IGN_F32 = 1, 2, 3, 4, 5
ROUND_FLOOR, ROUND_HALF_UP, ROUND_HALF_EVEN = 0, 1, 2

_DTYPE_CODE = {
  np.dtype(np.uint8): IGN_U8, np.dtype(np.bool_): IGN_U8, np.dtype(np.int8): IGN_U8,
  np.dtype(np.uint16): IGN_U16, np.dtype(np.int16): IGN_U16,
  np.dtype(np.uint32): IGN_U32, np.dtype(np.int32): IGN_U32,
  np.dtype(np.uint64): IGN_U64, np.dtype(np.int64): IGN_U64,
  np.dtype(np.float32): IGN_F32,
}
_CODE_DTYPE = {IGN_U8: np.uint8, IGN_U16: np.uint16, IGN_U32: np.uint32,
               IGN_U64: np.uint64, IGN_F32: np.float32}


class IgneousB200Error(RuntimeError):
  """Any non-zero status from the native library."""

  def __init__(self, status, message):
    super().__init__("libigneous_b200 status %d: %s" % (status, message))
    self.status = status


class NativeLibraryMissing(IgneousB200Error):
  def __init__(self, message):
    RuntimeError.__init__(self, message)
    self.status = None


def dtype_code(dtype):
  try:
    return _DTYPE_CODE[np.dtype(dtype)]
  except KeyError:
    raise NotImplementedError("igneous_b200: unsupported dtype %s" % np.dtype(dtype))


def require_unsigned(dtype, what):
  """Signed integer arrays share the unsigned kernels, which is exact for equality-only work
  (mode pooling, CCL on raw labels, remap) and WRONG for anything that orders or adds values:
  negative voxels would count as large positives.  Those operations refuse signed input."""
  dt = np.dtype(dtype)
  if dt.kind == "i":
    raise NotImplementedError("igneous_b200 %s: signed dtype %s is not supported (the kernels are unsigned; "
                              "negative values would be treated as large positives)" % (what, dt))


def code_dtype(code):
  return np.dtype(_CODE_DTYPE[code])


def lib_path():
  return os.environ.get(_LIB_ENV) or os.path.join(_HERE, "csrc", "libigneous_b200.so")


_SCALARS = {"int": ctypes.c_int, "uint32_t": ctypes.c_uint32, "uint64_t": ctypes.c_uint64,
            "int64_t": ctypes.c_int64, "float": ctypes.c_float, "double": ctypes.c_double}
_RETURNS = {"int": ctypes.c_int, "const char*": ctypes.c_char_p}
_PROTOTYPE = re.compile(r"IGN_API\s+([\w\s\*]+?)\s*\b(ign_\w+)\s*\(([^)]*)\)")


def _param_type(param):
  if "*" in param or "[" in param:
    return ctypes.c_void_p
  ctype = _SCALARS.get(" ".join(w for w in param.split()[:-1] if w != "const"))
  if ctype is None:
    raise ValueError("%s: no ctypes mapping for parameter %r" % (HEADER, param))
  return ctype


def prototypes():
  """{name: (restype, argtypes)} of every IGN_API function the header declares.  Every
  pointer or array parameter is c_void_p; a C type without a mapping raises ValueError."""
  with open(HEADER) as f:
    text = f.read()
  protos = {}
  for ret, name, params in _PROTOTYPE.findall(text):
    ret = " ".join(ret.split())
    if ret not in _RETURNS:
      raise ValueError("%s: no ctypes mapping for the return type %r of %s" % (HEADER, ret, name))
    params = [p.strip() for p in params.split(",")]
    protos[name] = (_RETURNS[ret], [] if params == ["void"] else [_param_type(p) for p in params])
  return protos


_lib = None
_lock = threading.Lock()


def load():
  """dlopen the native library and declare every function of the header on it (no GPU needed
  for this step).  A declared function the library does not export raises AttributeError."""
  global _lib
  if _lib is not None:
    return _lib
  with _lock:
    if _lib is not None:
      return _lib
    path = lib_path()
    if not os.path.exists(path):
      raise NativeLibraryMissing(
        "libigneous_b200.so not found at %s -- run `python -m igneous_b200.build` "
        "(there is no CPU fallback)" % path)
    lib = ctypes.CDLL(path)
    for name, (restype, argtypes) in prototypes().items():
      fn = getattr(lib, name)
      fn.restype, fn.argtypes = restype, argtypes
    _lib = lib
    return _lib


def check(status):
  if status == 0:
    return
  msg = load().ign_last_error().decode("utf-8", "replace")
  if status == -5:
    raise KeyError(msg)
  if status == -3:
    raise NotImplementedError("libigneous_b200: " + msg)
  if status == -4:
    raise MemoryError("libigneous_b200: " + msg)
  raise IgneousB200Error(status, msg)


def ptr(a):
  """address of a numpy array's buffer / raw int device pointer -> c_void_p"""
  if isinstance(a, np.ndarray):
    return ctypes.c_void_p(a.ctypes.data)
  if isinstance(a, DeviceBuffer):
    return ctypes.c_void_p(a.ptr)
  return ctypes.c_void_p(int(a) if a else None)


class DeviceBuffer:
  """Owned HBM allocation (ign_dev_alloc)."""

  def __init__(self, ctx, nbytes):
    self.ctx = ctx
    self.nbytes = int(nbytes)
    p = ctypes.c_void_p()
    check(ctx.lib.ign_dev_alloc(ctx.handle, self.nbytes, ctypes.byref(p)))
    self.ptr = p.value or 0

  def free(self):
    if self.ptr and self.ctx.handle:
      check(self.ctx.lib.ign_dev_free(self.ctx.handle, self.ptr))
    self.ptr = 0

  def offset(self, nbytes):
    return self.ptr + int(nbytes)

  def __del__(self):
    try:
      self.free()
    except Exception:
      pass


class Context:
  """One ign_ctx: a device, a stream, a scratch arena.  Not thread safe."""

  def __init__(self, device=None):
    self.lib = load()
    if device is None:
      device = int(os.environ.get(_DEV_ENV, os.environ.get("LOCAL_RANK", "0")))
    h = ctypes.c_void_p()
    check(self.lib.ign_init(device, ctypes.byref(h)))
    self.handle = h
    self.device = device

  # -- memory
  def alloc(self, nbytes):
    return DeviceBuffer(self, nbytes)

  def pinned_empty(self, shape, dtype, order="F"):
    """numpy array backed by pinned host memory (freed with the context)."""
    dtype = np.dtype(dtype)
    n = int(np.prod(shape)) if len(shape) else 1
    p = ctypes.c_void_p()
    check(self.lib.ign_host_alloc(self.handle, max(n * dtype.itemsize, 1), ctypes.byref(p)))
    buf = (ctypes.c_uint8 * max(n * dtype.itemsize, 1)).from_address(p.value)
    arr = np.frombuffer(buf, dtype=dtype, count=n).reshape(shape, order=order)
    self._pinned = getattr(self, "_pinned", [])
    self._pinned.append(p.value)
    return arr

  def h2d(self, dst, src_arr):
    check(self.lib.ign_h2d(self.handle, ptr(dst), ptr(src_arr), src_arr.nbytes))

  def d2h(self, dst_arr, src, nbytes=None):
    check(self.lib.ign_d2h(self.handle, ptr(dst_arr), ptr(src), dst_arr.nbytes if nbytes is None else nbytes))

  def d2d(self, dst, src, nbytes):
    check(self.lib.ign_d2d(self.handle, ptr(dst), ptr(src), nbytes))

  def memset(self, dst, byte, nbytes):
    check(self.lib.ign_memset(self.handle, ptr(dst), byte, nbytes))

  def sync(self):
    check(self.lib.ign_sync(self.handle))

  def set_priority(self, high=True):
    """Re-create the context's stream with the device's greatest / least stream priority."""
    check(self.lib.ign_stream_priority(self.handle, int(bool(high))))

  def to_device(self, arr):
    arr = np.asarray(arr)
    if not (arr.flags.f_contiguous or arr.flags.c_contiguous):
      arr = np.asfortranarray(arr)
    buf = self.alloc(arr.nbytes)
    self.h2d(buf, arr)
    self.sync()
    return buf

  def to_host(self, buf, shape, dtype, order="F"):
    out = np.empty(shape, dtype=dtype, order=order)
    self.d2h(out, buf)
    self.sync()
    return out

  # -- timers
  def timer_start(self, slot=0):
    check(self.lib.ign_timer_start(self.handle, slot))

  def timer_stop(self, slot=0):
    check(self.lib.ign_timer_stop(self.handle, slot))

  def timer_ms(self, slot=0):
    ms = ctypes.c_float()
    check(self.lib.ign_timer_ms(self.handle, slot, ctypes.byref(ms)))
    return float(ms.value)

  def launch_count(self):
    n = ctypes.c_uint64()
    check(self.lib.ign_launch_count(self.handle, ctypes.byref(n)))
    return int(n.value)

  def stream(self):
    s = ctypes.c_void_p()
    check(self.lib.ign_stream(self.handle, ctypes.byref(s)))
    return s.value or 0

  def close(self):
    if getattr(self, "handle", None):
      for p in getattr(self, "_pinned", []):
        self.lib.ign_host_free(self.handle, p)
      self._pinned = []
      self.lib.ign_destroy(self.handle)
      self.handle = None

  def __del__(self):
    try:
      self.close()
    except Exception:
      pass


_default_ctx = None


def default_context():
  """Process-wide context (one worker process <-> one GPU, SURVEY 8(b))."""
  global _default_ctx
  if _default_ctx is None:
    _default_ctx = Context()
  return _default_ctx


def device_count():
  n = ctypes.c_int(0)
  rc = load().ign_device_count(ctypes.byref(n))
  return int(n.value) if rc == 0 else 0


# ----------------------------------------------------------- array plumbing
def as_fortran_volume(img):
  """(x,y,z[,c]) array -> (F-contiguous array, sx, sy, nz) where the channel
  axis is folded into z (2x2x1 pooling never mixes z or c)."""
  img = np.asarray(img)
  if img.ndim == 2:
    img = img[:, :, np.newaxis]
  if img.ndim not in (3, 4):
    raise ValueError("expected a 2-, 3- or 4-D array, got ndim=%d" % img.ndim)
  arr = np.asfortranarray(img)
  sx, sy = arr.shape[0], arr.shape[1]
  nz = int(np.prod(arr.shape[2:]))
  return arr, sx, sy, nz


def void_pp(ptrs):
  arr = (ctypes.c_void_p * len(ptrs))(*[ctypes.c_void_p(int(p)) for p in ptrs])
  return arr
