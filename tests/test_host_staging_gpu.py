"""Every host-buffer entry point against its `_dev` twin: byte-identical outputs and equal returned
counts, the same number of kernel launches (the staging adds and drops none), and the same exception
type for a rejected argument, which returns before any launch."""
import ctypes as c

import numpy as np
import pytest

from igneous_b200 import _shim

pytestmark = pytest.mark.gpu

U8, U16, U32, U64, F32 = _shim.IGN_U8, _shim.IGN_U16, _shim.IGN_U32, _shim.IGN_U64, _shim.IGN_F32
SHAPES = [(37, 29, 11), (64, 48, 8)]  # odd extents; 37*29*11 bytes is not a multiple of 16


def _seg(shape, seed, dtype=np.uint32, ids=40):
  rng = np.random.default_rng(seed)
  coarse = rng.integers(0, ids, size=tuple((s + 3) // 4 for s in shape))
  seg = coarse.repeat(4, 0).repeat(4, 1).repeat(4, 2)[:shape[0], :shape[1], :shape[2]]
  seg[rng.random(shape) < 0.05] = 0
  return np.asfortranarray(seg.astype(dtype))


class Run:
  """One call of an entry point: host arrays for the host entry, device copies for the _dev entry."""

  def __init__(self, ctx, dev):
    self.ctx, self.dev, self.bufs, self.outs = ctx, dev, [], []

  def inp(self, arr):
    if not self.dev:
      return _shim.ptr(arr)
    b = self.ctx.to_device(arr)
    self.bufs.append(b)
    return _shim.ptr(b)

  def out(self, arr):
    """an output (or in-place) buffer, returned by result() as it is after the call"""
    arr = np.array(arr, order="F")
    if not self.dev:
      self.outs.append((arr, None))
      return _shim.ptr(arr)
    b = self.ctx.to_device(arr)
    self.bufs.append(b)
    self.outs.append((arr, b))
    return _shim.ptr(b)

  def result(self):
    got = [a if b is None else self.ctx.to_host(b, a.shape, a.dtype, order="F") for a, b in self.outs]
    for b in self.bufs:
      b.free()
    return got


def _both(ctx, call):
  """call(run, dev) -> list of returned counts, for the host and the _dev entry"""
  res = []
  for dev in (False, True):
    run = Run(ctx, dev)
    before = ctx.launch_count()
    counts = call(run, dev)
    launches = ctx.launch_count() - before
    res.append((run.result(), [int(v.value) for v in counts], launches))
  (h_out, h_n, h_l), (d_out, d_n, d_l) = res
  assert len(h_out) == len(d_out)
  for h, d in zip(h_out, d_out):
    assert h.tobytes() == d.tobytes()
  assert h_n == d_n
  assert h_l == d_l and h_l > 0
  return h_out, h_n


def _rejects(ctx, call):
  """both entries raise the same exception type, before any launch"""
  kinds = []
  for dev in (False, True):
    run = Run(ctx, dev)
    before = ctx.launch_count()
    with pytest.raises(Exception) as e:
      call(run, dev)
    assert ctx.launch_count() == before
    run.result()
    kinds.append(e.type)
  assert kinds[0] is kinds[1]


def _fn(ctx, name, dev):
  return getattr(ctx.lib, name + ("_dev" if dev else ""))


@pytest.mark.parametrize("shape", SHAPES)
def test_ccl6(ctx, shape):
  seg = _seg(shape, 1)

  def call(r, dev, dtype=U32):
    n = c.c_uint64(0)
    _shim.check(_fn(ctx, "ign_ccl6", dev)(ctx.handle, r.inp(seg), dtype, *shape, r.out(np.zeros(shape, np.uint32)), U32,
                                          c.byref(n)))
    return [n]
  _both(ctx, call)
  _rejects(ctx, lambda r, dev: call(r, dev, F32))


@pytest.mark.parametrize("shape", SHAPES)
def test_dust(ctx, shape):
  seg = _seg(shape, 2)

  def call(r, dev, dtype=U32):
    _shim.check(_fn(ctx, "ign_dust", dev)(ctx.handle, r.out(seg), dtype, *shape, 20))
    return []
  _both(ctx, call)
  _rejects(ctx, lambda r, dev: call(r, dev, F32))


@pytest.mark.parametrize("shape", SHAPES)
def test_ccl_task(ctx, shape):
  img = np.asfortranarray(np.random.default_rng(3).integers(0, 256, size=shape).astype(np.uint8))
  rails = [s // 2 for s in shape]

  def call(r, dev, dtype=U8):
    n = c.c_uint64(0)
    _shim.check(_fn(ctx, "ign_ccl_task", dev)(ctx.handle, r.inp(img), dtype, *shape, 1, 100.0, 1, 200.0, *rails, 3,
                                              1000, r.out(np.zeros(shape, np.uint64)), c.byref(n)))
    return [n]
  _both(ctx, call)
  _rejects(ctx, lambda r, dev: call(r, dev, 99))


@pytest.mark.parametrize("shape", SHAPES)
def test_pool_select(ctx, shape):
  img = np.asfortranarray(np.random.default_rng(4).integers(0, 256, size=shape).astype(np.uint8))

  def call(r, dev, mips=2):
    outs, ext = [], list(shape)
    for _ in range(max(mips, 1)):
      ext = [(e + 1) // 2 for e in ext]
      outs.append(r.out(np.zeros(ext, np.uint8)))
    _shim.check(_fn(ctx, "ign_pool_select", dev)(ctx.handle, r.inp(img), U8, *shape, 2, 2, 2, mips, 0,
                                                 _shim.void_pp([p.value for p in outs])))
    return []
  _both(ctx, call)
  _rejects(ctx, lambda r, dev: call(r, dev, 0))


@pytest.mark.parametrize("mode", [True, False])
@pytest.mark.parametrize("shape", SHAPES)
def test_pool_2x2x1(ctx, shape, mode):
  arr = _seg(shape, 5, np.uint32 if mode else np.uint16)
  dt = U32 if mode else U16

  def call(r, dev, mips=3):
    outs, (x, y, z) = [], shape
    for _ in range(max(mips, 1)):
      x, y = (x + 1) // 2, (y + 1) // 2
      outs.append(r.out(np.zeros((x, y, z), arr.dtype)))
    name = "ign_pool_mode_2x2x1" if mode else "ign_pool_avg_2x2x1"
    _shim.check(_fn(ctx, name, dev)(ctx.handle, r.inp(arr), dt, *shape, mips, 0,
                                    _shim.void_pp([p.value for p in outs])))
    return []
  _both(ctx, call)
  _rejects(ctx, lambda r, dev: call(r, dev, 33))


@pytest.mark.parametrize("shape", SHAPES)
def test_dilate_multilabel(ctx, shape):
  seg = _seg(shape, 6)

  def call(r, dev, dtype=U32):
    _shim.check(_fn(ctx, "ign_dilate_multilabel", dev)(ctx.handle, r.inp(seg), dtype, *shape,
                                                       r.out(np.zeros(shape, np.uint32))))
    return []
  _both(ctx, call)
  _rejects(ctx, lambda r, dev: call(r, dev, F32))


@pytest.mark.parametrize("shape", SHAPES)
def test_fill_holes(ctx, shape):
  seg = _seg(shape, 7, ids=6)

  def call(r, dev, dtype=U32):
    z = np.zeros(shape, np.uint32)
    _shim.check(_fn(ctx, "ign_fill_holes", dev)(ctx.handle, r.inp(seg), dtype, *shape, 1, 50, r.out(z), r.out(z)))
    return []
  _both(ctx, call)
  _rejects(ctx, lambda r, dev: call(r, dev, F32))


@pytest.mark.parametrize("shape", SHAPES)
def test_histogram(ctx, shape):
  img = np.random.default_rng(8).integers(0, 65536, size=int(np.prod(shape))).astype(np.uint16)
  start = np.random.default_rng(9).integers(0, 1000, size=65536).astype(np.uint64)  # added into

  def call(r, dev, dtype=U16):
    _shim.check(_fn(ctx, "ign_histogram", dev)(ctx.handle, r.inp(img), dtype, img.size, r.out(start)))
    return []
  _both(ctx, call)
  _rejects(ctx, lambda r, dev: call(r, dev, 99))


@pytest.mark.parametrize("shape", SHAPES)
def test_contrast_stretch(ctx, shape):
  img = np.asfortranarray(np.random.default_rng(10).integers(0, 256, size=shape).astype(np.uint8))
  lower = np.arange(shape[2], dtype=np.uint32) * 3
  upper = lower + 150
  upper[0] = lower[0]

  def call(r, dev, dtype=U8):
    _shim.check(_fn(ctx, "ign_contrast_stretch", dev)(ctx.handle, r.inp(img), dtype, *shape, 1, _shim.ptr(lower),
                                                      _shim.ptr(upper), 0.0, 65535.0, r.out(np.zeros(shape, np.uint16)),
                                                      U16))
    return []
  _both(ctx, call)
  _rejects(ctx, lambda r, dev: call(r, dev, U32))


@pytest.mark.parametrize("shape", SHAPES)
def test_quantize(ctx, shape):
  x = np.random.default_rng(11).uniform(-0.2, 1.2, size=int(np.prod(shape))).astype(np.float32)

  def call(r, dev, null_out=False):
    out = c.c_void_p(None) if null_out else r.out(np.zeros(x.size, np.uint8))
    _shim.check(_fn(ctx, "ign_quantize", dev)(ctx.handle, r.inp(x), x.size, out))
    return []
  _both(ctx, call)
  _rejects(ctx, lambda r, dev: call(r, dev, True))


@pytest.mark.parametrize("shape", SHAPES)
def test_clahe(ctx, shape):
  img = np.asfortranarray(np.random.default_rng(12).integers(0, 256, size=shape).astype(np.uint8))

  def call(r, dev, dtype=U8):
    _shim.check(_fn(ctx, "ign_clahe", dev)(ctx.handle, r.inp(img), dtype, *shape, 2.0, 4, 3,
                                           r.out(np.zeros(shape, np.uint8))))
    return []
  _both(ctx, call)
  _rejects(ctx, lambda r, dev: call(r, dev, U32))


@pytest.mark.parametrize("shape", SHAPES)
def test_renumber(ctx, shape):
  seg = _seg(shape, 13, np.uint64) * np.uint64(1 << 40)
  n = seg.size

  def call(r, dev, dtype=U64):
    k = c.c_uint64(0)
    _shim.check(_fn(ctx, "ign_renumber", dev)(ctx.handle, r.inp(seg), dtype, n, r.out(np.zeros(n, np.uint32)),
                                              r.out(np.zeros(20, np.uint64)), 20, c.byref(k)))
    return [k]
  _, (k,) = _both(ctx, call)
  assert k > 20  # the unique list is cut at its capacity
  _rejects(ctx, lambda r, dev: call(r, dev, F32))


@pytest.mark.parametrize("shape", SHAPES)
def test_remap(ctx, shape):
  seg = _seg(shape, 14)
  keys = np.arange(40, dtype=np.uint64)
  vals = (keys * 7 + 3) % 41

  def call(r, dev, dtype=U32, n_keys=keys.size):
    _shim.check(_fn(ctx, "ign_remap", dev)(ctx.handle, r.out(seg), dtype, seg.size, _shim.ptr(keys), _shim.ptr(vals),
                                           n_keys, 0))
    return []
  _both(ctx, call)
  _rejects(ctx, lambda r, dev: call(r, dev, F32, 0))


def _cseg_args(shape):
  return [*shape, 1, 8, 8, 8]


@pytest.mark.parametrize("shape", SHAPES)
def test_cseg(ctx, shape):
  seg = _seg(shape, 15)
  cap = 1 + 2 * 1024 + 3 * seg.size

  def encode(r, dev, dtype=U32):
    n = c.c_uint64(0)
    _shim.check(_fn(ctx, "ign_cseg_encode", dev)(ctx.handle, r.inp(seg), dtype, *_cseg_args(shape),
                                                 r.out(np.zeros(cap, np.uint32)), cap, c.byref(n)))
    return [n]
  (stream,), (n_words,) = _both(ctx, encode)
  stream = stream[:n_words]
  _rejects(ctx, lambda r, dev: encode(r, dev, U8))

  def decode(r, dev, dtype=U32):
    _shim.check(_fn(ctx, "ign_cseg_decode", dev)(ctx.handle, r.inp(stream), stream.size, dtype, *_cseg_args(shape),
                                                 r.out(np.zeros(shape, np.uint32))))
    return []
  (back,), _ = _both(ctx, decode)
  assert np.array_equal(back, seg)
  _rejects(ctx, lambda r, dev: decode(r, dev, U8))


def _export(ctx, m):
  nv, nf, nl = c.c_uint64(0), c.c_uint64(0), c.c_uint64(0)
  _shim.check(ctx.lib.ign_mesh_totals(m, c.byref(nv), c.byref(nf)))
  _shim.check(ctx.lib.ign_mesh_num_ids(m, c.byref(nl)))
  ids = np.zeros(nl.value, np.uint64)
  _shim.check(ctx.lib.ign_mesh_ids(m, _shim.ptr(ids), ids.size))
  out = [ids, np.zeros((nv.value, 3), np.float32), np.zeros((nf.value, 3), np.uint32),
         np.zeros(nl.value + 1, np.uint64), np.zeros(nl.value + 1, np.uint64)]
  res = (c.c_float * 3)(16.0, 16.0, 40.0)
  _shim.check(ctx.lib.ign_mesh_export(m, res, 1, *[_shim.ptr(a) for a in out[1:]]))
  return out


@pytest.mark.parametrize("shape", SHAPES)
def test_mesh_begin(ctx, shape):
  seg = _seg(shape, 16, ids=12)
  got = []

  def call(r, dev, sx=shape[0]):
    m = c.c_void_p()
    _shim.check(_fn(ctx, "ign_mesh_begin", dev)(ctx.handle, r.inp(seg), U32, sx, *shape[1:], c.byref(m)))
    try:
      got.append(_export(ctx, m))
    finally:
      ctx.lib.ign_mesh_free(m)
    return []
  _both(ctx, call)
  host, dev = got
  assert host[1].size > 0
  for h, d in zip(host, dev):
    assert h.tobytes() == d.tobytes()
  _rejects(ctx, lambda r, dev: call(r, dev, 0))
