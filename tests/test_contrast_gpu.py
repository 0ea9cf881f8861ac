"""GPU histogram, contrast stretch, quantize and CLAHE against numpy, tests/contrastref.py and
the recorded OpenCV fixtures; the contrast tasks end to end on file:// layers."""
import os
import random

import numpy as np
import pytest

import contrastref as R

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "clahe_cv2.npz")


@pytest.fixture(scope="module")
def C():
  from igneous_b200 import _shim, contrast
  _shim.default_context()
  return contrast


# ------------------------------------------------------------------ histogram
@pytest.mark.parametrize("dt", [np.uint8, np.uint16])
@pytest.mark.parametrize("shape", [(1,), (7, 3, 5), (257, 129, 3), (1001, 999, 2)])
def test_histogram_matches_bincount(C, dt, shape):
  rng = np.random.default_rng(hash((np.dtype(dt).itemsize, shape)) % 2**32)
  hi = 256 if dt == np.uint8 else 65536
  arr = rng.integers(0, hi, size=shape, dtype=np.int64).astype(dt)
  if arr.size > 100:
    arr.ravel()[: arr.size // 3] = 17  # a heavy bin
  want = np.bincount(arr.ravel(), minlength=hi).astype(np.uint64)
  assert np.array_equal(C.histogram(arr), want)
  # an unaligned view goes through the scalar head / tail path
  if arr.size > 3:
    tail = arr.ravel()[1:]
    assert np.array_equal(C.histogram(tail), np.bincount(tail, minlength=hi).astype(np.uint64))


@pytest.mark.parametrize("dt", [np.uint8, np.uint16])
def test_histogram_over_2_32_in_one_bin(C, dt):
  from igneous_b200 import _shim
  ctx = _shim.default_context()
  es = np.dtype(dt).itemsize
  n = (1 << 32) + 12345
  bins = 256 if es == 1 else 65536
  buf = ctx.alloc(n * es)
  hist = ctx.alloc(bins * 8)
  try:
    ctx.memset(buf, 7, n * es)  # every element 7 (u8) or 0x0707 (u16)
    ctx.memset(hist, 0, bins * 8)
    _shim.check(ctx.lib.ign_histogram_dev(ctx.handle, _shim.ptr(buf), _shim.dtype_code(dt), n, _shim.ptr(hist)))
    got = ctx.to_host(hist, (bins,), np.uint64)
  finally:
    buf.free()
    hist.free()
  v = 7 if es == 1 else 0x0707
  assert int(got[v]) == n
  assert int(got.sum()) == n


# -------------------------------------------------------------------- stretch
def _levels(rng, img, z, hs):
  return np.bincount(img[:, :, z].ravel(), minlength=hs).astype(np.uint64)


@pytest.mark.parametrize("dt,out_dt", [(np.uint8, np.uint8), (np.uint16, np.uint16), (np.uint16, np.float32),
                                       (np.uint8, np.uint16)])
@pytest.mark.parametrize("chans", [1, 3])
def test_stretch_bit_exact(C, dt, out_dt, chans):
  rng = np.random.default_rng(5 + chans)
  hs = 256 if dt == np.uint8 else 65536
  shape = (131, 77, 6, chans)
  img = np.asfortranarray(rng.normal(hs * 0.4, hs * 0.1, size=shape).clip(0, hs - 1).astype(dt))
  img[:, :, 2] = 0                 # a slice whose levels are all zero -> (0, 0): kept
  img[:, :, 3] = 33                # lower == upper: kept
  levels = [_levels(rng, img[..., 0], z, hs) for z in range(shape[2])]
  maxval_t = hs - 1
  top = np.iinfo(out_dt).max if np.dtype(out_dt).kind == "u" else maxval_t
  for lo_c, up_c, mn, mx in [(0.01, 0.01, None, None), (0.05, 0.2, 10, min(top, maxval_t) - 7), (0.0, 0.0, None, None)]:
    bounds = [R.clamping_values(lv, lo_c, 1 - up_c) for lv in levels]
    want = R.stretch(img, bounds, maxval_t, 0 if mn is None else mn, maxval_t if mx is None else mx, out_dt)
    got = C.stretch(img, levels, lo_c, up_c, minval=mn, maxval=mx, out_dtype=out_dt)
    assert got.dtype == np.dtype(out_dt) and got.shape == img.shape
    assert np.array_equal(got, want)


def test_stretch_3d_and_2d(C):
  rng = np.random.default_rng(9)
  img = rng.integers(0, 256, size=(33, 17, 3), dtype=np.uint8)
  levels = [np.bincount(img[:, :, z].ravel(), minlength=256).astype(np.uint64) for z in range(3)]
  bounds = [R.clamping_values(lv, 0.01, 0.99) for lv in levels]
  assert np.array_equal(C.stretch(img, levels, 0.01, 0.01), R.stretch(img, bounds, 255, 0, 255, np.uint8))
  assert np.array_equal(C.stretch(img[:, :, 0], levels[:1], 0.01, 0.01),
                        R.stretch(img[:, :, :1], bounds[:1], 255, 0, 255, np.uint8)[:, :, 0])


# ------------------------------------------------------------------- quantize
def test_quantize_matches_numpy(C):
  rng = np.random.default_rng(2)
  img = rng.random((97, 45, 7, 3), dtype=np.float32)
  img[:, 0, 0, 0] = np.arange(97, dtype=np.float32) / np.float32(255)  # exact multiples of 1/255
  img[0, 1, 0, 0] = 1.0
  img[1, 1, 0, 0] = 0.0
  want = (img[:, :, :, :1] * 255.0).astype(np.uint8)
  got = C.quantize(img)
  assert got.shape == want.shape and np.array_equal(got, want)


def test_quantize_saturates(C):
  v = np.array([-3.0, -0.001, np.nan, 1.0, 1.0001, 7.5, np.inf, -np.inf, 0.9999], np.float32).reshape(9, 1, 1, 1)
  assert np.array_equal(C.quantize(v), R.quantize(v))
  assert C.quantize(v).ravel().tolist() == [0, 0, 0, 255, 255, 255, 255, 0, 254]


# ---------------------------------------------------------------------- CLAHE
def test_clahe_fixtures(C):
  g = np.load(GOLDEN)
  n = sum(1 for k in g.files if k.startswith("in_"))
  for i in range(n):
    img = g["in_%d" % i]
    got = C.createCLAHE(float(g["clip_%d" % i]), tuple(int(v) for v in g["grid_%d" % i])).apply(img)
    assert np.array_equal(got, g["out_%d" % i]), i


@pytest.mark.parametrize("dt", [np.uint8, np.uint16])
@pytest.mark.parametrize("shape,grid,clip", [
  ((64, 64, 3), (8, 8), 40.0), ((131, 77, 4), (8, 8), 2.5), ((77, 131, 2), (3, 5), 0.0),
  ((5, 3, 2), (8, 8), 1.0), ((1, 1, 1), (1, 1), 40.0), ((2064, 2064, 2), (8, 8), 40.0),
  ((1031, 2064, 8), (8, 8), 40.0)])
def test_clahe_stack_matches_ref(C, dt, shape, grid, clip):
  rng = np.random.default_rng(shape[0] * 7 + shape[1])
  hs = 256 if dt == np.uint8 else 65536
  stack = np.asfortranarray(rng.normal(hs * 0.45, hs * 0.12, size=shape).clip(0, hs - 1).astype(dt))
  stack[: shape[0] // 4, : shape[1] // 5] = 0
  if shape[0] * shape[1] > 10 ** 6:
    stack[:, :, 1] = 1000 % hs  # one constant slice: a tile of more than 2^16 equal pixels
  got = C.clahe(stack, clip, grid)
  zs = range(shape[2]) if shape[0] * shape[1] < 10 ** 6 else (0, 1, shape[2] - 1)
  for z in zs:
    assert np.array_equal(got[:, :, z], R.clahe(stack[:, :, z], clip, grid)), z


def test_dev_entries_refuse_misaligned_buffers(C):
  """The _dev entries check element alignment before launching anything."""
  from igneous_b200 import _shim
  ctx = _shim.default_context()
  buf, hist = ctx.alloc(4096), ctx.alloc(65536 * 8)
  try:
    with pytest.raises(_shim.IgneousB200Error) as e:
      _shim.check(ctx.lib.ign_histogram_dev(ctx.handle, buf.ptr + 1, _shim.IGN_U16, 100, _shim.ptr(hist)))
    assert e.value.status == -2
    with pytest.raises(_shim.IgneousB200Error):
      _shim.check(ctx.lib.ign_clahe_dev(ctx.handle, buf.ptr + 1, _shim.IGN_U16, 8, 8, 1, 40.0, 2, 2, _shim.ptr(buf)))
    with pytest.raises(_shim.IgneousB200Error):
      _shim.check(ctx.lib.ign_quantize_dev(ctx.handle, buf.ptr + 2, 16, buf.ptr + 2048))
    # an odd uint8 offset is fine: the head before the first 16-byte boundary is counted by scalar loads
    ctx.memset(buf, 5, 4096)
    ctx.memset(hist, 0, 256 * 8)
    _shim.check(ctx.lib.ign_histogram_dev(ctx.handle, buf.ptr + 3, _shim.IGN_U8, 4000, _shim.ptr(hist)))
    got = ctx.to_host(hist, (256,), np.uint64)
    assert int(got[5]) == 4000 and int(got.sum()) == 4000
  finally:
    buf.free()
    hist.free()


def test_stretch_uint32_output(C):
  rng = np.random.default_rng(12)
  img = rng.integers(0, 65536, size=(65, 33, 3), dtype=np.int64).astype(np.uint16)
  levels = [np.bincount(img[:, :, z].ravel(), minlength=65536).astype(np.uint64) for z in range(3)]
  bounds = [R.clamping_values(lv, 0.01, 0.99) for lv in levels]
  want = R.stretch(img, bounds, 65535, 0, 4294967040, np.uint32)
  assert np.array_equal(C.stretch(img, levels, 0.01, 0.01, maxval=4294967040, out_dtype=np.uint32), want)
