"""igneous_b200.edt against tests/edtref.py (the rule of DESIGN.md §5d restated with scipy):
bit-exact for integer anisotropy, where every squared distance here is below 2^24, and within
1e-5 relative otherwise; edt == np.sqrt(edtsq) bit for bit.  Seeded Voronoi segmentations at odd
and prime shapes in 1, 2 and 3 dimensions, every label dtype, bool and signed input, both memory
orders and both borders; lines of 10,007 voxels along each axis; all-zero volumes, one label
filling the volume and every voxel its own label in closed form; u64 labels that differ only in
their high bits; ign_edt_dev against ign_edt; and a block volume past 2^32 voxels checked in
closed form on the planes and lines at the 2^32-element boundary and the volume's edges."""
import ctypes as c

import numpy as np
import pytest
from scipy.spatial import cKDTree

import edtref

pytestmark = pytest.mark.gpu

EXACT = [(1.0, 1.0, 1.0), (4.0, 4.0, 40.0)]
INEXACT = (4.5, 7.25, 40.3)
IGN_U8, IGN_F32 = 1, 5


def voronoi(shape, seed, pitch=6):
  """seeded Voronoi cells of about pitch^ndim voxels, numbered 1..; every seventh cell is label 0"""
  rng = np.random.default_rng(seed)
  k = max(2, int(np.prod(shape)) // pitch ** len(shape))
  pts = rng.random((k, len(shape))) * np.array(shape)
  grid = np.indices(shape).reshape(len(shape), -1).T + 0.5
  _, idx = cKDTree(pts).query(grid)
  lab = (idx + 1) * (idx % 7 != 0)
  return lab.reshape(shape).astype(np.uint64)


def check(got, labels, a, black_border):
  """compares with the reference; bit-exact (and returns True) for integer anisotropy when every
  finite squared distance is below 2^24, else within 1e-5 relative"""
  want = edtref.edtsq(labels, a, black_border)
  assert got.dtype == np.float32 and got.shape == want.shape
  assert np.array_equal(np.isinf(got), np.isinf(want))
  fin = np.isfinite(want)
  if all(float(v).is_integer() for v in a) and not np.any(want[fin] >= 2**24):
    np.testing.assert_array_equal(got, want)
    return True
  assert np.all(np.abs(got[fin] - want[fin]) <= 1e-5 * want[fin])
  return False


def _both(labels, a, black_border, ctx):
  """edtsq against the reference and edt against np.sqrt(edtsq); returns whether edtsq was exact"""
  from igneous_b200 import edt
  sq = edt.edtsq(labels, anisotropy=a, black_border=black_border, ctx=ctx)
  exact = check(sq, labels, a, black_border)
  d = edt.edt(labels, anisotropy=a, black_border=black_border, ctx=ctx)
  assert d.dtype == np.float32
  np.testing.assert_array_equal(d.view(np.uint32), np.sqrt(sq).view(np.uint32))
  return exact


@pytest.mark.parametrize("shape", [(1009,), (97, 61), (41, 37, 29), (31, 1, 23), (1, 53, 19)])
@pytest.mark.parametrize("a", EXACT + [INEXACT])
@pytest.mark.parametrize("black_border", [False, True])
def test_voronoi_segmentations(ctx, shape, a, black_border):
  labels = voronoi(shape, seed=sum(shape)).astype(np.uint32)
  assert _both(labels, a[:len(shape)], black_border, ctx) == (a != INEXACT)


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.uint32, np.uint64, np.int8, np.int16, np.int32, np.int64])
@pytest.mark.parametrize("order", ["F", "C"])
@pytest.mark.parametrize("black_border", [False, True])
def test_dtypes_and_orders(ctx, dtype, order, black_border):
  labels = voronoi((43, 31, 17), seed=5)
  if np.dtype(dtype).itemsize == 8:
    labels = labels + np.uint64(2**40)  # high bits in use; 0 stays 0 below
    labels[voronoi((43, 31, 17), seed=5) == 0] = 0
  labels = np.asarray(labels.astype(dtype), order=order)
  if np.dtype(dtype).kind == "i":
    labels[labels == 3] = -3  # a negative label is just another value
  assert _both(labels, (4.0, 4.0, 40.0), black_border, ctx)


@pytest.mark.parametrize("black_border", [False, True])
def test_bool(ctx, black_border):
  rng = np.random.default_rng(7)
  labels = rng.random((37, 23, 11)) < 0.8
  _both(labels, (1.0, 1.0, 1.0), black_border, ctx)
  _both(labels, INEXACT, black_border, ctx)
  _both(labels[:, 3, :], (2.0, 5.0), black_border, ctx)


@pytest.mark.parametrize("shape", [(10007, 3, 3), (3, 10007, 3), (3, 3, 10007), (10007,), (2, 10007)])
@pytest.mark.parametrize("black_border", [False, True])
def test_long_lines(ctx, shape, black_border):
  rng = np.random.default_rng(len(shape) + shape[0])
  ax = int(np.argmax(shape))
  # runs of a few hundred voxels along the long axis (label 0 among them), the same on every line
  # but one, which holds one label from end to end
  runs = np.cumsum(rng.random(shape[ax]) < 0.004) % 5
  labels = np.broadcast_to(runs.reshape([-1 if i == ax else 1 for i in range(len(shape))]), shape).astype(np.uint16)
  if len(shape) > 1:
    labels[tuple(slice(None) if i == ax else 0 for i in range(len(shape)))] = 9
  assert _both(labels, (1.0, 1.0, 1.0)[:len(shape)], black_border, ctx)
  _both(labels, (4.0, 4.0, 40.0)[:len(shape)], black_border, ctx)
  _both(labels, INEXACT[:len(shape)], black_border, ctx)


def _closed_one_label(shape, a, black_border):
  if not black_border:
    return np.full(shape, np.inf, np.float32)
  g = np.indices(shape)
  return np.min([(ai * np.minimum(gi + 1, n - gi)) ** 2 for gi, n, ai in zip(g, shape, a)], axis=0).astype(np.float32)


@pytest.mark.parametrize("shape", [(45, 34, 23), (1, 1, 1), (7, 1, 5), (29,), (13, 8)])
def test_zero_one_label_and_distinct(ctx, shape):
  from igneous_b200 import edt
  a = (4.0, 4.0, 40.0)[:len(shape)]
  for bb in (False, True):
    np.testing.assert_array_equal(edt.edtsq(np.zeros(shape, np.uint32), a, bb, ctx=ctx), np.zeros(shape, np.float32))
    got = edt.edtsq(np.full(shape, 7, np.uint8), a, bb, ctx=ctx)
    np.testing.assert_array_equal(got, _closed_one_label(shape, a, bb))
    # every voxel its own label: the smallest a_i^2 over the axes along which it has a neighbour
    # (every axis with black_border)
    distinct = np.arange(1, int(np.prod(shape)) + 1, dtype=np.uint32).reshape(shape)
    want = np.full(shape, np.inf, np.float32)
    for ai, n in zip(a, shape):
      if n > 1 or bb:
        want = np.minimum(want, np.float32(ai * ai))
    np.testing.assert_array_equal(edt.edtsq(distinct, a, bb, ctx=ctx), want)
    np.testing.assert_array_equal(edt.edtsq(np.asfortranarray(distinct), a, bb, ctx=ctx), want)


def test_u64_high_bits_stay_distinct(ctx):
  from igneous_b200 import edt
  labels = np.ones((6, 5, 4), dtype=np.uint64)
  labels[3:] = 2**32 + 1
  got = edt.edtsq(labels, ctx=ctx)
  np.testing.assert_array_equal(got[:, 0, 0], np.array([9, 4, 1, 1, 4, 9], np.float32))
  check(got, labels, (1.0, 1.0, 1.0), False)
  assert np.all(np.isinf(edt.edtsq(np.full((4, 4), 2**32 + 1, np.uint64), ctx=ctx)))


def test_edt_dev_matches_host_entry(ctx):
  from igneous_b200 import _shim
  labels = np.asfortranarray(voronoi((67, 45, 33), seed=11).astype(np.uint32))
  a = (c.c_float * 3)(4.5, 7.25, 40.3)
  for bb, sq in ((0, 1), (1, 0)):
    host = np.empty(labels.shape, np.float32, order="F")
    _shim.check(ctx.lib.ign_edt(ctx.handle, _shim.ptr(labels), _shim.IGN_U32, *labels.shape, a, bb, sq,
                                _shim.ptr(host)))
    d_in = ctx.to_device(labels)
    d_out = ctx.alloc(labels.size * 4)
    _shim.check(ctx.lib.ign_edt_dev(ctx.handle, _shim.ptr(d_in), _shim.IGN_U32, *labels.shape, a, bb, sq,
                                    _shim.ptr(d_out)))
    dev = ctx.to_host(d_out, labels.shape, np.float32)
    np.testing.assert_array_equal(dev.view(np.uint32), host.view(np.uint32))
    d_in.free()
    d_out.free()


def test_refusals(ctx):
  from igneous_b200 import edt, _shim
  lab = np.ones((4, 4, 4), np.uint32)
  with pytest.raises(NotImplementedError):
    edt.edt(lab, voxel_graph=np.ones((4, 4, 4), np.uint8), ctx=ctx)
  with pytest.raises(NotImplementedError):
    edt.edt(lab.astype(np.float32), ctx=ctx)
  with pytest.raises(ValueError):
    edt.edt(lab, anisotropy=(1, 1), ctx=ctx)
  with pytest.raises(ValueError):
    edt.edt(lab, anisotropy=(1, 0, 1), ctx=ctx)
  with pytest.raises(ValueError):
    edt.edt(np.ones((2, 2, 2, 2), np.uint8), ctx=ctx)
  bad = (c.c_float * 3)(1.0, float("inf"), 1.0)  # +inf only on an axis of extent 1
  out = np.empty(64, np.float32)
  with pytest.raises(_shim.IgneousB200Error):
    _shim.check(ctx.lib.ign_edt(ctx.handle, _shim.ptr(lab), _shim.IGN_U32, 4, 4, 4, bad, 1, 1, _shim.ptr(out)))
  assert edt.edt(np.zeros((0, 3), np.uint8), ctx=ctx).shape == (0, 3)


# ------------------------------------------------------------ past 2^32 voxels
BIG = (4099, 1031, 1093)  # 4.6e9 voxels, element 2^32 in plane 1016; rows not a multiple of 32
BLOCK = (37, 29, 23)
BIG_A = (4.0, 4.0, 40.0)


def _block_labels(shape, x, y, z):
  return ((x // BLOCK[0]) + (y // BLOCK[1]) + (z // BLOCK[2])) % 3


def _block_want(x, y, z, black_border):
  """closed form of the block volume: face-adjacent boxes always differ, so a voxel's nearest other
  label lies straight across the nearest boundary face"""
  lab = _block_labels(BIG, x, y, z)
  d = edtref.block_edtsq((x, y, z), BIG, BLOCK, BIG_A, black_border)
  return np.where(lab == 0, np.float32(0), d)


@pytest.fixture
def big_ctx():
  """a context of its own, so that its scratch arena and buffers go with it"""
  from igneous_b200 import _shim
  ctx = _shim.Context()
  bufs = []
  try:
    yield ctx, bufs
  finally:
    for b in bufs:
      b.free()
    ctx.close()


@pytest.mark.parametrize("black_border", [False, True])
def test_block_volume_past_2_32_voxels(big_ctx, black_border):
  from igneous_b200 import _shim
  ctx, bufs = big_ctx
  sx, sy, sz = BIG
  assert sx * sy * sz > 2**32
  lab = ctx.alloc(sx * sy * sz)
  out = ctx.alloc(sx * sy * sz * 4)
  bufs += [lab, out]
  xs, ys = np.meshgrid(np.arange(sx), np.arange(sy), indexing="ij")
  planes = {}
  for z in range(sz):  # one upload per layer of boxes, device copies for the rest
    key = z // BLOCK[2]
    if key in planes:
      ctx.d2d(lab.offset(z * sx * sy), planes[key], sx * sy)
    else:
      ctx.h2d(lab.offset(z * sx * sy), np.asfortranarray(_block_labels(BIG, xs, ys, z).astype(np.uint8)))
      planes[key] = lab.offset(z * sx * sy)
  ctx.sync()
  a = (c.c_float * 3)(*BIG_A)

  def run(squared):
    _shim.check(ctx.lib.ign_edt_dev(ctx.handle, _shim.ptr(lab), IGN_U8, *BIG, a, int(black_border), squared,
                                    _shim.ptr(out)))
    ctx.sync()

  run(1)
  zb = 2**32 // (sx * sy)  # the plane holding element 2^32
  plane = np.empty((sx, sy), np.float32, order="F")
  for z in sorted({0, 1, zb - 1, zb, zb + 1, sz - 2, sz - 1}):
    ctx.d2h(plane, out.offset(z * sx * sy * 4))
    ctx.sync()
    np.testing.assert_array_equal(plane, _block_want(xs, ys, z, black_border), err_msg="plane z=%d" % z)
  # z-lines at the volume's edges and through element 2^32 and its neighbours
  xb, yb = (2**32 % (sx * sy)) % sx, (2**32 % (sx * sy)) // sx
  box = ctx.alloc(3 * 3 * sz * 4)
  bufs.append(box)
  zs = np.arange(sz)
  for x0, y0 in ((0, 0), (sx - 3, sy - 3), (0, sy - 3), (max(0, xb - 1), max(0, yb - 1))):
    _shim.check(ctx.lib.ign_copy_box_dev(ctx.handle, _shim.ptr(out), IGN_F32, *BIG, x0, y0, 0, 3, 3, sz,
                                         _shim.ptr(box)))
    got = ctx.to_host(box, (3, 3, sz), np.float32)
    g = np.meshgrid(np.arange(x0, x0 + 3), np.arange(y0, y0 + 3), zs, indexing="ij")
    np.testing.assert_array_equal(got, _block_want(*g, black_border), err_msg="lines at (%d, %d)" % (x0, y0))
  # the rooted transform on the plane of element 2^32
  run(0)
  ctx.d2h(plane, out.offset(zb * sx * sy * 4))
  ctx.sync()
  np.testing.assert_array_equal(plane.view(np.uint32), np.sqrt(_block_want(xs, ys, zb, black_border)).view(np.uint32))
