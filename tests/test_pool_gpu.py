"""GPU parity: pooling kernels (through the C ABI) vs the CPU oracle."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _seg(rng, shape, dtype, nlab=5):
  # blocky labels (3x3 in xy) plus 30% noise so that ties and majorities both occur
  small = rng.integers(0, nlab, size=((shape[0] + 2) // 3, (shape[1] + 2) // 3) + tuple(shape[2:]))
  big = np.repeat(np.repeat(small, 3, axis=0), 3, axis=1)[:shape[0], :shape[1]]
  noise = rng.integers(0, nlab, size=shape)
  out = np.where(rng.random(shape) < 0.3, noise, big)
  if np.dtype(dtype).itemsize == 8:
    out = out.astype(np.uint64) * np.uint64(0x100000001)
  return np.asfortranarray(out.astype(dtype))


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.uint32, np.uint64])
@pytest.mark.parametrize("shape,num_mips", [
  ((128, 128, 64), 1),    # BASELINE config C1
  ((256, 64, 5), 4),      # fused multi-mip
  ((64, 48, 3), 3),       # sy not divisible by 16 -> mixed fused/generic
  ((37, 21, 2), 3),       # odd extents -> generic path
  ((16, 16, 1), 5),       # deeper than the extent
])
def test_mode_pool_matches_oracle(ctx, oracle, dtype, shape, num_mips):
  from igneous_b200 import tinybrain
  rng = np.random.default_rng(hash((np.dtype(dtype).itemsize, shape, num_mips)) % (1 << 32))
  img = _seg(rng, shape, dtype)
  got = tinybrain.downsample_segmentation(img, (2, 2, 1), num_mips=num_mips)
  want = oracle.downsample_segmentation(img, (2, 2, 1), num_mips=num_mips)
  assert len(got) == num_mips
  for g, w in zip(got, want):
    assert g.dtype == w.dtype and g.shape == w.shape and g.flags.f_contiguous
    assert np.array_equal(g, w)


def test_mode_pool_kats_gpu(ctx):
  from igneous_b200 import tinybrain
  from test_oracle import MODE_KATS
  for dtype in (np.uint8, np.uint32, np.uint64):
    for (a, b, c, d), want in MODE_KATS:
      img = np.zeros((2, 2, 1), dtype=dtype, order="F")
      img[0, 0, 0], img[1, 0, 0], img[0, 1, 0], img[1, 1, 0] = a, b, c, d
      out, = tinybrain.downsample_segmentation(img, (2, 2, 1))
      assert out[0, 0, 0] == want
    # same KATs through the vectorised path (tile them to a 64x64 image)
    img = np.zeros((64, 64, 2), dtype=dtype, order="F")
    wants = np.zeros((32, 32, 2), dtype=dtype)
    for i, ((a, b, c, d), want) in enumerate(MODE_KATS * 128):
      x, y = i % 32, (i // 32) % 32
      img[2 * x, 2 * y, :], img[2 * x + 1, 2 * y, :] = a, b
      img[2 * x, 2 * y + 1, :], img[2 * x + 1, 2 * y + 1, :] = c, d
      wants[x, y, :] = want
    out, = tinybrain.downsample_segmentation(img, (2, 2, 1))
    assert np.array_equal(out, wants)


def test_mode_pool_sparse_and_4d(ctx, oracle):
  from igneous_b200 import tinybrain
  rng = np.random.default_rng(7)
  img = _seg(rng, (64, 32, 4, 2), np.uint32, nlab=3)
  for sparse in (False, True):
    got = tinybrain.downsample_segmentation(img, (2, 2, 1, 1), num_mips=2, sparse=sparse)
    want = oracle.downsample_segmentation(img, (2, 2, 1, 1), num_mips=2, sparse=sparse)
    for g, w in zip(got, want):
      assert g.shape == w.shape and np.array_equal(g, w)


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.uint32])
@pytest.mark.parametrize("shape,num_mips", [
  ((512, 512, 8), 5),     # C2 shape class: 5-level pyramid, group of 4 + 1
  ((64, 64, 3), 4),
  ((48, 40, 2), 3),       # generic path (not a multiple of 16)
  ((37, 21, 2), 6),       # odd extents, mirrored edges, two groups
])
@pytest.mark.parametrize("rounding", [0, 1, 2])
def test_avg_pool_matches_oracle(ctx, oracle, dtype, shape, num_mips, rounding):
  from igneous_b200 import tinybrain
  rng = np.random.default_rng(11)
  hi = np.iinfo(dtype).max
  img = np.asfortranarray(rng.integers(0, hi, size=shape, dtype=dtype, endpoint=True))
  got = tinybrain.downsample_with_averaging(img, (2, 2, 1), num_mips=num_mips, rounding=rounding)
  want = oracle.downsample_with_averaging(img, (2, 2, 1), num_mips=num_mips, rounding=rounding)
  for g, w in zip(got, want):
    assert g.shape == w.shape and np.array_equal(g, w)


def test_avg_pool_f32_within_tolerance(ctx, oracle):
  from igneous_b200 import tinybrain
  rng = np.random.default_rng(12)
  img = np.asfortranarray(rng.random((65, 33, 3), dtype=np.float32))
  got = tinybrain.downsample_with_averaging(img, (2, 2, 1), num_mips=3)
  want = oracle.downsample_with_averaging(img, (2, 2, 1), num_mips=3)
  for g, w in zip(got, want):
    # same operation order, no FMA contraction on either side: bit exact
    assert np.array_equal(g, w)


def test_pool_invariants_large(ctx):
  """Size-independent properties at a size the oracle would take minutes for."""
  from igneous_b200 import tinybrain
  data = np.zeros((1024, 1024, 16), dtype=np.uint32, order="F")
  i = 1
  for x in range(16):
    for y in range(16):
      data[64 * x:64 * (x + 1), 64 * y:64 * (y + 1), :] = i
      i += 1
  mips = tinybrain.downsample_segmentation(data, (2, 2, 1), num_mips=5)
  cur = data
  for m in mips:
    cur = cur[::2, ::2, :]
    assert np.array_equal(m, cur)
  const = np.full((512, 512, 4), 173, dtype=np.uint8, order="F")
  for m in tinybrain.downsample_with_averaging(const, (2, 2, 1), num_mips=5):
    assert (m == 173).all()


def test_unsupported_factor_raises(ctx):
  from igneous_b200 import tinybrain
  with pytest.raises(NotImplementedError):
    tinybrain.downsample_segmentation(np.zeros((4, 4, 4), np.uint8), (3, 3, 1))
  with pytest.raises(NotImplementedError):
    tinybrain.downsample_with_averaging(np.zeros((4, 4, 4), np.uint64), (2, 2, 2))


def test_synth_matches_oracle(ctx, oracle):
  """The on-device benchmark volume generator is bit-identical to the oracle's."""
  import ctypes as c
  from igneous_b200 import _shim
  shape, off = (70, 45, 33), (-7, 11, 2048)
  for dtype, pitch, ids, base in ((np.uint32, 16, 1 << 20, 0), (np.uint64, 24, 5, 1 << 32)):
    d = ctx.alloc(int(np.prod(shape)) * np.dtype(dtype).itemsize)
    _shim.check(ctx.lib.ign_synth_seg_dev(ctx.handle, _shim.ptr(d), _shim.dtype_code(dtype), shape[0], shape[1],
                                          shape[2], off[0], off[1], off[2], pitch, ids, 3, base))
    got = ctx.to_host(d, shape, dtype)
    want = oracle.synth_seg(shape, pitch=pitch, num_ids=ids, seed=3, offset=off, dtype=dtype, id_base=base)
    assert np.array_equal(got, want)
    d.free()
  d = ctx.alloc(int(np.prod(shape)))
  _shim.check(ctx.lib.ign_synth_image_dev(ctx.handle, _shim.ptr(d), shape[0], shape[1], shape[2], 1, 2, 3, 9))
  assert np.array_equal(ctx.to_host(d, shape, np.uint8), oracle.synth_image(shape, seed=9, offset=(1, 2, 3)))


@pytest.mark.parametrize("op,name", [(0, "min"), (1, "max"), (2, "stride")])
@pytest.mark.parametrize("factor", [(2, 2, 1), (2, 2, 2), (1, 2, 2)])
@pytest.mark.parametrize("dtype", [np.uint8, np.uint32, np.float32])
def test_min_max_striding_pooling(ctx, oracle, op, name, factor, dtype):
  """DownsampleMethods MIN / MAX / STRIDING (igneous/types.py:9-11), SURVEY 8(f) row 3."""
  from igneous_b200 import tinybrain
  rng = np.random.default_rng(31)
  shape = (37, 22, 9)
  img = rng.random(shape).astype(np.float32) if dtype == np.float32 else rng.integers(0, 250, size=shape).astype(dtype)
  img = np.asfortranarray(img)
  fn = [tinybrain.downsample_with_min_pooling, tinybrain.downsample_with_max_pooling,
        tinybrain.downsample_with_striding][op]
  got = fn(img, factor, num_mips=3)
  want = oracle.downsample_select(img, factor, num_mips=3, op=name)
  for g, w in zip(got, want):
    assert g.shape == w.shape and g.dtype == w.dtype and np.array_equal(g, w)


@pytest.mark.parametrize("factor", [(2, 2, 2), (1, 2, 2), (2, 1, 2), (2, 1, 1), (1, 1, 2)])
@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.uint32, np.uint64])
@pytest.mark.parametrize("sparse", [False, True])
def test_block_mode_pooling(ctx, oracle, factor, dtype, sparse):
  """downsample_segmentation with a non-(2,2,1) factor (2x2x2 = --volumetric), SURVEY 8(f) row 3."""
  from igneous_b200 import tinybrain
  rng = np.random.default_rng(7)
  for shape, hi in (((37, 22, 9), 4), ((16, 16, 16), 3), ((5, 1, 7), 2)):
    img = np.asfortranarray(rng.integers(0, hi, size=shape).astype(dtype))
    if dtype == np.uint64:
      img[img > 0] += np.uint64(1 << 40)
    got = tinybrain.downsample_segmentation(img, factor, num_mips=3, sparse=sparse)
    want = oracle.downsample_segmentation(img, factor, num_mips=3, sparse=sparse)
    for g, w in zip(got, want):
      assert g.shape == w.shape and g.dtype == w.dtype and np.array_equal(g, w)


@pytest.mark.parametrize("factor", [(2, 2, 2), (1, 2, 2), (2, 1, 1)])
@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.uint32, np.float32])
@pytest.mark.parametrize("rounding", [0, 1, 2])
def test_block_average_pooling(ctx, oracle, factor, dtype, rounding):
  from igneous_b200 import tinybrain
  rng = np.random.default_rng(8)
  for shape in ((37, 22, 9), (16, 16, 16), (1, 5, 3)):
    if dtype == np.float32:
      img = rng.random(shape).astype(np.float32)
    else:
      img = rng.integers(0, np.iinfo(dtype).max, size=shape, endpoint=True).astype(dtype)
    img = np.asfortranarray(img)
    got = tinybrain.downsample_with_averaging(img, factor, num_mips=3, rounding=rounding)
    want = oracle.downsample_with_averaging(img, factor, num_mips=3, rounding=rounding)
    for g, w in zip(got, want):
      assert g.shape == w.shape and g.dtype == w.dtype and np.array_equal(g, w)


def test_block_pooling_4d_and_221_consistency(ctx, oracle):
  """Channels are pooled independently; (2,2,1) through the generic entry point equals the
  tuned pyramid for mode pooling (COUNTLESS pick on planar blocks)."""
  import ctypes as c
  from igneous_b200 import tinybrain, _shim
  rng = np.random.default_rng(9)
  img = np.asfortranarray(rng.integers(0, 5, size=(20, 14, 6, 2)).astype(np.uint8))
  got = tinybrain.downsample_segmentation(img, (2, 2, 2), num_mips=2)
  want = oracle.downsample_segmentation(img, (2, 2, 2), num_mips=2)
  for g, w in zip(got, want):
    assert g.shape == w.shape and np.array_equal(g, w)
  vol = np.asfortranarray(rng.integers(0, 4, size=(33, 18, 5)).astype(np.uint32))
  tuned = tinybrain.downsample_segmentation(vol, (2, 2, 1), num_mips=2)
  generic = tinybrain._select(vol, (2, 2, 1), 2, tinybrain._OP_MODE, None)
  for g, w in zip(generic, tuned):
    assert np.array_equal(g, w)


@pytest.mark.parametrize("factor", [(2, 2, 1), (2, 2, 2)])
@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.uint32, np.float32])
@pytest.mark.parametrize("rounding", [0, 1, 2])
def test_sparse_average_pooling(ctx, oracle, factor, dtype, rounding):
  """downsample_with_averaging(sparse=True): mean of the non-zero samples."""
  from igneous_b200 import tinybrain
  rng = np.random.default_rng(10)
  for shape in ((37, 22, 9), (16, 16, 4)):
    if dtype == np.float32:
      img = rng.random(shape).astype(np.float32)
    else:
      img = rng.integers(1, np.iinfo(dtype).max, size=shape, endpoint=True).astype(dtype)
    img[rng.random(shape) < 0.6] = 0
    img = np.asfortranarray(img)
    got = tinybrain.downsample_with_averaging(img, factor, num_mips=3, sparse=True, rounding=rounding)
    want = oracle.downsample_with_averaging(img, factor, num_mips=3, sparse=True, rounding=rounding)
    for g, w in zip(got, want):
      assert g.shape == w.shape and g.dtype == w.dtype and np.array_equal(g, w)
