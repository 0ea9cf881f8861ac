"""GPU parity: CCL / dust kernels (through the C ABI) vs the CPU oracle and
the reference's own structural known answers (test/test_ccl_tasks.py)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _blobs(rng, shape, nlab, dtype, p_bg=0.3):
  # smooth random blobs: threshold a low-pass field, label by a second field
  small = rng.integers(0, nlab + 1, size=tuple((s + 3) // 4 for s in shape))
  big = np.repeat(np.repeat(np.repeat(small, 4, 0), 4, 1), 4, 2)[:shape[0], :shape[1], :shape[2]]
  noise = rng.random(shape) < p_bg
  out = np.where(noise, 0, big)
  if np.dtype(dtype).itemsize == 8:
    out = out.astype(np.uint64) * np.uint64((1 << 32) + 7)
  return np.asfortranarray(out.astype(dtype))


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.uint32, np.uint64])
@pytest.mark.parametrize("shape", [(64, 64, 64), (33, 29, 17), (129, 7, 5), (1, 1, 1), (5, 1, 3), (70, 65, 3)])
def test_ccl_matches_oracle_bit_exact(ctx, oracle, dtype, shape):
  from igneous_b200 import cc3d
  rng = np.random.default_rng(abs(hash((shape, np.dtype(dtype).itemsize))) % (1 << 32))
  labels = _blobs(rng, shape, 3, dtype)
  got, n = cc3d.connected_components(labels, connectivity=6, out_dtype=np.uint64, return_N=True)
  want, n_want = oracle.connected_components(labels, return_N=True)
  assert n == n_want
  assert got.dtype == np.uint64 and got.shape == labels.shape
  # same numbering convention (first voxel in raster order): bit exact
  assert np.array_equal(got, want)
  # and therefore canonical relabelling is the identity (test_ccl_tasks.py:246-249)
  assert np.array_equal(oracle.renumber(got)[0], got)


def test_ccl_random_noise_worst_case(ctx, oracle):
  # every voxel its own component: exercises the candidate-overflow retry
  from igneous_b200 import cc3d
  rng = np.random.default_rng(5)
  labels = np.asfortranarray(rng.integers(1, 1 << 30, size=(40, 37, 21), dtype=np.uint32))
  got, n = cc3d.connected_components(labels, connectivity=6, out_dtype=np.uint32, return_N=True)
  want, n_want = oracle.connected_components(labels, return_N=True)
  assert n == n_want and np.array_equal(got, want)


def test_ccl_bool_and_binary_long_runs(ctx, oracle):
  from igneous_b200 import cc3d
  rng = np.random.default_rng(6)
  field = rng.random((96, 50, 20)) < 0.62  # near the percolation threshold: deep merge trees
  got, n = cc3d.connected_components(field, connectivity=6, out_dtype=np.uint64, return_N=True)
  want, n_want = oracle.connected_components(field, return_N=True)
  assert n == n_want and np.array_equal(got, want)
  snake = np.zeros((100, 64, 4), dtype=np.uint8, order="F")
  for y in range(0, 64, 2):  # one serpentine component: worst-case tree depth
    snake[:, y, 0] = 1
    snake[99 if (y // 2) % 2 == 0 else 0, y + 1, 0] = 1
  got, n = cc3d.connected_components(snake, connectivity=6, return_N=True)
  assert n == 1 and np.array_equal(got != 0, snake != 0)


def test_ccl_checker_reference_kat(ctx):
  # test/test_ccl_tasks.py:20-30,188-208: 512x512x128 uint8, 64^3 blocks 1..128
  from igneous_b200 import cc3d
  data = np.zeros((512, 512, 128), dtype=np.uint8, order="F")
  i = 1
  for x in range(8):
    for y in range(8):
      for z in range(2):
        data[64 * x:64 * (x + 1), 64 * y:64 * (y + 1), 64 * z:64 * (z + 1)] = i
        i += 1
  cc, n = cc3d.connected_components(data, connectivity=6, out_dtype=np.uint64, return_N=True)
  assert n == 128
  uniq, counts = np.unique(cc, return_counts=True)
  assert np.array_equal(uniq, np.arange(1, 129)) and (counts == 64 ** 3).all()
  cc, n = cc3d.connected_components(data <= 255, connectivity=6, return_N=True)
  assert n == 1 and (cc == 1).all()
  assert not cc3d.dust(data, 64 ** 3 + 1, connectivity=6).any()
  assert np.array_equal(cc3d.dust(data, 64 ** 3, connectivity=6), data)


@pytest.mark.parametrize("dtype", [np.uint8, np.uint32, np.uint64])
@pytest.mark.parametrize("threshold", [1, 5, 40, 10 ** 9])
def test_dust_matches_oracle(ctx, oracle, dtype, threshold):
  from igneous_b200 import cc3d
  rng = np.random.default_rng(9)
  labels = _blobs(rng, (48, 40, 24), 4, dtype, p_bg=0.45)
  want = oracle.dust(labels, threshold)
  got = cc3d.dust(labels, threshold, connectivity=6, in_place=False)
  assert np.array_equal(got, want)
  work = labels.copy(order="F")
  res = cc3d.dust(work, threshold, connectivity=6, in_place=True)
  assert res is work and np.array_equal(work, want)


def test_ccl_synthetic_voronoi_1024_properties(ctx, oracle):
  """Size-independent properties on a chunk the oracle needs minutes for:
  (1) idempotence: CCL of the CCL output is the identity;
  (2) every output id maps to exactly one input label;
  (3) a 128^3 corner agrees with the oracle after canonical renumbering."""
  from igneous_b200 import cc3d
  seg = oracle.synth_seg((128, 128, 64), pitch=32, num_ids=4)
  big = np.asfortranarray(np.tile(seg, (4, 4, 4)))  # 512x512x256
  cc, n = cc3d.connected_components(big, connectivity=6, out_dtype=np.uint32, return_N=True)
  assert cc.max() == n
  cc2, n2 = cc3d.connected_components(cc, connectivity=6, out_dtype=np.uint32, return_N=True)
  assert n2 == n and np.array_equal(cc2, cc)
  pairs = np.unique(np.stack([cc.ravel()[::7], big.ravel()[::7]], axis=1), axis=0)
  assert len(np.unique(pairs[:, 0])) == len(pairs)
  want, n_want = oracle.connected_components(big, return_N=True)
  assert n == n_want and np.array_equal(cc, want)


def test_ccl_rejects_other_connectivity(ctx):
  from igneous_b200 import cc3d
  with pytest.raises(NotImplementedError):
    cc3d.connected_components(np.zeros((4, 4, 4), np.uint8), connectivity=26)


@pytest.mark.parametrize("shape", [(64, 48, 40), (33, 29, 17), (70, 65, 9), (40, 40, 40), (260, 20, 19)])
@pytest.mark.parametrize("dtype", [np.uint8, np.uint64])
def test_volume_ccl_equals_whole_volume(ctx, oracle, shape, dtype):
  """ign_ccl6_volume_dev (begin + finish, the halves a multi-GPU run links in between) must
  be bit-identical to a single whole-volume CCL (and to the oracle)."""
  import ctypes as c
  from igneous_b200 import _shim
  rng = np.random.default_rng(21)
  labels = _blobs(rng, shape, 3, dtype, p_bg=0.2)
  want, n_want = oracle.connected_components(labels, return_N=True)
  d_in = ctx.to_device(labels)
  d_out = ctx.alloc(labels.size * 4)
  n = c.c_uint64(0)
  _shim.check(ctx.lib.ign_ccl6_volume_dev(ctx.handle, _shim.ptr(d_in), _shim.dtype_code(dtype), shape[0], shape[1],
                                          shape[2], _shim.ptr(d_out), _shim.IGN_U32, c.byref(n)))
  got = ctx.to_host(d_out, shape, np.uint32)
  assert n.value == n_want
  assert np.array_equal(got, want.astype(np.uint32))


def test_ccl_device_resident_properties_1024(ctx):
  """BASELINE config C3 size (1024^3, uint64 ids >= 2^32, ~5.7k objects), device resident:
  idempotence (CCL of the CCL output is the identity), component count stable across
  slab splits, every id in 1..N used.  The oracle needs minutes at this size."""
  import ctypes as c
  from igneous_b200 import _shim
  S = 1024
  n = S ** 3
  d_in = ctx.alloc(n * 8)
  d_cc = ctx.alloc(n * 4)
  d_cc2 = ctx.alloc(n * 4)
  try:
    _shim.check(ctx.lib.ign_synth_seg_dev(ctx.handle, _shim.ptr(d_in), _shim.IGN_U64, S, S, S, 0, 0, 0, 64, 4096, 0,
                                          1 << 32))
    n1, n2, n3 = c.c_uint64(0), c.c_uint64(0), c.c_uint64(0)
    args = (S, S, S)
    _shim.check(ctx.lib.ign_ccl6_dev(ctx.handle, _shim.ptr(d_in), _shim.IGN_U64, *args, _shim.ptr(d_cc), _shim.IGN_U32,
                                     c.byref(n1)))
    _shim.check(ctx.lib.ign_ccl6_dev(ctx.handle, _shim.ptr(d_cc), _shim.IGN_U32, *args, _shim.ptr(d_cc2), _shim.IGN_U32,
                                     c.byref(n2)))
    assert n1.value == n2.value and 4000 < n1.value < 8000
    a = ctx.to_host(d_cc, (S, S, 64), np.uint32)   # first 64 z-planes
    b = ctx.to_host(d_cc2, (S, S, 64), np.uint32)
    assert np.array_equal(a, b)
    # the begin / finish halves must give the same labelling as the single call
    _shim.check(ctx.lib.ign_ccl6_volume_dev(ctx.handle, _shim.ptr(d_in), _shim.IGN_U64, *args, _shim.ptr(d_cc2),
                                            _shim.IGN_U32, c.byref(n3)))
    assert n3.value == n1.value
    assert np.array_equal(ctx.to_host(d_cc2, (S, S, 64), np.uint32), a)
    tail = np.empty((S, S, 8), dtype=np.uint32, order="F")
    ctx.d2h(tail, d_cc.ptr + (S - 8) * S * S * 4)
    tail2 = np.empty((S, S, 8), dtype=np.uint32, order="F")
    ctx.d2h(tail2, d_cc2.ptr + (S - 8) * S * S * 4)
    ctx.sync()
    assert np.array_equal(tail, tail2) and int(max(a.max(), tail.max())) <= n1.value
  finally:
    d_in.free(); d_cc.free(); d_cc2.free()


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.uint32, np.uint64])
def test_ccl_tma_and_cooperative_fill_match_oracle(ctx, oracle, monkeypatch, dtype):
  """The mask kernel stages tiles by TMA when the row pitch is 16-byte aligned and by
  cooperative loads otherwise (IGN_CCL_NO_TMA=1 forces the latter): same ids as the oracle
  from both, on aligned volumes with full and partial tiles, long runs and dense noise (the
  tile-run overflow path of k_ccl_tiles), and on unaligned row pitches."""
  from igneous_b200 import cc3d
  rng = np.random.default_rng(0)
  vols = [oracle.synth_seg((512, 64, 40), pitch=16, num_ids=9).astype(dtype),
          rng.integers(0, 3, size=(256, 16, 24)).astype(dtype),
          rng.integers(0, 3, size=(1024, 16, 16)).astype(dtype),
          oracle.synth_seg((300, 40, 20), pitch=16, num_ids=5).astype(dtype),
          oracle.synth_seg((129, 33, 17), pitch=8, num_ids=5).astype(dtype)]
  for v in vols:
    v = np.asfortranarray(v)
    want, wn = oracle.connected_components(v, return_N=True)
    for no_tma in (False, True):
      for pair in ("0", "1"):  # 1: x-adjacent tile pairs with whole-sector mask writes (the default for 2048+ voxel rows)
        if no_tma:
          monkeypatch.setenv("IGN_CCL_NO_TMA", "1")
        else:
          monkeypatch.delenv("IGN_CCL_NO_TMA", raising=False)
        monkeypatch.setenv("IGN_CCL_PAIR", pair)
        got, n = cc3d.connected_components(v, connectivity=6, out_dtype=np.uint64, return_N=True)
        assert n == wn and np.array_equal(got, want), (v.shape, no_tma, pair)
  monkeypatch.delenv("IGN_CCL_NO_TMA", raising=False)
  monkeypatch.delenv("IGN_CCL_PAIR", raising=False)
