"""tests/edtref.py (the CPU statement of the distance-transform rule) against the rule's definition,
an O(N^2) search over every voxel pair, on tiny volumes: 1-, 2- and 3-D, both borders, integer and
non-integer anisotropy, the +inf case; and the block volumes' closed form against the reference."""
import numpy as np
import pytest

import edtref

ANISO = {1: [(1.0,), (2.5,)], 2: [(1.0, 1.0), (3.0, 1.0), (1.5, 7.25)],
         3: [(1.0, 1.0, 1.0), (4.0, 4.0, 40.0), (4.5, 7.25, 40.3)]}


def _volumes(ndim, seed):
  rng = np.random.default_rng(seed)
  shape = {1: (13,), 2: (7, 6), 3: (6, 5, 4)}[ndim]
  yield rng.integers(0, 3, size=shape).astype(np.uint8)                    # many small runs
  coarse = rng.integers(1, 4, size=tuple(-(-s // 3) for s in shape))
  yield np.kron(coarse, np.ones((3,) * ndim, dtype=np.int64))[tuple(slice(0, s) for s in shape)].astype(np.uint32)
  v = np.full(shape, 5, dtype=np.uint16)                                     # one label, one hole
  v[tuple(s // 2 for s in shape)] = 0
  yield v


@pytest.mark.parametrize("ndim", [1, 2, 3])
@pytest.mark.parametrize("black_border", [False, True])
def test_reference_matches_brute_force(ndim, black_border):
  for ai, a in enumerate(ANISO[ndim]):
    for vol in _volumes(ndim, 10 * ndim + ai):
      want = edtref.brute_edtsq(vol, a, black_border)
      got = edtref.edtsq(vol, a, black_border)
      if all(float(x).is_integer() for x in a):
        np.testing.assert_array_equal(got, want)
      else:
        np.testing.assert_allclose(got, want, rtol=1e-6)


@pytest.mark.parametrize("ndim", [1, 2, 3])
def test_one_label_filling_the_volume(ndim):
  vol = np.full({1: (9,), 2: (5, 4), 3: (4, 3, 5)}[ndim], 7, dtype=np.uint8)
  a = ANISO[ndim][-1]
  assert np.all(np.isinf(edtref.edtsq(vol, a, False)))
  want = edtref.brute_edtsq(vol, a, True)
  assert np.all(np.isfinite(want))
  np.testing.assert_allclose(edtref.edtsq(vol, a, True), want, rtol=1e-6)


def test_all_zero_and_distinct_labels():
  assert not np.any(edtref.edtsq(np.zeros((4, 3, 2), np.uint8), (2, 3, 5)))
  vol = np.arange(1, 25, dtype=np.uint32).reshape((4, 3, 2))
  np.testing.assert_array_equal(edtref.edtsq(vol, (2.0, 3.0, 5.0)), np.full(vol.shape, 4.0, np.float32))
  np.testing.assert_array_equal(edtref.edtsq(vol, (2.0, 3.0, 5.0)), edtref.brute_edtsq(vol, (2.0, 3.0, 5.0)))


def test_u64_labels_differing_in_high_bits():
  vol = np.array([[1, 1, 2**32 + 1, 2**32 + 1]], dtype=np.uint64)
  want = np.array([[4, 1, 1, 4]], dtype=np.float32)
  np.testing.assert_array_equal(edtref.edtsq(vol), want)
  np.testing.assert_array_equal(edtref.brute_edtsq(vol), want)


@pytest.mark.parametrize("black_border", [False, True])
def test_block_closed_form(black_border):
  shape, block, a = (23, 17, 11), (5, 4, 3), (4.0, 4.0, 40.0)
  g = np.indices(shape)
  lab = ((g[0] // block[0]) + (g[1] // block[1]) + (g[2] // block[2])) % 3
  want = np.where(lab == 0, np.float32(0), edtref.block_edtsq(g, shape, block, a, black_border))
  np.testing.assert_array_equal(edtref.edtsq(lab.astype(np.uint8), a, black_border), want)
