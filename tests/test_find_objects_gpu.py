"""igneous_b200.spatial_index.find_objects against scipy.ndimage.find_objects, exactly: dense
labels with gaps, one label filling the volume, every voxel its own label, labels only on faces,
edges and corners, rows of 1, 31, 33 and 4100 voxels, every label dtype, both memory orders,
max_label below and above the largest label, empty volumes and a renumbered synthetic
segmentation; and the refusals."""
import numpy as np
import pytest
import scipy.ndimage

pytestmark = pytest.mark.gpu


def _check(labels, max_label=0):
  from igneous_b200 import spatial_index
  got = spatial_index.find_objects(labels, max_label=max_label)
  want = scipy.ndimage.find_objects(labels, max_label=max_label)
  assert len(got) == len(want)
  assert got == want


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.uint32, np.uint64])
@pytest.mark.parametrize("order", ["F", "C"])
def test_random_labels_with_gaps(dtype, order):
  rng = np.random.default_rng(1)
  labels = rng.choice(np.array([0, 1, 2, 5, 9, 17, 200, 201, 255], dtype=dtype), size=(37, 29, 11))
  _check(np.asarray(labels, order=order))


@pytest.mark.parametrize("order", ["F", "C"])
def test_blocky_labels(order):
  # segmentation-like: runs along every axis, a few hundred labels, most of them missing
  rng = np.random.default_rng(2)
  coarse = rng.integers(0, 400, size=(9, 7, 5)).astype(np.uint32) * 3
  labels = np.kron(coarse, np.ones((13, 11, 7), dtype=np.uint32))[:111, :70, :33]
  _check(np.asarray(labels, order=order))


def test_one_label_fills_the_volume():
  _check(np.full((300, 70, 20), 7, dtype=np.uint32, order="F"))


@pytest.mark.parametrize("order", ["F", "C"])
def test_every_voxel_its_own_label(order):
  labels = np.arange(1, 64 * 48 * 40 + 1, dtype=np.uint32).reshape((64, 48, 40), order=order)
  _check(labels)
  rng = np.random.default_rng(3)
  _check(rng.permutation(labels.ravel()).reshape(labels.shape, order=order))


def test_faces_edges_and_corners():
  shape = (45, 34, 23)
  labels = np.zeros(shape, dtype=np.uint16, order="F")
  labels[0, :, :] = 1
  labels[-1, :, :] = 2
  labels[:, 0, :] = 3
  labels[:, -1, 5:9] = 4
  labels[:, :, 0] = 5
  labels[:, :, -1] = 6
  labels[0, 0, :] = 7
  labels[-1, -1, :] = 8
  labels[:, 0, -1] = 9
  for i, c in enumerate([(0, 0, 0), (44, 0, 0), (0, 33, 0), (0, 0, 22), (44, 33, 22), (44, 33, 0)]):
    labels[c] = 10 + i
  labels[44, 0, 22] = 10  # label 10 at two opposite corners
  _check(labels)


@pytest.mark.parametrize("shape", [(1, 40, 30), (31, 17, 9), (33, 17, 9), (4100, 3, 2), (4096, 2, 1),
                                   (70, 1, 13), (70, 13, 1), (1, 1, 1), (2, 1, 1)])
def test_row_lengths_and_thin_volumes(shape):
  rng = np.random.default_rng(sum(shape))
  _check(np.asfortranarray(rng.integers(0, 6, size=shape).astype(np.uint32)))
  # long runs along x with changes at odd positions
  runs = np.asfortranarray(np.cumsum(rng.random(shape) < 0.05, axis=0).astype(np.uint32) % 7)
  _check(runs)


def test_u64_labels():
  rng = np.random.default_rng(5)
  labels = np.asfortranarray(rng.choice(np.array([0, 1, 3, 4, 2**32 - 1, 2**40, 2**64 - 1], dtype=np.uint64),
                                        size=(20, 6, 5)))
  _check(labels, max_label=3)  # labels above max_label, 2^32 and more included, are ignored
  _check(np.asfortranarray(np.where(labels > 4, np.uint64(2), labels)))


def test_bool_input():
  rng = np.random.default_rng(6)
  labels = rng.random((17, 9, 4)) < 0.3
  from igneous_b200 import spatial_index
  assert spatial_index.find_objects(labels) == scipy.ndimage.find_objects(labels.view(np.uint8))


@pytest.mark.parametrize("max_label", [1, 4, 9, 40])
def test_max_label_below_and_above(max_label):
  rng = np.random.default_rng(7)
  labels = np.asfortranarray(rng.integers(0, 10, size=(23, 19, 7)).astype(np.uint16))
  _check(labels, max_label=max_label)


def test_all_zero_and_empty():
  from igneous_b200 import spatial_index
  _check(np.zeros((5, 6, 7), dtype=np.uint32))
  _check(np.zeros((5, 6, 7), dtype=np.uint8), max_label=3)
  _check(np.zeros((0, 6, 7), dtype=np.uint32), max_label=3)
  assert spatial_index.find_objects(np.zeros((0, 6, 7), dtype=np.uint32)) == []
  assert spatial_index.find_objects(np.zeros((4, 0, 2), dtype=np.uint64), max_label=2) == [None, None]


def test_renumbered_synthetic_segmentation_449():
  from igneous_b200 import fastremap
  from oracle import oracle as O
  seg = O.synth_seg((449, 449, 449), pitch=24, num_ids=1 << 20, seed=3)
  small, mapping = fastremap.renumber(seg)
  _check(small)
  _check(np.ascontiguousarray(small.T).T)  # the same data through a C-order copy of the transpose


def test_refusals():
  from igneous_b200 import spatial_index
  big = np.zeros((4, 4, 4), dtype=np.uint64)
  big[1, 2, 3] = 2**32
  with pytest.raises(NotImplementedError, match="renumber"):
    spatial_index.find_objects(big)
  with pytest.raises(NotImplementedError, match="renumber"):
    spatial_index.find_objects(np.ones((4, 4, 4), dtype=np.uint8), max_label=2**32)
  with pytest.raises(ValueError):
    spatial_index.find_objects(np.ones((4, 4), dtype=np.uint32))
  with pytest.raises(NotImplementedError):
    spatial_index.find_objects(np.ones((4, 4, 4), dtype=np.int32))
