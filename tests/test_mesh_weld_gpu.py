"""GPU: the mesher's triangle order, vertex order, faces, per-label offsets and ids, exactly as the
numpy restatement in mcref.py, on volumes that reach the corners of the weld: more than 2^16
labels in one task (three or more digit passes of the label sort), one-voxel-thick dimensions, a
1023 x 2 x 2 task, one label everywhere and checkerboards."""
import numpy as np
import pytest

import mcref

pytestmark = pytest.mark.gpu

RES = (4.0, 5.0, 40.0)


def _check(data):
  from igneous_b200 import zmesh
  ids, tri_off, vert_off, verts, faces = mcref.mesh(data)
  m = zmesh.Mesher(RES)
  m.mesh(data)
  present = [l for l in range(1, len(ids) + 1) if tri_off[l + 1] > tri_off[l]]
  assert m.ids() == [int(ids[l - 1]) for l in present]
  if not present:
    return
  gv, gf, voff, foff, _ = m._exported(False)
  assert np.array_equal(voff, np.append(vert_off[present], vert_off[-1]))
  assert np.array_equal(foff, np.append(tri_off[present], tri_off[-1]))
  assert gf.shape == faces.shape and np.array_equal(gf, faces)
  want = (verts.astype(np.float32) * np.float32(0.5)) * np.array(RES, dtype=np.float32)
  assert gv.shape == want.shape and np.array_equal(gv, want)


def test_more_than_2_16_labels_in_one_task(ctx):
  rng = np.random.default_rng(7)
  data = np.asfortranarray(rng.integers(1, 2**40, size=(60, 50, 40), dtype=np.uint64))
  data[rng.random(data.shape) < 0.05] = 0
  assert len(np.unique(data)) > 65536
  _check(data)


@pytest.mark.parametrize("shape", [(2, 31, 17), (29, 2, 23), (19, 27, 2), (2, 2, 40), (2, 2, 2)])
def test_one_voxel_thick_dimensions(ctx, shape):
  rng = np.random.default_rng(sum(shape))
  _check(np.asfortranarray(rng.integers(0, 5, size=shape, dtype=np.uint32)))


def test_1023_by_2_by_2(ctx):
  rng = np.random.default_rng(1023)
  _check(np.asfortranarray(rng.integers(0, 4, size=(1023, 2, 2), dtype=np.uint32)))


def test_one_label_everywhere_and_padded(ctx):
  _check(np.ones((20, 21, 22), dtype=np.uint32, order="F"))
  data = np.zeros((20, 21, 22), dtype=np.uint32, order="F")
  data[1:-1, 1:-1, 1:-1] = 9
  _check(data)


@pytest.mark.parametrize("labels", [(0, 1), (1, 2), (3, 0, 7)])
def test_checkerboard(ctx, labels):
  x, y, z = np.indices((17, 18, 19))
  data = np.asarray(labels, dtype=np.uint32)[(x + y + z) % len(labels)]
  _check(np.asfortranarray(data))


def test_random_multilabel_blocks(ctx):
  rng = np.random.default_rng(3)
  small = rng.integers(0, 40, size=(12, 11, 10), dtype=np.uint32)
  data = np.asfortranarray(np.kron(small, np.ones((4, 4, 4), dtype=np.uint32))[:45, :41, :38])
  _check(data)
