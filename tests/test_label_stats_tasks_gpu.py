"""SpatialIndexTask and CountVoxelsTask end to end through their creators and LocalTaskQueue on
file:// segmentation layers: a non-zero voxel_offset, a task grid that does not divide the
volume, labels of 2^63 and above, a deleted chunk read with fill_missing=True, and .spatial
files written with and without gzip.  Every .spatial file is compared with a CPU restatement of
the reference task (numpy renumber + scipy.ndimage.find_objects), every voxel-count file with
np.unique over its box."""
import os

import numpy as np
import pytest
import scipy.ndimage

pytestmark = pytest.mark.gpu

OFFSET = (7, 13, 3)
SHAPE = (520, 70, 36)
CHUNK = (64, 32, 12)


def _layer(tmp_path, resolution, name="seg"):
  from igneous_b200._compat import CloudFiles, CloudVolume
  rng = np.random.default_rng(11)
  pool = np.array([0, 0, 1, 2, 77, 2**32 + 5, 2**63, 2**63 + 1, 2**64 - 1] + list(range(1000, 1040)), dtype=np.uint64)
  coarse = rng.choice(pool, size=(40, 10, 6))
  data = np.kron(coarse, np.ones((13, 7, 6), dtype=np.uint64))[:SHAPE[0], :SHAPE[1], :SHAPE[2]]
  data = np.asfortranarray(data)
  path = "file://" + str(tmp_path / name)
  vol = CloudVolume.from_numpy(data[..., np.newaxis], vol_path=path, resolution=resolution, voxel_offset=OFFSET,
                               chunk_size=CHUNK, layer_type="segmentation")
  # one chunk deleted: read as zeros under fill_missing=True
  lo = np.asarray(OFFSET) + np.asarray(CHUNK) * (2, 1, 1)
  box = "%d-%d_%d-%d_%d-%d" % (lo[0], lo[0] + CHUNK[0], lo[1], lo[1] + CHUNK[1], lo[2], lo[2] + CHUNK[2])
  CloudFiles(path).delete(vol.key + "/" + box)
  data[lo[0] - OFFSET[0]:lo[0] - OFFSET[0] + CHUNK[0], lo[1] - OFFSET[1]:lo[1] - OFFSET[1] + CHUNK[1],
       lo[2] - OFFSET[2]:lo[2] - OFFSET[2] + CHUNK[2]] = 0
  return path, data


def _reference_spatial_index(data, resolution_vec, shape, offset):
  """igneous/tasks/spatial_index.py:44-69 restated on the host: clamp, +1 high overlap (zeros past
  the dataset edge), numpy renumber, scipy find_objects, boxes shifted by the task offset."""
  from igneous_b200._compat import Bbox, Vec
  ds = Bbox(OFFSET, np.asarray(OFFSET) + np.asarray(SHAPE))
  bounds = Bbox.clamp(Bbox(Vec(*offset), Vec(*shape) + Vec(*offset)), ds)
  lo = np.asarray(bounds.minpt) - np.asarray(OFFSET)
  hi = np.asarray(bounds.maxpt) + 1 - np.asarray(OFFSET)
  img = np.zeros(tuple(hi - lo), dtype=data.dtype)
  src = data[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]]
  img[:src.shape[0], :src.shape[1], :src.shape[2]] = src
  uniq = np.unique(img)
  uniq = uniq[uniq != 0]
  renum = np.where(img == 0, 0, np.searchsorted(uniq, img) + 1)
  out = {}
  for i, slc in enumerate(scipy.ndimage.find_objects(renum)):
    if slc is None:
      continue
    b = np.array([s.start for s in slc] + [s.stop for s in slc], dtype=np.int64) + np.tile(np.asarray(offset), 2)
    b = b * np.tile(np.asarray(resolution_vec, dtype=np.float32), 2)
    out[str(int(uniq[i]))] = b.astype(resolution_vec.dtype).tolist()
  name = (bounds.astype(resolution_vec.dtype) * resolution_vec).to_filename(0)
  return name, out


@pytest.mark.parametrize("resolution,compress", [((4, 4, 40), None), ((4.5, 3.25, 40.5), "gzip")])
@pytest.mark.parametrize("kind", ["mesh", "skeletons"])
def test_spatial_index_tasks(tmp_path, resolution, compress, kind):
  from igneous_b200 import task_creation as tc
  from igneous_b200._compat import CloudFiles, CloudVolume, LocalTaskQueue
  path, data = _layer(tmp_path, resolution)
  shape = (200, 48, 24)
  if kind == "mesh":
    itr = tc.create_spatial_index_mesh_tasks(path, shape=shape, fill_missing=True, compress=compress)
  else:
    itr = tc.create_spatial_index_skeleton_tasks(path, shape=shape, fill_missing=True, compress=compress)
  todo = list(itr)
  assert len(todo) == 3 * 2 * 2
  LocalTaskQueue().insert(todo)
  subdir = "mesh_mip_0_err_40" if kind == "mesh" else "skeletons_mip_0"
  res = CloudVolume(path).resolution
  cf = CloudFiles(path)
  names = set()
  labels_seen = set()
  for t in todo:
    name, want = _reference_spatial_index(data, res, t.keywords["shape"], t.keywords["offset"])
    key = "%s/%s.spatial" % (subdir, name)
    assert os.path.exists(os.path.join(path[len("file://"):], key + (".gz" if compress else "")))
    assert cf.get_json(key) == want
    names.add(name)
    labels_seen.update(want)
  assert len(names) == len(todo)
  assert {"9223372036854775808", "18446744073709551615"} <= labels_seen


def test_spatial_index_all_zero_region_writes_empty(tmp_path):
  from igneous_b200 import tasks
  from igneous_b200._compat import CloudFiles, CloudVolume
  path = "file://" + str(tmp_path / "zero")
  CloudVolume.from_numpy(np.zeros((40, 30, 20, 1), dtype=np.uint32), vol_path=path, resolution=(8, 8, 40),
                         voxel_offset=(5, 0, 0), chunk_size=(32, 32, 16), layer_type="segmentation")
  tasks.SpatialIndexTask(path, (64, 64, 64), (5, 0, 0), "mesh_mip_0_err_40", 0, compress=None)
  assert CloudFiles(path).get_json("mesh_mip_0_err_40/40-360_0-240_0-800.spatial") == {}


def test_voxel_counting_tasks(tmp_path):
  from igneous_b200 import task_creation as tc
  from igneous_b200._compat import Bbox, CloudFiles, CloudVolume, LocalTaskQueue
  path, data = _layer(tmp_path, (4, 4, 40))
  todo = list(tc.create_voxel_counting_tasks(path, mip=0, fill_missing=True))
  assert len(todo) == 2  # 512^3 tasks: x is split at 512 and the second task is clamped to 8 voxels
  LocalTaskQueue().insert(todo)
  key = CloudVolume(path).key
  cf = CloudFiles(path)
  total = {}
  for t in todo:
    offset = np.asarray(t.keywords["offset"])
    shape = np.asarray(t.keywords["shape"])
    box = Bbox(offset, offset + shape)
    lo = offset - np.asarray(OFFSET)
    hi = lo + shape
    u, c = np.unique(data[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]], return_counts=True)
    want = {str(int(a)): int(b) for a, b in zip(u, c)}
    got = cf.get_json("%s/stats/voxel_counts/%s.json" % (key, box.to_filename()))
    assert got == want
    for k, v in got.items():
      total[k] = total.get(k, 0) + v
  u, c = np.unique(data, return_counts=True)
  assert total == {str(int(a)): int(b) for a, b in zip(u, c)}
  assert "0" in total and "18446744073709551615" in total
