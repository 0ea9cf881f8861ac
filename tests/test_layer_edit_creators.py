"""Blackout, touch and deletion creators without a GPU: task grids, bounds and shapes under the reference's
rules, provenance, the refusals raised before anything is written, DeleteTask itself (it only removes
files) and the exports.  tests/test_layer_edit_gpu.py runs the blackout and touch tasks."""
import json
import os

import numpy as np
import pytest


def _layer(tmp_path, size=(512, 512, 128), chunk=(64, 64, 64), dtype="uint8", layer="image", name="vol",
           mips=1, sharded_mip=None, fill=True):
  """a raw layer with `mips` scales (2x2x1 each), every chunk written from the host (no GPU needed)"""
  from igneous_b200 import sharding
  from igneous_b200._compat import CloudVolume
  path = "file://" + str(tmp_path / name)
  info = CloudVolume.create_new_info(1, layer, dtype, "raw", (4, 4, 40), (0, 0, 0), size, chunk)
  vol = CloudVolume(path, info=info)
  for m in range(1, mips):
    vol.add_resolution((4 * 2 ** m, 4 * 2 ** m, 40))
  if sharded_mip is not None:
    s = vol.scales[sharded_mip]
    s["sharding"] = sharding.create_sharded_image_info(s["size"], s["chunk_sizes"][0], "raw", dtype)
  vol.commit_info()
  if fill:
    for m in range(mips):
      if m == sharded_mip:
        continue
      vol.mip = m
      vol[vol.bounds] = np.full(tuple(vol.volume_size) + (1,), 7, dtype=dtype)
  return path


def _files(path):
  """the layer's files, named without their .gz suffix"""
  root = path[len("file://"):]
  names = (os.path.relpath(os.path.join(d, f), root) for d, _, fs in os.walk(root) for f in fs)
  return sorted(n[:-3] if n.endswith(".gz") else n for n in names)


def _provenance(path):
  p = os.path.join(path[len("file://"):], "provenance")
  if not os.path.exists(p):
    return None
  with open(p) as f:
    return json.load(f)


def _offsets(tasks):
  return sorted(tuple(int(v) for v in t.keywords["offset"]) for t in tasks)


def test_exports():
  import igneous_b200
  import igneous_b200.task_creation as tc
  import igneous_b200.tasks as tasks
  for name in ("BlackoutTask", "TouchTask", "DeleteTask"):
    assert name in igneous_b200._TASK_NAMES and getattr(igneous_b200, name) is getattr(tasks, name)
  for name in ("create_blackout_tasks", "create_touch_tasks", "create_deletion_tasks", "compute_rois"):
    assert callable(getattr(tc, name))


@pytest.mark.parametrize("non_aligned", [False, True])
def test_blackout_grid_off_the_chunk_grid(tmp_path, non_aligned):
  import igneous_b200.task_creation as tc
  from igneous_b200._compat import Bbox
  path = _layer(tmp_path, fill=False)
  tasks = tc.create_blackout_tasks(path, Bbox((10, 20, 5), (100, 130, 70)), shape=(64, 64, 64), value=3,
                                   non_aligned_writes=non_aligned)
  if non_aligned:  # the bounds as given: a 2 x 2 x 2 grid from (10, 20, 5)
    assert tasks.bounds == Bbox((10, 20, 5), (100, 130, 70))
    assert _offsets(tasks)[0] == (10, 20, 5) and _offsets(tasks)[-1] == (74, 84, 69) and len(tasks) == 8
  else:  # expanded to whole 64^3 chunks
    assert tasks.bounds == Bbox((0, 0, 0), (128, 192, 128))
    assert len(tasks) == 2 * 3 * 2 and _offsets(tasks)[-1] == (64, 128, 64)
  kw = list(tasks)[0].keywords
  assert kw["value"] == 3 and kw["non_aligned_writes"] == non_aligned and kw["mip"] == 0
  assert list(kw["shape"]) == [64, 64, 64]  # the task clamps, not the creator


def test_blackout_bounds_at_mip0_used_at_mip1(tmp_path):
  import igneous_b200.task_creation as tc
  from igneous_b200._compat import Bbox
  path = _layer(tmp_path, mips=2, fill=False)
  tasks = tc.create_blackout_tasks(path, Bbox((10, 20, 5), (100, 130, 70)), mip=1, shape=(64, 64, 64))
  # (5, 10, 5)-(50, 65, 70) at mip 1, expanded to its 64^3 chunks
  assert tasks.bounds == Bbox((0, 0, 0), (64, 128, 128))
  tasks = tc.create_blackout_tasks(path, Bbox((10, 20, 5), (100, 131, 70)), mip=1, non_aligned_writes=True)
  assert tasks.bounds == Bbox((5, 10, 5), (50, 66, 70))
  # clamped to the mip's bounds
  tasks = tc.create_blackout_tasks(path, Bbox((300, 0, 0), (2000, 64, 64)), mip=1)
  assert tasks.bounds == Bbox((128, 0, 0), (256, 64, 64))


def test_blackout_provenance_is_not_committed(tmp_path):
  """as in the reference: on_finish appends to the volume in memory and writes nothing"""
  import igneous_b200.task_creation as tc
  from igneous_b200._compat import Bbox
  path = _layer(tmp_path, fill=False)
  before = _files(path)
  list(tc.create_blackout_tasks(path, Bbox((0, 0, 0), (64, 64, 64))))
  assert _files(path) == before and _provenance(path) is None


def test_touch_grid_and_provenance(tmp_path):
  import igneous_b200.task_creation as tc
  from igneous_b200._compat import Bbox
  path = _layer(tmp_path, size=(600, 600, 200), fill=False)
  tasks = tc.create_touch_tasks(path, shape=(256, 256, 64))
  assert tasks.bounds == Bbox((0, 0, 0), (600, 600, 200)) and len(tasks) == 3 * 3 * 4
  shapes = {tuple(int(v) for v in t.keywords["offset"]): list(t.keywords["shape"]) for t in tasks}
  assert shapes[(0, 0, 0)] == [256, 256, 64]
  assert shapes[(512, 512, 192)] == [88, 88, 8]  # clamped to the volume's far edge
  prov = _provenance(path)["processing"]
  assert len(prov) == 1 and prov[0]["method"] == {"task": "TouchTask", "mip": 0, "shape": [256, 256, 64],
                                                  "bounds": [[0, 0, 0], [600, 600, 200]]}


def test_touch_bounds_are_read_at_mip0(tmp_path):
  """the reference moves `bounds` from mip 0 to `mip`, its default (the bounds at `mip`) included"""
  import igneous_b200.task_creation as tc
  from igneous_b200._compat import Bbox
  path = _layer(tmp_path, mips=2, fill=False)
  assert tc.create_touch_tasks(path, mip=1).bounds == Bbox((0, 0, 0), (128, 128, 128))
  assert tc.create_touch_tasks(path, mip=1, bounds=Bbox((0, 0, 0), (512, 512, 128))).bounds == \
      Bbox((0, 0, 0), (256, 256, 128))


def test_deletion_shapes_and_provenance(tmp_path):
  import igneous_b200.task_creation as tc
  from igneous_b200._compat import Bbox
  path = _layer(tmp_path, size=(600, 600, 200), mips=2, fill=False)
  tasks = tc.create_deletion_tasks(path, num_mips=2)
  assert list(tasks.shape) == [256, 256, 64] and tasks.bounds == Bbox((0, 0, 0), (600, 600, 200))
  listed = list(tasks)  # provenance is committed once the iterator is exhausted
  shapes = {tuple(int(v) for v in t.keywords["offset"]): list(t.keywords["shape"]) for t in listed}
  assert shapes[(0, 0, 0)] == [256, 256, 64] and shapes[(512, 256, 192)] == [88, 256, 8]
  assert listed[0].keywords["mip"] == 0 and listed[0].keywords["num_mips"] == 2
  assert list(tc.create_deletion_tasks(path, mip=1, num_mips=3).shape) == [512, 512, 64]
  assert list(tc.create_deletion_tasks(path, shape=(100, 100, 100)).shape) == [100, 100, 100]
  listed = list(tc.create_deletion_tasks(path, bounds=Bbox((0, 0, 0), (300, 300, 64)), num_mips=1))
  assert {list(t.keywords["shape"])[0] for t in listed} == {128, 44}
  prov = _provenance(path)["processing"]
  assert [p["method"] for p in prov] == [
    {"task": "DeleteTask", "mip": 0, "num_mips": 2, "shape": [256, 256, 64]},
    {"task": "DeleteTask", "mip": 0, "num_mips": 1, "shape": [128, 128, 64]}]
  assert all(p["by"] is not None and p["date"] for p in prov)


def _round(v, c):
  """the nearest multiple of c, halves to the even multiple (np.round)"""
  q, r = divmod(v, c)
  return c * (q + (1 if 2 * r > c or (2 * r == c and q % 2) else 0))


def test_delete_task_removes_the_rounded_boxes(tmp_path):
  """DeleteTask at mips 0-2: per mip the box is mapped down, rounded to the nearest chunk boundaries and
  clamped, and exactly the chunk files inside it are gone"""
  from igneous_b200._compat import CloudVolume
  from igneous_b200.tasks import DeleteTask
  path = _layer(tmp_path, size=(512, 512, 128), chunk=(32, 32, 32), mips=4)
  vol = CloudVolume(path)
  before = _files(path)
  lo, hi = np.array([40, 70, 0]), np.array([250, 300, 80])
  DeleteTask(path, shape=hi - lo, offset=lo, mip=0, num_mips=2)
  gone = set()
  for m in range(3):
    f = np.array([2 ** m, 2 ** m, 1])
    a = [_round(int(v), 32) for v in lo // f]
    b = [min(_round(int(-(-v // ff)), 32), int(s)) for v, ff, s in zip(hi, f, vol.volume_size_at(m))]
    for z in range(a[2], b[2], 32):
      for y in range(a[1], b[1], 32):
        for x in range(a[0], b[0], 32):
          gone.add("%s/%d-%d_%d-%d_%d-%d" % (vol.key_at(m), x, x + 32, y, y + 32, z, z + 32))
  assert gone and {g.split("/")[0] for g in gone} == {vol.key_at(m) for m in range(3)}
  assert set(before) - set(_files(path)) == gone and set(_files(path)) <= set(before)


def test_round_to_chunk_size():
  from igneous_b200._compat import Bbox
  got = Bbox((16, 47, 48), (80, 96, 97)).round_to_chunk_size((32, 32, 32), offset=(0, 0, 0))
  assert got == Bbox((0, 32, 64), (64, 96, 96))
  assert Bbox((21, 0, 0), (60, 1, 1)).round_to_chunk_size((10, 1, 1), offset=(5, 0, 0)) == Bbox((25, 0, 0), (65, 1, 1))


@pytest.mark.parametrize("dtype,value", [("uint8", 256), ("uint8", -1), ("uint8", 1.5), ("uint16", 70000),
                                         ("uint64", 2 ** 64), ("float32", 1e39)])
def test_blackout_refuses_values_the_dtype_cannot_hold(tmp_path, dtype, value):
  import igneous_b200.task_creation as tc
  from igneous_b200._compat import Bbox
  from igneous_b200.tasks import BlackoutTask
  path = _layer(tmp_path, size=(128, 128, 64), dtype=dtype)
  before = _files(path)
  with pytest.raises(ValueError):
    BlackoutTask(path, 0, (64, 64, 64), (0, 0, 0), value=value)
  with pytest.raises(ValueError):
    tc.create_blackout_tasks(path, Bbox((0, 0, 0), (64, 64, 64)), value=value)
  assert _files(path) == before


def test_blackout_and_delete_refuse_sharded_scales(tmp_path):
  import igneous_b200.task_creation as tc
  from igneous_b200._compat import Bbox
  from igneous_b200.tasks import BlackoutTask, DeleteTask
  path = _layer(tmp_path, size=(256, 256, 64), mips=2, sharded_mip=1)
  before = _files(path)
  with pytest.raises(NotImplementedError):
    BlackoutTask(path, 1, (64, 64, 64), (0, 0, 0))
  with pytest.raises(NotImplementedError):
    tc.create_blackout_tasks(path, Bbox((0, 0, 0), (64, 64, 64)), mip=1)
  with pytest.raises(NotImplementedError):  # mip 0 is not sharded, mip 1 is in range
    DeleteTask(path, (64, 64, 64), (0, 0, 0), mip=0, num_mips=1)
  with pytest.raises(NotImplementedError):
    tc.create_deletion_tasks(path, mip=0, num_mips=1)
  assert _files(path) == before


def test_non_aligned_blackout_without_the_flag_raises_the_storage_error(tmp_path):
  from igneous_b200.tasks import BlackoutTask
  path = _layer(tmp_path, size=(128, 128, 64))
  before = _files(path)
  with pytest.raises(ValueError, match="chunk aligned"):
    BlackoutTask(path, 0, (40, 64, 64), (10, 0, 0), value=1)
  assert _files(path) == before


def test_compute_rois_refuses_signed_layers(tmp_path):
  """an int16 layer with negative voxels: refused before anything is read or written (the threshold kernel
  compares unsigned, so a negative voxel would count as above every threshold)"""
  import igneous_b200.task_creation as tc
  from igneous_b200._compat import CloudVolume
  path = _layer(tmp_path, size=(64, 64, 16), chunk=(32, 32, 16), dtype="int16", fill=False)
  vol = CloudVolume(path)
  vol[vol.bounds] = np.full((64, 64, 16, 1), -3, dtype=np.int16)
  before = _files(path)
  with pytest.raises(NotImplementedError, match="signed"):
    tc.compute_rois(path, suppress_faint_voxels=0)
  assert _files(path) == before and "rois" not in CloudVolume(path).info["scales"][0]
