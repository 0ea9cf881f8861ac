"""The contrast / CLAHE / quantize task creators and LuminanceLevelsTask's patch selection on the
file:// stand-in: task counts, offsets and shapes, the extra z task of the levels iterator, the
destination info and provenance.  Nothing here runs a kernel."""
import math
import random

import numpy as np
import pytest

from igneous_b200 import task_creation as tc
from igneous_b200 import tasks
from igneous_b200._compat import Bbox, CloudFiles, CloudVolume


def _layer(tmp_path, shape, dtype, chunk, offset=(0, 0, 0), channels=1, name="src"):
  path = "file://" + str(tmp_path / name)
  CloudVolume.from_numpy(np.zeros(tuple(shape) + (channels,), dtype=dtype), vol_path=path, resolution=(4, 4, 40),
                         voxel_offset=offset, chunk_size=chunk, layer_type="image")
  return path


def _kw(t):
  return t.keywords if hasattr(t, "keywords") else None


# ------------------------------------------------------------- levels creator
def test_luminance_levels_tasks_inclusive_z(tmp_path):
  src = _layer(tmp_path, (300, 200, 5), np.uint8, (64, 64, 5), offset=(10, 20, 3))
  itr = tc.create_luminance_levels_tasks(src, coverage_factor=0.25)
  assert len(itr) == 5
  got = list(itr)
  assert len(got) == 6  # range(minpt.z, maxpt.z + 1)
  assert all(isinstance(t, tasks.LuminanceLevelsTask) for t in got)
  assert [int(t.offset.z) for t in got] == list(range(3, 9))
  assert all(list(map(int, t.offset[:2])) == [10, 20] for t in got)
  assert all(list(map(int, t.shape)) == [300, 200, 1] for t in got)
  assert all(t.coverage_factor == 0.25 and t.mip == 0 and t.levels_path is None for t in got)
  # the last task's box clamps to nothing in z: it writes no levels file (and runs no kernel)
  random.seed(1)
  got[-1].execute()
  assert not CloudFiles(src).exists("levels/0/8")
  assert CloudVolume(src).provenance.processing[-1]["method"]["task"] == "LuminanceLevelsTask"


def test_luminance_levels_tasks_bounds(tmp_path):
  src = _layer(tmp_path, (300, 200, 6), np.uint16, (64, 64, 3))
  got = list(tc.create_luminance_levels_tasks(src, levels_path=src, bounds=Bbox((0, 64, 2), (128, 200, 4))))
  assert [int(t.offset.z) for t in got] == [2, 3, 4]
  assert all(list(map(int, t.shape)) == [128, 136, 1] and list(map(int, t.offset[:2])) == [0, 64] for t in got)


# ----------------------------------------------------------- patch selection
def _replay_selection(seed, shape, offset, coverage, dataset):
  """The sampling rule written out: N distinct patch indices drawn with random.randint on a
  2048 x 2048 grid over the task's (x, y) extent, in draw order of a set, clamped to the
  dataset and dropped when empty."""
  random.seed(seed)
  total = int(math.ceil(shape[0] * shape[1] * shape[2] / (2048 * 2048)))
  n = int(math.ceil(total * coverage))
  picked = set()
  while len(picked) < n:
    picked.add(random.randint(0, total - 1))
  gridx = int(math.ceil(shape[0] / 2048))
  boxes = []
  for i in picked:
    lo = np.array([(i % gridx) * 2048, (i // gridx) * 2048, 0]) + np.array(offset)
    hi = lo + np.array([2048, 2048, 1])
    lo, hi = np.clip(lo, dataset[0], dataset[1]), np.clip(hi, dataset[0], dataset[1])
    if np.all(hi > lo):
      boxes.append((lo.tolist(), hi.tolist()))
  return boxes


@pytest.mark.parametrize("dataset_max", [(4300, 4200, 10), (4196, 4200, 10)])
@pytest.mark.parametrize("seed", [0, 7, 12345])
def test_levels_patch_selection_replays_seeded_random(seed, dataset_max):
  shape, offset, coverage = (5000, 4500, 1), (100, 50, 7), 0.5
  dataset = ((0, 0, 0), dataset_max)
  t = tasks.LuminanceLevelsTask("file:///nowhere", None, shape, offset, coverage, 0)
  random.seed(seed)
  got = [(list(map(int, b.minpt)), list(map(int, b.maxpt))) for b in t.select_bounding_boxes(Bbox(*dataset))]
  want = _replay_selection(seed, shape, offset, coverage, dataset)
  assert got == want
  assert len(want) <= 3
  # patches in the third column start at x = 4196: clamped short by the first dataset, dropped by the second
  xs = [b[0][0] for b in got]
  if dataset_max[0] == 4196:
    assert 4196 not in xs
  else:
    assert all(b[1][0] == 4300 for b in got if b[0][0] == 4196)


def test_levels_patch_selection_draws_until_distinct():
  # 6 patches at coverage 1: every index once, however many draws repeat
  t = tasks.LuminanceLevelsTask("file:///nowhere", None, (5000, 4500, 1), (0, 0, 0), 1.0, 0)
  random.seed(3)
  boxes = t.select_bounding_boxes(Bbox((0, 0, 0), (10000, 10000, 1)))
  assert sorted((int(b.minpt.x), int(b.minpt.y)) for b in boxes) == \
      [(x, y) for x in (0, 2048, 4096) for y in (0, 2048)] and len(boxes) == 6


# ------------------------------------------------- contrast normalization creator
def test_contrast_normalization_tasks(tmp_path):
  src = _layer(tmp_path, (300, 200, 10), np.uint8, (64, 64, 5))
  dest = "file://" + str(tmp_path / "dest")
  itr = tc.create_contrast_normalization_tasks(src, dest, clip_fraction=(0.01, 0.02), minval=3, maxval=250,
                                               translate=(0, 0, 0))
  got = list(itr)
  assert len(itr) == 2 and len(got) == 2
  assert all(isinstance(t, tasks.ContrastNormalizationTask) for t in got)
  # (2048, 2048, chunk z) shrunk to whole chunks, clamped to the bounds
  assert all(list(map(int, t.shape)) == [300, 200, 5] for t in got)
  assert [list(map(int, t.offset)) for t in got] == [[0, 0, 0], [0, 0, 5]]
  t = got[0]
  assert (t.lower_clip_fraction, t.upper_clip_fraction, t.minval, t.maxval) == (0.01, 0.02, 3, 250)
  assert t.levels_path == src and t.src_path == src and t.dest_path == dest
  dv = CloudVolume(dest)
  sv = CloudVolume(src)
  assert dv.info["data_type"] == "uint8" and dv.info["num_channels"] == 1
  assert dv.scales[0] == sv.scales[0]
  assert len(dv.available_mips) > 1  # downsample scales of the task shape
  assert all(s["chunk_sizes"] == [[64, 64, 5]] for s in dv.scales)
  assert dv.provenance.processing[-1]["method"]["task"] == "ContrastNormalizationTask"
  assert dv.provenance.processing[-1]["method"]["bounds"] == [[0, 0, 0], [300, 200, 10]]


def test_contrast_normalization_tasks_keep_existing_dest(tmp_path):
  src = _layer(tmp_path, (300, 200, 10), np.uint8, (64, 64, 5))
  dest = _layer(tmp_path, (300, 200, 10), np.uint16, (32, 32, 10), name="dest")
  got = list(tc.create_contrast_normalization_tasks(src, dest, shape=(128, 128, 10)))
  assert len(got) == 3 * 2
  assert sorted({(int(t.offset.x), int(t.offset.y)) for t in got}) == \
      [(x, y) for x in (0, 128, 256) for y in (0, 128)]
  assert CloudVolume(dest).info["data_type"] == "uint16"


def test_default_task_shape_shrinks_to_chunks(tmp_path):
  src = _layer(tmp_path, (3000, 2100, 8), np.uint8, (600, 700, 4))
  dest = "file://" + str(tmp_path / "dest")
  got = list(tc.create_clahe_tasks(src, dest))
  # 2048 shrinks to whole chunks: 1800 (3 x 600) in x, 1400 (2 x 700) in y
  assert all(list(map(int, t.keywords["shape"])) == [1800, 1400, 4] for t in got)
  assert len(got) == 2 * 2 * 2


# ---------------------------------------------------------------- CLAHE creator
def test_clahe_tasks(tmp_path):
  src = _layer(tmp_path, (300, 200, 6), np.uint16, (64, 64, 3))
  dest = "file://" + str(tmp_path / "dest")
  got = list(tc.create_clahe_tasks(src, dest, clip_limit=2.5, tile_grid_size=(4, 6), fill_missing=True))
  assert len(got) == 2
  kw = [_kw(t) for t in got]
  assert all(t.func is tasks.CLAHETask for t in got)
  assert [list(map(int, k["offset"])) for k in kw] == [[0, 0, 0], [0, 0, 3]]
  assert all(list(map(int, k["shape"])) == [300, 200, 3] for k in kw)
  assert all(k["clip_limit"] == 2.5 and k["tile_grid_size"] == (4, 6) and k["fill_missing"] for k in kw)
  dv = CloudVolume(dest)
  assert dv.info["data_type"] == "uint16" and dv.scales[0] == CloudVolume(src).scales[0]
  assert dv.provenance.processing[-1]["method"]["task"] == "CLAHETask"


# ------------------------------------------------------------- quantize creator
def test_quantized_affinity_info(tmp_path):
  src = _layer(tmp_path, (256, 256, 16), np.float32, (64, 64, 16), channels=3)
  info = tc.create_quantized_affinity_info(src, None, (128, 128, 16), 0, (32, 32, 8), "raw")
  assert info["num_channels"] == 1 and info["data_type"] == "uint8" and info["type"] == "image"
  assert len(info["scales"]) == 1
  assert info["scales"][0]["chunk_sizes"] == [[32, 32, 8]] and info["scales"][0]["encoding"] == "raw"


def test_quantize_tasks(tmp_path):
  src = _layer(tmp_path, (256, 256, 16), np.float32, (64, 64, 16), channels=3)
  dest = "file://" + str(tmp_path / "q")
  itr = tc.create_quantize_tasks(src, dest, shape=(128, 128, 16), chunk_size=(32, 32, 8))
  got = list(itr)
  assert len(got) == 4 and all(t.func is tasks.QuantizeTask for t in got)
  kw = [_kw(t) for t in got]
  assert sorted(tuple(k["offset"]) for k in kw) == [(0, 0, 0), (0, 128, 0), (128, 0, 0), (128, 128, 0)]
  assert all(k["shape"] == [128, 128, 16] and isinstance(k["shape"][0], int) for k in kw)
  assert all(k["source_layer_path"] == src and k["dest_layer_path"] == dest and k["mip"] == 0 for k in kw)
  dv = CloudVolume(dest)
  assert dv.info["data_type"] == "uint8" and dv.info["num_channels"] == 1
  assert len(dv.available_mips) > 1 and all(s["chunk_sizes"] == [[32, 32, 8]] for s in dv.scales)
  assert dv.provenance.processing[-1]["method"]["task"] == "QuantizeTask"


def test_quantize_tasks_bounds_expand_to_chunks(tmp_path):
  src = _layer(tmp_path, (256, 256, 16), np.float32, (64, 64, 16), channels=3)
  dest = "file://" + str(tmp_path / "q")
  got = list(tc.create_quantize_tasks(src, dest, shape=(64, 64, 16), chunk_size=(32, 32, 8),
                                      bounds=Bbox((40, 10, 0), (100, 70, 16))))
  # (40..100, 10..70) snapped to 32-voxel chunks: (32..128, 0..96) -> 2 x 2 tasks of 64
  assert sorted(tuple(t.keywords["offset"]) for t in got) == [(32, 0, 0), (32, 64, 0), (96, 0, 0), (96, 64, 0)]
