"""LuminanceLevelsTask, ContrastNormalizationTask, CLAHETask and QuantizeTask end to end on
file:// layers, checked against numpy, tests/contrastref.py and the averaging pyramid."""
import copy
import json
import random

import numpy as np
import pytest

import contrastref as R

pytestmark = pytest.mark.gpu


def _layer(tmp_path, data, name, chunk, layer_type="image"):
  from igneous_b200._compat import CloudVolume
  path = "file://" + str(tmp_path / name)
  CloudVolume.from_numpy(data, vol_path=path, resolution=(4, 4, 40), chunk_size=chunk, layer_type=layer_type)
  return path


def _empty_like(tmp_path, src, name, **changes):
  from igneous_b200 import downsample_scales
  from igneous_b200._compat import CloudVolume
  info = copy.deepcopy(CloudVolume(src).info)
  info.update(changes)
  path = "file://" + str(tmp_path / name)
  CloudVolume(path, info=info).commit_info()
  shape = CloudVolume(path).meta.volume_size(0)
  downsample_scales.create_downsample_scales(path, 0, shape, preserve_chunk_size=True)
  return path


def test_levels_then_contrast_normalization(tmp_path):
  from igneous_b200 import tasks, tinybrain
  from igneous_b200._compat import CloudFiles, CloudVolume
  rng = np.random.default_rng(4)
  shape = (256, 192, 4)
  img = rng.normal(90, 25, size=shape + (1,)).clip(0, 255).astype(np.uint8)
  img[:40, :, 1] = 0
  img[:, :, 3] = 200  # one level only: lower == upper, the slice keeps its values
  src = _layer(tmp_path, img, "src", (64, 64, 4))
  random.seed(7)
  for z in range(shape[2]):
    tasks.LuminanceLevelsTask(src, None, (256, 192, 1), (0, 0, z), 1.0, 0).execute()
  cf = CloudFiles(src)
  for z in range(shape[2]):
    got = json.loads(cf.get("levels/0/%d" % z).decode("utf8"))
    assert got["levels"] == np.bincount(img[:, :, z].ravel(), minlength=256).tolist()
    assert got["num_patches"] == 1 and got["patch_size"] == [256, 192, 1]
  dest = _empty_like(tmp_path, src, "dest")
  task = tasks.ContrastNormalizationTask(src, dest, None, shape, (0, 0, 0), 0, 0.01, False, (0, 0, 0), None, None)
  task.execute()
  levels = task.fetch_z_levels(CloudVolume(src).meta.bounds(0))
  bounds = [R.clamping_values(lv, 0.01, 0.99) for lv in levels]
  want0 = R.stretch(img, bounds, 255, 0, 255, np.uint8)
  cv = CloudVolume(dest)
  assert np.array_equal(cv[cv.meta.bounds(0)], want0)
  mips = tinybrain.downsample_with_averaging(want0, (2, 2, 1), num_mips=len(cv.available_mips) - 1)
  assert len(mips) >= 1
  for m, want in enumerate(mips, start=1):
    cv.mip = m
    assert np.array_equal(cv[cv.meta.bounds(m)], want), m
  with pytest.raises(Exception, match="were not defined"):
    tasks.ContrastNormalizationTask(src, dest, "file://" + str(tmp_path / "nowhere"), shape, (0, 0, 0), 0, 0.01, False,
                                    (0, 0, 0), None, None).execute()


def test_clahe_task_at_dataset_edge(tmp_path):
  from igneous_b200 import tasks
  from igneous_b200._compat import CloudVolume
  rng = np.random.default_rng(8)
  img = rng.normal(110, 30, size=(300, 200, 2, 1)).clip(0, 255).astype(np.uint8)
  src = _layer(tmp_path, img, "src", (8, 8, 2))
  dest = _empty_like(tmp_path, src, "dest")
  tasks.CLAHETask(src, dest, 0, False, (256, 256, 2), (128, 128, 0), clip_limit=40.0, tile_grid_size=(8, 8))
  # the box (128..300, 128..200) enlarged by 8 voxels and clamped: (120..300, 120..200)
  want = R.clahe_stack(img[120:300, 120:200, :, 0], 40.0, (8, 8))[8:, 8:]
  cv = CloudVolume(dest)
  assert np.array_equal(cv[128:300, 128:200, 0:2][..., 0], want)


def test_quantize_task(tmp_path):
  from igneous_b200 import tasks, tinybrain
  from igneous_b200._compat import CloudVolume
  rng = np.random.default_rng(9)
  aff = rng.random((128, 128, 4, 3), dtype=np.float32)
  src = _layer(tmp_path, aff, "aff", (64, 64, 4))
  dest = _empty_like(tmp_path, src, "q", num_channels=1, data_type="uint8")
  tasks.QuantizeTask(src, dest, (128, 128, 4), (0, 0, 0), 0)
  want0 = (aff[..., :1] * 255.0).astype(np.uint8)
  cv = CloudVolume(dest)
  assert np.array_equal(cv[cv.meta.bounds(0)], want0)
  cv.mip = 1
  assert np.array_equal(cv[cv.meta.bounds(1)], tinybrain.downsample_with_averaging(want0, (2, 2, 1), num_mips=1)[0])


def test_levels_sampled_patches_follow_seeded_random(tmp_path):
  """A slice larger than one 2048 x 2048 patch in x and y, sampled at coverage 0.5: the levels
  file holds the histogram of exactly the patches a seeded `random` picks, clamped to the dataset
  (the patch at x = 4096 is 204 voxels wide)."""
  import math
  from igneous_b200 import tasks
  from igneous_b200._compat import CloudFiles
  rng = np.random.default_rng(10)
  img = rng.integers(0, 256, size=(4300, 2300, 1, 1), dtype=np.int64).astype(np.uint8)
  src = _layer(tmp_path, img, "big", (1024, 1024, 1))
  shape = (4300, 2300, 1)
  random.seed(24)
  tasks.LuminanceLevelsTask(src, None, shape, (0, 0, 0), 0.5, 0).execute()
  # replay the draws.  The number of patch indices comes from the area, ceil(4300 * 2300 / 2048^2) = 3,
  # not from the 3 x 2 grid, so (as in the reference) only the first row of patches is ever sampled;
  # ceil(3 * 0.5) = 2 of them are picked
  total = math.ceil(4300 * 2300 / 2048 ** 2)
  n = math.ceil(total * 0.5)
  assert (total, n) == (3, 2)
  random.seed(24)
  picked = set()
  while len(picked) < n:
    picked.add(random.randint(0, total - 1))
  want = np.zeros(256, np.uint64)
  area, biggest = 0, (0, None)
  for i in picked:
    x0, y0 = (i % 3) * 2048, (i // 3) * 2048
    patch = img[x0:min(x0 + 2048, 4300), y0:min(y0 + 2048, 2300), 0, 0]
    want += np.bincount(patch.ravel(), minlength=256).astype(np.uint64)
    area += patch.size
  got = json.loads(CloudFiles(src).get("levels/0/0").decode("utf8"))
  assert got["levels"] == want.tolist()
  assert got["num_patches"] == 2
  assert 2 in picked  # seed 24 draws the edge patch, clamped to x = 4096..4300
  assert got["coverage_ratio"] == area / (4300 * 2300)
  assert math.prod(got["patch_size"]) == max(
    min(2048, 4300 - (i % 3) * 2048) * min(2048, 2300 - (i // 3) * 2048) for i in picked)
