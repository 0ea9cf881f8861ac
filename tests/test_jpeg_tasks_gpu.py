"""Image tasks on `jpeg` layers: each run on a jpeg layer and on a raw layer holding the jpeg layer's
decoded pixels.  Every jpeg output chunk must be the jpeg round trip of the raw output chunk."""
import copy

import numpy as np
import pytest

from igneous_b200 import codecs

pytestmark = pytest.mark.gpu


def em_like(shape, seed):
  rng = np.random.default_rng(seed)
  sx, sy, sz = shape
  x = np.arange(sx)[:, None, None] / 11.0
  y = np.arange(sy)[None, :, None] / 8.0
  z = np.arange(sz)[None, None, :] / 4.0
  v = 130 + 50 * np.sin(x + 0.4 * z) * np.cos(y - 0.2 * z) - 70 * (np.abs(np.sin(0.6 * x + 0.5 * y)) < 0.1)
  return (v + rng.normal(0, 10, shape)).clip(0, 255).astype(np.uint8)[..., None]


def pair(tmp_path, img, chunk, offset=(0, 0, 0)):
  """(jpeg layer path, raw layer path holding the jpeg layer's decoded pixels)"""
  from igneous_b200._compat import CloudVolume
  jp = "file://" + str(tmp_path / "jpeg")
  rp = "file://" + str(tmp_path / "raw")
  CloudVolume.from_numpy(img, vol_path=jp, resolution=(4, 4, 40), voxel_offset=offset, chunk_size=chunk,
                         layer_type="image", encoding="jpeg")
  jv = CloudVolume(jp)
  assert jv.scales[0]["encoding"] == "jpeg"
  decoded = jv[jv.bounds]
  assert decoded.shape == img.shape and np.abs(decoded.astype(int) - img).mean() < 8
  CloudVolume.from_numpy(decoded, vol_path=rp, resolution=(4, 4, 40), voxel_offset=offset, chunk_size=chunk,
                         layer_type="image")
  return jp, rp


def assert_round_trips(jpeg_path, raw_path, mip):
  from igneous_b200._compat import CloudVolume
  jv, rv = CloudVolume(jpeg_path, mip=mip), CloudVolume(raw_path, mip=mip)
  assert jv.scales[mip]["encoding"] == "jpeg" and rv.scales[mip]["encoding"] == "raw"
  quality = int(jv.scales[mip].get("jpeg_quality", 85))
  got, raw = jv[jv.bounds], rv[rv.bounds]
  n = 0
  for c in rv._chunks(mip, rv.bounds):
    sl = tuple(slice(int(a - o), int(b - o)) for a, b, o in zip(c.minpt, c.maxpt, rv.bounds.minpt))
    block = np.asfortranarray(raw[sl])
    want = codecs.jpeg_decode(codecs.jpeg_encode(block, quality), block.shape)
    assert np.array_equal(got[sl], want), (mip, c)
    n += 1
  assert n > 0


def test_downsampling_tasks_on_a_jpeg_layer(ctx, tmp_path):
  from igneous_b200 import task_creation as tc
  from igneous_b200._compat import CloudVolume, LocalTaskQueue
  img = em_like((256, 192, 16), 1)
  jp, rp = pair(tmp_path, img, (64, 64, 8), offset=(8, 16, 0))
  LocalTaskQueue(parallel=1).insert_all(tc.create_downsampling_tasks(jp, mip=0, num_mips=2, encoding="jpeg"))
  LocalTaskQueue(parallel=1).insert_all(tc.create_downsampling_tasks(rp, mip=0, num_mips=2))
  mips = len(CloudVolume(rp).available_mips)
  assert mips >= 2 and len(CloudVolume(jp).available_mips) == mips
  for m in range(1, mips):
    assert_round_trips(jp, rp, m)


def copy_layer(tmp_path, src, name):
  """An empty layer with src's info and its downsample scales."""
  from igneous_b200 import downsample_scales
  from igneous_b200._compat import CloudVolume
  path = "file://" + str(tmp_path / name)
  CloudVolume(path, info=copy.deepcopy(CloudVolume(src).info)).commit_info()
  downsample_scales.create_downsample_scales(path, 0, CloudVolume(path).meta.volume_size(0), preserve_chunk_size=True)
  return path


def test_transfer_task_jpeg_to_jpeg(ctx, tmp_path):
  from igneous_b200 import tasks
  from igneous_b200._compat import CloudVolume
  img = em_like((128, 128, 8), 2)
  jp, rp = pair(tmp_path, img, (64, 64, 8))
  dj, dr = copy_layer(tmp_path, jp, "tj"), copy_layer(tmp_path, rp, "tr")
  tasks.TransferTask(jp, dj, 0, (128, 128, 8), (0, 0, 0))
  tasks.TransferTask(rp, dr, 0, (128, 128, 8), (0, 0, 0))
  mips = len(CloudVolume(dr).available_mips)
  assert mips >= 2
  for m in range(mips):
    assert_round_trips(dj, dr, m)


def test_clahe_task_jpeg_to_jpeg(ctx, tmp_path):
  from igneous_b200 import tasks
  img = em_like((160, 128, 4), 3)
  jp, rp = pair(tmp_path, img, (32, 32, 4))
  dests = []
  for src, name in ((jp, "cj"), (rp, "cr")):
    dests.append(copy_layer(tmp_path, src, name))
    tasks.CLAHETask(src, dests[-1], 0, False, (128, 128, 4), (32, 0, 0), clip_limit=40.0, tile_grid_size=(8, 8))
  from igneous_b200._compat import CloudVolume as CV
  jv, rv = CV(dests[0]), CV(dests[1])
  box = (slice(32, 160), slice(0, 128), slice(0, 4))
  got, raw = jv[box], rv[box]
  for x in range(32, 160, 32):
    for y in range(0, 128, 32):
      block = np.asfortranarray(raw[x - 32:x, y:y + 32])
      want = codecs.jpeg_decode(codecs.jpeg_encode(block), block.shape)
      assert np.array_equal(got[x - 32:x, y:y + 32], want), (x, y)


def test_image_shard_downsample_jpeg(ctx, tmp_path):
  from igneous_b200 import task_creation as tc
  from igneous_b200._compat import LocalTaskQueue
  img = em_like((128, 128, 16), 4)
  jp, rp = pair(tmp_path, img, (32, 32, 16))
  LocalTaskQueue(parallel=1).insert_all(tc.create_image_shard_downsample_tasks(jp, mip=0, num_mips=1, encoding="jpeg"))
  LocalTaskQueue(parallel=1).insert_all(tc.create_image_shard_downsample_tasks(rp, mip=0, num_mips=1))
  assert_round_trips(jp, rp, 1)


def test_image_shard_downsample_jpeg_png_top_is_refused(ctx, tmp_path):
  from igneous_b200 import task_creation as tc
  from igneous_b200._compat import LocalTaskQueue
  jp, _ = pair(tmp_path, em_like((128, 128, 16), 5), (32, 32, 16))
  with pytest.raises(NotImplementedError, match="png"):
    LocalTaskQueue(parallel=1).insert_all(tc.create_image_shard_downsample_tasks(jp, mip=0, num_mips=2, encoding="jpeg"))
