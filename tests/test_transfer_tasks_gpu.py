"""Transfer tasks end to end on file:// layers: the cases of the reference's test/test_transfer_tasks.py
on random uint8 images with 64^3 source chunks, plus segmentation transfers into
compressed_segmentation layers, each mip checked against the oracle and every stored file against the
one-chunk encoder."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _layer(tmp_path, data, name, chunk=(64, 64, 64), layer="image", encoding="raw", offset=(0, 0, 0)):
  from igneous_b200._compat import CloudVolume
  path = "file://" + str(tmp_path / name)
  vol = CloudVolume(path, info=CloudVolume.create_new_info(data.shape[3], layer, data.dtype, encoding, (1, 1, 1),
                                                           offset, data.shape[:3], chunk))
  vol.commit_info()
  vol[vol.bounds] = data
  return path


def _image(shape, seed=0):
  return np.random.default_rng(seed).integers(0, 256, tuple(shape) + (1,), dtype=np.uint8)


def _run(tasks):
  from igneous_b200._compat import LocalTaskQueue
  LocalTaskQueue(parallel=1).insert_all(tasks)


@pytest.mark.parametrize("size", [(512, 512, 128), (600, 600, 200)])
def test_vanilla(ctx, oracle, tmp_path, size):
  import igneous_b200.task_creation as tc
  from igneous_b200._compat import CloudVolume
  img = _image(size)
  src = _layer(tmp_path, img, "src")
  dest = "file://" + str(tmp_path / "dest")
  _run(tc.create_transfer_tasks(src, dest, shape=(512, 512, 64)))
  cv = CloudVolume(dest)
  assert np.array_equal(cv[cv.bounds], img)
  want = oracle.downsample_with_averaging(img, (2, 2, 1, 1), num_mips=len(cv.available_mips) - 1)
  for m in range(1, len(cv.available_mips)):
    cv.mip = m
    assert np.array_equal(cv[cv.bounds], want[m - 1])


def test_rechunk_five_scales(ctx, oracle, tmp_path):
  import igneous_b200.task_creation as tc
  from igneous_b200._compat import CloudVolume
  img = _image((512, 512, 128), 1)
  src = _layer(tmp_path, img, "src")
  dest = "file://" + str(tmp_path / "dest")
  _run(tc.create_transfer_tasks(src, dest, chunk_size=(50, 50, 50), shape=(800, 800, 50)))
  cv = CloudVolume(dest)
  assert len(cv.available_mips) == 5
  assert list(cv.meta.chunk_size(0)) == [50, 50, 50]
  want = oracle.downsample_with_averaging(img, (2, 2, 1, 1), num_mips=4)
  assert np.array_equal(cv[cv.bounds], img)
  for m in range(1, 5):
    cv.mip = m
    assert np.array_equal(cv[cv.bounds], want[m - 1])


@pytest.mark.parametrize("chunk", [(50, 50, 50), (64, 64, 64)])
def test_skip_downsamples(ctx, tmp_path, chunk):
  """64^3 is the file-copy path: the destination's files are the source's, byte for byte"""
  import igneous_b200.task_creation as tc
  from igneous_b200._compat import CloudVolume, CloudFiles
  img = _image((512, 512, 128), 2)
  src = _layer(tmp_path, img, "src")
  dest = "file://" + str(tmp_path / "dest")
  _run(tc.create_transfer_tasks(src, dest, chunk_size=chunk, skip_downsamples=True, shape=(200, 200, 50)
                                if chunk[0] == 50 else (256, 256, 64)))
  cv = CloudVolume(dest)
  assert len(cv.available_mips) == 1
  assert np.array_equal(cv[cv.bounds], img)
  if chunk == (64, 64, 64):
    a, b = CloudFiles(src), CloudFiles(dest)
    names = [n for n in a.list("1_1_1")]
    assert names and names == b.list("1_1_1")
    assert all(a.get(n) == b.get(n) for n in names)


def test_cropped_off_the_chunk_grid(ctx, tmp_path):
  """a destination cropped to 500^2 at the source's origin: its edge chunks are 52 wide and named by its
  own bounds, so both tasks re-cut them instead of copying the source's 64-wide files"""
  import igneous_b200.task_creation as tc
  from igneous_b200._compat import Bbox, CloudFiles, CloudVolume
  img = _image((512, 512, 128), 7)
  src = _layer(tmp_path, img, "src")
  crop = Bbox((0, 0, 0), (500, 500, 128))
  dest, sh = "file://" + str(tmp_path / "dest"), "file://" + str(tmp_path / "sharded")
  _run(tc.create_transfer_tasks(src, dest, skip_downsamples=True, cutout=True, bounds=crop, shape=(256, 256, 64)))
  _run(tc.create_image_shard_transfer_tasks(src, sh, cutout=True, bounds=crop, memory_target=int(2 ** 23)))
  for path in (dest, sh):
    cv = CloudVolume(path)
    assert list(cv.meta.volume_size(0)) == [500, 500, 128]
    assert np.array_equal(cv[cv.bounds], img[:500, :500])
  names = CloudFiles(dest).list("1_1_1")
  assert "1_1_1/448-500_0-64_0-64" in names and not any("448-512" in n for n in names)


def test_dest_voxel_offset(ctx, tmp_path):
  import igneous_b200.task_creation as tc
  from igneous_b200._compat import CloudVolume
  img = _image((512, 512, 128), 3)
  src = _layer(tmp_path, img, "src")
  dest = "file://" + str(tmp_path / "dest")
  _run(tc.create_transfer_tasks(src, dest, dest_voxel_offset=(100, 100, 100), shape=(512, 512, 64)))
  cv = CloudVolume(dest)
  assert list(cv.bounds.minpt) == [100, 100, 100]
  assert np.array_equal(cv[cv.bounds], img)


def test_subset_translate(ctx, oracle, tmp_path):
  """a 256x256x64 destination at the origin takes the source's [128, 384) x [128, 384) x [64, 128)"""
  import copy
  import igneous_b200.task_creation as tc
  from igneous_b200._compat import CloudVolume
  img = _image((512, 512, 128), 4)
  src = _layer(tmp_path, img, "src")
  dest = "file://" + str(tmp_path / "dest")
  dv = CloudVolume(dest, info=copy.deepcopy(CloudVolume(src).info))
  dv.scales[0]["size"] = [256, 256, 64]
  dv.commit_info()
  _run(tc.create_transfer_tasks(src, dest, chunk_size=(64, 64, 64), translate=(-128, -128, -64)))
  cv = CloudVolume(dest)
  sub = img[128:384, 128:384, 64:128]
  assert len(cv.available_mips) == 3
  assert np.array_equal(cv[cv.bounds], sub)
  want = oracle.downsample_with_averaging(sub, (2, 2, 1, 1), num_mips=2)
  for m in (1, 2):
    cv.mip = m
    assert np.array_equal(cv[cv.bounds], want[m - 1])


def test_image_shard_transfer_and_round_trip(ctx, tmp_path):
  import igneous_b200.task_creation as tc
  from igneous_b200._compat import CloudVolume
  img = _image((600, 600, 200), 5)
  src = _layer(tmp_path, img, "src")
  sh = "file://" + str(tmp_path / "sharded")
  _run(tc.create_image_shard_transfer_tasks(src, sh, memory_target=int(2 ** 23)))
  cv = CloudVolume(sh)
  assert cv.scales[0].get("sharding")
  assert np.array_equal(cv[cv.bounds], img)
  back = "file://" + str(tmp_path / "sharded2")  # sharded -> sharded: the encoded chunks are copied
  _run(tc.create_image_shard_transfer_tasks(sh, back, memory_target=int(2 ** 23)))
  assert np.array_equal(CloudVolume(back)[CloudVolume(back).bounds], img)
  rechunked = "file://" + str(tmp_path / "sharded3")  # rechunked: built on the device
  _run(tc.create_image_shard_transfer_tasks(sh, rechunked, chunk_size=(50, 50, 50), memory_target=int(2 ** 23)))
  assert np.array_equal(CloudVolume(rechunked)[CloudVolume(rechunked).bounds], img)


def test_sharded_jpeg_round_trip(ctx, tmp_path):
  """sharded source -> jpeg -> jpeg: the second transfer reproduces the first's pixels"""
  import igneous_b200.task_creation as tc
  from igneous_b200._compat import CloudVolume
  img = _image((512, 512, 128), 6)
  src = _layer(tmp_path, img, "src")
  sh = "file://" + str(tmp_path / "sharded")
  _run(tc.create_image_shard_transfer_tasks(src, sh, memory_target=int(2 ** 23)))
  j1, j2 = "file://" + str(tmp_path / "j1"), "file://" + str(tmp_path / "j2")
  _run(tc.create_image_shard_transfer_tasks(sh, j1, encoding="jpeg", memory_target=int(2 ** 23)))  # re-encoded
  _run(tc.create_image_shard_transfer_tasks(j1, j2, encoding="jpeg", memory_target=int(2 ** 23)))  # copied
  a, b = CloudVolume(j1), CloudVolume(j2)
  first = a[a.bounds]
  assert np.abs(first.astype(int) - img.astype(int)).mean() < 40
  assert np.array_equal(b[b.bounds], first)


@pytest.mark.parametrize("dtype", [np.uint32, np.uint64])
@pytest.mark.parametrize("block", [(8, 8, 8), (4, 4, 2)])
@pytest.mark.parametrize("nc", [1, 2])
def test_segmentation_to_cseg(ctx, oracle, tmp_path, dtype, block, nc):
  import igneous_b200.task_creation as tc
  from igneous_b200 import codecs
  from igneous_b200._compat import CloudVolume, CloudFiles
  big = 2 ** 33 if dtype == np.uint64 else 2 ** 20
  seg = np.stack([oracle.synth_seg((256, 256, 64), pitch=16, num_ids=64).astype(dtype) + dtype(big + k)
                  for k in range(nc)], axis=3)
  src = _layer(tmp_path, seg, "src", layer="segmentation")
  dest = "file://" + str(tmp_path / "dest")
  tc.create_transfer_tasks(src, dest, shape=(256, 256, 64), encoding="compressed_segmentation")  # writes the info
  cv = CloudVolume(dest)
  for s in cv.scales:
    s["compressed_segmentation_block_size"] = list(block)
  cv.commit_info()
  _run(tc.create_transfer_tasks(src, dest, shape=(256, 256, 64), encoding="compressed_segmentation",
                                truncate_scales=False))
  cv = CloudVolume(dest)
  assert np.array_equal(cv[cv.bounds], seg)
  want = oracle.downsample_segmentation(seg, (2, 2, 1, 1), num_mips=len(cv.available_mips) - 1)
  cf = CloudFiles(dest)
  for m in range(len(cv.available_mips)):
    cv.mip = m
    vol = cv[cv.bounds]
    if m:
      assert np.array_equal(vol, want[m - 1])
    for c in cv._chunks(m, cv.bounds):
      rel = c - cv.bounds.minpt
      assert cf.get(cv._chunk_name(m, c)) == codecs.cseg_encode(vol[rel.to_slices()], cv._cseg_block(m))
