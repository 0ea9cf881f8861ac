"""create_transfer_tasks / create_image_shard_transfer_tasks without a GPU: info edits, task grids,
task shapes from memory_target, shard specs, provenance and the refusals raised before anything is
written.  The tasks themselves are only built, never run (tests/test_transfer_tasks_gpu.py runs them)."""
import json
import os

import numpy as np
import pytest


def _src(tmp_path, size=(512, 512, 128), chunk=(64, 64, 64), dtype="uint8", layer="image", offset=(0, 0, 0),
         encoding="raw", name="src"):
  from igneous_b200._compat import CloudVolume
  path = "file://" + str(tmp_path / name)
  info = CloudVolume.create_new_info(1, layer, dtype, encoding, (4, 4, 40), offset, size, chunk)
  info["mesh"] = "mesh"
  info["skeletons"] = "skeletons"
  CloudVolume(path, info=info).commit_info()
  return path


def _info(path):
  with open(os.path.join(path[len("file://"):], "info")) as f:
    return json.load(f)


def _kwargs(task):
  return task.keywords


def test_memory_target_shape_known_answer():
  """the reference docstring's example: uint64, 128x128x64 chunks, 3 GB, (2,2,1) -> 2048x2048x64"""
  from igneous_b200.downsample_scales import downsample_shape_from_memory_target as f
  assert list(f(8, 128, 128, 64, (2, 2, 1), 3e9)) == [2048, 2048, 64]
  # one mip more would need 4/3 * 8 * 4096^2 * 64 bytes = 11.5 GB
  assert list(f(8, 128, 128, 64, (2, 2, 1), 11.4e9)) == [2048, 2048, 64]
  assert list(f(8, 128, 128, 64, (2, 2, 1), 11.5e9)) == [4096, 4096, 64]
  assert list(f(8, 128, 128, 64, (2, 2, 1), 3e9, max_mips=2)) == [512, 512, 64]
  # non-square chunks: every axis has its own doubling count
  assert list(f(1, 256, 128, 64, (2, 2, 1), 3.5e9)) == [8192, 2048, 64]
  assert list(f(4, 128, 128, 64, (2, 2, 2), 3.5e9)) == [1024, 1024, 256]
  assert list(f(1, 128, 128, 64, (2, 2, 2), 3.5e9)) == [2048, 2048, 512]
  assert list(f(1, 64, 64, 64, (1, 1, 1), 64 ** 3 * 9)) == [192, 192, 64]
  for bad in ((1, 64, 64, 64, (2, 2, 1), 0), (1, 0, 64, 64, (2, 2, 1), 1e9), (8, 128, 128, 64, (2, 2, 1), 1e6),
              (1, 64, 64, 64, (2, 1, 1), 1e9)):
    with pytest.raises(ValueError):
      f(*bad)


def test_vanilla_grid_and_info(tmp_path):
  import igneous_b200.task_creation as tc
  src = _src(tmp_path)
  dest = "file://" + str(tmp_path / "dest")
  tasks = tc.create_transfer_tasks(src, dest, shape=(256, 256, 64))
  assert len(tasks) == 2 * 2 * 2
  info = _info(dest)
  assert [s["size"] for s in info["scales"]][:2] == [[512, 512, 128], [256, 256, 128]]
  assert info["scales"][0]["chunk_sizes"] == [[64, 64, 64]]
  assert info["mesh"] == "mesh"
  kw = _kwargs(list(tasks)[0])
  assert kw["compress"] == "gzip" and list(kw["translate"]) == [0, 0, 0] and kw["factor"] == (2, 2, 1)
  offsets = sorted(tuple(int(v) for v in _kwargs(t)["offset"]) for t in tasks)
  assert offsets[0] == (0, 0, 0) and offsets[-1] == (256, 256, 64)


def test_memory_target_sets_the_shape(tmp_path):
  import igneous_b200.task_creation as tc
  src = _src(tmp_path, size=(4096, 4096, 128), chunk=(128, 128, 64), dtype="uint64", layer="segmentation")
  dest = "file://" + str(tmp_path / "dest")
  tasks = tc.create_transfer_tasks(src, dest, memory_target=int(3e9))
  assert list(tasks.shape) == [2048, 2048, 64]
  assert len(tasks) == 2 * 2 * 2


def test_rechunk_encoding_and_level(tmp_path):
  import igneous_b200.task_creation as tc
  src = _src(tmp_path)
  dest = "file://" + str(tmp_path / "dest")
  tasks = tc.create_transfer_tasks(src, dest, chunk_size=(50, 50, 50), shape=(200, 200, 50), encoding="jpeg",
                                   encoding_level=70)
  info = _info(dest)
  assert info["scales"][0]["chunk_sizes"] == [[50, 50, 50]]
  assert info["scales"][0]["encoding"] == "jpeg" and info["scales"][0]["jpeg_quality"] == 70
  assert all(s["encoding"] == "jpeg" for s in info["scales"])
  assert _kwargs(list(tasks)[0])["compress"] is False  # jpeg is stored without gzip


def test_dest_voxel_offset_and_translate(tmp_path):
  import igneous_b200.task_creation as tc
  src = _src(tmp_path)
  dest = "file://" + str(tmp_path / "dest")
  tasks = tc.create_transfer_tasks(src, dest, shape=(512, 512, 64), dest_voxel_offset=(100, 100, 100))
  info = _info(dest)
  assert info["scales"][0]["voxel_offset"] == [100, 100, 100]
  assert list(_kwargs(list(tasks)[0])["translate"]) == [100, 100, 100]
  assert tasks.bounds.minpt.tolist() == [100, 100, 100]


def test_skip_downsamples_truncate_and_clean_info(tmp_path):
  import igneous_b200.task_creation as tc
  from igneous_b200 import downsample_scales
  src = _src(tmp_path)
  downsample_scales.create_downsample_scales(src, 0, (512, 512, 64), preserve_chunk_size=True)
  dest = "file://" + str(tmp_path / "dest")
  tasks = tc.create_transfer_tasks(src, dest, shape=(256, 256, 64), skip_downsamples=True, clean_info=True)
  info = _info(dest)
  assert len(info["scales"]) == 1
  assert "mesh" not in info and "skeletons" not in info
  assert _kwargs(list(tasks)[0])["factor"] == (1, 1, 1)
  dest2 = "file://" + str(tmp_path / "dest2")
  tc.create_transfer_tasks(src, dest2, shape=(256, 256, 64), skip_downsamples=True, truncate_scales=False)
  assert len(_info(dest2)["scales"]) == len(_info(src)["scales"])


def test_cutout_bounds(tmp_path):
  import igneous_b200.task_creation as tc
  from igneous_b200._compat import Bbox
  src = _src(tmp_path)
  dest = "file://" + str(tmp_path / "dest")
  tasks = tc.create_transfer_tasks(src, dest, shape=(128, 128, 64), cutout=True,
                                   bounds=Bbox((128, 128, 64), (384, 384, 128)), translate=(0, 0, 0))
  info = _info(dest)
  assert info["scales"][0]["voxel_offset"] == [128, 128, 64]
  assert info["scales"][0]["size"] == [256, 256, 64]
  assert tasks.bounds.minpt.tolist() == [128, 128, 64] and tasks.bounds.maxpt.tolist() == [384, 384, 128]
  assert len(tasks) == 4


def test_provenance(tmp_path):
  import igneous_b200.task_creation as tc
  from igneous_b200._compat import CloudVolume
  src = _src(tmp_path)
  dest = "file://" + str(tmp_path / "dest")
  tasks = tc.create_transfer_tasks(src, dest, shape=(512, 512, 128))
  tasks.on_finish()
  for p in (dest, src):
    job = CloudVolume(p).provenance.processing[-1]["method"]
    assert job["task"] == "TransferTask" and job["src"] == src and job["dest"] == dest
  tasks = tc.create_transfer_tasks(src, dest + "2", shape=(512, 512, 128), no_src_update=True)
  n = len(CloudVolume(src).provenance.processing)
  tasks.on_finish()
  assert len(CloudVolume(src).provenance.processing) == n


def test_image_shard_transfer_spec_and_grid(tmp_path):
  import igneous_b200.task_creation as tc
  from igneous_b200 import sharding, shards
  from igneous_b200._compat import CloudVolume
  src = _src(tmp_path, size=(512, 512, 128))
  dest = "file://" + str(tmp_path / "dest")
  tasks = tc.create_image_shard_transfer_tasks(src, dest, memory_target=int(2 ** 22))
  info = _info(dest)
  spec = info["scales"][0]["sharding"]
  want = sharding.create_sharded_image_info(dataset_size=[512, 512, 128], chunk_size=[64, 64, 64], encoding="raw",
                                            dtype="uint8", uncompressed_shard_bytesize=int(2 ** 22),
                                            data_encoding="gzip")
  assert spec == json.loads(json.dumps(want))
  shape = shards.image_shard_shape_from_spec(spec, [512, 512, 128], [64, 64, 64])
  assert list(tasks.shape) == list(shape)
  assert len(tasks) == int(np.prod(np.ceil(np.array([512, 512, 128]) / np.array(shape))))
  assert _kwargs(list(tasks)[0])["mip"] == 0
  tasks.on_finish()
  assert CloudVolume(dest).provenance.processing[-1]["method"]["task"] == "ImageShardTransferTask"
  jp = "file://" + str(tmp_path / "jp")
  tc.create_image_shard_transfer_tasks(src, jp, encoding="jpeg")
  assert _info(jp)["scales"][0]["sharding"]["data_encoding"] == "raw"  # jpeg: compress="auto" -> no gzip


@pytest.mark.parametrize("kwargs", [{"agglomerate": True}, {"timestamp": 5}, {"stop_layer": 2}, {"encoding": "png"},
                                    {"encoding": "jxl"}, {"encoding": "jpegxl"}, {"encoding": "compresso"},
                                    {"encoding": "crackle"}, {"encoding": "fpzip"}, {"encoding": "kempressed"},
                                    {"encoding": "zfpc"}, {"compress": "br"}])
@pytest.mark.parametrize("sharded", [False, True])
def test_refusals_write_nothing(tmp_path, kwargs, sharded):
  import igneous_b200.task_creation as tc
  src = _src(tmp_path)
  dest = tmp_path / "dest"
  fn = tc.create_image_shard_transfer_tasks if sharded else tc.create_transfer_tasks
  with pytest.raises(NotImplementedError):
    fn(src, "file://" + str(dest), **kwargs)
  assert not dest.exists()


@pytest.mark.parametrize("sharded", [False, True])
@pytest.mark.parametrize("layer", ["source", "destination"])
def test_refuses_unsupported_layer_encodings(tmp_path, sharded, layer):
  """an unsupported encoding already in the source scale, or in an existing destination scale that the
  request keeps, is refused before anything is written"""
  import igneous_b200.task_creation as tc
  src = _src(tmp_path, encoding="png" if layer == "source" else "raw")
  dest = _src(tmp_path, encoding="compresso", name="dest") if layer == "destination" else \
      "file://" + str(tmp_path / "dest")
  before = _info(dest) if layer == "destination" else None
  fn = tc.create_image_shard_transfer_tasks if sharded else tc.create_transfer_tasks
  with pytest.raises(NotImplementedError, match=layer):
    fn(src, dest)
  if layer == "source":
    assert not (tmp_path / "dest").exists()
  else:
    assert _info(dest) == before


def test_file_copy_needs_the_same_chunk_grid(tmp_path):
  """a destination cropped off the chunk grid names and sizes its edge chunks by its own bounds: the
  file copy is not taken, and transfer_to refuses it"""
  from igneous_b200._compat import Bbox, CloudVolume
  from igneous_b200.tasks.image import _same_chunks
  import igneous_b200.task_creation as tc
  src = _src(tmp_path)
  dest = "file://" + str(tmp_path / "dest")
  tc.create_transfer_tasks(src, dest, skip_downsamples=True, cutout=True, bounds=Bbox((0, 0, 0), (500, 500, 128)))
  s, d = CloudVolume(src), CloudVolume(dest)
  assert list(d.meta.volume_size(0)) == [500, 500, 128]
  assert not _same_chunks(s, d, 0)
  with pytest.raises(ValueError, match="chunk grid"):
    s.image.transfer_to(dest, d.meta.bounds(0), 0)
  assert not (tmp_path / "dest" / "1_1_1").exists()
  same = "file://" + str(tmp_path / "same")
  tc.create_transfer_tasks(src, same, skip_downsamples=True)
  assert _same_chunks(s, CloudVolume(same), 0)


def test_select_compression_by_encoding():
  import igneous_b200.task_creation as tc
  assert tc._select_compression_by_encoding("raw") == "gzip"
  assert tc._select_compression_by_encoding("compressed_segmentation") == "gzip"
  assert tc._select_compression_by_encoding("JPEG") is False
