"""create_sharded_skeletons_from_unsharded_tasks without a GPU: the device hash is replaced by the host
specification's (the kernel itself is checked in test_sharded_skeletons_gpu.py), so the info edits, the
.labels files, the tasks, the provenance, the file-name rule and the refusals run on any machine."""
import copy
import json
import os

import numpy as np
import pytest

import igneous_b200
from igneous_b200 import labelshard, tasks
from igneous_b200 import task_creation as tc
from igneous_b200._compat import CloudFiles, CloudVolume
from igneous_b200.sharding import LabelShardingSpecification

ATTRS = [{"id": "radius", "data_type": "float32", "num_components": 1},
         {"id": "vertex_types", "data_type": "uint8", "num_components": 1},
         {"id": "thickness", "data_type": "float64", "num_components": 2}]


def host_hash(labels, preshift_bits, minishard_bits, shard_bits, ctx=None):
  spec = LabelShardingSpecification({"preshift_bits": preshift_bits, "minishard_bits": minishard_bits,
                                     "shard_bits": shard_bits})
  labels = np.asarray(labels, dtype=np.uint64)
  shards, minis = spec.locate_many(labels)
  order = np.lexsort((labels, minis, shards))
  loc = (shards << np.uint64(minishard_bits)) | minis
  s = shards[order]
  heads = np.flatnonzero(np.r_[True, s[1:] != s[:-1]]) if len(s) else np.zeros(0, np.int64)
  return labels[order], loc[order], np.r_[heads, len(s)].astype(np.uint64), s[heads]


@pytest.fixture
def layer(tmp_path, monkeypatch):
  monkeypatch.setattr(labelshard, "shard_hash", host_hash)
  path = "file://" + str(tmp_path / "seg")
  CloudVolume.from_numpy(np.zeros((8, 8, 8), np.uint64), path, resolution=(4, 4, 40), layer_type="segmentation")
  vol = CloudVolume(path)
  vol.info["skeletons"] = "skel"
  vol.commit_info()
  vol = CloudVolume(path)
  vol.skeleton.meta.info["vertex_attributes"] = copy.deepcopy(ATTRS)
  vol.skeleton.meta.info["mip"] = 0
  vol.skeleton.meta.commit_info()
  return path


def put_labels(path, labels, compress="gzip"):
  cf = CloudFiles(CloudVolume(path).skeleton.path)
  for l in labels:
    cf.put(str(l), b"blob", compress=compress)


def files(root):
  out = {}
  for d, _, fs in os.walk(root):
    for f in fs:
      with open(os.path.join(d, f), "rb") as fh:
        out[os.path.relpath(os.path.join(d, f), root)] = fh.read()
  return out


def test_info_labels_tasks_and_provenance(layer, tmp_path):
  rng = np.random.default_rng(1)
  labels = sorted(set(rng.integers(1, 2 ** 64 - 1, 300, dtype=np.uint64, endpoint=True).tolist()) | {1, 2 ** 32})
  put_labels(layer, labels)
  cf = CloudFiles(CloudVolume(layer).skeleton.path)
  cf.put("5:0-32_0-32_0-320", b"fragment", compress="gzip")   # a fragment: not a label
  cf.put("17.spatial", b"{}", compress="gzip")                # not a label
  cf.put("12x", b"", compress=None)
  cf.put("sub/44", b"", compress=None)
  got = tc.create_sharded_skeletons_from_unsharded_tasks(layer, layer, shard_index_bytes=64,
                                                         minishard_index_bytes=192, skel_dir="skel_sharded",
                                                         data_encoding="raw")
  dest = CloudVolume(layer, skel_dir="skel_sharded")
  info = dest.skeleton.meta.info
  assert [a["id"] for a in info["vertex_attributes"]] == ["radius", "thickness"]
  assert info["sharding"] == {"@type": "neuroglancer_uint64_sharded_v1", "preshift_bits": 0,
                              "hash": "murmurhash3_x86_128", "minishard_bits": 2, "shard_bits": 4,
                              "minishard_index_encoding": "gzip", "data_encoding": "raw"}
  assert info["mip"] == 0 and info["@type"] == "neuroglancer_skeletons"
  spec = LabelShardingSpecification(info["sharding"])
  dcf = CloudFiles(dest.skeleton.path)
  seen = []
  shard_nos = sorted(int(n[:-len(".labels")]) for n in dcf.list() if n.endswith(".labels"))
  assert [int(t.keywords["shard_no"]) for t in got] == shard_nos and len(got) > 4
  for t in got:
    assert t.func is tasks.ShardedFromUnshardedSkeletonMergeTask
    assert t.keywords == {"src": layer, "dest": layer, "shard_no": t.keywords["shard_no"], "skel_dir": "skel_sharded"}
    assert os.path.exists(os.path.join(dest.skeleton.path[len("file://"):], t.keywords["shard_no"] + ".labels.gz"))
    mine = dcf.get_json(t.keywords["shard_no"] + ".labels")
    assert all(spec.locate(l)[0] == int(t.keywords["shard_no"]) for l in mine)
    assert mine == sorted(mine, key=lambda l: (spec.locate(l)[1], l))
    seen += mine
  assert sorted(seen) == labels
  prov = json.loads(CloudFiles(layer).get("provenance"))["processing"][-1]
  assert prov["method"] == {"task": "ShardedFromUnshardedSkeletonMergeTask", "src": layer, "dest": layer,
                            "preshift_bits": 0, "minishard_bits": 2, "shard_bits": 4, "skel_dir": "skel_sharded"}
  # the source's info is untouched
  assert [a["id"] for a in CloudVolume(layer).skeleton.meta.info["vertex_attributes"]] == [a["id"] for a in ATTRS]


def test_no_labels_gives_no_tasks(layer):
  got = tc.create_sharded_skeletons_from_unsharded_tasks(layer, layer, skel_dir="out")
  assert got == []
  assert CloudVolume(layer, skel_dir="out").skeleton.meta.info["sharding"]["shard_bits"] == 0


def test_refusals_write_nothing(layer, tmp_path):
  put_labels(layer, [3, 4])
  before = files(str(tmp_path))
  with pytest.raises(ValueError, match="source"):
    tc.create_sharded_skeletons_from_unsharded_tasks(layer, layer)
  with pytest.raises(ValueError, match="source"):
    tc.create_sharded_skeletons_from_unsharded_tasks(layer, layer, skel_dir="skel/./")
  with pytest.raises(ValueError, match="encoding"):
    tc.create_sharded_skeletons_from_unsharded_tasks(layer, layer, skel_dir="out", data_encoding="zstd")
  with pytest.raises(ValueError, match="encoding"):
    tc.create_sharded_skeletons_from_unsharded_tasks(layer, layer, skel_dir="out", minishard_index_encoding="br")
  with pytest.raises(ValueError, match="source"):
    tasks.ShardedFromUnshardedSkeletonMergeTask(layer, layer, "0")
  assert files(str(tmp_path)) == before
  CloudFiles(CloudVolume(layer).skeleton.path).put("9.zstd", b"", compress=None)
  before = files(str(tmp_path))
  with pytest.raises(NotImplementedError, match="zstd"):
    tc.create_sharded_skeletons_from_unsharded_tasks(layer, layer, skel_dir="out")
  assert files(str(tmp_path)) == before


def test_task_without_labels_file_or_with_a_missing_label(layer, tmp_path):
  put_labels(layer, [3, 4, 5])
  (t,) = tc.create_sharded_skeletons_from_unsharded_tasks(layer, layer, skel_dir="out")
  dest = CloudVolume(layer, skel_dir="out")
  dcf = CloudFiles(dest.skeleton.path)
  with pytest.raises(FileNotFoundError, match="7.labels"):
    tasks.ShardedFromUnshardedSkeletonMergeTask(layer, layer, "7", skel_dir="out")
  dcf.put_json("0.labels", [3, 77, 4], compress="gzip")
  before = files(str(tmp_path))
  with pytest.raises(FileNotFoundError, match="label 77"):
    t()
  dcf.put_json("0.labels", [], compress="gzip")
  before = files(str(tmp_path))
  t()  # an empty list writes nothing
  assert files(str(tmp_path)) == before


def test_exports():
  assert igneous_b200.ShardedFromUnshardedSkeletonMergeTask is tasks.ShardedFromUnshardedSkeletonMergeTask
  assert tc.ShardedFromUnshardedSkeletonMergeTask is tasks.ShardedFromUnshardedSkeletonMergeTask
  assert igneous_b200.create_sharded_skeletons_from_unsharded_tasks is tc.create_sharded_skeletons_from_unsharded_tasks
  assert "ShardedFromUnshardedSkeletonMergeTask" in igneous_b200.__all__
