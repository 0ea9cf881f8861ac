"""Mesh manifests, and the transfer and deletion of mesh and skeleton layers, without a GPU: these tasks only
list, group, copy and delete files (DESIGN.md §5m).  The manifest tests restate the reference's
test_mesh_manifests_filesystem and test_mesh_manifests_prefixes (test/test_tasks.py:506-600)."""
import json
import os

import numpy as np
import pytest

import igneous_b200
from igneous_b200 import labelshard, tasks
from igneous_b200 import task_creation as tc
from igneous_b200._compat import Bbox, CloudFiles, CloudVolume, LocalTaskQueue
from igneous_b200.sharding import LabelShardingSpecification, pack_shard
from igneous_b200.tasks import MeshTask

MESH_DIR = "mesh_mip_3_error_40"


def files(root):
  """{relative path: bytes} of every file under root"""
  out = {}
  for d, _, fs in os.walk(root):
    for f in fs:
      with open(os.path.join(d, f), "rb") as fh:
        out[os.path.relpath(os.path.join(d, f), root)] = fh.read()
  return out


def run(task_list):
  LocalTaskQueue().insert_all(task_list)


def segmentation_layer(tmp_path, name="seg", **info):
  path = "file://" + str(tmp_path / name)
  CloudVolume.from_numpy(np.zeros((8, 8, 8), np.uint32), path, resolution=(4, 4, 40), layer_type="segmentation")
  vol = CloudVolume(path)
  vol.info.update(info)
  vol.commit_info()
  return path


def touch_fragments(directory, n_segids=100, n_lods=2, n_fragids=5):
  os.makedirs(directory, exist_ok=True)
  for segid in range(n_segids):
    for lod in range(n_lods):
      for fragid in range(n_fragids):
        open(os.path.join(directory, "%d:%d:%d" % (segid, lod, fragid)), "wb").close()


def manifest(directory, name):
  with open(os.path.join(directory, name)) as f:
    return json.load(f)


# ------------------------------------------------------------------ manifests
def test_mesh_manifests_filesystem(tmp_path):
  layer_path = "file://" + str(tmp_path)
  directory = str(tmp_path / MESH_DIR)
  CloudFiles(layer_path).put_json("info", {"mesh": MESH_DIR})
  touch_fragments(directory)
  tasks.MeshManifestFilesystemTask(layer_path=layer_path, lod=0)
  for segid in range(100):
    assert os.path.exists(os.path.join(directory, "%d:0" % segid))
    assert not os.path.exists(os.path.join(directory, "%d:1" % segid))
  tasks.MeshManifestFilesystemTask(layer_path=layer_path, lod=1)
  for segid in range(100):
    assert os.path.exists(os.path.join(directory, "%d:0" % segid))
    assert os.path.exists(os.path.join(directory, "%d:1" % segid))
  content = manifest(directory, "50:0")
  content["fragments"].sort()
  assert content == {"fragments": ["50:0:0", "50:0:1", "50:0:2", "50:0:3", "50:0:4"]}
  assert sorted(manifest(directory, "7:1")["fragments"]) == ["7:1:%d" % i for i in range(5)]


def test_mesh_manifests_prefixes(tmp_path):
  layer_path = "file://" + str(tmp_path)
  directory = str(tmp_path / MESH_DIR)
  CloudFiles(layer_path).put_json("info", {"mesh": MESH_DIR})
  touch_fragments(directory)
  for i in range(10):
    tasks.MeshManifestPrefixTask(layer_path=layer_path, prefix=str(i), lod=0)
  for segid in range(100):
    assert os.path.exists(os.path.join(directory, "%d:0" % segid))
    assert not os.path.exists(os.path.join(directory, "%d:1" % segid))
  for i in range(10):
    tasks.MeshManifestPrefixTask(layer_path=layer_path, prefix=str(i), lod=1)
  for segid in range(100):
    assert os.path.exists(os.path.join(directory, "%d:1" % segid))
  assert manifest(directory, "50:0") == {"fragments": ["50:0:0", "50:0:1", "50:0:2", "50:0:3", "50:0:4"]}


def test_manifests_name_gzipped_fragments_and_skip_other_files(tmp_path):
  layer_path = "file://" + str(tmp_path)
  cf = CloudFiles(layer_path)
  cf.put_json("info", {"mesh": "m"})
  frags = ["3:0:0-64_0-64_0-64", "3:0:64-128_0-64_0-64", "3:1:0-64_0-64_0-64", "31:0:0-64_0-64_0-64"]
  for name in frags:
    cf.put("m/" + name, b"fragment", compress="gzip")
  cf.put_json("m/info", {"@type": "neuroglancer_legacy_mesh"})
  cf.put_json("m/3:0", {"fragments": ["stale"]})                       # an existing manifest
  cf.put_json("m/31:0", {"fragments": ["stale"]})
  cf.put_json("m/0-64_0-64_0-64.spatial", {"3": [0, 0, 0, 1, 1, 1]}, compress="gzip")
  os.makedirs(str(tmp_path / "m" / "5:0:dir"))                         # not a regular file
  want = {"m/3:0": {"fragments": ["3:0:0-64_0-64_0-64", "3:0:64-128_0-64_0-64"]},
          "m/31:0": {"fragments": ["31:0:0-64_0-64_0-64"]}}
  for t in (lambda: tasks.MeshManifestFilesystemTask(layer_path),
            lambda: [tasks.MeshManifestPrefixTask(layer_path, p) for p in ("3:", "31")]):
    t()
    got = {k: cf.get_json(k) for k in want}
    assert {k: {"fragments": sorted(v["fragments"])} for k, v in got.items()} == want
    assert not os.path.exists(str(tmp_path / "m" / "5:0"))
    # manifests are stored uncompressed, next to the gzipped fragments
    assert os.path.isfile(str(tmp_path / "m" / "3:0")) and not os.path.exists(str(tmp_path / "m" / "3:0.gz"))
    assert cf.get_json("m/info") == {"@type": "neuroglancer_legacy_mesh"}
    cf.put_json("m/3:0", {"fragments": ["stale"]})
    cf.put_json("m/31:0", {"fragments": ["stale"]})
  # lod 1 and an explicit mesh_dir
  tasks.MeshManifestFilesystemTask(layer_path, lod=1, mesh_dir="m")
  assert cf.get_json("m/3:1") == {"fragments": ["3:1:0-64_0-64_0-64"]}


@pytest.mark.parametrize("compress", ("gzip", None))
def test_single_task_manifest_equals_generate_manifests(tmp_path, compress):
  """A layer meshed by one task: the merged manifests are those MeshTask(generate_manifests=True) writes.
  The task's upload step is called directly with stand-in fragment bytes, so no mesh is computed."""
  path = segmentation_layer(tmp_path, mesh="mesh")
  t = MeshTask(shape=(64, 64, 64), offset=(0, 0, 0), layer_path=path, generate_manifests=True, compress=compress)
  t._mesh_dir, t._bounds = "mesh", Bbox((0, 0, 0), (8, 8, 8))
  t._upload_individuals({3: b"a", 17: b"bb", 1234: b"ccc"}, True)
  cf = CloudFiles(path)
  names = ["mesh/3:0", "mesh/17:0", "mesh/1234:0"]
  want = {n: cf.get_json(n) for n in names}
  assert want["mesh/17:0"] == {"fragments": ["17:0:0-8_0-8_0-8"]}
  for creator_path in (path, "gs://bucket/layer"):
    cf.delete(names)
    manifest_tasks = tc.create_mesh_manifest_tasks(creator_path, magnitude=2)
    if creator_path != path:  # the prefix route, run here against the file:// layer
      manifest_tasks = [lambda p=t.keywords["prefix"]: tasks.MeshManifestPrefixTask(path, p) for t in manifest_tasks]
    run(manifest_tasks)
    assert {n: cf.get_json(n) for n in names} == want


def test_manifest_task_without_mesh_dir_writes_nothing(tmp_path):
  layer_path = "file://" + str(tmp_path)
  CloudFiles(layer_path).put_json("info", {"scales": []})
  touch_fragments(str(tmp_path / "mesh"), 3, 1, 1)
  before = files(str(tmp_path))
  for t in (tasks.MeshManifestFilesystemTask, lambda p: tasks.MeshManifestPrefixTask(p, "1")):
    with pytest.raises(ValueError, match="mesh_dir"):
      t(layer_path)
  with pytest.raises(ValueError, match="mesh_dir"):
    tasks.MeshManifestPrefixTask("file://" + str(tmp_path / "nolayer"), "1")
  assert files(str(tmp_path)) == before
  tasks.MeshManifestPrefixTask(layer_path, "1", mesh_dir="mesh")
  assert CloudFiles(layer_path).get_json("mesh/1:0") == {"fragments": ["1:0:0"]}


# ------------------------------------------------------------ creator prefixes
def decimal(m):
  """every string of m decimal digits, in order"""
  return ["%0*d" % (m, i) for i in range(10 ** m)]


def hexadecimal(m):
  return ["%0*x" % (m, i) for i in range(16 ** m)]


@pytest.mark.parametrize("magnitude", (1, 2, 3))
def test_manifest_creator_prefixes(tmp_path, magnitude):
  got = tc.create_mesh_manifest_tasks("gs://bucket/layer", magnitude=magnitude, mesh_dir="m")
  prefixes = [t.keywords["prefix"] for t in got]
  short = ["%d:" % i for i in range(1, 10 ** (magnitude - 1))]
  assert prefixes == short + [str(i) for i in range(10 ** (magnitude - 1), 10 ** magnitude)]
  assert len(got) == len(prefixes) == 10 ** magnitude - 1
  assert {(t.func, t.keywords["layer_path"], t.keywords["mesh_dir"]) for t in got} == {
    (tasks.MeshManifestPrefixTask, "gs://bucket/layer", "m")}
  for path in ("file://" + str(tmp_path), str(tmp_path)):
    (t,) = tc.create_mesh_manifest_tasks(path, magnitude=magnitude)
    assert t.func is tasks.MeshManifestFilesystemTask and t.keywords == {"layer_path": path, "mesh_dir": None}
  with pytest.raises(AssertionError):
    tc.create_mesh_manifest_tasks("gs://bucket/layer", magnitude=0)
  with pytest.raises(AssertionError):
    tc.create_mesh_manifest_tasks("gs://bucket/layer", magnitude=1.5)


def deletion_prefixes(m):
  return ["0"] + ["%d:" % i for i in range(1, 10 ** (m - 1))] + [str(i) for i in range(10 ** (m - 1), 10 ** m)]


@pytest.mark.parametrize("magnitude", (1, 2, 3))
@pytest.mark.parametrize("kind", ("mesh", "skeleton"))
def test_deletion_creator_prefixes_info_and_provenance(tmp_path, magnitude, kind):
  path = segmentation_layer(tmp_path, mesh="m", skeletons="s")
  cf = CloudFiles(path)
  for sub in ("m", "s"):
    cf.put_json(sub + "/info", {"@type": "x", "sharding": None})
  create = tc.create_mesh_deletion_tasks if kind == "mesh" else tc.create_skeleton_deletion_tasks
  got = create(path, magnitude)
  sub, other = ("m", "s") if kind == "mesh" else ("s", "m")
  assert not cf.exists(sub + "/info") and cf.exists(other + "/info")
  assert [t.keywords["prefix"] for t in got] == deletion_prefixes(magnitude)
  assert len(got) == 10 ** magnitude
  task = tasks.DeleteMeshFilesTask if kind == "mesh" else tasks.DeleteSkeletonFilesTask
  key, dir_key = ("layer_path", "mesh_dir") if kind == "mesh" else ("cloudpath", "skel_dir")
  assert all(t.func is task and t.keywords["cloudpath"] == path and t.keywords[dir_key] is None for t in got)
  (prov,) = cf.get_json("provenance")["processing"]
  assert prov["method"] == {"task": task.__name__, key: path, dir_key: None}
  # a sharded directory: one task over every file
  cf.put_json("x/info", {"@type": "x", "sharding": {"@type": "neuroglancer_uint64_sharded_v1"}})
  got = create(path, magnitude, "x")
  assert [(t.keywords["prefix"], t.keywords[dir_key]) for t in got] == [("", "x")]
  assert not cf.exists("x/info")
  assert len(cf.get_json("provenance")["processing"]) == 2
  assert cf.get_json("provenance")["processing"][1]["method"][dir_key] == "x"


@pytest.mark.parametrize("kind", ("mesh", "skeleton"))
def test_deletion_creator_refuses_magnitude_zero(tmp_path, kind):
  path = segmentation_layer(tmp_path, mesh="m", skeletons="s")
  CloudFiles(path).put_json("m/info", {"@type": "x"})
  CloudFiles(path).put_json("s/info", {"@type": "x"})
  before = files(str(tmp_path))
  create = tc.create_mesh_deletion_tasks if kind == "mesh" else tc.create_skeleton_deletion_tasks
  with pytest.raises(ValueError, match="magnitude"):
    create(path, magnitude=0)
  with pytest.raises(AssertionError):
    create(path, magnitude=-1)
  assert files(str(tmp_path)) == before


@pytest.mark.parametrize("magnitude", (1, 2, 3))
@pytest.mark.parametrize("sharded", (False, True))
@pytest.mark.parametrize("kind", ("mesh", "skeleton"))
def test_xfer_creator_prefixes_and_info(tmp_path, magnitude, sharded, kind):
  src = segmentation_layer(tmp_path, "src", mesh="m", skeletons="s")
  dest = segmentation_layer(tmp_path, "dest", mesh="dm", skeletons="ds")
  src_info = {"@type": "x", "sharding": {"@type": "neuroglancer_uint64_sharded_v1"} if sharded else None}
  CloudFiles(src).put_json(("m" if kind == "mesh" else "s") + "/info", src_info)
  create = tc.create_xfer_meshes_tasks if kind == "mesh" else tc.create_xfer_skeleton_tasks
  got = create(src, dest, magnitude=magnitude)
  digits = hexadecimal if sharded else decimal
  suffix = ("." if sharded else ":0") if kind == "mesh" else ""
  want = digits(magnitude) + [p + suffix for i in range(1, magnitude) for p in digits(i)]
  assert [t.keywords["prefix"] for t in got] == want
  base = 16 if sharded else 10
  assert len(got) == sum(base ** i for i in range(1, magnitude + 1))
  task, dir_key, sub = ((tasks.TransferMeshFilesTask, "mesh_dir", "dm") if kind == "mesh"
                        else (tasks.TransferSkeletonFilesTask, "skel_dir", "ds"))
  assert all(t.func is task and (t.keywords["src"], t.keywords["dest"], t.keywords[dir_key]) == (src, dest, sub)
             for t in got)
  assert CloudFiles(dest).get_json(sub + "/info") == src_info
  # an explicit directory wins over the destination's info
  got = create(src, dest, "elsewhere", magnitude)
  assert {t.keywords[dir_key] for t in got} == {"elsewhere"}
  assert CloudFiles(dest).get_json("elsewhere/info") == src_info


@pytest.mark.parametrize("kind", ("mesh", "skeleton"))
def test_xfer_creator_refusals_write_nothing(tmp_path, kind):
  src = segmentation_layer(tmp_path, "src", mesh="m", skeletons="s")
  bare = segmentation_layer(tmp_path, "bare")
  nowhere = "file://" + str(tmp_path / "nowhere")
  create = tc.create_xfer_meshes_tasks if kind == "mesh" else tc.create_xfer_skeleton_tasks
  before = files(str(tmp_path))
  with pytest.raises(ValueError, match="no info"):
    create(src, nowhere)
  with pytest.raises(ValueError, match="no info"):
    create(src, nowhere, "d")
  with pytest.raises(ValueError, match="mesh" if kind == "mesh" else "skeletons"):
    create(src, bare)
  assert files(str(tmp_path)) == before


# ------------------------------------------------------------- transfers and deletions
def mesh_files(cf, sub):
  """a mesh directory: gzipped fragments of several lods and label lengths, raw manifests, spatial index files"""
  stored = {}
  for name in ("1:0:0-64_0-64_0-64", "5:0:0-64_0-64_0-64", "5:1:0-64_0-64_0-64", "12:0:0-64_0-64_0-64",
               "12:1:64-128_0-64_0-64", "150:0:0-64_0-64_0-64", "1234:0:64-128_0-64_0-64"):
    cf.put("%s/%s" % (sub, name), name.encode() * 3, compress="gzip")
    stored[name + ".gz"] = None
  for name in ("1:0", "5:0", "12:0", "150:0", "1234:0"):
    cf.put_json("%s/%s" % (sub, name), {"fragments": [name + ":0-64_0-64_0-64"]})
    stored[name] = None
  for name in ("0-64_0-64_0-64.spatial", "64-128_0-64_0-64.spatial", "128-192_0-64_0-64.spatial",
               "1024-1088_0-64_0-64.spatial"):
    cf.put_json("%s/%s" % (sub, name), {"1": [0, 0, 0, 1, 1, 1]}, compress="gzip")
    stored[name + ".gz"] = None
  return set(stored)


def test_mesh_transfer_is_byte_identical_except_the_kept_quirks(tmp_path):
  src = segmentation_layer(tmp_path, "src", mesh="m")
  dest = segmentation_layer(tmp_path, "dest", mesh="dm")
  cf = CloudFiles(src)
  cf.put_json("m/info", {"@type": "neuroglancer_legacy_mesh", "mip": 0})
  names = mesh_files(cf, "m")
  got = tc.create_xfer_meshes_tasks(src, dest)
  run(got)
  src_files, dest_files = files(str(tmp_path / "src" / "m")), files(str(tmp_path / "dest" / "dm"))
  # an unsharded source's prefixes miss lod > 0 files of labels 1-9 and spatial files from a one-digit coordinate
  missed = {"5:1:0-64_0-64_0-64.gz", "0-64_0-64_0-64.spatial.gz"}
  assert set(dest_files) == (names - missed) | {"info"}
  assert all(dest_files[n] == src_files[n] for n in names - missed)
  assert json.loads(dest_files["info"]) == {"@type": "neuroglancer_legacy_mesh", "mip": 0}
  # the tasks alone (the info is the creator's), to an explicit directory
  for t in got:
    tasks.TransferMeshFilesTask(src, dest, t.keywords["prefix"], mesh_dir="other")
  other = files(str(tmp_path / "dest" / "other"))
  assert set(other) == names - missed and all(other[n] == src_files[n] for n in other)


def test_sharded_mesh_transfer_and_deletion(tmp_path):
  src = segmentation_layer(tmp_path, "src", mesh="m")
  dest = segmentation_layer(tmp_path, "dest", mesh="dm")
  cf = CloudFiles(src)
  cf.put_json("m/info", {"@type": "neuroglancer_multilod_draco", "sharding": {"@type": "neuroglancer_uint64_sharded_v1"}})
  for name in ("0.shard", "b.shard", "1a.shard", "3f0.shard"):
    cf.put("m/" + name, os.urandom(40), compress=None)
  run(tc.create_xfer_meshes_tasks(src, dest))
  src_files, dest_files = files(str(tmp_path / "src" / "m")), files(str(tmp_path / "dest" / "dm"))
  assert dest_files == src_files
  run(tc.create_mesh_deletion_tasks(src))
  assert files(str(tmp_path / "src" / "m")) == {}


def test_mesh_deletion_leaves_only_the_kept_quirks(tmp_path):
  path = segmentation_layer(tmp_path, mesh="m")
  cf = CloudFiles(path)
  cf.put_json("m/info", {"@type": "neuroglancer_legacy_mesh"})
  mesh_files(cf, "m")
  cf.put_json("other/keep", {})
  deleted = tc.create_mesh_deletion_tasks(path)
  assert not cf.exists("m/info")
  run(deleted)
  # a spatial file whose first coordinate has 1 to magnitude - 1 digits: "64-" is neither "64:" nor 3 digits
  assert set(files(str(tmp_path / "seg" / "m"))) == {"64-128_0-64_0-64.spatial.gz"}
  assert cf.exists("other/keep") and cf.exists("info")


def skeleton_blob(segid, nv=3):
  """a precomputed skeleton with one float32 `radius` attribute: a path of nv vertices"""
  v = np.arange(nv * 3, dtype=np.float32).reshape(nv, 3) + segid
  e = np.stack([np.arange(nv - 1), np.arange(1, nv)], axis=1).astype(np.uint32)
  return (np.array([nv, nv - 1], np.uint32).tobytes() + v.tobytes() + e.tobytes()
          + np.full(nv, segid % 7, np.float32).tobytes())


SKELETON_INFO = {"@type": "neuroglancer_skeletons", "transform": [1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0],
                 "vertex_attributes": [{"id": "radius", "data_type": "float32", "num_components": 1}],
                 "sharding": None, "spatial_index": None, "mip": 0}


def skeleton_files(cf, sub):
  cf.put_json(sub + "/info", SKELETON_INFO)
  for segid in (5, 12, 345, 6789):
    cf.put("%s/%d" % (sub, segid), skeleton_blob(segid), compress="gzip")
  for name in ("5:0-64_0-64_0-64", "12:64-128_0-64_0-64", "345:0-64_0-64_0-64"):
    cf.put("%s/%s" % (sub, name), b"fragment " + name.encode(), compress="gzip")
  for name in ("0-64_0-64_0-64.spatial", "8-16_0-64_0-64.spatial", "64-128_0-64_0-64.spatial"):
    cf.put_json("%s/%s" % (sub, name), {"5": [0, 0, 0, 1, 1, 1]}, compress="gzip")


def test_skeleton_transfer_and_deletion(tmp_path):
  src = segmentation_layer(tmp_path, "src", skeletons="s")
  dest = segmentation_layer(tmp_path, "dest", skeletons="ds")
  cf = CloudFiles(src)
  skeleton_files(cf, "s")
  src_files = files(str(tmp_path / "src" / "s"))
  got = tc.create_xfer_skeleton_tasks(src, dest)
  assert len(got) == 110
  run(got)
  # the plain one-digit prefixes reach every file, spatial files from a one-digit coordinate included
  assert files(str(tmp_path / "dest" / "ds")) == src_files
  vol = CloudVolume(dest)
  for segid in (5, 12, 345, 6789):
    assert vol.skeleton.get(segid).vertices[0, 0] == segid
  run(tc.create_skeleton_deletion_tasks(src))
  # labels 1-9 are final skeletons named "5" (no colon), and "8-" is neither "8:" nor two digits
  assert set(files(str(tmp_path / "src" / "s"))) == {"5.gz", "8-16_0-64_0-64.spatial.gz"}
  assert (json.loads(CloudFiles(src).get("provenance"))["processing"][-1]["method"]
          == {"task": "DeleteSkeletonFilesTask", "cloudpath": src, "skel_dir": None})


def host_hash(labels, preshift_bits, minishard_bits, shard_bits, ctx=None):
  """labelshard.shard_hash restated with the host specification"""
  spec = LabelShardingSpecification({"preshift_bits": preshift_bits, "minishard_bits": minishard_bits,
                                     "shard_bits": shard_bits})
  labels = np.asarray(labels, dtype=np.uint64)
  shards, minis = spec.locate_many(labels)
  order = np.lexsort((labels, minis, shards))
  loc = (shards << np.uint64(minishard_bits)) | minis
  s = shards[order]
  heads = np.flatnonzero(np.r_[True, s[1:] != s[:-1]]) if len(s) else np.zeros(0, np.int64)
  return labels[order], loc[order], np.r_[heads, len(s)].astype(np.uint64), s[heads]


def test_sharded_skeleton_layer_transfers_with_hex_prefixes(tmp_path, monkeypatch):
  """A sharded layer laid out by create_sharded_skeletons_from_unsharded_tasks (its shards packed on the
  host, as the task packs them) is copied whole and read back label by label at the destination."""
  monkeypatch.setattr(labelshard, "shard_hash", host_hash)
  src = segmentation_layer(tmp_path, "src", skeletons="s")
  dest = segmentation_layer(tmp_path, "dest", skeletons="ds")
  cf = CloudFiles(src)
  cf.put_json("s/info", SKELETON_INFO)
  labels = list(range(1, 400, 3)) + [2 ** 40 + 7]
  for segid in labels:
    cf.put("s/%d" % segid, skeleton_blob(segid), compress="gzip")
  merge = tc.create_sharded_skeletons_from_unsharded_tasks(src, src, shard_index_bytes=64, minishard_index_bytes=48,
                                                           skel_dir="sharded", data_encoding="raw")
  vol = CloudVolume(src, skel_dir="sharded")
  spec = LabelShardingSpecification(vol.skeleton.meta.info["sharding"])
  assert spec.shard_bits == 4  # shard files 0.shard ... f.shard
  scf = CloudFiles(vol.skeleton.meta.layerpath)
  for t in merge:
    ids = scf.get_json(t.keywords["shard_no"] + ".labels")
    _, minis = spec.locate_many(ids)
    scf.put(spec.shard_filename(int(t.keywords["shard_no"])),
            pack_shard(spec.minishard_bits, spec.minishard_index_encoding, minis, ids,
                       [skeleton_blob(i) for i in ids]), compress=None)
  assert vol.skeleton.meta.is_sharded() and any(n[0] in "abcdef" for n in scf.list())
  vol.info["skeletons"] = "sharded"  # the transfer copies the source layer's own skeleton directory
  vol.commit_info()
  xfer = tc.create_xfer_skeleton_tasks(src, dest, skel_dir="copy")
  assert len(xfer) == 256 + 16
  run(xfer)
  assert files(str(tmp_path / "dest" / "copy")) == files(str(tmp_path / "src" / "sharded"))
  got = CloudVolume(dest, skel_dir="copy")
  assert got.skeleton.meta.is_sharded()
  for segid in labels:
    s = got.skeleton.get(segid)
    assert np.array_equal(s.vertices, np.arange(9, dtype=np.float32).reshape(3, 3) + segid)
    assert len(s.edges) == 2
  run(tc.create_skeleton_deletion_tasks(src, skel_dir="sharded"))
  assert files(str(tmp_path / "src" / "sharded")) == {}


def test_exports():
  names = ("MeshManifestPrefixTask", "MeshManifestFilesystemTask", "TransferMeshFilesTask", "DeleteMeshFilesTask",
           "TransferSkeletonFilesTask", "DeleteSkeletonFilesTask")
  for n in names:
    assert getattr(igneous_b200, n) is getattr(tasks, n) and n in igneous_b200.__all__
  for n in ("create_mesh_manifest_tasks", "create_mesh_deletion_tasks", "create_xfer_meshes_tasks",
            "create_skeleton_deletion_tasks", "create_xfer_skeleton_tasks"):
    assert getattr(igneous_b200, n) is getattr(tc, n) and n in igneous_b200.__all__
