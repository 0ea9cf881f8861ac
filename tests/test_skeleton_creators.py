"""create_skeletonizing_tasks and the skeleton source of the file:// stand-in: the task grid, the overlap,
spatial_grid_shape and will_postprocess on both sides of the volume size, the skeleton info edits, the
frag_path info, provenance, every refused option, the import surface, and cv.skeleton.get on a blob
written by a plain numpy encoder.  Nothing here runs a kernel."""
import gzip
import os

import numpy as np
import pytest

import igneous_b200
from igneous_b200 import task_creation as tc
from igneous_b200 import tasks
from igneous_b200._compat import CloudFiles, CloudVolume


def _layer(tmp_path, shape=(300, 200, 70), offset=(10, 20, 3), resolution=(4, 4, 40), name="seg"):
  path = "file://" + str(tmp_path / name)
  info = CloudVolume.create_new_info(1, "segmentation", np.uint64, "raw", resolution, offset, shape, (64, 64, 32))
  CloudVolume(path, info=info).commit_info()
  return path


def encode(vertices, edges, attributes=()):
  """neuroglancer precomputed skeleton: nv, ne, vertices, edges, then each vertex attribute in order"""
  vertices, edges = np.asarray(vertices, np.float32), np.asarray(edges, np.uint32)
  parts = [np.array([len(vertices), len(edges)], np.uint32).tobytes(), vertices.tobytes(), edges.tobytes()]
  return b"".join(parts + [np.asarray(a).tobytes() for a in attributes])


def test_grid_overlap_and_will_postprocess(tmp_path):
  path = _layer(tmp_path)
  got = list(tc.create_skeletonizing_tasks(path, mip=0, shape=(128, 128, 64)))
  assert len(got) == 3 * 2 * 2
  assert [list(map(int, t.bounds.minpt)) for t in got[:4]] == [[10, 20, 3], [138, 20, 3], [266, 20, 3], [10, 148, 3]]
  assert all(list(map(int, t.bounds.size3())) == [129, 129, 65] for t in got)
  assert all(list(map(int, t.index_bounds.size3())) == [128, 128, 64] for t in got)
  assert all(t.will_postprocess is True and t.mip == 0 for t in got)
  assert all(t.teasar_params == {"scale": 10, "const": 10} and t.dust_threshold == 1000 for t in got)
  # one task covering the whole volume: nothing to merge
  one = list(tc.create_skeletonizing_tasks(path, mip=0, shape=(300, 200, 70)))
  assert len(one) == 1 and one[0].will_postprocess is False
  assert list(map(int, one[0].bounds.size3())) == [301, 201, 71]
  # larger than the volume on every axis: still one task, still no merge
  big = list(tc.create_skeletonizing_tasks(path, mip=0, shape=(512, 512, 512)))
  assert len(big) == 1 and big[0].will_postprocess is False
  # one axis too short is enough to need the merge
  assert list(tc.create_skeletonizing_tasks(path, mip=0, shape=(300, 200, 69)))[0].will_postprocess is True


def test_info_edits_and_provenance(tmp_path):
  path = _layer(tmp_path)
  list(tc.create_skeletonizing_tasks(path, mip=0, shape=(128, 128, 64), dust_threshold=50, object_ids=[3, 4]))
  vol = CloudVolume(path)
  assert vol.info["skeletons"] == "skeletons_mip_0"
  info = CloudFiles(path).get_json("skeletons_mip_0/info")
  assert info["@type"] == "neuroglancer_skeletons" and info["mip"] == 0
  assert info["spatial_index"] == {"resolution": [4, 4, 40], "chunk_size": [512, 512, 2560]}
  # cloudvolume's default attributes, as recalled, with the integer one left out
  assert info["vertex_attributes"] == [{"id": "radius", "data_type": "float32", "num_components": 1}]
  assert vol.skeleton.meta.info == info and vol.skeleton.spatial_index is vol.mesh.spatial_index
  method = vol.provenance.processing[-1]["method"]
  assert method["task"] == "SkeletonTask" and method["cloudpath"] == path and method["shape"] == [128, 128, 64]
  assert method["dust_threshold"] == 50 and method["object_ids"] == [3, 4] and method["will_postprocess"] is True
  assert method["sharded"] is False and method["fill_holes"] == 0 and method["teasar_params"] == {"scale": 10,
                                                                                                  "const": 10}


def test_existing_directory_and_info_are_kept(tmp_path):
  path = _layer(tmp_path)
  vol = CloudVolume(path)
  vol.info["skeletons"] = "skels"
  vol.commit_info()
  CloudFiles(path).put_json("skels/info", {
    "@type": "neuroglancer_skeletons", "transform": [2, 0, 0, 0, 0, 2, 0, 0, 0, 0, 2, 0], "spatial_index": None,
    "vertex_attributes": [{"id": "radius", "data_type": "float32", "num_components": 1},
                          {"id": "vertex_types", "data_type": "uint8", "num_components": 1},
                          {"id": "cross_sectional_area", "data_type": "float32", "num_components": 1}]})
  list(tc.create_skeletonizing_tasks(path, mip=0, shape=(128, 128, 64), spatial_index=False))
  info = CloudFiles(path).get_json("skels/info")
  assert CloudVolume(path).info["skeletons"] == "skels"
  assert info["transform"] == [2, 0, 0, 0, 0, 2, 0, 0, 0, 0, 2, 0] and info["spatial_index"] is None
  assert [a["id"] for a in info["vertex_attributes"]] == ["radius"]


def test_frag_path_info(tmp_path):
  path = _layer(tmp_path)
  plain = str(tmp_path / "frags")
  list(tc.create_skeletonizing_tasks(path, mip=0, shape=(128, 128, 64), frag_path=plain))
  assert CloudFiles(plain).get_json("info") == CloudFiles(path).get_json("skeletons_mip_0/info")
  # a frag_path holding a volume gets the info under the layer's skeleton directory
  other = _layer(tmp_path, name="other")
  t = list(tc.create_skeletonizing_tasks(path, mip=0, shape=(128, 128, 64), frag_path=other))[0]
  assert CloudFiles(other).get_json("skeletons_mip_0/info") == CloudFiles(path).get_json("skeletons_mip_0/info")
  vol = CloudVolume(path)
  assert t.fragment_path(vol) == CloudFiles(other).join(other, "skeletons_mip_0")
  t.frag_path = plain
  assert t.fragment_path(vol) == plain
  t.frag_path = None
  assert t.fragment_path(vol) == path + "/skeletons_mip_0"


@pytest.mark.parametrize("option", [
  dict(sharded=True), dict(dust_global=True), dict(synapses=[((1, 2, 3), 5, 1)]), dict(cross_sectional_area=True),
  dict(fix_autapses=True), dict(timestamp=12345), dict(root_ids_cloudpath="file:///x"), dict(fix_avocados=True),
  dict(fill_holes=1)])
def test_refusals(tmp_path, option):
  path = _layer(tmp_path)
  with pytest.raises(NotImplementedError, match="igneous_b200 create_skeletonizing_tasks"):
    tc.create_skeletonizing_tasks(path, mip=0, **option)
  assert "skeletons" not in CloudVolume(path).info  # refused before any write
  with pytest.raises(NotImplementedError, match="igneous_b200 SkeletonTask"):
    tasks.SkeletonTask(path, (64, 64, 64), (0, 0, 0), 0, {}, False, **option)


def test_import_surface():
  assert igneous_b200.SkeletonTask is tasks.SkeletonTask
  assert "SkeletonTask" in igneous_b200.__all__
  from igneous_b200.kimimaro import export_skeletons, skeletonize  # noqa: F401
  t = tasks.SkeletonTask("file:///x", (65, 65, 65), (1, 2, 3), 0, {}, True, spatial_grid_shape=(64, 64, 64),
                         progress=True, parallel=4)
  assert list(map(int, t.bounds.maxpt)) == [66, 67, 68] and list(map(int, t.index_bounds.maxpt)) == [65, 66, 67]
  assert t.strip_integer_attributes is True and t.spatial_index is True and t.dry_run is False


@pytest.mark.parametrize("attributes", ["default", "radius_only"])
def test_skeleton_get_decodes_the_info_attributes(tmp_path, attributes):
  path = _layer(tmp_path)
  vol = CloudVolume(path)
  vol.info["skeletons"] = "sk"
  vol.commit_info()
  rng = np.random.default_rng(5)
  v = rng.normal(size=(7, 3)).astype(np.float32)
  e = np.array([[0, 1], [1, 2], [2, 3], [3, 4], [4, 5], [5, 6]], np.uint32)
  r = rng.random(7).astype(np.float32)
  t = np.arange(7, dtype=np.uint8)
  if attributes == "radius_only":
    CloudFiles(path).put_json("sk/info", {"@type": "neuroglancer_skeletons", "vertex_attributes": [
      {"id": "radius", "data_type": "float32", "num_components": 1}]})
    blob = encode(v, e, [r])
  else:  # no info file: cloudvolume's default attributes
    blob = encode(v, e, [r, t])
  CloudFiles(path).put("sk/2", blob, compress="gzip")
  assert os.path.exists(str(tmp_path / "seg" / "sk" / "2.gz"))
  s = CloudVolume(path).skeleton.get(2)
  assert s.id == 2 and np.array_equal(s.vertices, v) and np.array_equal(s.edges, e) and np.array_equal(s.radii, r)
  assert s.vertices.dtype == np.float32 and s.edges.dtype == np.uint32 and s.vertex_types.dtype == np.uint8
  assert np.array_equal(s.vertex_types, t if attributes == "default" else np.zeros(7, np.uint8))
  assert CloudVolume(path).skeleton.path == path + "/sk"
  CloudFiles(path).put("sk/3", gzip.decompress(gzip.compress(blob))[:-3])
  with pytest.raises(ValueError):
    CloudVolume(path).skeleton.get(3)
  with pytest.raises(FileNotFoundError):
    CloudVolume(path).skeleton.get(4)
