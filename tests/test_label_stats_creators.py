"""The spatial-index and voxel-counting task creators on the file:// stand-in: task counts,
shapes and offsets, the mesh and skeleton info edits, default directory names and provenance.
Nothing here runs a kernel."""
import numpy as np

from igneous_b200 import task_creation as tc
from igneous_b200._compat import CloudFiles, CloudVolume


def _layer(tmp_path, shape=(300, 200, 70), offset=(10, 20, 3), resolution=(4, 4, 40), name="seg"):
  path = "file://" + str(tmp_path / name)
  info = CloudVolume.create_new_info(1, "segmentation", np.uint64, "raw", resolution, offset, shape, (64, 64, 32))
  CloudVolume(path, info=info).commit_info()
  return path


def test_spatial_index_mesh_tasks_grid_and_info(tmp_path):
  path = _layer(tmp_path)
  itr = tc.create_spatial_index_mesh_tasks(path, shape=(128, 128, 64), compress=None)
  assert len(itr) == 3 * 2 * 2
  got = list(itr)
  kw = [t.keywords for t in got]
  assert [list(map(int, k["offset"])) for k in kw[:4]] == [[10, 20, 3], [138, 20, 3], [266, 20, 3], [10, 148, 3]]
  assert all(list(map(int, k["shape"])) == [128, 128, 64] for k in kw)
  assert all(k["subdir"] == "mesh_mip_0_err_40" and k["precision"] == 0 and k["mip"] == 0 and
             k["fill_missing"] is False and k["compress"] is None and k["cloudpath"] == path for k in kw)
  assert all(t.func.__name__ == "SpatialIndexTask" for t in got)
  vol = CloudVolume(path)
  assert vol.info["mesh"] == "mesh_mip_0_err_40"
  assert CloudFiles(path).get_json("mesh_mip_0_err_40/info") == {
    "@type": "neuroglancer_legacy_mesh", "mip": 0, "chunk_size": [128, 128, 64],
    "spatial_index": {"resolution": [4, 4, 40], "chunk_size": [512, 512, 2560]}}
  prov = vol.provenance.processing[-1]["method"]
  assert prov == {"task": "SpatialIndexTask", "cloudpath": path, "shape": [128, 128, 64], "mip": 0,
                  "subdir": "mesh_mip_0_err_40", "fill_missing": False, "compress": None}


def test_spatial_index_mesh_tasks_keep_existing_directory_and_type(tmp_path):
  path = _layer(tmp_path)
  vol = CloudVolume(path)
  vol.info["mesh"] = "meshes"
  vol.commit_info()
  cf = CloudFiles(path)
  cf.put_json("meshes/info", {"@type": "neuroglancer_multilod_draco", "mip": 2, "vertex_quantization_bits": 16})
  list(tc.create_spatial_index_mesh_tasks(path, shape=(448, 448, 448), mip=0))
  info = cf.get_json("meshes/info")
  assert info["@type"] == "neuroglancer_multilod_draco" and info["mip"] == 2 and info["vertex_quantization_bits"] == 16
  assert info["chunk_size"] == [448, 448, 448]
  assert info["spatial_index"] == {"resolution": [4, 4, 40], "chunk_size": [1792, 1792, 17920]}
  # an explicit directory wins, but the layer's own entry is left as it was
  list(tc.create_spatial_index_mesh_tasks(path, mesh_dir="other"))
  assert CloudVolume(path).info["mesh"] == "meshes"
  assert cf.get_json("other/info")["@type"] == "neuroglancer_legacy_mesh"


def test_spatial_index_info_written_only_on_change(tmp_path):
  path = _layer(tmp_path)
  tc.create_spatial_index_skeleton_tasks(path, shape=(100, 100, 100))
  fn = str(tmp_path / "seg" / "skeletons_mip_0" / "info")
  before = open(fn, "rb").read()
  import os
  os.utime(fn, (0, 0))
  tc.create_spatial_index_skeleton_tasks(path, shape=(100, 100, 100))
  assert os.path.getmtime(fn) == 0 and open(fn, "rb").read() == before
  tc.create_spatial_index_skeleton_tasks(path, shape=(50, 100, 100))
  assert os.path.getmtime(fn) != 0


def test_spatial_index_skeleton_tasks(tmp_path):
  path = _layer(tmp_path, resolution=(8, 8, 40))
  vol = CloudVolume(path)
  vol.add_resolution((16, 16, 40))
  vol.commit_info()
  itr = tc.create_spatial_index_skeleton_tasks(path, mip=1, fill_missing=True)
  assert len(itr) == 1  # mip 1 is 150 x 100 x 70, inside one 448^3 task
  (t,) = list(itr)
  assert t.keywords["subdir"] == "skeletons_mip_1" and t.keywords["mip"] == 1 and t.keywords["fill_missing"] is True
  assert t.keywords["compress"] == "gzip"
  assert list(map(int, t.keywords["offset"])) == [5, 10, 3]
  vol = CloudVolume(path)
  assert vol.info["skeletons"] == "skeletons_mip_1"
  assert vol.skeleton.spatial_index is vol.mesh.spatial_index
  assert CloudFiles(path).get_json("skeletons_mip_1/info") == {
    "@type": "neuroglancer_skeletons", "mip": 1, "chunk_size": [448, 448, 448],
    "spatial_index": {"resolution": [16, 16, 40], "chunk_size": [7168, 7168, 17920]}}
  method = vol.provenance.processing[-1]["method"]
  assert method["task"] == "SpatialIndexTask" and method["subdir"] == "skeletons_mip_1" and method["mip"] == 1


def test_voxel_counting_tasks(tmp_path):
  path = _layer(tmp_path, shape=(1100, 520, 70), offset=(-3, 5, 0))
  itr = tc.create_voxel_counting_tasks(path, mip=0, fill_missing=True, agglomerate=True, timestamp=17)
  assert len(itr) == 3 * 2 * 1
  got = list(itr)
  kw = [t.keywords for t in got]
  assert [list(map(int, k["offset"])) for k in kw] == [[-3, 5, 0], [509, 5, 0], [1021, 5, 0],
                                                     [-3, 517, 0], [509, 517, 0], [1021, 517, 0]]
  assert [list(map(int, k["shape"])) for k in kw] == [[512, 512, 70], [512, 512, 70], [76, 512, 70],
                                                    [512, 8, 70], [512, 8, 70], [76, 8, 70]]
  assert all(k["agglomerate"] is True and k["timestamp"] == 17 and k["fill_missing"] is True and k["mip"] == 0
             for k in kw)
  assert all(t.func.__name__ == "CountVoxelsTask" for t in got)
  method = CloudVolume(path).provenance.processing[-1]["method"]
  assert method == {"task": "CountVoxelsTask", "cloudpath": path, "mip": 0, "shape": [512, 512, 512],
                    "fill_missing": True, "agglomerate": True, "timestamp": 17}


def test_import_surface():
  import igneous_b200
  from igneous_b200 import tasks
  assert igneous_b200.SpatialIndexTask is tasks.SpatialIndexTask
  assert igneous_b200.CountVoxelsTask is tasks.CountVoxelsTask
  for name in ("create_spatial_index_mesh_tasks", "create_spatial_index_skeleton_tasks",
               "create_voxel_counting_tasks"):
    assert callable(getattr(tc, name))
