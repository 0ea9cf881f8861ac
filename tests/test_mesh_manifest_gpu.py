"""The legacy mesh stage end to end: a 2x2x2 grid of GPU MeshTasks over a segmentation whose labels cross the
task faces, then the manifest merge, a transfer to a second layer and the deletion of the mesh directory
(DESIGN.md §5m)."""
import json
import os
import re

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SHAPE = (128, 128, 128)
TASK = (64, 64, 64)


def files(root):
  out = {}
  for d, _, fs in os.walk(root):
    for f in fs:
      with open(os.path.join(d, f), "rb") as fh:
        out[os.path.relpath(os.path.join(d, f), root)] = fh.read()
  return out


def test_mesh_grid_manifests_transfer_and_deletion(ctx, oracle, tmp_path):
  import igneous_b200.task_creation as tc
  from igneous_b200 import tasks, zmesh
  from igneous_b200._compat import CloudFiles, CloudVolume, LocalTaskQueue
  seg = oracle.synth_seg(SHAPE, pitch=16, num_ids=150, seed=3)  # labels 1-150: one to three digits
  src = "file://" + str(tmp_path / "src")
  CloudVolume.from_numpy(seg, src, resolution=(1, 1, 1), chunk_size=(64, 64, 64), layer_type="segmentation")
  grid = tc.create_meshing_tasks(src, mip=0, shape=TASK, mesh_dir="mesh")
  assert len(grid) == 8
  LocalTaskQueue().insert_all(grid)
  cf = CloudFiles(src)

  fragments = {}  # label -> its fragment names, as stored without the .gz suffix
  for name in cf.list("mesh/"):
    m = re.fullmatch(r"mesh/(\d+):0:(\d+)-(\d+)_(\d+)-(\d+)_(\d+)-(\d+)", name)
    if m:
      fragments.setdefault(int(m.group(1)), set()).add(name[len("mesh/"):])
  # every label meshed in a task's own box has that task's fragment, and no label outside its box (with the
  # one voxel of high padding) does
  for off in np.ndindex(2, 2, 2):
    lo = np.asarray(off) * np.asarray(TASK)
    core = set(np.unique(seg[lo[0]:lo[0] + 64, lo[1]:lo[1] + 64, lo[2]:lo[2] + 64]).tolist()) - {0}
    padded = set(np.unique(seg[lo[0]:lo[0] + 65, lo[1]:lo[1] + 65, lo[2]:lo[2] + 65]).tolist()) - {0}
    box = "%d-%d_%d-%d_%d-%d" % (lo[0], lo[0] + 64, lo[1], lo[1] + 64, lo[2], lo[2] + 64)
    meshed = {l for l, names in fragments.items() if "%d:0:%s" % (l, box) in names}
    assert core <= meshed <= padded
  # labels cross task faces, so several tasks mesh them
  assert all(np.any((np.take(seg, 63, a) == np.take(seg, 64, a)) & (np.take(seg, 64, a) != 0)) for a in range(3))
  assert max(len(v) for v in fragments.values()) >= 2
  assert any(l < 10 for l in fragments) and any(l >= 100 for l in fragments)

  (merge,) = tc.create_mesh_manifest_tasks(src)
  LocalTaskQueue().insert_all([merge])
  manifests = {}
  for label, names in fragments.items():
    got = cf.get_json("mesh/%d:0" % label)["fragments"]
    assert len(got) == len(set(got)) and set(got) == names, label
    manifests[label] = got
    for name in got:
      mesh = zmesh.Mesh.from_precomputed(cf.get("mesh/" + name))
      assert len(mesh.faces) > 0 and len(mesh.vertices) > 0
  assert sorted(n for n in cf.list("mesh/") if re.fullmatch(r"mesh/\d+:0", n)) == \
      sorted("mesh/%d:0" % l for l in fragments)

  # the prefix route writes the same manifests, in listing order
  for label in fragments:
    cf.delete("mesh/%d:0" % label)
  for t in tc.create_mesh_manifest_tasks("gs://bucket/layer"):
    tasks.MeshManifestPrefixTask(src, t.keywords["prefix"])
  for label, got in manifests.items():
    assert cf.get_json("mesh/%d:0" % label)["fragments"] == sorted(got)

  dest = "file://" + str(tmp_path / "dest")
  CloudVolume.from_numpy(np.zeros(SHAPE, np.uint32), dest, resolution=(1, 1, 1), chunk_size=(64, 64, 64),
                         layer_type="segmentation")
  vol = CloudVolume(dest)
  vol.info["mesh"] = "copied"
  vol.commit_info()
  LocalTaskQueue().insert_all(tc.create_xfer_meshes_tasks(src, dest))
  src_files, dest_files = files(str(tmp_path / "src" / "mesh")), files(str(tmp_path / "dest" / "copied"))
  # an unsharded transfer misses the spatial index files whose first coordinate has one digit
  missed = {n for n in src_files if re.fullmatch(r"0-64_\d+-\d+_\d+-\d+\.spatial\.gz", n)}
  assert len(missed) == 4
  assert set(dest_files) == set(src_files) - missed
  assert all(dest_files[n] == src_files[n] for n in dest_files)
  assert json.loads(dest_files["info"])["@type"] == "neuroglancer_legacy_mesh"

  LocalTaskQueue().insert_all(tc.create_mesh_deletion_tasks(src))
  # at magnitude 3 the deletion leaves the spatial index files whose first coordinate is 64
  left = set(files(str(tmp_path / "src" / "mesh")))
  assert left == {n for n in src_files if n.startswith("64-128_") and n.endswith(".spatial.gz")}
  assert len(left) == 4
