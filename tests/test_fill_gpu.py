"""ign_fill_holes / ign_dilate_multilabel (fastmorph shim) bit-exact against the serial C oracle
(oracle_fill/) and, on the hand-built volumes, the numpy transcription (tests/fillref.py); and
MeshTask(fill_holes=N) end to end."""
import numpy as np
import pytest

import fillref as F
import oracle_fill as C

pytestmark = pytest.mark.gpu

LEVELS = (1, 2, 3, 4, 50, 103)


def _gpu_level(X, level):
  from igneous_b200 import fastmorph
  X0 = fastmorph.dilate(X) if level >= 3 else X
  return fastmorph.fill_holes_v2(X0, fix_borders=level >= 2,
                                 merge_threshold=1.0 if level <= 3 else 1.0 - 0.01 * (level - 3))


def _check(X, level, numpy_ref=False):
  got_f, got_h = _gpu_level(X, level)
  refs = [C.fill_level(X, level)] + ([F.fill_level(X, level)] if numpy_ref else [])
  assert got_f.dtype == X.dtype and got_h.dtype == X.dtype
  for want_f, want_h in refs:
    assert np.array_equal(got_f, want_f), ("filled", level, int((got_f != want_f).sum()))
    assert np.array_equal(got_h, want_h), ("holes", level, int((got_h != want_h).sum()))


@pytest.mark.parametrize("name", sorted(F.kats()))
def test_kats_bit_exact(ctx, name):
  X = F.kats()[name]
  for level in LEVELS + (12, 13):
    _check(X, level, numpy_ref=True)


def test_two_cycle_at_60_percent(ctx):
  from igneous_b200 import fastmorph
  X = F.kats()["cycle2"]
  got = fastmorph.fill_holes_v2(X, merge_threshold=0.40)
  want = C.fill_holes(X, p=60)
  assert np.array_equal(want[0], F.fill_holes(X, p=60)[0])
  assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
  assert (got[0][X == 2] == 1).all()


def test_dilate_bit_exact(ctx):
  from igneous_b200 import fastmorph
  rng = np.random.default_rng(0)
  for shape in ((5, 5, 5), (33, 17, 9), (70, 1, 13), (1, 1, 40)):
    for dtype in (np.uint8, np.uint16, np.uint32, np.uint64):
      X = rng.integers(1, 4, size=shape).astype(dtype)
      X[rng.random(shape) < 0.6] = 0
      X = np.asfortranarray(X)
      assert np.array_equal(fastmorph.dilate(X), C.dilate(X)), (shape, dtype)
      assert np.array_equal(fastmorph.dilate(X), F.dilate(X)), (shape, dtype)


def _as(X, dtype):
  if dtype == np.uint8:
    return np.asfortranarray(np.where(X == 0, 0, X % 251 + 1).astype(dtype))
  if dtype == np.uint16:
    return np.asfortranarray(np.where(X == 0, 0, X % 65000 + 1).astype(dtype))
  return np.asfortranarray(X.astype(dtype))


@pytest.mark.parametrize("shape,dtype", [
  ((17, 17, 17), np.uint32), ((64, 64, 64), np.uint16), ((65, 33, 17), np.uint8), ((40, 1, 30), np.uint32),
  ((1, 37, 29), np.uint16), ((97, 80, 71), np.uint32), ((129, 129, 129), np.uint32), ((100, 90, 80), np.uint64)])
def test_random_volumes(ctx, shape, dtype):
  X = _as(F.random_volume(shape, seed=sum(shape)), dtype)
  for level in LEVELS:
    _check(X, level)


def test_random_259_cubed(ctx):
  X = F.random_volume((259, 259, 259), seed=259, pitch=16)
  for level in (1, 2, 4, 103):
    _check(X, level)


def test_u64_extremes(ctx):
  from igneous_b200 import fastmorph
  X = F.kats()["organelle_floating"].astype(np.uint64)
  X[X == 3] = (1 << 64) - 2
  X[X == 7] = 1 << 40
  f, h = fastmorph.fill_holes_v2(X)
  wf, wh = C.fill_holes(X)
  assert np.array_equal(f, wf) and np.array_equal(h, wh) and (h == (1 << 40)).sum() == 8
  X[0, 0, 0] = (1 << 64) - 1
  with pytest.raises(NotImplementedError):
    fastmorph.fill_holes_v2(X)


def _layer(tmp_path, data):
  from igneous_b200._compat import CloudVolume
  path = "file://" + str(tmp_path / "layer")
  CloudVolume.from_numpy(data, vol_path=path, resolution=(1, 1, 1), voxel_offset=(0, 0, 0), chunk_size=(64, 64, 64),
                         layer_type="segmentation", max_mip=0)
  cv = CloudVolume(path)
  cv.info["mesh"] = "mesh"
  cv.commit_info()
  return path


def _euler(mesh):
  f = mesh.faces.astype(np.int64)
  e = np.sort(np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]), axis=1)
  edges = np.unique(e[:, 0] * (1 << 32) + e[:, 1]).size
  return len(np.unique(f)) - edges + len(f)


def _cell_with_organelle():
  x, y, z = np.meshgrid(*[np.arange(64)] * 3, indexing="ij")
  d = np.sqrt((x - 31.5) ** 2 + (y - 31.5) ** 2 + (z - 31.5) ** 2)
  data = np.zeros((64, 64, 64, 1), dtype=np.uint32)
  data[(d < 24) & (d >= 18), 0] = 5     # hollow cell L
  data[d < 8, 0] = 9                    # organelle M floating in the cavity
  return data


def test_mesh_task_fill_holes(ctx, tmp_path):
  from igneous_b200.tasks import MeshTask
  from igneous_b200._compat import CloudFiles
  from igneous_b200 import zmesh
  path = _layer(tmp_path, _cell_with_organelle())
  cf = CloudFiles(path)
  frags = {}
  for level in (0, 1):
    for simp in (0, 100):
      d = "m%d_%d" % (level, simp)
      MeshTask(shape=(64, 64, 64), offset=(0, 0, 0), layer_path=path, mip=0, fill_holes=level,
               simplification_factor=simp, mesh_dir=d).execute()
      frags[level, simp] = {seg: cf.get("%s/%d:0:0-64_0-64_0-64" % (d, seg)) for seg in (5, 9)}
  assert _euler(zmesh.Mesh.from_precomputed(frags[0, 0][5])) == 4   # outer and inner surface of the shell
  assert _euler(zmesh.Mesh.from_precomputed(frags[1, 0][5])) == 2   # the cavity is filled: one surface
  for simp in (0, 100):
    assert frags[1, simp][9] is not None and frags[0, simp][9] == frags[1, simp][9]


def test_create_meshing_tasks_fill_holes_2(ctx, tmp_path):
  import igneous_b200.task_creation as tc
  from igneous_b200._compat import CloudFiles, LocalTaskQueue
  data = _cell_with_organelle()
  data[2:6, 2:6, 2:6, 0] = 3            # a solid object with nothing to fill
  path = _layer(tmp_path, data)
  tasks = tc.create_meshing_tasks(path, mip=0, shape=(32, 64, 64), fill_holes=2, mesh_dir="mf")
  assert len(tasks) == 2
  LocalTaskQueue().insert_all(tasks)
  names = CloudFiles(path).list("mf/")
  for want in ("mf/3:0:0-32_0-64_0-64", "mf/5:0:0-32_0-64_0-64", "mf/5:0:32-64_0-64_0-64",
               "mf/9:0:0-32_0-64_0-64", "mf/9:0:32-64_0-64_0-64"):
    assert want in names, (want, names)


def test_mesh_task_fill_holes_concatenates_hole_and_filled_meshes(ctx, tmp_path):
  """Label 9 has one component inside the cell (a hole) and one outside it (stays in filled):
  its fragment is the filled mesh with the hole mesh appended (Mesh.concatenate, mesh.py:237-241).
  Unsimplified, that is the same triangles as meshing both components together at level 0."""
  from igneous_b200.tasks import MeshTask
  from igneous_b200._compat import CloudFiles
  from igneous_b200 import zmesh
  data = _cell_with_organelle()
  data[52:60, 52:60, 52:60, 0] = 9      # a second, visible component of the organelle's label
  path = _layer(tmp_path, data)
  cf = CloudFiles(path)
  got = {}
  for level in (0, 1):
    MeshTask(shape=(64, 64, 64), offset=(0, 0, 0), layer_path=path, mip=0, fill_holes=level,
             simplification_factor=0, mesh_dir="c%d" % level).execute()
    got[level] = zmesh.Mesh.from_precomputed(cf.get("c%d/9:0:0-64_0-64_0-64" % level))
  assert _euler(got[1]) == 4           # two closed surfaces in one fragment
  tri = {lv: sorted(tuple(sorted(map(tuple, t.tolist()))) for t in m.vertices[m.faces]) for lv, m in got.items()}
  assert len(got[0].faces) == len(got[1].faces) and tri[0] == tri[1]
  # the filled component comes first, the hole component is appended
  n_out = int((got[1].vertices.min(axis=1) > 45).sum())
  assert n_out > 0 and (got[1].vertices[:n_out].min(axis=1) > 45).all()
