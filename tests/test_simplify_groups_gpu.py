"""E2 of k_simp_labels gives each winner one group of 8 lanes (16 or 32 when a ring holds more than 8 or 16
faces), which runs its flip tests, link condition, collapse and re-costs with no barrier in between.
IGN_SIMP_GROUP=16|32 sets the narrowest group, so that the wider sweeps take every winner.  Meshes stay
bit-identical to the oracle for every group width and selection-pass cap, on shared-memory, hybrid and
global-memory labels and on labels that migrate between size classes; the counters do not depend on the
width, and ign_mesh_simplify_groups shows which sweeps ran."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

GROUPS = (None, 16, 32)


def _setenv(monkeypatch, name, value):
  if value is None:
    monkeypatch.delenv(name, raising=False)
  else:
    monkeypatch.setenv(name, str(value))


def _counters(m, fn, n):
  from igneous_b200 import _shim
  out = (ctypes.c_uint32 * n)()
  _shim.check(getattr(m._ctx.lib, fn)(m._handle, out))
  return list(out)


def _simplified(seg, res, factor, max_error, centered):
  from igneous_b200 import zmesh
  m = zmesh.Mesher(res)
  m.mesh(seg)
  meshes = {int(i): m.get(i, reduction_factor=factor, max_error=max_error, voxel_centered=centered) for i in m.ids()}
  counters = {fn: _counters(m, fn, n) for fn, n in (("ign_mesh_simplify_stats", 6), ("ign_mesh_simplify_costs", 3),
                                                   ("ign_mesh_simplify_passes", 2), ("ign_mesh_simplify_migrations", 3))}
  return meshes, counters, _counters(m, "ign_mesh_simplify_groups", 3)


_WANT = {}


def _run(oracle, monkeypatch, name, seg, res, factor, max_error, centered, wcap):
  key = (name, factor, max_error)
  if key not in _WANT:
    tl, tv = oracle.marching_cubes(seg)
    _WANT[key] = oracle.simplify_welded(oracle.WeldedMeshes(tl, tv), res, factor, max_error, centered)[0]
  want = _WANT[key]
  monkeypatch.delenv("IGN_SIMP_GMEM", raising=False)
  _setenv(monkeypatch, "IGN_SIMP_WCAP", wcap)
  runs = {}
  try:
    for g in GROUPS:
      _setenv(monkeypatch, "IGN_SIMP_GROUP", g)
      got, counters, groups = _simplified(seg, res, factor, max_error, centered)
      assert got.keys() == want.keys(), g
      for k in want:
        wv, wf = want[k]
        assert np.array_equal(got[k].vertices, wv) and np.array_equal(got[k].faces, wf), (g, k)
      runs[g] = (counters, groups)
  finally:
    monkeypatch.delenv("IGN_SIMP_GROUP", raising=False)
    monkeypatch.delenv("IGN_SIMP_WCAP", raising=False)
  counters, groups = runs[None]
  for g in GROUPS:
    assert runs[g][0] == counters, (g, runs[g][0], counters)
    assert sum(runs[g][1]) == sum(groups), (g, runs[g][1], groups)  # the same winners, whatever the width
  assert groups[0] > 0, groups
  assert runs[16][1][0] == 0 and runs[16][1][1] > 0, runs[16][1]
  assert runs[32][1][:2] == [0, 0] and runs[32][1][2] == sum(groups), runs[32][1]
  return counters, groups


@pytest.fixture(scope="module")
def bench_block(oracle):
  # a 129^3 block of the benchmark's mip-2 MeshTask volume: synth_seg pitch 64, seed 0, two 2x2x1 mode mips
  seg = oracle.synth_seg((516, 516, 129), pitch=64, num_ids=1 << 20, seed=0)
  return np.asfortranarray(oracle.downsample_segmentation(seg, (2, 2, 1), num_mips=2)[1].astype(np.uint32))


@pytest.mark.parametrize("wcap", [None, 8])
def test_groups_bench_block(ctx, oracle, monkeypatch, bench_block, wcap):
  _, groups = _run(oracle, monkeypatch, "bench", bench_block, (16, 16, 40), 100, 40.0, True, wcap)
  assert groups[1] + groups[2] > 0, groups  # rings over 8 faces took the wider sweeps


@pytest.mark.parametrize("wcap", [None, 8])
def test_groups_migrating_labels(ctx, oracle, monkeypatch, bench_block, wcap):
  # factor 10: labels shrink into the 512- and 256-thread classes and resume there
  counters, _ = _run(oracle, monkeypatch, "bench", bench_block, (16, 16, 40), 10, 8.0, True, wcap)
  resumed = counters["ign_mesh_simplify_migrations"]
  assert resumed[1] > 0 and resumed[2] > 0, resumed


@pytest.mark.parametrize("wcap", [None, 8])
def test_groups_size_classes(ctx, oracle, monkeypatch, wcap):
  # 57 labels from 490 to 35,550 faces, in all three size classes and on the global-memory path
  seg = np.asfortranarray(oracle.synth_seg((128, 128, 96), pitch=32, num_ids=64).astype(np.uint32))
  counters, _ = _run(oracle, monkeypatch, "classes", seg, (16, 16, 40), 100, 40.0, True, wcap)
  stats = counters["ign_mesh_simplify_stats"]
  assert min(stats[3:]) > 0 and stats[2] > 0, stats


# a closed box of (n - 2)^3 voxels: its faces in shared memory (n = 30), in global memory with keys, flags and
# states in shared memory (hybrid, n = 40), or everything in global memory (n = 64)
@pytest.mark.parametrize("wcap", [None, 8])
@pytest.mark.parametrize("n,memory", [(30, [1, 0]), (40, [0, 1]), (64, [0, 1])])
def test_groups_box(ctx, oracle, monkeypatch, n, memory, wcap):
  data = np.zeros((n, n, n), dtype=np.uint32, order="F")
  data[1:-1, 1:-1, 1:-1] = 1
  counters, _ = _run(oracle, monkeypatch, "box%d" % n, data, (1, 1, 1), 100, 40.0, False, wcap)
  assert counters["ign_mesh_simplify_stats"][1:3] == memory, counters
