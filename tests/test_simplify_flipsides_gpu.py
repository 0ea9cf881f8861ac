"""E2 of k_simp_labels flip-tests the faces of both rings of a winner that survive the collapse; a flip on
either side rejects the winner.  The re-costs after a collapse take the kept vertex's new quadric and position
from the lane group's registers (sl_recost_k) instead of reloading them.  The IGN_SIMP_TRACE summary counts
the winners rejected by flips on the u side only, the v side only and both.  Meshes stay bit-identical to the
oracle at every group width (IGN_SIMP_GROUP=8|16|32), and neither the simplifier counters nor the
rejections depend on the width."""
import ctypes
import re

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

_FLIPS = re.compile(r"winners rejected by E2 flip tests: (\d+) on the u side only, (\d+) on the v side only, (\d+) on both")


def _counters(m, fn, n):
  from igneous_b200 import _shim
  out = (ctypes.c_uint32 * n)()
  _shim.check(getattr(m._ctx.lib, fn)(m._handle, out))
  return list(out)


@pytest.fixture(scope="module")
def bench_block(oracle):
  # a 129^3 block of the benchmark's mip-2 MeshTask volume: synth_seg pitch 64, seed 0, two 2x2x1 mode mips
  seg = oracle.synth_seg((516, 516, 129), pitch=64, num_ids=1 << 20, seed=0)
  return np.asfortranarray(oracle.downsample_segmentation(seg, (2, 2, 1), num_mips=2)[1].astype(np.uint32))


@pytest.fixture(scope="module")
def bench_want(oracle, bench_block):
  tl, tv = oracle.marching_cubes(bench_block)
  return oracle.simplify_welded(oracle.WeldedMeshes(tl, tv), (16, 16, 40), 100, 40.0, True)[0]


_RUNS = {}


def _run(monkeypatch, capfd, seg, want, group):
  """Simplify `seg` at the narrowest group width `group` with the trace on; check every mesh against the
  oracle and return the counters and the flip-test trace (rejected u side only, v side only, both)."""
  from igneous_b200 import zmesh
  if group in _RUNS:
    return _RUNS[group]
  monkeypatch.delenv("IGN_SIMP_GMEM", raising=False)
  monkeypatch.delenv("IGN_SIMP_WCAP", raising=False)
  monkeypatch.setenv("IGN_SIMP_GROUP", str(group))
  monkeypatch.setenv("IGN_SIMP_TRACE", "1")
  capfd.readouterr()
  try:
    m = zmesh.Mesher((16, 16, 40))
    m.mesh(seg)
    got = {int(i): m.get(i, reduction_factor=100, max_error=40.0, voxel_centered=True) for i in m.ids()}
  finally:
    monkeypatch.delenv("IGN_SIMP_GROUP", raising=False)
    monkeypatch.delenv("IGN_SIMP_TRACE", raising=False)
  err = capfd.readouterr().err
  assert got.keys() == want.keys(), group
  for k in want:
    wv, wf = want[k]
    assert np.array_equal(got[k].vertices, wv) and np.array_equal(got[k].faces, wf), (group, k)
  counters = {fn: _counters(m, fn, n) for fn, n in (("ign_mesh_simplify_stats", 6), ("ign_mesh_simplify_costs", 3),
                                                   ("ign_mesh_simplify_passes", 2), ("ign_mesh_simplify_migrations", 3))}
  groups = _counters(m, "ign_mesh_simplify_groups", 3)
  lines = _FLIPS.findall(err)
  assert lines, err[-2000:]
  flips = [sum(int(x[i]) for x in lines) for i in range(3)]
  _RUNS[group] = (counters, groups, flips)
  return _RUNS[group]


@pytest.mark.parametrize("group", [8, 16, 32])
def test_flipsides_bench_block(ctx, monkeypatch, capfd, bench_block, bench_want, group):
  counters, groups, flips = _run(monkeypatch, capfd, bench_block, bench_want, group)
  ref_counters, ref_groups, ref_flips = _run(monkeypatch, capfd, bench_block, bench_want, 8)
  assert counters == ref_counters, (group, counters, ref_counters)
  assert sum(groups) == sum(ref_groups), (group, groups, ref_groups)
  assert flips == ref_flips, (group, flips, ref_flips)  # the same winners flip, whatever the width
  assert counters["ign_mesh_simplify_costs"][1] > 0 and counters["ign_mesh_simplify_costs"][2] == 0, counters


def test_flipsides_one_sided_rejections(ctx, monkeypatch, capfd, bench_block, bench_want):
  # winners rejected only by a flip of a u-side face, and only by one of a v-side face
  _, _, flips = _run(monkeypatch, capfd, bench_block, bench_want, 8)
  assert flips[0] > 0 and flips[1] > 0, flips
