"""The simplifier caches each edge's cost in the format of the label's key.  A label whose 3T half-edge ids fit
16 bits (3T <= 65536: 32-bit keys) keeps only the key's 16 cost bits, three per face in one 8-byte word; a
larger label (64-bit keys) keeps the float costs.  Labels on both sides of the boundary (3T = 65,535 and
65,538) run next to a shared-memory label that migrates to smaller size classes, with their topology in
shared memory / hybrid and with IGN_SIMP_GMEM=1 in global memory; the meshes stay bit-identical to the
oracle and the key pass never meets an edge without a cost."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _simplified(seg, factor, max_error):
  from igneous_b200 import _shim, zmesh
  m = zmesh.Mesher((16, 16, 40))
  m.mesh(seg)
  meshes = {int(i): m.get(i, reduction_factor=factor, max_error=max_error, voxel_centered=True) for i in m.ids()}
  stats = (ctypes.c_uint32 * 6)()
  _shim.check(m._ctx.lib.ign_mesh_simplify_stats(m._handle, stats))
  resumed = (ctypes.c_uint32 * 3)()
  _shim.check(m._ctx.lib.ign_mesh_simplify_migrations(m._handle, resumed))
  costs = (ctypes.c_uint32 * 3)()
  _shim.check(m._ctx.lib.ign_mesh_simplify_costs(m._handle, costs))
  return meshes, list(stats), list(resumed), list(costs)


def _volume(dents):
  # label 1: a 40 x 40 x 119 box in the volume's corner (an open surface: its face count can be odd), with
  # voxels taken out of its corner edges to set the count; label 2: a closed 28^3 box (9,404 faces)
  seg = np.zeros((72, 44, 124), dtype=np.uint32, order="F")
  seg[0:40, 0:40, 0:119] = 1
  for p in dents:
    seg[p] = 0
  seg[42:70, 8:36, 20:48] = 2
  return seg


@pytest.mark.parametrize("factor,max_error", [(100, 40.0), (10, 8.0)])
@pytest.mark.parametrize("dents,three_t", [([(0, 0, 20)], 65535), ([(0, 0, 0), (39, 0, 0)], 65538)])
def test_cost_format_boundary_bit_exact(ctx, oracle, monkeypatch, dents, three_t, factor, max_error):
  seg = _volume(dents)
  tl, tv = oracle.marching_cubes(seg)
  W = oracle.WeldedMeshes(tl, tv)
  assert W.ids() == [1, 2]
  assert [int(3 * (b - a)) for a, b in zip(W.f0, W.f1)] == [three_t, 28212]
  want, _ = oracle.simplify_welded(W, (16, 16, 40), factor, max_error, True)
  monkeypatch.delenv("IGN_SIMP_WCAP", raising=False)
  for gmem in (False, True):
    if gmem:
      monkeypatch.setenv("IGN_SIMP_GMEM", "1")
    else:
      monkeypatch.delenv("IGN_SIMP_GMEM", raising=False)
    got, st, resumed, costs = _simplified(seg, factor, max_error)
    monkeypatch.delenv("IGN_SIMP_GMEM", raising=False)
    assert got.keys() == want.keys()
    for k in want:
      wv, wf = want[k]
      assert np.array_equal(got[k].vertices, wv) and np.array_equal(got[k].faces, wf), (k, gmem)
    assert costs[2] == 0, costs  # the key pass never meets an edge without a cost
    if gmem:
      assert st[1:3] == [0, 2] and resumed == [0, 0, 0], (st, resumed)
    else:
      # label 1 keeps its faces in global memory (hybrid), label 2 runs in shared memory and migrates
      assert st[1:3] == [1, 1] and resumed[1] + resumed[2] > 0, (st, resumed)
