"""The simplifier caches the float cost of every edge.  k_simp_ecost costs every edge before the first round,
and each collapse re-costs the edges of the vertex it moved right after it moved (E2d), so the key pass of a
round only posts cached keys and never evaluates a cost.  Meshes stay bit-identical to the oracle on the
benchmark block, on a volume with labels in every size class, and on closed boxes whose flat faces park
many edges (topology in shared memory, in hybrid and in global memory), also with rounds split into several
selection passes (IGN_SIMP_WCAP=8)."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _simplified(seg, res, factor, max_error, centered):
  from igneous_b200 import _shim, zmesh
  m = zmesh.Mesher(res)
  m.mesh(seg)
  meshes = {int(i): m.get(i, reduction_factor=factor, max_error=max_error, voxel_centered=centered) for i in m.ids()}
  stats = (ctypes.c_uint32 * 6)()
  _shim.check(m._ctx.lib.ign_mesh_simplify_stats(m._handle, stats))
  costs = (ctypes.c_uint32 * 3)()
  _shim.check(m._ctx.lib.ign_mesh_simplify_costs(m._handle, costs))
  return meshes, list(stats), list(costs)


def _check(oracle, monkeypatch, seg, res, factor, max_error, centered, wcap):
  tl, tv = oracle.marching_cubes(seg)
  W = oracle.WeldedMeshes(tl, tv)
  want, _ = oracle.simplify_welded(W, res, factor, max_error, centered)
  if wcap:
    monkeypatch.setenv("IGN_SIMP_WCAP", str(wcap))
  else:
    monkeypatch.delenv("IGN_SIMP_WCAP", raising=False)
  monkeypatch.delenv("IGN_SIMP_GMEM", raising=False)
  got, stats, costs = _simplified(seg, res, factor, max_error, centered)
  monkeypatch.delenv("IGN_SIMP_WCAP", raising=False)
  assert got.keys() == want.keys()
  for k in want:
    wv, wf = want[k]
    assert np.array_equal(got[k].vertices, wv) and np.array_equal(got[k].faces, wf), k
  # every canonical half-edge (u < v) of the input is costed once before the first round
  f = np.asarray(W.faces, dtype=np.int64).reshape(-1, 3)
  canonical = int((f[:, 0] < f[:, 1]).sum() + (f[:, 1] < f[:, 2]).sum() + (f[:, 2] < f[:, 0]).sum())
  assert costs[0] == canonical, (costs, canonical)
  assert costs[1] > 0, costs  # collapses re-cost the edges of the vertices they move
  assert costs[2] == 0, costs  # the key pass never meets an edge without a cost
  return stats


@pytest.fixture(scope="module")
def bench_block(oracle):
  # a 129^3 block of the benchmark's mip-2 MeshTask volume: synth_seg pitch 64, seed 0, two 2x2x1 mode mips
  seg = oracle.synth_seg((516, 516, 129), pitch=64, num_ids=1 << 20, seed=0)
  return np.asfortranarray(oracle.downsample_segmentation(seg, (2, 2, 1), num_mips=2)[1].astype(np.uint32))


@pytest.mark.parametrize("wcap", [None, 8])
def test_costs_bench_block(ctx, oracle, monkeypatch, bench_block, wcap):
  _check(oracle, monkeypatch, bench_block, (16, 16, 40), 100, 40.0, True, wcap)


@pytest.mark.parametrize("wcap", [None, 8])
def test_costs_size_classes(ctx, oracle, monkeypatch, wcap):
  # 57 labels from 490 to 35,550 faces, in all three size classes and on the global-memory path
  seg = np.asfortranarray(oracle.synth_seg((128, 128, 96), pitch=32, num_ids=64).astype(np.uint32))
  stats = _check(oracle, monkeypatch, seg, (16, 16, 40), 100, 40.0, True, wcap)
  assert min(stats[3:]) > 0 and stats[2] > 0, stats


# a closed box of (n - 2)^3 voxels: about 9,400 faces run in shared memory, about 17,300 keep their faces in
# global memory with keys, flags and states in shared memory (hybrid), 46,124 run wholly in global memory
@pytest.mark.parametrize("wcap", [None, 8])
@pytest.mark.parametrize("n,smem", [(30, True), (40, False), (64, False)])
def test_costs_box(ctx, oracle, monkeypatch, n, smem, wcap):
  data = np.zeros((n, n, n), dtype=np.uint32, order="F")
  data[1:-1, 1:-1, 1:-1] = 1
  stats = _check(oracle, monkeypatch, data, (1, 1, 1), 100, 40.0, False, wcap)
  assert stats[1:3] == ([1, 0] if smem else [0, 1]), stats
