"""A shared-memory label of k_simp_labels whose alive faces and vertices come to fit the next smaller
size class continues there (1024 -> 512 -> 256 threads): its state is compacted, its faces and vertices
renumbered, and the keys, cached costs, positions and quadrics are still addressed by the original ids.
The meshes stay bit-identical to the oracle, and each label still counts once, in the class it started in."""
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
  return meshes, list(stats), list(resumed)


def _assert_same(got, want):
  assert got.keys() == want.keys()
  for k in want:
    wv, wf = want[k]
    assert np.array_equal(got[k].vertices, wv) and np.array_equal(got[k].faces, wf), k


@pytest.fixture(scope="module")
def bench_block(oracle):
  # a 129^3 block of the benchmark's mip-2 MeshTask volume: synth_seg pitch 64, seed 0, two 2x2x1 mode mips
  seg = oracle.synth_seg((516, 516, 129), pitch=64, num_ids=1 << 20, seed=0)
  return np.asfortranarray(oracle.downsample_segmentation(seg, (2, 2, 1), num_mips=2)[1].astype(np.uint32))


@pytest.mark.parametrize("factor,max_error", [(100, 40.0), (10, 8.0)])
def test_migration_bench_block_bit_exact(ctx, oracle, bench_block, monkeypatch, factor, max_error):
  monkeypatch.delenv("IGN_SIMP_GMEM", raising=False)
  tl, tv = oracle.marching_cubes(bench_block)
  want, _ = oracle.simplify_welded(oracle.WeldedMeshes(tl, tv), (16, 16, 40), factor, max_error, True)
  got, st, resumed = _simplified(bench_block, factor, max_error)
  _assert_same(got, want)
  n_full, n_half = st[3], st[4]
  assert st[3] + st[4] + st[5] == st[1] + st[2] == len(want), st
  assert resumed[0] == 0 and resumed[1] > 0 and resumed[2] > 0, (st, resumed)
  assert resumed[1] <= n_full and resumed[2] <= n_full + n_half, (st, resumed)
  if factor == 100:
    # more labels resumed in the 256-thread class than started in the 512-thread one: some of them
    # started in the 1024-thread class and migrated twice
    assert resumed[2] > n_half, (st, resumed)


@pytest.mark.parametrize("factor,max_error", [(100, 40.0), (10, 8.0)])
def test_migration_size_class_volume_bit_exact(ctx, oracle, monkeypatch, factor, max_error):
  # the 57-label volume of test_simplify_classes_gpu.py: labels in every class, and over 16,384 faces
  # (global-memory path, which never migrates)
  seg = np.asfortranarray(oracle.synth_seg((128, 128, 96), pitch=32, num_ids=64).astype(np.uint32))
  tl, tv = oracle.marching_cubes(seg)
  want, _ = oracle.simplify_welded(oracle.WeldedMeshes(tl, tv), (16, 16, 40), factor, max_error, True)
  monkeypatch.delenv("IGN_SIMP_GMEM", raising=False)
  got, st, resumed = _simplified(seg, factor, max_error)
  _assert_same(got, want)
  assert resumed[0] == 0 and resumed[1] + resumed[2] > 0, (st, resumed)
  assert resumed[1] <= st[3] - st[2], (st, resumed)  # only shared-memory labels of the full class
  monkeypatch.setenv("IGN_SIMP_GMEM", "1")
  got_g, st_g, resumed_g = _simplified(seg, factor, max_error)
  monkeypatch.delenv("IGN_SIMP_GMEM", raising=False)
  _assert_same(got_g, want)
  assert resumed_g == [0, 0, 0] and st_g[3:] == st[3:], (st_g, resumed_g)
