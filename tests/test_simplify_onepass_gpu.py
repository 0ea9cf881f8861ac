"""k_simp_labels validates the winners of a round in as few passes as the label's shared memory allows: a
shared-memory label takes as many winners per pass as its size class's budget leaves room for, and a round
with more winners than that runs further passes.  IGN_SIMP_WCAP=n caps the winners per pass so that the
extra passes run on any volume.  The meshes are bit-identical to the oracle whatever the cap, in shared
and in global memory, and the cap never changes the class a label runs in."""
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
  passes = (ctypes.c_uint32 * 2)()
  _shim.check(m._ctx.lib.ign_mesh_simplify_passes(m._handle, passes))
  return meshes, list(stats), list(passes)


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


@pytest.fixture(scope="module")
def class_volume(oracle):
  # the 57-label volume of test_simplify_classes_gpu.py: labels in every class, and over 16,384 faces
  return np.asfortranarray(oracle.synth_seg((128, 128, 96), pitch=32, num_ids=64).astype(np.uint32))


@pytest.mark.parametrize("volume", ["bench_block", "class_volume"])
@pytest.mark.parametrize("gmem", [False, True])
def test_winner_capacity_bit_exact(ctx, oracle, request, monkeypatch, volume, gmem):
  seg = request.getfixturevalue(volume)
  tl, tv = oracle.marching_cubes(seg)
  want, _ = oracle.simplify_welded(oracle.WeldedMeshes(tl, tv), (16, 16, 40), 100, 40.0, True)
  monkeypatch.delenv("IGN_SIMP_WCAP", raising=False)
  if gmem:
    monkeypatch.setenv("IGN_SIMP_GMEM", "1")
  else:
    monkeypatch.delenv("IGN_SIMP_GMEM", raising=False)
  got, st, passes = _simplified(seg, 100, 40.0)
  _assert_same(got, want)
  multi = {}
  for cap in (8, 32):
    monkeypatch.setenv("IGN_SIMP_WCAP", str(cap))
    got_c, st_c, passes_c = _simplified(seg, 100, 40.0)
    _assert_same(got_c, want)
    assert st_c == st, (cap, st_c, st)  # the cap changes no label's class or memory path
    # winners rejected for a ring over 32 faces are the same ones whatever the cap
    assert passes_c[1] == passes[1], (cap, passes_c, passes)
    multi[cap] = passes_c[0]
  monkeypatch.delenv("IGN_SIMP_WCAP", raising=False)
  monkeypatch.delenv("IGN_SIMP_GMEM", raising=False)
  # a smaller cap splits more rounds, and the default capacity splits fewer than either
  assert multi[8] >= multi[32] > passes[0], (multi, passes)
