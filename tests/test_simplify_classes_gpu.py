"""k_simp_labels runs each label in the smallest CTA whose shared-memory budget holds it (1024 threads
alone on an SM, 512 threads two per SM, 256 threads four per SM).  A volume with labels in every size
class: each class runs, and every mesh is bit-identical to the oracle, with the topology in shared
memory and on the global-memory path (IGN_SIMP_GMEM=1)."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _simplified(seg, factor, max_error):
  from igneous_b200 import zmesh
  m = zmesh.Mesher((16, 16, 40))
  m.mesh(seg)
  meshes = {int(i): m.get(i, reduction_factor=factor, max_error=max_error, voxel_centered=True) for i in m.ids()}
  stats = (ctypes.c_uint32 * 6)()
  from igneous_b200 import _shim
  _shim.check(m._ctx.lib.ign_mesh_simplify_stats(m._handle, stats))
  return meshes, list(stats)


@pytest.mark.parametrize("factor,max_error", [(100, 40.0), (10, 8.0)])
def test_simplify_size_classes_bit_exact(ctx, oracle, monkeypatch, factor, max_error):
  # 57 labels from 490 to 35,550 faces: 6 fit a 256-thread CTA, 12 a 512-thread one, 39 need the whole SM
  seg = np.asfortranarray(oracle.synth_seg((128, 128, 96), pitch=32, num_ids=64).astype(np.uint32))
  tl, tv = oracle.marching_cubes(seg)
  want, _ = oracle.simplify_welded(oracle.WeldedMeshes(tl, tv), (16, 16, 40), factor, max_error, True)
  monkeypatch.delenv("IGN_SIMP_GMEM", raising=False)
  smem, st = _simplified(seg, factor, max_error)
  rounds, n_smem, n_gmem, n_full, n_half, n_quarter = st
  assert n_full > 0 and n_half > 0 and n_quarter > 0, st
  assert n_full + n_half + n_quarter == n_smem + n_gmem == len(want)
  assert n_gmem > 0  # labels over 16,384 faces keep their faces in global memory
  monkeypatch.setenv("IGN_SIMP_GMEM", "1")
  gmem, st_g = _simplified(seg, factor, max_error)
  monkeypatch.delenv("IGN_SIMP_GMEM", raising=False)
  assert st_g[1] == 0 and st_g[2] == len(want) and st_g[3:] == st[3:], st_g
  assert smem.keys() == gmem.keys() == want.keys()
  for k in want:
    wv, wf = want[k]
    for got in (smem[k], gmem[k]):
      assert np.array_equal(got.vertices, wv) and np.array_equal(got.faces, wf), k
