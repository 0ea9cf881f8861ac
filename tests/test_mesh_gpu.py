"""GPU parity: marching cubes + weld (through the C ABI) vs the CPU oracle."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _compare_all_labels(oracle, mesher, data, resolution, voxel_centered):
  tl, tv = oracle.marching_cubes(data)
  want_ids = sorted(int(i) for i in np.unique(tl))
  assert sorted(mesher.ids()) == want_ids
  for lab in want_ids:
    got = mesher.get(lab, reduction_factor=0, voxel_centered=voxel_centered)
    wv, wf = oracle.mesh_for_label(tl, tv, lab, resolution=resolution, voxel_centered=voxel_centered)
    # the product already emits the canonical order: compare raw first
    assert got.vertices.shape == wv.shape and got.faces.shape == wf.shape
    assert np.abs(got.vertices - wv).max() <= 1e-5 * max(1.0, float(np.abs(wv).max()))
    assert np.array_equal(got.vertices, wv)       # same f32 operation order: bit exact
    assert np.array_equal(got.faces, wf)          # identical triangle topology and order
    cv1, cf1 = oracle.canonicalise_mesh(got.vertices, got.faces)
    cv2, cf2 = oracle.canonicalise_mesh(wv, wf)
    assert np.array_equal(cf1, cf2) and np.array_equal(cv1, cv2)


def test_mc_box_kat_gpu(ctx):
  # reference mesh test volume (test/test_tasks.py:413-415): 62^3 box in 64^3
  from igneous_b200 import zmesh
  data = np.zeros((64, 64, 64), dtype=np.uint32, order="F")
  data[1:-1, 1:-1, 1:-1] = 1
  m = zmesh.Mesher((1, 1, 1))
  m.mesh(data)
  assert m.ids() == [1]
  mesh = m.get(1, reduction_factor=0, voxel_centered=False)
  assert mesh.faces.shape == (46124, 3) and mesh.vertices.shape == (23064, 3)
  v, f = mesh.vertices.astype(np.float64), mesh.faces
  vol = np.einsum("ij,ij->i", v[f[:, 0]], np.cross(v[f[:, 1]], v[f[:, 2]])).sum() / 6
  n = 62
  assert abs(vol - ((n - 1) ** 3 + 3 * (n - 1) ** 2 + 1.5 * (n - 1) + 1 / 6)) < 1e-3
  binary = mesh.to_precomputed()
  assert len(binary) == 4 + 12 * 23064 + 12 * 46124
  back = zmesh.Mesh.from_precomputed(binary)
  assert back == mesh


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.uint32, np.uint64])
def test_mc_random_multilabel_matches_oracle(ctx, oracle, dtype):
  from igneous_b200 import zmesh
  rng = np.random.default_rng(3)
  data = np.zeros((23, 19, 17), dtype=dtype, order="F")
  vals = np.array([0, 7, 9, 250], dtype=dtype)
  if np.dtype(dtype).itemsize == 8:
    vals = np.array([0, 7, 1 << 40, (1 << 63) + 5], dtype=np.uint64)
  data[1:-1, 1:-1, 1:-1] = vals[rng.integers(0, 4, size=(21, 17, 15))]
  res = (4.0, 4.0, 40.0)
  m = zmesh.Mesher(res)
  m.mesh(data)
  for vc in (False, True):
    _compare_all_labels(oracle, m, data, res, vc)


def test_mc_synthetic_segmentation_unpadded(ctx, oracle):
  # open surfaces at the chunk border (no zero padding), realistic labels
  from igneous_b200 import zmesh
  seg = oracle.synth_seg((65, 65, 33), pitch=16, num_ids=1 << 20)
  m = zmesh.Mesher((16, 16, 40))
  m.mesh(seg)
  _compare_all_labels(oracle, m, seg, (16, 16, 40), True)


def test_mc_empty_and_degenerate(ctx):
  from igneous_b200 import zmesh
  m = zmesh.Mesher((1, 1, 1))
  m.mesh(np.zeros((8, 8, 8), dtype=np.uint32))
  assert m.ids() == []
  m.mesh(np.full((8, 8, 8), 5, dtype=np.uint32))  # no surface inside the chunk
  assert m.ids() == []
  m.mesh(np.ones((1, 5, 5), dtype=np.uint8))
  assert m.ids() == []
  with pytest.raises(KeyError):
    m.get(3)


def test_mc_properties_at_task_size(ctx):
  """257^3 task (BASELINE config C4 task shape + overlap): every label's mesh
  has only valid indices, no degenerate faces, and interior labels are closed."""
  from igneous_b200 import zmesh, _shim
  n = 257
  d = ctx.alloc(n ** 3 * 4)
  _shim.check(ctx.lib.ign_synth_seg_dev(ctx.handle, _shim.ptr(d), _shim.IGN_U32, n, n, n, 0, 0, 0, 64, 1 << 20, 0, 0))
  seg = ctx.to_host(d, (n, n, n), np.uint32)
  d.free()
  m = zmesh.Mesher((16, 16, 40))
  m.mesh(seg)
  ids = m.ids()
  assert len(ids) > 50
  inner = set(np.unique(seg[1:-1, 1:-1, 1:-1])) - set(np.unique(np.concatenate([
    seg[0].ravel(), seg[-1].ravel(), seg[:, 0].ravel(), seg[:, -1].ravel(),
    seg[:, :, 0].ravel(), seg[:, :, -1].ravel()])))
  checked = 0
  for lab in ids:
    mesh = m.get(lab, voxel_centered=True)
    f = mesh.faces
    assert f.max() < len(mesh.vertices)
    assert (f[:, 0] != f[:, 1]).all() and (f[:, 1] != f[:, 2]).all() and (f[:, 0] != f[:, 2]).all()
    if lab in inner and checked < 10:
      e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]).astype(np.int64)
      fwd = e[:, 0] * (1 << 32) + e[:, 1]
      bwd = e[:, 1] * (1 << 32) + e[:, 0]
      assert np.array_equal(np.sort(fwd), np.sort(bwd))  # closed + consistently oriented
      checked += 1
  assert checked > 0


def _closed(f):
  e = np.concatenate([f[:, [0, 1]], f[:, [1, 2]], f[:, [2, 0]]]).astype(np.int64)
  return np.array_equal(np.sort(e[:, 0] * (1 << 32) + e[:, 1]), np.sort(e[:, 1] * (1 << 32) + e[:, 0]))


def test_simplify_box_matches_oracle_bit_exact(ctx, oracle):
  """62^3 box (reference mesh test volume): the GPU simplifier reproduces the
  CPU restatement of the same round-based algorithm bit for bit (parity with
  zmesh's own simplifier is unpinned, see DESIGN.md)."""
  from igneous_b200 import zmesh
  data = np.zeros((64, 64, 64), dtype=np.uint32, order="F")
  data[1:-1, 1:-1, 1:-1] = 1
  m = zmesh.Mesher((1, 1, 1))
  m.mesh(data)
  got = m.get(1, reduction_factor=100, max_error=40, voxel_centered=False)
  tl, tv = oracle.marching_cubes(data)
  want, rounds = oracle.simplify_welded(oracle.WeldedMeshes(tl, tv), (1, 1, 1), 100, 40.0, False)
  wv, wf = want[1]
  assert got.faces.shape == wf.shape and got.vertices.shape == wv.shape
  assert np.array_equal(got.faces, wf) and np.array_equal(got.vertices, wv)
  assert len(got.faces) <= 46124 // 100 + 2 and len(got.faces) >= 0.8 * (46124 // 100)
  assert _closed(got.faces)
  v = got.vertices.astype(np.float64)
  vol = np.einsum("ij,ij->i", v[got.faces[:, 0]], np.cross(v[got.faces[:, 1]], v[got.faces[:, 2]])).sum() / 6
  assert abs(vol - 238235.6667) < 1e-3 * 238235  # flat faces: volume preserved


@pytest.mark.parametrize("factor,max_error", [(100, 40.0), (4, 1e9), (10, 8.0)])
def test_simplify_multilabel_matches_oracle(ctx, oracle, factor, max_error):
  from igneous_b200 import zmesh
  seg = oracle.synth_seg((49, 45, 41), pitch=16, num_ids=1 << 20)
  res = (16, 16, 40)
  m = zmesh.Mesher(res)
  m.mesh(seg)
  tl, tv = oracle.marching_cubes(seg)
  W = oracle.WeldedMeshes(tl, tv)
  want, rounds = oracle.simplify_welded(W, res, factor, max_error, True)
  assert sorted(m.ids()) == sorted(want.keys())
  before = {l: len(W.get(l)[1]) for l in W.ids()}
  for lab in m.ids():
    got = m.get(lab, reduction_factor=factor, max_error=max_error, voxel_centered=True)
    wv, wf = want[lab]
    assert got.vertices.shape == wv.shape and got.faces.shape == wf.shape, lab
    assert np.abs(got.vertices - wv).max(initial=0) <= 1e-5 * max(1.0, float(np.abs(wv).max(initial=0)))
    assert np.array_equal(got.vertices, wv) and np.array_equal(got.faces, wf), lab
    assert len(got.faces) <= before[lab]
  total_after = sum(len(f) for v, f in want.values())
  assert total_after < sum(before.values())
  with pytest.raises(ValueError):
    m.get(m.ids()[0], reduction_factor=factor + 1, max_error=max_error)


def test_simplify_shared_and_global_memory_classes_bit_exact(ctx, oracle, monkeypatch):
  """k_simp_labels keeps a label's topology in shared memory when it fits and otherwise runs the
  same code on the global-memory arrays (IGN_SIMP_GMEM=1 forces that class): identical meshes
  from both, and both identical to the oracle."""
  from igneous_b200 import zmesh

  def meshes(seg, factor):
    m = zmesh.Mesher((16, 16, 40))
    m.mesh(seg)
    return {int(i): m.get(i, reduction_factor=factor, max_error=40.0, voxel_centered=True) for i in m.ids()}

  for shape, pitch, factor in (((96, 80, 64), 24, 10), ((128, 128, 64), 32, 100)):
    seg = np.asfortranarray(oracle.synth_seg(shape, pitch=pitch, num_ids=9).astype(np.uint32))
    monkeypatch.delenv("IGN_SIMP_GMEM", raising=False)
    smem = meshes(seg, factor)
    monkeypatch.setenv("IGN_SIMP_GMEM", "1")
    gmem = meshes(seg, factor)
    monkeypatch.delenv("IGN_SIMP_GMEM", raising=False)
    tl, tv = oracle.marching_cubes(seg)
    want, _ = oracle.simplify_welded(oracle.WeldedMeshes(tl, tv), (16, 16, 40), factor, 40.0, True)
    assert smem.keys() == gmem.keys() == want.keys()
    for k in smem:
      assert np.array_equal(smem[k].vertices, gmem[k].vertices)
      assert np.array_equal(smem[k].faces, gmem[k].faces)
      assert np.array_equal(smem[k].vertices, want[k][0]) and np.array_equal(smem[k].faces, want[k][1])
