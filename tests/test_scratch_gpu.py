"""The per-context scratch arena: frames nest on a held CCL volume, the arena grows inside a call
without moving what earlier takes hold, and every error exit releases what the call took."""
import ctypes as c

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

RES = (16, 16, 40)


def _fresh():
  from igneous_b200 import _shim
  return _shim.Context()


def _ccl_dev(ctx, labels, out_dtype):
  from igneous_b200 import _shim
  d_in = ctx.to_device(labels)
  d_out = ctx.alloc(labels.size * np.dtype(out_dtype).itemsize)
  n = c.c_uint64(0)
  try:
    _shim.check(ctx.lib.ign_ccl6_dev(ctx.handle, _shim.ptr(d_in), _shim.dtype_code(labels.dtype), *labels.shape,
                                     _shim.ptr(d_out), _shim.dtype_code(out_dtype), c.byref(n)))
    return ctx.to_host(d_out, labels.shape, out_dtype), n.value
  finally:
    d_in.free()
    d_out.free()


def _meshes(ctx, seg, factor=10, max_error=8.0):
  from igneous_b200 import zmesh
  m = zmesh.Mesher(RES, ctx=ctx)
  m.mesh(seg)
  got = {int(i): m.get(i, reduction_factor=factor, max_error=max_error, voxel_centered=True) for i in m.ids()}
  m.clear()
  return got


def _assert_oracle_meshes(oracle, seg, got, factor=10, max_error=8.0):
  tl, tv = oracle.marching_cubes(seg)
  want, _ = oracle.simplify_welded(oracle.WeldedMeshes(tl, tv), RES, factor, max_error, True)
  assert got.keys() == want.keys()
  for k, (wv, wf) in want.items():
    assert np.array_equal(got[k].vertices, wv) and np.array_equal(got[k].faces, wf), k


def test_ccl_nests_on_held_volume(oracle):
  """A CCL whose run-capacity retry outgrows the arena runs while another volume holds its masks."""
  from igneous_b200 import _shim
  ctx = _fresh()
  rng = np.random.default_rng(5)
  a = np.asfortranarray(rng.integers(0, 3, size=(64, 48, 40)).astype(np.uint32))
  b = np.asfortranarray(rng.integers(0, 256, size=(96, 96, 96)).astype(np.uint8))  # mean x-run ~1 voxel
  want_a, n_a = oracle.connected_components(a, return_N=True)
  want_b, n_b = oracle.connected_components(b, return_N=True)
  d_a = ctx.to_device(a)
  d_out = ctx.alloc(a.size * 4)
  vol = c.c_void_p()
  n_local = c.c_uint64(0)
  null = c.c_void_p(None)
  try:
    _shim.check(ctx.lib.ign_ccl6_volume_begin_dev(ctx.handle, _shim.ptr(d_a), _shim.IGN_U32, *a.shape, null, null, null,
                                                  null, c.byref(vol), c.byref(n_local)))
    got_b, got_n_b = _ccl_dev(ctx, b, np.uint32)
    _shim.check(ctx.lib.ign_ccl6_volume_finish_dev(vol, null, n_local.value, _shim.ptr(d_out), _shim.IGN_U32))
    got_a = ctx.to_host(d_out, a.shape, np.uint32)
  finally:
    d_a.free()
    d_out.free()
  assert got_n_b == n_b and np.array_equal(got_b, want_b.astype(np.uint32))
  assert n_local.value == n_a and np.array_equal(got_a, want_a.astype(np.uint32))
  ctx.close()


def test_arena_grows_inside_mesh_and_simplify(oracle):
  """A larger task than the arena holds grows it during the weld and the simplification."""
  ctx = _fresh()
  small = np.asfortranarray(oracle.synth_seg((48, 48, 40), pitch=16, num_ids=12).astype(np.uint32))
  large = np.asfortranarray(oracle.synth_seg((128, 128, 96), pitch=32, num_ids=64).astype(np.uint32))
  first = _meshes(ctx, small)
  _assert_oracle_meshes(oracle, small, first)
  _assert_oracle_meshes(oracle, large, _meshes(ctx, large))
  again = _meshes(ctx, small)
  assert first.keys() == again.keys()
  for k in first:
    assert first[k].vertices.tobytes() == again[k].vertices.tobytes()
    assert first[k].faces.tobytes() == again[k].faces.tobytes()
  ctx.close()


def test_error_exits_release_the_arena(oracle):
  """A KeyError from remap and a failed CCL leave the arena as they found it."""
  from igneous_b200 import _shim
  ctx = _fresh()
  rng = np.random.default_rng(9)
  arr = np.asfortranarray(rng.integers(0, 8, size=(32, 32, 16)).astype(np.uint32))
  keys = np.arange(7, dtype=np.uint64)  # label 7 is missing
  d_arr = ctx.to_device(arr)
  try:
    with pytest.raises(KeyError):
      _shim.check(ctx.lib.ign_remap_dev(ctx.handle, _shim.ptr(d_arr), _shim.IGN_U32, arr.size, _shim.ptr(keys),
                                        _shim.ptr(keys), keys.size, 0))
  finally:
    d_arr.free()
  noise = np.asfortranarray(rng.integers(0, 256, size=(96, 96, 96)).astype(np.uint8))  # > 65,535 components
  with pytest.raises(_shim.IgneousB200Error):
    _ccl_dev(ctx, noise, np.uint16)
  seg = np.asfortranarray(oracle.synth_seg((48, 48, 40), pitch=16, num_ids=12).astype(np.uint32))
  _assert_oracle_meshes(oracle, seg, _meshes(ctx, seg))
  ctx.close()
