"""igneous_b200.kimimaro.skeletonize against the rule of DESIGN.md §5f, bit for bit: the expected skeleton is
built by tests/teasarref.py's pipeline with the serial C checkers standing in for the solvers
(oracle_geodesic: heap Dijkstra for the fields, teasar_oracle.c for the loop) and scipy / tests/edtref.py
for the objects and the distance to the boundary.  Both fix_branching modes, three anisotropies, shapes off
the brick grid, every dtype and both memory orders, a pitch-16 synthetic segmentation, a label in several
parts, dust_threshold, object_ids, max_paths, extra targets, fix_borders targets, random capsule-tree
neurites with many rounds and a full 449^3 chunk; every skeleton a tree of 26-neighbour edges; all labels in
one call against one call per label; refusals."""
import ctypes

import numpy as np
import pytest

import oracle_geodesic as G
import teasarref as T
from igneous_b200 import kimimaro

pytestmark = pytest.mark.gpu

NB = dict(fix_borders=False)


def c_geodesic(lab, sources, anisotropy=(1, 1, 1), weights=None, parents=False):
  return G.geodesic(lab, np.asarray(sources, np.uint64), 26, anisotropy, weights, parents)


def expected(lab, anisotropy=(1, 1, 1), params=None, dust_threshold=0, object_ids=None, fix_branching=True,
             before=(), after=(), fix_borders=False):
  p = dict(kimimaro.DEFAULT_TEASAR_PARAMS)
  p.update(params or {})
  return T.skeletonize(np.asarray(lab), anisotropy, float(p["scale"]), float(p["const"]), p["pdrf_scale"],
                       p["pdrf_exponent"], p["max_paths"], dust_threshold, object_ids, fix_branching, before, after,
                       fix_borders, geodesic=c_geodesic, run_loop=G.teasar)


def run(ctx, lab, anisotropy=(1, 1, 1), params=None, dust_threshold=0, **kw):
  kw = {**NB, **kw}
  return kimimaro.skeletonize(lab, teasar_params=params or {}, anisotropy=anisotropy, dust_threshold=dust_threshold,
                              ctx=ctx, **kw)


def assert_same(got, want):
  assert sorted(got) == sorted(want)
  for l, s in got.items():
    v, e, r = want[l]
    assert s.id == l
    for x, y in ((s.vertices, v), (s.edges, e), (s.radii, r)):
      assert x.dtype == y.dtype and x.shape == y.shape and np.array_equal(x, y), l
    assert s.vertex_types.dtype == np.uint8 and not s.vertex_types.any()


def assert_trees(got, anisotropy):
  a = np.asarray(anisotropy, np.float32)
  for s in got.values():
    vox = np.rint(s.vertices / a).astype(np.int64)
    if len(s.edges):
      assert np.abs(vox[s.edges[:, 0]] - vox[s.edges[:, 1]]).max() <= 1
    assert len(s.edges) < len(s.vertices)


def blobs(shape, seed, labels=4, block=3):
  rng = np.random.default_rng(seed)
  coarse = rng.integers(0, labels + 1, size=[(n + block - 1) // block for n in shape])
  return np.asfortranarray(np.kron(coarse, np.ones((block,) * 3, int))[:shape[0], :shape[1], :shape[2]]
                           .astype(np.uint32))


@pytest.mark.parametrize("fix_branching", [True, False])
@pytest.mark.parametrize("anisotropy,params", [((1, 1, 1), {"scale": 1.5, "const": 1}),
                                               ((16, 16, 40), {"scale": 1.5, "const": 20}),
                                               ((1.1, 0.7, 3.3), {"scale": 2, "const": 0.5})])
@pytest.mark.parametrize("shape", [(37, 11, 9), (33, 9, 17)])
def test_matches_the_checker(ctx, shape, anisotropy, params, fix_branching):
  lab = blobs(shape, hash(shape) % 1000)
  got = run(ctx, lab, anisotropy, params, fix_branching=fix_branching)
  assert_same(got, expected(lab, anisotropy, params, fix_branching=fix_branching))
  assert_trees(got, anisotropy)
  stats = (ctypes.c_uint64 * 4)()
  ctx.lib.ign_teasar_last_stats(stats)
  assert stats[0] >= 1 and stats[1] >= 1 and stats[3] >= stats[0]


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.uint64, np.int32, np.bool_])
@pytest.mark.parametrize("order", ["C", "F"])
def test_dtypes_and_orders(ctx, dtype, order):
  lab = blobs((20, 13, 11), 5, labels=1 if dtype == np.bool_ else 4)
  want = expected(lab, params={"scale": 1, "const": 1})
  cast = np.asarray(lab.astype(dtype), order=order)
  if dtype == np.uint64:
    cast = np.where(cast != 0, cast + np.uint64(1 << 40), 0).astype(np.uint64, order=order)
    want = {l + (1 << 40): s for l, s in want.items()}
  got = run(ctx, cast, params={"scale": 1, "const": 1})
  if dtype == np.bool_:
    want = {1: want[1]}
  assert_same(got, want)


def test_synthetic_segmentation(ctx, oracle):
  seg = np.asfortranarray(oracle.synth_seg((96, 80, 40), pitch=16, num_ids=40).astype(np.uint32))
  params = {"scale": 4, "const": 40}
  for fb in (True, False):
    got = run(ctx, seg, (16, 16, 40), params, fix_branching=fb)
    assert_same(got, expected(seg, (16, 16, 40), params, fix_branching=fb))
    assert_trees(got, (16, 16, 40))


def test_label_in_several_parts_dust_and_object_ids(ctx):
  lab = np.zeros((30, 12, 10), np.uint32)
  lab[1:8, 1:5, 1:5] = 7
  lab[12:20, 2:9, 2:8] = 7
  lab[25:27, 1:3, 1:3] = 7        # 8 voxels: dust at 10
  lab[1:29, 8:11, 6:9] = 3
  params = {"scale": 1, "const": 1}
  for dust in (0, 10):
    got = run(ctx, lab, params=params, dust_threshold=dust)
    assert_same(got, expected(lab, params=params, dust_threshold=dust))
  got = run(ctx, lab, params=params, object_ids=[7])
  assert_same(got, expected(lab, params=params, object_ids=[7]))
  # all labels in one call give what one call per label gives
  full = run(ctx, lab, params=params)
  for l in (3, 7):
    assert_same({l: full[l]}, {l: (s.vertices, s.edges, s.radii) for s in [run(ctx, lab, params=params,
                                                                                 object_ids=[l])[l]]})


@pytest.mark.parametrize("max_paths", [1, 2])
def test_max_paths(ctx, max_paths):
  lab = blobs((25, 19, 9), 9, labels=2, block=2)
  params = {"scale": 0.5, "const": 0, "max_paths": max_paths}
  assert_same(run(ctx, lab, params=params), expected(lab, params=params))


@pytest.mark.parametrize("fix_branching", [True, False])
def test_extra_targets(ctx, fix_branching):
  lab = blobs((24, 17, 10), 13, labels=3)
  pts = np.argwhere(lab != 0)
  rng = np.random.default_rng(1)
  before = [tuple(int(c) for c in p) for p in pts[rng.choice(len(pts), 5, replace=False)]]
  after = [tuple(int(c) for c in p) for p in pts[rng.choice(len(pts), 5, replace=False)]]
  params = {"scale": 1, "const": 2}
  got = run(ctx, lab, params=params, fix_branching=fix_branching, extra_targets_before=before,
            extra_targets_after=after)
  assert_same(got, expected(lab, params=params, fix_branching=fix_branching, before=before, after=after))


def test_refusals(ctx):
  lab = blobs((12, 10, 8), 2)
  for kw in ({"fill_holes": True}, {"fix_avocados": True}, {"voxel_graph": np.zeros_like(lab)}):
    with pytest.raises(NotImplementedError):
      run(ctx, lab, **kw)
  for bad in ({"scale": -1}, {"const": float("inf")}):
    with pytest.raises(ValueError):
      run(ctx, lab, params=bad)
  z = tuple(int(c) for c in np.argwhere(lab == 0)[0])
  with pytest.raises(ValueError):
    run(ctx, lab, extra_targets_before=[z])
  big = np.ones((40, 40, 40), np.uint32)
  with pytest.raises(NotImplementedError, match="label 1 "):
    run(ctx, big, params={"soma_detection_threshold": 5})
  assert run(ctx, np.zeros((5, 5, 5), np.uint8)) == {}


@pytest.mark.parametrize("anisotropy", [(1, 1, 1), (16, 16, 40), (1.1, 0.7, 3.3)])
def test_border_targets_match_scipy_and_edtref(ctx, anisotropy):
  lab = blobs((37, 11, 9), 21, labels=3, block=2)
  obj, k = T.objects_of(lab)
  want = T.border_targets(obj, k, anisotropy)
  n = obj.size
  d_obj, d_out = ctx.to_device(np.asfortranarray(obj)), ctx.alloc(8 * 2 * (37 * 11 + 37 * 9 + 11 * 9))
  cnt = ctypes.c_uint64(0)
  from igneous_b200 import _shim
  _shim.check(ctx.lib.ign_teasar_border_targets_dev(ctx.handle, _shim.ptr(d_obj), *obj.shape, k,
                                                    (ctypes.c_float * 3)(*anisotropy), _shim.ptr(d_out),
                                                    2 * (37 * 11 + 37 * 9 + 11 * 9), ctypes.byref(cnt)))
  got = np.empty(int(cnt.value), np.uint64)
  ctx.d2h(got, d_out, got.nbytes)
  ctx.sync()
  d_obj.free()
  d_out.free()
  assert n and got.tolist() == want and len(want) > 6


@pytest.mark.parametrize("fix_branching", [True, False])
def test_fix_borders_default_call(ctx, fix_branching):
  lab = blobs((40, 17, 12), 31, labels=3)
  params = {"scale": 1, "const": 2}
  pts = np.argwhere(lab != 0)
  before = [tuple(int(c) for c in pts[len(pts) // 2])]
  got = kimimaro.skeletonize(lab, params, anisotropy=(16, 16, 40), dust_threshold=0, fix_branching=fix_branching,
                             extra_targets_before=before, ctx=ctx)
  assert_same(got, expected(lab, (16, 16, 40), params, fix_branching=fix_branching, before=before,
                            fix_borders=True))
  assert_trees(got, (16, 16, 40))


@pytest.mark.parametrize("fix_borders", [False, True])
def test_capsule_tree_neurites(ctx, fix_borders):
  lab = T.capsule_trees((160, 150, 70), 14, seed=4, anisotropy=(16, 16, 40))
  params = {"scale": 1, "const": 20}
  for fb in (True, False):
    got = run(ctx, lab, (16, 16, 40), params, fix_branching=fb, fix_borders=fix_borders)
    stats = (ctypes.c_uint64 * 4)()
    ctx.lib.ign_teasar_last_stats(stats)
    assert_same(got, expected(lab, (16, 16, 40), params, fix_branching=fb, fix_borders=fix_borders))
    assert_trees(got, (16, 16, 40))
    assert stats[0] >= 8 and stats[1] >= 4 * len(got)  # several rounds and paths per object


def test_full_449_chunk(ctx, oracle):
  seg = np.asfortranarray(oracle.synth_seg((449, 449, 449), pitch=16, num_ids=1 << 20).astype(np.uint32))
  want = T.skeletonize_modes(seg, (16, 16, 40), 4.0, 500.0, dust_threshold=1000, fix_borders=True,
                             geodesic=c_geodesic, run_loop=G.teasar)
  for fb in (True, False):
    got = kimimaro.skeletonize(seg, {"scale": 4, "const": 500}, anisotropy=(16, 16, 40), dust_threshold=1000,
                               fix_branching=fb, ctx=ctx)
    assert len(got) > 20000
    assert_same(got, want[fb])
