"""The serial C checker of the TEASAR loop (oracle_geodesic/teasar_oracle.c) against the heapq restatement
tests/teasarref.py (no shared code), on random small volumes in both fix_branching modes, and the
restatement on hand-built volumes of known answer.  No GPU."""
import numpy as np
import pytest

import oracle_geodesic as G
import teasarref as T


def c_geodesic(lab, sources, anisotropy=(1, 1, 1), weights=None, parents=False):
  return G.geodesic(lab, np.asarray(sources, np.uint64), 26, anisotropy, weights, parents)


def blobs(shape, seed, labels=3, block=2):
  rng = np.random.default_rng(seed)
  coarse = rng.integers(0, labels + 1, size=[(n + block - 1) // block for n in shape])
  return np.kron(coarse, np.ones((block,) * 3, int))[:shape[0], :shape[1], :shape[2]].astype(np.uint32)


def same(a, b):
  assert sorted(a) == sorted(b)
  for l in a:
    for x, y in zip(a[l], b[l]):
      assert x.dtype == y.dtype and np.array_equal(x, y), l


@pytest.mark.parametrize("fix_branching", [True, False])
@pytest.mark.parametrize("seed,anisotropy", [(0, (1, 1, 1)), (1, (1.1, 0.7, 3.3)), (2, (16, 16, 40))])
def test_checker_matches_restatement(seed, anisotropy, fix_branching):
  lab = blobs((9, 8, 6), seed)
  kw = dict(anisotropy=anisotropy, scale=1.5, const=float(min(anisotropy)), fix_branching=fix_branching)
  got = T.skeletonize(lab, geodesic=c_geodesic, run_loop=G.teasar, **kw)
  want = T.skeletonize(lab, **kw)
  same(got, want)
  assert got


def test_targets_and_max_paths_match_restatement():
  lab = blobs((10, 7, 5), 7, labels=2)
  pts = np.argwhere(lab != 0)
  rng = np.random.default_rng(3)
  before = [tuple(p) for p in pts[rng.choice(len(pts), 3, replace=False)]]
  after = [tuple(p) for p in pts[rng.choice(len(pts), 3, replace=False)]]
  for mp in (None, 1, 2):
    kw = dict(scale=1.0, const=1.0, max_paths=mp, before=before, after=after)
    same(T.skeletonize(lab, geodesic=c_geodesic, run_loop=G.teasar, **kw), T.skeletonize(lab, **kw))


def tree_ok(verts, edges):
  n = len(verts)
  assert len(edges) == n - 1
  parent = list(range(n))

  def find(i):
    while parent[i] != i:
      i = parent[i]
    return i
  for a, b in edges:
    assert np.abs(verts[a] - verts[b]).max() <= 1  # 26-neighbours at anisotropy 1
    ra, rb = find(a), find(b)
    assert ra != rb
    parent[ra] = rb


def test_straight_tube_is_one_path_along_its_axis():
  lab = np.zeros((20, 5, 5), np.uint32)
  lab[:, 1:4, 1:4] = 1
  v, e, r = T.skeletonize(lab, scale=1, const=1)[1]
  tree_ok(v, e)
  deg = np.bincount(e.ravel(), minlength=len(v))
  assert (deg == 1).sum() == 2 and sorted(v[:, 0]) == list(range(20))  # one path, end to end
  inner = (v[:, 0] >= 2) & (v[:, 0] <= 17)
  assert np.all(v[inner, 1:] == 2)  # on the axis away from the ends, where it turns to the farthest corners


def test_y_has_three_ends_and_one_junction():
  lab = np.zeros((21, 21, 3), np.uint32)
  for i in range(11):
    lab[10, i, 1] = 1                  # stem
    lab[10 - i, 10 + i, 1] = 1         # left arm
    lab[10 + i, 10 + i, 1] = 1         # right arm
  v, e, r = T.skeletonize(lab, scale=0, const=0)[1]
  tree_ok(v, e)
  deg = np.bincount(e.ravel(), minlength=len(v))
  assert sorted(deg[deg != 2]) == [1, 1, 1, 3]


def test_const_larger_than_the_object_gives_one_path():
  lab = blobs((8, 8, 6), 11, labels=1, block=8)
  lab[:] = 1
  lab[2:6, 2:6, :] = 0
  lab[0, 0, 0] = 1
  v, e, r = T.skeletonize(lab, scale=0, const=100)[1]
  tree_ok(v, e)
  deg = np.bincount(e.ravel(), minlength=len(v))
  assert (deg == 1).sum() == 2  # a single path: two ends


def test_max_paths_one():
  lab = np.zeros((21, 21, 3), np.uint32)
  for i in range(11):
    lab[10, i, 1] = lab[10 - i, 10 + i, 1] = lab[10 + i, 10 + i, 1] = 1
  v, e, r = T.skeletonize(lab, scale=0, const=0, max_paths=1)[1]
  deg = np.bincount(e.ravel(), minlength=len(v))
  assert (deg == 1).sum() == 2 and len(v) == 21
