"""The serial C checker of the geodesic rule (oracle_geodesic/) against the numpy / heapq restatement
(tests/geodesicref.py, no shared code) on small volumes, bit for bit: each connectivity, representable
and non-representable anisotropy, field weights with zeros, several labels and sources, parents; and
against scipy.sparse.csgraph.dijkstra on a unit-weight 6-connected mask, where float64 and float32
agree exactly.  Runs without a GPU."""
import numpy as np
import pytest
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import dijkstra

import geodesicref
import oracle_geodesic as G


def blobs(shape, seed, labels=3):
  """random label volume: blocks of 3^3 voxels of labels 0..labels, so that objects are connected in places"""
  rng = np.random.default_rng(seed)
  coarse = rng.integers(0, labels + 1, size=[(n + 2) // 3 for n in shape])
  return np.kron(coarse, np.ones((3, 3, 3), int))[:shape[0], :shape[1], :shape[2]].astype(np.uint32)


def first_voxels(lab):
  """one source per label: its first voxel in F order"""
  flat = lab.ravel(order="F")
  return [int(np.flatnonzero(flat == l)[0]) for l in np.unique(flat[flat != 0])]


def same_bits(a, b):
  return a.dtype == b.dtype and a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("connectivity", [6, 18, 26])
@pytest.mark.parametrize("anisotropy", [(1, 1, 1), (4, 4, 40), (1.1, 0.7, 3.3)])
def test_euclidean_matches_the_restatement(connectivity, anisotropy):
  lab = blobs((11, 9, 7), seed=connectivity)
  src = first_voxels(lab)
  vox = [np.unravel_index(s, lab.shape, order="F") for s in src]
  want, wpar = geodesicref.geodesic(lab, vox, connectivity, anisotropy, parents=True)
  got, gpar = G.geodesic(lab, src, connectivity, anisotropy, parents=True)
  assert same_bits(got, want) and np.array_equal(gpar, wpar)
  assert np.isinf(got[lab == 0]).all() and (got[np.unravel_index(src, lab.shape, order="F")] == 0).all()


@pytest.mark.parametrize("connectivity", [6, 26])
def test_field_weights_match_the_restatement(connectivity):
  rng = np.random.default_rng(3)
  lab = blobs((10, 8, 6), seed=5, labels=2)
  w = (rng.random(lab.shape) * 10).astype(np.float32)
  src = first_voxels(lab)
  vox = [np.unravel_index(s, lab.shape, order="F") for s in src]
  want, wpar = geodesicref.geodesic(lab, vox, connectivity, weights=w, parents=True)
  got, gpar = G.geodesic(lab, src, connectivity, weights=w, parents=True)
  assert same_bits(got, want) and np.array_equal(gpar, wpar)
  # weights with zeros: distances agree; parents exist only where no plateau is entered from a higher index
  w[rng.random(lab.shape) < 0.3] = 0
  assert same_bits(G.geodesic(lab, src, connectivity, weights=w), geodesicref.geodesic(lab, vox, connectivity, weights=w))


def test_zero_weight_plateau_and_the_guard():
  """a row of zero weights: everything is at distance 0.  From a source at the low end every voxel's
  parent is the voxel before it; from a source at the high end no voxel has a predecessor of lower
  (distance, index), and both the checker and the restatement say so instead of writing a cycle."""
  lab = np.ones((6, 1, 1), np.uint8)
  w = np.zeros((6, 1, 1), np.float32)
  dist, par = G.geodesic(lab, [0], 6, weights=w, parents=True)
  assert (dist == 0).all() and par.ravel().tolist() == [0, 1, 2, 3, 4, 5]
  assert np.array_equal(par, geodesicref.geodesic(lab, [(0, 0, 0)], 6, weights=w, parents=True)[1])
  with pytest.raises(G.NoParent):
    G.geodesic(lab, [5], 6, weights=w, parents=True)
  with pytest.raises(ValueError):
    geodesicref.geodesic(lab, [(5, 0, 0)], 6, weights=w, parents=True)


def test_unit_mask_matches_scipy():
  rng = np.random.default_rng(9)
  mask = rng.random((12, 10, 8)) < 0.75
  mask[0, 0, 0] = True
  idx = np.arange(mask.size).reshape(mask.shape, order="F")
  rows, cols = [], []
  for ax in range(3):
    a = [slice(None)] * 3
    b = [slice(None)] * 3
    a[ax], b[ax] = slice(0, -1), slice(1, None)
    both = mask[tuple(a)] & mask[tuple(b)]
    rows.append(idx[tuple(a)][both])
    cols.append(idx[tuple(b)][both])
  rows, cols = np.concatenate(rows), np.concatenate(cols)
  graph = coo_matrix((np.ones(rows.size), (rows, cols)), shape=(mask.size, mask.size)).tocsr()
  want = dijkstra(graph, directed=False, indices=0).reshape(mask.shape, order="F")
  want[~mask] = np.inf
  got = G.geodesic(mask.astype(np.uint8), [0], 6)
  assert np.array_equal(got, want.astype(np.float32))


def test_refused_sources_and_disconnected_parts():
  lab = np.zeros((7, 3, 1), np.uint16)
  lab[:3] = 5
  lab[4:] = 5  # the same label on both sides of a wall of zeros
  dist, par = G.geodesic(lab, [0], 26, parents=True)
  assert np.isfinite(dist[:3]).all() and np.isinf(dist[3:]).all() and not par[3:].any()
  with pytest.raises(ValueError):
    G.geodesic(lab, [3], 26)
  with pytest.raises(ValueError):
    G.geodesic(lab, [lab.size], 26)


def test_penalty_field_restatement():
  lab = np.array([[[1, 1, 2, 0]]], np.uint32).reshape(4, 1, 1)
  dbf = np.array([1, 2, 3, 0], np.float32).reshape(4, 1, 1)
  daf = np.array([0, 5, 0, np.inf], np.float32).reshape(4, 1, 1)
  p = geodesicref.pdrf(lab, dbf, daf, scale=10, exponent=2)
  t = np.float32(1) - np.float32(1) / (np.float32(1.01) * np.float32(2))
  assert p[0, 0, 0] == np.float32(10) * (t * t) and p[3, 0, 0] == 0
  t = np.float32(1) - np.float32(2) / (np.float32(1.01) * np.float32(2))
  assert p[1, 0, 0] == np.float32(10) * (t * t) + np.float32(1)
  t = np.float32(1) - np.float32(3) / (np.float32(1.01) * np.float32(3))
  assert p[2, 0, 0] == np.float32(10) * (t * t)  # a one-voxel label: max daf is 0 and the second term drops
