"""The two checkers of the cross-sectional area rule (DESIGN.md §5i) -- oracle_xsection's serial C and
tests/xsectionref.py's numpy -- against each other and against closed forms, without a GPU: solid boxes
whose section is the plane across the whole box, a one-voxel line, the contact bits, parallel tubes of one
label, a neighbouring label, and the normals of straight, kinked, branched, lone and cyclic skeletons."""
import itertools

import numpy as np
import pytest

import oracle_xsection as X
import xsectionref as R

REL = 2.0 ** -20
ANISO = [(1, 1, 1), (16, 16, 40), (1.1, 0.7, 3.3)]


def both(lab, voxels, point_labels, normals, a):
  """(area, contacts) of the C checker, after checking the numpy checker agrees"""
  ca, cc, _ = X.sections(lab, voxels, point_labels, normals, a)
  pa, pc = R.sections(lab, voxels, point_labels, normals, a)
  assert np.array_equal(cc, pc)
  np.testing.assert_allclose(pa, ca, rtol=REL, atol=0)
  return ca, cc


def box_section(n, lo, hi, p):
  """area of {x in [lo, hi] : n.(x - p) = 0}, by inclusion-exclusion over the corners of the one box"""
  n, lo, hi, p = (np.asarray(v, np.float64) for v in (n, lo, hi, p))
  nz = np.nonzero(n)[0]
  zero = np.prod([hi[i] - lo[i] for i in range(3) if n[i] == 0])
  m = len(nz)
  if m == 1:
    return zero
  f = 0.0
  for ups in itertools.product((0, 1), repeat=m):
    corner = sum(abs(n[i]) * ((hi[i] if up else lo[i]) if n[i] > 0 else -(lo[i] if up else hi[i]))
                 for i, up in zip(nz, ups))
    w = np.dot(np.abs(n), np.where(n >= 0, p, -p)) - corner
    if w > 0:
      f += (-1) ** sum(ups) * w ** (m - 1)
  return zero * f * np.linalg.norm(n) / (np.prod(np.abs(n[nz])) * (2 if m == 3 else 1))


@pytest.mark.parametrize("a", ANISO)
def test_plane_across_a_box_is_the_box_section(a):
  lab = np.zeros((14, 13, 12), np.uint16)
  lo, hi = np.array([2, 3, 2]), np.array([11, 9, 10])  # inclusive voxel ranges, away from every face
  lab[lo[0]:hi[0] + 1, lo[1]:hi[1] + 1, lo[2]:hi[2] + 1] = 7
  av = np.asarray(a, np.float64)
  size = (hi - lo + 1) * av
  for c in [(5, 6, 6), (2, 3, 2), (11, 9, 10)]:
    area, cont = both(lab, [c], [7], [(1.0 * a[0], 0, 0)], a)
    assert cont[0] == 0
    np.testing.assert_allclose(area[0], size[1] * size[2], rtol=REL)
  # oblique planes through inner voxels: the union of the voxel boxes is the box, and a voxel the plane only
  # touches adds nothing
  for c, n in [((6, 6, 6), (1, 2, 0)), ((5, 6, 5), (1, 2, 3)), ((7, 5, 6), (-3, 1, 2)), ((6, 6, 6), (2, -1, 1))]:
    nn = np.asarray(n, np.float64) * av
    area, _ = both(lab, [c], [7], [nn], a)
    want = box_section(nn, (lo - 0.5) * av, (hi + 0.5) * av, np.asarray(c) * av)
    np.testing.assert_allclose(area[0], want, rtol=REL)


@pytest.mark.parametrize("k,Z", [(2, 5), (4, 3)])
def test_diagonal_plane_through_a_square_prism(k, Z):
  side = 2 * k + 1
  lab = np.zeros((side + 4, side + 4, Z + 4), np.uint8)
  lab[2:2 + side, 2:2 + side, 2:2 + Z] = 1
  c = (2 + k, 2 + k, 2 + Z // 2)
  area, _ = both(lab, [c], [1], [(1.0, 1.0, 0.0)], (1, 1, 1))
  np.testing.assert_allclose(area[0], side * np.sqrt(2) * Z, rtol=REL)


@pytest.mark.parametrize("a", ANISO)
def test_one_voxel_line(a):
  lab = np.zeros((20, 5, 6), np.uint32)
  lab[1:19, 2, 3] = 3
  vox = np.array([(x, 2, 3) for x in range(1, 19)])
  edges = np.array([(i, i + 1) for i in range(len(vox) - 1)])
  for w in (1, 5):
    nc = X.normals(vox, edges, a, w)
    assert np.array_equal(nc, R.normals(vox, edges, a, w))
    assert np.all(nc[:, 1:] == 0) and np.all(nc[:, 0] != 0)
    area, cont = both(lab, vox, [3] * len(vox), nc, a)
    np.testing.assert_allclose(area, np.float32(a[1] * a[2]), rtol=REL)
    assert not cont.any()


def test_contact_bits():
  lab = np.zeros((10, 9, 8), np.uint8)
  lab[0:6, 4:9, 2:6] = 1  # touches x = 0 and y = sy - 1
  area, cont = both(lab, [(2, 6, 3)], [1], [(0, 0, 1.0)], (1, 1, 1))
  assert cont[0] == 0b1001
  assert area[0] == 30
  area, cont = both(lab, [(2, 6, 3)], [1], [(1.0, 0, 0)], (1, 1, 1))
  assert cont[0] == 0b1000  # the plane x = 2 meets y = sy - 1 only


def test_parallel_tubes_of_one_label_count_apart():
  lab = np.zeros((16, 12, 7), np.uint32)
  lab[:, 2:5, 2:5] = 9
  lab[:, 6:9, 2:5] = 9  # one voxel of background between them
  area, _ = both(lab, [(8, 3, 3), (8, 7, 3)], [9, 9], [(1.0, 0, 0), (1.0, 0, 0)], (1, 1, 1))
  assert list(area) == [9, 9]
  lab[:, 5, 3] = 9  # a bridge joins them
  area, _ = both(lab, [(8, 3, 3)], [9], [(1.0, 0, 0)], (1, 1, 1))
  assert area[0] == 19


def test_other_labels_do_not_count():
  lab = np.zeros((12, 10, 10), np.uint16)
  lab[:, 3:6, 3:6] = 1
  lab[:, 6:9, 3:6] = 2  # touching the tube
  lab[:, 3:6, 6] = 2
  area, _ = both(lab, [(6, 4, 4)], [1], [(1.0, 0, 0)], (1, 1, 1))
  assert area[0] == 9
  # a vertex whose voxel holds another label, and a zero normal, give nothing
  area, cont = both(lab, [(6, 7, 4), (6, 4, 4)], [1, 1], [(1.0, 0, 0), (0, 0, 0)], (1, 1, 1))
  assert list(area) == [0, 0] and list(cont) == [0, 0]


def normals_both(vox, edges, a, w):
  nc = X.normals(vox, edges, a, w)
  assert np.array_equal(nc, R.normals(vox, edges, a, w))
  return nc


@pytest.mark.parametrize("a", [(1, 1, 1), (1.1, 0.7, 3.3)])
def test_normals_straight_and_kinked(a):
  av = np.asarray(a, np.float64)
  line = np.array([(x, 4, 2) for x in range(6)])
  chain = np.array([(i, i + 1) for i in range(5)])
  assert np.array_equal(normals_both(line, chain, a, 3), np.tile([-3 * a[0], 0, 0], (6, 1)))
  # an L: 0..3 along x, then 4..6 along y; vertex 6 is the root and the path runs 0 -> 6
  L = np.array([(0, 0, 0), (1, 0, 0), (2, 0, 0), (3, 0, 0), (3, 1, 0), (3, 2, 0), (3, 3, 0)])
  edges = np.array([(i, i + 1) for i in range(6)])
  Xs, Ys = np.array([-1, 0, 0]), np.array([0, -1, 0])
  want = {  # (x steps, y steps) per vertex, from the step sequence X X X Y Y Y (Y) padded symmetrically
    1: [(1, 0), (1, 0), (1, 0), (0, 1), (0, 1), (0, 1), (0, 1)],
    3: [(3, 0), (3, 0), (2, 1), (1, 2), (0, 3), (0, 3), (0, 3)],
    4: [(4, 0), (4, 0), (3, 1), (2, 2), (1, 3), (0, 4), (0, 4)],
    5: [(5, 0), (4, 1), (3, 2), (2, 3), (1, 4), (0, 5), (0, 5)],
  }
  for w, rows in want.items():
    expect = np.array([(nx * Xs + ny * Ys) * av for nx, ny in rows])
    assert np.array_equal(normals_both(L, edges, a, w), expect), w


def test_normals_of_a_y_a_lone_vertex_and_a_cycle():
  # Y: centre 0, arm 1-2-3 along +x, arm 4-5 along +y, arm 6 along -y; root 3 (farthest from 0)
  vox = np.array([(5, 5, 5), (6, 5, 5), (7, 5, 5), (8, 5, 5), (5, 6, 5), (5, 7, 5), (5, 4, 5), (1, 1, 1)])
  edges = np.array([(0, 1), (1, 2), (2, 3), (0, 4), (4, 5), (0, 6)])
  n1 = normals_both(vox, edges, (1, 1, 1), 1)
  d = lambda u, p: vox[u] - vox[p]
  assert np.array_equal(n1[:7], [d(0, 1), d(1, 2), d(2, 3), d(2, 3), d(4, 0), d(5, 4), d(6, 0)])
  assert np.array_equal(n1[7], [0, 0, 0])  # the lone vertex
  n3 = normals_both(vox, edges, (1, 1, 1), 3)
  assert np.array_equal(n3[0], d(6, 0) + d(0, 1) + d(1, 2))  # 0 lies on the path of the shallower leaf 6
  assert np.array_equal(n3[4], d(5, 4) + d(4, 0) + d(0, 1))
  assert np.array_equal(n3[3], d(1, 2) + d(2, 3) + d(2, 3))
  # a square: root 2 (farthest from 0), parents 1 -> 2, 3 -> 2, 0 -> 1 (the lower of 1 and 3)
  sq = np.array([(0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0)])
  cyc = np.array([(0, 1), (1, 2), (2, 3), (3, 0)])
  n = normals_both(sq, cyc, (2, 3, 5), 1)
  a = np.array([2, 3, 5])
  assert np.array_equal(n, [(sq[0] - sq[1]) * a, (sq[1] - sq[2]) * a, (sq[3] - sq[2]) * a, (sq[3] - sq[2]) * a])


def test_zero_window_sum_falls_back_to_the_own_step():
  # a hairpin: the steps of a 2-window cancel at the turn
  vox = np.array([(0, 0, 0), (1, 0, 0), (0, 0, 0), (0, 1, 0), (0, 2, 0)])
  edges = np.array([(0, 1), (1, 2), (2, 3), (3, 4)])
  n = normals_both(vox, edges, (1, 1, 1), 2)
  assert np.array_equal(n[1], vox[1] - vox[2])


def test_checkers_agree_on_random_trees():
  rng = np.random.default_rng(5)
  lab = np.zeros((24, 22, 20), np.uint32)
  lab[3:21, 4:18, 2:18] = 1
  lab[8:14, 6:12, :] = 2
  for _ in range(6):
    V = int(rng.integers(2, 30))
    vox = np.clip(np.cumsum(rng.integers(-1, 2, (V, 3)), 0) + [12, 11, 10], 0, [23, 21, 19])
    edges = np.array([(i, int(rng.integers(0, i))) for i in range(1, V)])
    for w in (1, 4):
      n = normals_both(vox, edges, (1.1, 0.7, 3.3), w)
      both(lab, vox, lab[tuple(vox.T)], n, (1.1, 0.7, 3.3))
