"""The hole-filling rule (DESIGN.md "Hole filling") in its numpy transcription, tests/fillref.py,
pinned on hand-built volumes and against scipy.ndimage.binary_fill_holes.  No GPU."""
import numpy as np
import pytest
from scipy import ndimage

import fillref as F

KATS = F.kats()
CELL = 3


def _cavity(X, lo, hi):
  return np.s_[lo:hi, lo:hi, lo:hi]


def test_hollow_cell():
  X = KATS["hollow_cell"]
  filled, holes = F.fill_holes(X)
  want = X.copy()
  want[_cavity(X, 4, 12)] = CELL
  assert np.array_equal(filled, want)
  assert not holes.any()


@pytest.mark.parametrize("name,organelles", [("organelle_floating", [7]), ("organelle_wall", [7]),
                                             ("organelles_touching", [7, 8])])
def test_organelles_become_holes(name, organelles):
  X = KATS[name]
  filled, holes = F.fill_holes(X)
  want = X.copy()
  want[_cavity(X, 4, 12)] = CELL
  assert np.array_equal(filled, want)
  assert np.array_equal(holes, np.where(np.isin(X, organelles), X, 0))


def test_nested_shells():
  X = KATS["nested_three"]
  filled, holes = F.fill_holes(X)
  assert (filled[1:23, 1:23, 1:23] == 2).all() and (filled[0] == 0).all()
  assert np.array_equal(holes, np.where(np.isin(X, [4, 6]), X, 0))


def test_cavity_open_to_a_face_needs_fix_borders():
  X = KATS["open_to_face"]
  assert np.array_equal(F.fill_level(X, 1)[0], X)
  filled, holes = F.fill_level(X, 2)
  want = X.copy()
  want[0:10, 4:12, 4:12] = 5
  assert np.array_equal(filled, want) and not holes.any()


def test_floating_object_on_the_border_is_left_alone():
  X = np.zeros((12, 12, 12), np.uint32)
  X[0:4, 3:7, 3:7] = 4
  X[1:3, 4:6, 4:6] = 6   # enclosed by 4 except on the x = 0 face
  for level in (1, 2):
    filled, _ = F.fill_level(X, level)
    assert (filled[X == 4] == 4).all()


def test_threshold_fills_at_13_not_12():
  X = KATS["threshold"]
  for level in (1, 2, 3, 12):
    assert F.fill_level(X, level)[0][10, 10, 10] == 0, level
  for level in (13, 14, 50):
    assert F.fill_level(X, level)[0][10, 10, 10] == 3, level


def test_two_cycle_of_candidates():
  """Equal areas: the larger root (B, first voxel later in Fortran order) is absorbed into A."""
  X = KATS["cycle2"]
  filled, holes = F.fill_holes(X, p=60)
  want = X.copy()
  want[X == 2] = 1
  assert np.array_equal(filled, want)
  assert np.array_equal(holes, np.where(X == 2, 2, 0))
  # below the threshold nothing merges and nothing is enclosed
  assert np.array_equal(F.fill_holes(X, p=58)[0], X)


def test_triangle_resolves_in_pairs():
  """Three bars with equal pairwise contacts: 1 and 2 point at each other (2 points at the lower
  root of two equal contacts) and 2 is absorbed; the pair and 3 then point at each other."""
  X = KATS["triangle"]
  comp, N, value = F.components(X)
  w, wo = F.contacts(comp)
  ids = {int(v): c for c, v in enumerate(value) if v in (1, 2, 3)}
  assert w[(ids[1], ids[2])] == w[(ids[1], ids[3])] == w[(ids[2], ids[3])]
  root = F.merge(N, w, wo, 80)
  assert root[ids[2]] == ids[1] and root[ids[3]] == ids[1]
  assert F.merge(N, w, wo, 77) == list(range(N + 1))


@pytest.mark.parametrize("seed", [11, 12])
def test_candidate_targets_form_no_cycle_longer_than_two(seed):
  """Contacts are symmetric, so along a cycle of targets the weights cannot fall and ties go to
  the lower root: only 2-cycles exist, and the rule's longer-cycle fallback never runs."""
  X = F.random_volume((40, 40, 40), seed, pitch=8)
  comp, N, value = F.components(X)
  w, wo = F.contacts(comp)
  nbrs = {}
  for (a, b), c in w.items():
    nbrs.setdefault(a, {})[b] = c
    nbrs.setdefault(b, {})[a] = c
  target = {r: min(nb, key=lambda u: (-nb[u], u)) for r, nb in nbrs.items() if not wo.get(r)}
  for r in target:
    seen, v = [], r
    while v in target and v not in seen:
      seen.append(v)
      v = target[v]
    if v in seen:
      assert len(seen) - seen.index(v) <= 2


def test_dilation_ties_and_counts():
  X = np.zeros((5, 5, 5), np.uint32)
  X[1, 2, 2] = 9
  X[3, 2, 2] = 9
  X[2, 1, 2] = 4
  X[2, 3, 2] = 4
  X[0, 0, 0] = 7
  D = F.dilate(X)
  assert D[2, 2, 2] == 4                 # 2 vs 2: the smaller label
  assert D[1, 1, 1] == 4 and D[0, 1, 0] == 7 and D[4, 4, 4] == 0
  assert np.array_equal(D[X != 0], X[X != 0])
  X[2, 2, 1] = 9
  assert F.dilate(X)[2, 2, 2] == 9       # 3 vs 2


@pytest.mark.parametrize("seed", [1, 2, 3, 4])
def test_matches_scipy_fill_for_single_component_labels(seed):
  X = F.single_component_labels(F.random_volume((40, 36, 33), seed))
  filled, holes = F.fill_holes(X)
  assert np.array_equal(filled, F.scipy_fill(X))
  assert np.array_equal(holes, np.where((filled != X) & (X != 0), X, 0))


@pytest.mark.parametrize("seed", [5, 6])
def test_random_volumes_fill_something(seed):
  X = F.random_volume((48, 48, 40), seed)
  for level in (1, 4, 103):
    filled, holes = F.fill_level(X, level)
    assert (holes != 0).any() or (filled != X).any()


@pytest.mark.parametrize("seed", [7, 8, 9])
def test_lowlink_equals_separator_definition(seed):
  X = F.random_volume((48, 48, 40), seed)
  for p in (0, 50):
    comp, N, value = F.components(X)
    w, wo = F.contacts(comp)
    root = F.merge(N, w, wo, p) if p else list(range(N + 1))
    regions = sorted(set(root[1:]))
    edges = {(min(root[a], root[b]), max(root[a], root[b])) for a, b in w if root[a] != root[b]}
    touch = {root[a] for a in wo}
    want = F.fillers_bruteforce(regions, edges, touch, value)
    assert want or p  # merging at 50 % may leave nothing enclosed
    assert F.fillers_lowlink(regions, edges, touch, value) == want


def test_create_meshing_tasks_rejects_fill_level_104():
  from igneous_b200.task_creation import create_meshing_tasks
  with pytest.raises(AssertionError):
    create_meshing_tasks("file:///nonexistent-layer", 0, fill_holes=104)
  with pytest.raises(AssertionError):
    create_meshing_tasks("file:///nonexistent-layer", 0, fill_holes=-1)


def test_merge_threshold_must_be_whole_percent():
  from igneous_b200 import fastmorph
  assert fastmorph.merge_threshold_pct(1.0) == 100
  assert fastmorph.merge_threshold_pct(1.0 - 0.01 * 100) == 0
  assert all(fastmorph.merge_threshold_pct(1.0 - 0.01 * (lv - 3)) == 103 - lv for lv in range(3, 104))
  for bad in (0.995, 1.01, -0.01):
    with pytest.raises(ValueError):
      fastmorph.merge_threshold_pct(bad)
