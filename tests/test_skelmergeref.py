"""The skeleton merge rule of DESIGN.md §5h: the numpy restatement (tests/skelmergeref.py) on hand-built
skeletons of known answer, and the serial C checker (oracle_skeleton/merge_oracle.c) against the restatement
on random fragment sets (no shared code).  No GPU."""
import numpy as np
import pytest

import oracle_skeleton as C
import skelmergeref as R
from igneous_b200 import kimimaro
from igneous_b200._compat import Bbox


def sk(v, e, r=None, t=None):
  v = np.asarray(v, np.float32).reshape(-1, 3)
  r = np.ones(len(v), np.float32) if r is None else np.asarray(r, np.float32)
  t = np.zeros(len(v), np.uint8) if t is None else np.asarray(t, np.uint8)
  return v, np.asarray(e, np.uint32).reshape(-1, 2), r, t


def path(points, r=0.1):
  return sk(points, [(i, i + 1) for i in range(len(points) - 1)], np.full(len(points), r))


def edges(s):
  return [tuple(map(int, x)) for x in s[1]]


def coords(s):
  return [tuple(map(float, x)) for x in s[0]]


def test_duplicates_keep_the_first_fragment_and_sort():
  a = sk([[2, 0, 0], [1, 0, 0]], [(0, 1)], r=[5, 6], t=[1, 2])
  b = sk([[1, 0, 0], [3, 0, 0], [-0.0, 0, 0]], [(0, 1), (0, 2)], r=[7, 8, 9], t=[3, 4, 5])
  v, e, r, t = R.fuse([a, b], [None, None])
  assert coords((v,)) == [(0, 0, 0), (1, 0, 0), (2, 0, 0), (3, 0, 0)]
  assert np.signbit(v[0, 0])  # the bits of the first occurrence
  assert r.tolist() == [9, 6, 5, 8] and t.tolist() == [5, 2, 1, 4]
  assert edges((v, e)) == [(0, 1), (1, 2), (1, 3)]


def test_self_loops_duplicates_and_lone_vertices_go():
  v, e, r, t = R.consolidate(sk([[0, 0, 0], [0, 0, 0], [1, 0, 0], [5, 5, 5]], [(0, 1), (1, 2), (2, 0), (0, 2)]))
  assert coords((v,)) == [(0, 0, 0), (1, 0, 0)] and edges((v, e)) == [(0, 1)]
  assert len(R.consolidate(sk([[0, 0, 0], [0, 0, 0]], [(0, 1)]))[0]) == 0


def test_crop_and_the_zero_volume_box():
  s = path([[0, 0, 0], [5, 5, 5], [10, 10, 10], [15, 5, 5]])
  assert R.crop_box((0, 0, 0), (20, 20, 20), 0, (1, 1, 1)) is None
  box = R.crop_box((0, 0, 0), (20, 20, 20), 5, (1, 1, 1))
  v, e, _, _ = R.crop(s, box)
  assert coords((v,)) == [(5, 5, 5), (10, 10, 10), (15, 5, 5)] and edges((v, e)) == [(0, 1), (1, 2)]
  assert R.crop_box((0, 0, 0), (20, 20, 20), 10, (1, 1, 1)) is None  # volume 0: uncropped
  assert R.crop_box((0, 0, 0), (20, 20, 20), 3, (1, 1, 4)) is None
  # the product's crop box agrees
  assert kimimaro.crop_box(Bbox((0, 0, 0), (20, 20, 20)), 10, (1, 1, 1)) is None
  assert np.array_equal(kimimaro.crop_box(Bbox((0, 0, 0), (20, 20, 40)), 2, (1, 2, 3)), [2, 4, 6, 18, 16, 34])


def test_dust_just_under_and_over():
  s = path([[0, 0, 0], [10, 0, 0], [20, 0, 0]])
  assert len(R.postprocess(s, dust_threshold=20.5, tick_threshold=0)[0]) == 0
  assert len(R.postprocess(s, dust_threshold=19.5, tick_threshold=0)[0]) == 3
  assert len(R.postprocess(s, dust_threshold=0, tick_threshold=0)[0]) == 3


def test_loop_without_branches_goes():
  s = sk([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0]], [(0, 1), (1, 2), (2, 3), (3, 0)], r=[0.1] * 4)
  assert len(R.postprocess(s, 0, 0)[0]) == 0


def test_loop_with_one_branch_becomes_a_spoke():
  # square 0-1-2-3 with a tail at 0: the branch is 0, the farthest cycle vertex is 2
  s = sk([[0, 0, 0], [1, 0, 0], [1, 1, 0], [0, 1, 0], [-5, 0, 0]], [(0, 1), (1, 2), (2, 3), (3, 0), (0, 4)],
         r=[0.1] * 5)
  v, e, _, _ = R.postprocess(s, 0, 0)
  assert coords((v,)) == [(-5, 0, 0), (0, 0, 0), (1, 1, 0)] and edges((v, e)) == [(0, 1), (1, 2)]


def test_loop_with_two_branches_keeps_the_shorter_arc_and_the_tie():
  # hexagon with tails at vertices 0 and 2: arcs of 2 and 4 edges
  ring = [[2, 0, 0], [1, 1.7, 0], [-1, 1.7, 0], [-2, 0, 0], [-1, -1.7, 0], [1, -1.7, 0]]
  s = sk(ring + [[9, 0, 0], [-1, 9, 0]], [(i, (i + 1) % 6) for i in range(6)] + [(0, 6), (2, 7)], r=[0.01] * 8)
  v, e, _, _ = R.postprocess(s, 0, 0)
  assert len(e) == len(v) - 1 == 4
  assert (1.0, 1.7000000476837158, 0.0) in coords((v,)) and (-2.0, 0.0, 0.0) not in coords((v,))
  # tails at 0 and 3: equal arcs; the one holding the smaller index is kept
  s = sk(ring + [[9, 0, 0], [-9, 0, 0]], [(i, (i + 1) % 6) for i in range(6)] + [(0, 6), (3, 7)], r=[0.01] * 8)
  # consolidated order by x: the lower arc's interior holds index 2 = (-1, -1.7), the upper arc's 3 and 5
  v, e, _, _ = R.postprocess(s, 0, 0)
  assert len(e) == len(v) - 1 == 5
  y = float(np.float32(1.7))
  assert (-1.0, -y, 0.0) in coords((v,)) and (-1.0, y, 0.0) not in coords((v,))


def test_loop_with_three_branches_drops_the_longest_edge():
  tri = [[0, 0, 0], [4, 0, 0], [0, 3, 0]]
  s = sk(tri + [[-9, 0, 0], [9, 0, 0], [0, 9, 0]], [(0, 1), (1, 2), (2, 0), (0, 3), (1, 4), (2, 5)], r=[0.01] * 6)
  v, e, _, _ = R.postprocess(s, 0, 0)
  assert len(e) == 5
  pts = coords((v,))
  assert (pts.index((0, 3, 0)), pts.index((4, 0, 0))) not in edges((v, e))  # the hypotenuse (length 5) went
  assert tuple(sorted((pts.index((4, 0, 0)), pts.index((0, 3, 0))))) not in edges((v, e))


def test_pieces_join_inside_the_radii_and_not_beyond():
  a, b = path([[0, 0, 0], [10, 0, 0]], r=1.0), path([[11.5, 0, 0], [20, 0, 0]], r=1.0)
  v, e, _, _ = R.fuse([a, b], [None, None])
  got = R.postprocess((v, e, np.full(len(v), 1.0, np.float32), np.zeros(len(v), np.uint8)), 0, 0)
  assert edges(got) == [(0, 1), (1, 2), (2, 3)]
  got = R.postprocess((v, e, np.full(len(v), 0.7, np.float32), np.zeros(len(v), np.uint8)), 0, 0)
  assert edges(got) == [(0, 1), (2, 3)]


def test_a_y_loses_its_short_tick_only():
  # trunk 0..100 on x, a short tick of 5 and a long one of 50 at the branch (100, 0, 0)
  s = sk([[0, 0, 0], [100, 0, 0], [100, 5, 0], [100, -50, 0]], [(0, 1), (1, 2), (1, 3)], r=[0.01] * 4)
  v, e, _, _ = R.postprocess(s, 0, 10)
  assert coords((v,)) == [(0, 0, 0), (100, -50, 0), (100, 0, 0)] and len(e) == 2
  v, e, _, _ = R.postprocess(s, 0, 4)
  assert len(v) == 4


def test_a_plain_path_is_never_trimmed():
  s = path([[0, 0, 0], [1, 0, 0], [2, 0, 0]], r=0.01)
  assert len(R.postprocess(s, 0, 1e9)[0]) == 3


def test_max_cable_length_skips_postprocessing():
  s = path([[0, 0, 0], [10, 0, 0], [20, 0, 0]])
  assert len(R.merge([s], dust_threshold=100, tick_threshold=0, max_cable_length=15)[0]) == 3
  assert len(R.merge([s], dust_threshold=100, tick_threshold=0, max_cable_length=25)[0]) == 0
  assert len(R.merge([s], dust_threshold=100, tick_threshold=0)[0]) == 0


class _S:
  def __init__(self, v, e, r, t):
    self.vertices, self.edges, self.radii, self.vertex_types = v, e, r, t


def random_batch(seed, labels=6):
  """fragments of random trees on a coarse grid: shared vertices across fragments, loops, near pieces"""
  rng = np.random.default_rng(seed)
  out = {}
  for l in range(labels):
    frags = []
    for _ in range(int(rng.integers(1, 4))):
      n = int(rng.integers(2, 25))
      v = rng.integers(0, 6, size=(n, 3)).astype(np.float32) * np.float32(3.5)
      parent = [int(rng.integers(0, i)) for i in range(1, n)]
      e = [(i, p) for i, p in zip(range(1, n), parent)]
      e += [tuple(int(x) for x in rng.integers(0, n, 2)) for _ in range(int(rng.integers(0, 4)))]
      r = rng.uniform(0.5, 4.0, n).astype(np.float32)
      t = rng.integers(0, 5, n).astype(np.uint8)
      lo = rng.integers(0, 6, 3) * 3
      box = Bbox(lo, lo + 12) if rng.random() < 0.5 else None
      frags.append((box, _S(v, np.array(e, np.uint32).reshape(-1, 2), r, t)))
    out[int(rng.integers(1, 1 << 40)) if l % 2 else l + 1] = frags
  return out


def signed_zero_batch(seed, labels=6):
  """random_batch with about half of its zero coordinates written as -0.0: the same positions then occur
  with both signs, in either order"""
  rng = np.random.default_rng(seed + 1000)
  batch = random_batch(seed, labels)
  for frags in batch.values():
    for _, f in frags:
      v = f.vertices.copy()
      flip = (v == 0) & (rng.random(v.shape) < 0.5)
      v[flip] = np.float32(-0.0)
      f.vertices = v
  return batch


def ref_batch(batch, crop, dust, tick, max_cable, vertex_types=True):
  blobs = []
  for frags in batch.values():
    sks = [(f.vertices, f.edges, f.radii, f.vertex_types) for _, f in frags]
    boxes = [None if b is None else R.crop_box(b.minpt, b.maxpt, crop, (1, 1, 1)) for b, _ in frags]
    blobs.append(R.encode(R.merge(sks, boxes, dust, tick, max_cable), vertex_types))
  return blobs


def split(buf, table):
  return [bytes(buf[int(o):int(o) + 8 + 16 * int(nv) + 8 * int(ne) + int(nv)]) for _, o, nv, ne in table]


@pytest.mark.parametrize("seed", range(8))
@pytest.mark.parametrize("crop,dust,tick,max_cable", [(0, 0, 0, None), (1, 30, 0, None), (0, 0, 12, None),
                                                      (2, 20, 10, None), (0, 10, 8, 60.5)])
def test_checker_matches_restatement(seed, crop, dust, tick, max_cable):
  batch = random_batch(seed)
  _, packed = kimimaro.pack_fragments(batch, crop=crop)
  buf, table = C.merge(packed, dust, tick, max_cable)
  assert table[:, 0].tolist() == list(range(len(batch)))
  assert split(buf, table) == ref_batch(batch, crop, dust, tick, max_cable)


@pytest.mark.parametrize("seed", range(4))
def test_checker_matches_restatement_on_signed_zeros(seed):
  batch = signed_zero_batch(seed)
  _, packed = kimimaro.pack_fragments(batch)
  assert np.signbit(packed["vertices"][packed["vertices"] == 0]).any()
  buf, table = C.merge(packed, 0, 0, None)
  assert split(buf, table) == ref_batch(batch, 0, 0, 0, None)


def test_checker_refusals():
  batch = random_batch(0, labels=2)
  _, packed = kimimaro.pack_fragments(batch)
  bad = dict(packed, edges=packed["edges"].copy())
  bad["edges"][0, 1] = packed["frag_vert"][1]
  with pytest.raises(ValueError, match="outside its fragment"):
    C.merge(bad)
  bad = dict(packed, vertices=packed["vertices"].copy())
  bad["vertices"][3, 2] = np.nan
  with pytest.raises(ValueError, match="non-finite"):
    C.merge(bad)
