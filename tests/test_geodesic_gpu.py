"""igneous_b200.dijkstra3d and igneous_b200.teasar against the serial C checker of DESIGN.md §5e
(oracle_geodesic/), bit for bit: distances and parents at each connectivity, representable and
non-representable anisotropy, shapes that are not brick multiples, every label dtype (u64 labels that
differ only in their high bits), both memory orders and 1-D / 2-D input; all labels in one call against
one call per label; a serpentine corridor; a label in two parts; field weights (random, with zeros, a
float32 plateau that needs the parent rule's guard, and one it refuses); path_from_parents;
the per-label argmax; teasar.fields against a restatement built from edt, the checker and the formula;
refusals; and a volume past 2^32 voxels in closed form."""
import ctypes as c

import numpy as np
import pytest

import geodesicref
import oracle_geodesic as G

pytestmark = pytest.mark.gpu

ANISO = [(1.0, 1.0, 1.0), (4.0, 4.0, 40.0), (1.1, 0.7, 3.3)]
SHAPES = [(33, 29, 17), (129, 7, 5), (1, 1, 1), (5, 1, 3), (70, 65, 3)]


def blobs(shape, seed, labels=4, block=3):
  """blocks of block^3 voxels of random labels 0..labels: several objects, some in more than one part"""
  rng = np.random.default_rng(seed)
  coarse = rng.integers(0, labels + 1, size=[(n + block - 1) // block for n in shape])
  full = np.kron(coarse, np.ones((block,) * 3, int))[:shape[0], :shape[1], :shape[2]]
  return np.asfortranarray(full.astype(np.uint32))


def first_voxels(lab):
  """linear F-order index of the first voxel of every non-zero label (uint64)"""
  flat = lab.ravel(order="F")
  ids, first = np.unique(flat, return_index=True)
  return np.sort(first[ids != 0]).astype(np.uint64)


def bits(a):
  return np.asarray(a).view(np.uint32)


def check_parents(par, dist, lab, src, connectivity, weights=None, anisotropy=(1, 1, 1)):
  """the invariants of a parent field, without the checker: a parent is a neighbour of the same label,
  fl32(d[parent] + w) == d[q], and every walk ends at a source in fewer steps than the label has voxels"""
  shape = lab.shape
  flat_p, flat_d, flat_l = (v.ravel(order="F") for v in (par, dist, lab))
  reached = np.isfinite(flat_d) & (flat_l != 0)
  is_src = np.zeros(lab.size, bool)
  is_src[np.asarray(src, dtype=np.int64)] = True
  assert np.array_equal(flat_p != 0, reached & ~is_src)
  q = np.flatnonzero(flat_p)
  p = flat_p[q].astype(np.int64) - 1
  assert np.array_equal(flat_l[p], flat_l[q])
  delta = np.stack(np.unravel_index(p, shape, order="F")) - np.stack(np.unravel_index(q, shape, order="F"))
  assert np.abs(delta).max(initial=0) <= 1 and (np.abs(delta).sum(0) <= {6: 1, 18: 2, 26: 3}[connectivity]).all()
  if weights is not None:
    w = weights.ravel(order="F")[q]
  else:
    length = dict(geodesicref.neighbours(connectivity, anisotropy))
    w = np.array([length[tuple(d)] for d in delta.T.tolist()], np.float32)
  assert np.array_equal(flat_d[p] + w, flat_d[q])
  hops, at = 0, q.copy()
  counts = np.bincount(flat_l.astype(np.int64))
  while at.size:
    at = flat_p[at].astype(np.int64) - 1
    at = at[~is_src[at]]
    hops += 1
    assert hops < counts.max()
  return True


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("anisotropy", ANISO, ids=["iso", "4-4-40", "inexact"])
@pytest.mark.parametrize("connectivity", [6, 18, 26])
def test_euclidean_fields_and_parents_match_the_checker(ctx, shape, anisotropy, connectivity):
  from igneous_b200 import _shim
  lab = blobs(shape, seed=sum(shape) + connectivity)
  if not lab.any():
    lab[...] = 3
  src = first_voxels(lab)
  want, wpar = G.geodesic(lab, src, connectivity, anisotropy, parents=True)
  got = np.empty(shape, np.float32, order="F")
  par = np.empty(shape, np.uint32, order="F")
  a = (c.c_float * 3)(*anisotropy)
  _shim.check(ctx.lib.ign_geodesic(ctx.handle, _shim.ptr(lab), _shim.IGN_U32, *shape, connectivity, a, None,
                                   _shim.ptr(src), src.size, _shim.ptr(got), _shim.ptr(par)))
  assert np.array_equal(bits(got), bits(want))
  assert np.array_equal(par, wpar)
  assert check_parents(par, got, lab, src, connectivity, anisotropy=anisotropy)
  from igneous_b200 import dijkstra3d
  assert np.array_equal(bits(dijkstra3d.euclidean_distance_field(lab, None, anisotropy, connectivity, source_indices=src, ctx=ctx)),
                        bits(want))


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.uint64, np.int8, np.int64, np.bool_])
@pytest.mark.parametrize("order", ["F", "C"])
def test_dtypes_and_orders(ctx, dtype, order):
  from igneous_b200 import dijkstra3d
  small = blobs((37, 21, 13), seed=3)
  lab = small.astype(np.uint64)
  if np.dtype(dtype).itemsize == 8:
    lab = np.where(small == 0, 0, (lab << np.uint64(40)) + np.uint64(5))  # the labels differ only above bit 40
  if dtype == np.bool_:
    small = (small != 0).astype(np.uint32)
    lab = small
  lab = np.asarray(lab.astype(dtype), order=order)
  if np.dtype(dtype).kind == "i":
    lab[small == 3] = -3  # a negative label is just another value
  vox = [np.unravel_index(int(i), small.shape, order="F") for i in first_voxels(small)]
  want = G.geodesic(small, first_voxels(small), 26, (4, 4, 40))
  got = dijkstra3d.euclidean_distance_field(lab, vox, (4, 4, 40), 26, ctx=ctx)
  assert got.flags.c_contiguous == lab.flags.c_contiguous
  assert np.array_equal(bits(np.asfortranarray(got)), bits(want))
  # {label: voxel} names the same sources
  by_label = {lab[v].item(): v for v in vox}
  assert np.array_equal(bits(dijkstra3d.euclidean_distance_field(lab, by_label, (4, 4, 40), ctx=ctx)), bits(got))


def test_u64_high_bits_stay_distinct(ctx):
  from igneous_b200 import dijkstra3d
  lab = np.ones((8, 3, 2), np.uint64)
  lab[4:] = 2**32 + 1
  got = dijkstra3d.euclidean_distance_field(lab, (0, 0, 0), connectivity=6, ctx=ctx)
  assert np.array_equal(got[:4, 0, 0], np.arange(4, dtype=np.float32)) and np.isinf(got[4:]).all()


def test_one_and_two_dimensions(ctx):
  from igneous_b200 import dijkstra3d
  rng = np.random.default_rng(2)
  row = (rng.random(300) < 0.97).astype(np.uint8)
  row[100] = 1
  got = dijkstra3d.euclidean_distance_field(row, 100, anisotropy=2.5, ctx=ctx)
  assert np.array_equal(bits(got), bits(G.geodesic(row, [100], 6, (2.5, 1, 1))))
  plane = blobs((61, 47, 1), seed=8)[:, :, 0]
  src = first_voxels(plane[:, :, None])
  for conn2, conn3 in ((4, 6), (8, 18)):
    want = G.geodesic(plane, src, conn3, (3, 5, 1))
    for arr in (np.asfortranarray(plane), np.ascontiguousarray(plane)):
      vox = [np.unravel_index(int(i), plane.shape, order="F") for i in src]
      got = dijkstra3d.euclidean_distance_field(arr, vox, (3, 5), conn2, ctx=ctx)
      assert np.array_equal(bits(np.asfortranarray(got)), bits(want))
  with pytest.raises(ValueError):
    dijkstra3d.euclidean_distance_field(plane, (0, 0), connectivity=26, ctx=ctx)


def test_all_labels_in_one_call_equal_one_call_per_label(ctx):
  from igneous_b200 import dijkstra3d
  rng = np.random.default_rng(4)
  # every voxel of a 4^3 block grid its own object: 385 labels in one call
  coarse = rng.permutation(11 * 7 * 5).reshape(11, 7, 5) + 1
  lab = np.asfortranarray(np.kron(coarse, np.ones((4, 4, 4), int)).astype(np.uint32))
  src = first_voxels(lab)
  every = dijkstra3d.euclidean_distance_field(lab, None, (4, 4, 40), 26, source_indices=src, ctx=ctx)
  flat = lab.ravel(order="F")
  for s in src[::29]:
    l = flat[int(s)]
    one = dijkstra3d.euclidean_distance_field(lab == l, None, (4, 4, 40), 26, source_indices=[int(s)], ctx=ctx)
    assert np.array_equal(bits(one[lab == l]), bits(every[lab == l])) and np.isinf(one[lab != l]).all()
  assert np.array_equal(bits(every), bits(G.geodesic(lab, src, 26, (4, 4, 40))))


def test_serpentine_corridor(ctx):
  from igneous_b200 import dijkstra3d, _shim
  snake = np.zeros((100, 64, 4), dtype=np.uint8, order="F")
  for y in range(0, 64, 2):  # one corridor one voxel wide, 3,200 voxels long: the most rounds per voxel
    snake[:, y, 0] = 1
    snake[99 if (y // 2) % 2 == 0 else 0, y + 1, 0] = 1
  for connectivity in (6, 26):
    want, wpar = G.geodesic(snake, [0], connectivity, parents=True)
    w = np.ones(snake.shape, np.float32, order="F")
    got = dijkstra3d.distance_field(w, (0, 0, 0), connectivity, labels=snake, ctx=ctx)
    stats = (c.c_uint64 * 3)()
    _shim.check(ctx.lib.ign_geodesic_last_stats(stats))
    assert stats[0] >= 32 * 3 and stats[1] >= stats[0] and stats[2] >= stats[0] // 8
    assert np.array_equal(bits(dijkstra3d.euclidean_distance_field(snake, (0, 0, 0), connectivity=connectivity,
                                                                   ctx=ctx)), bits(want))
    assert np.array_equal(dijkstra3d.parental_field(w, (0, 0, 0), connectivity, labels=snake, ctx=ctx),
                          G.geodesic(snake, [0], connectivity, weights=w, parents=True)[1])
    if connectivity == 6:
      assert np.array_equal(bits(got), bits(want)) and got[snake != 0].max() == 99 * 32 + 63
  cap = c.c_uint64(0)
  _shim.check(ctx.lib.ign_geodesic_round_cap(100, 64, 4, c.byref(cap)))
  assert cap.value == 100 * 64 * 4 + 1


def test_label_in_two_parts(ctx):
  from igneous_b200 import dijkstra3d
  lab = np.zeros((40, 12, 9), np.uint16)
  lab[:19] = 7
  lab[21:] = 7
  lab[19:21, :, :4] = 9
  w = np.ones(lab.shape, np.float32)
  dist = dijkstra3d.distance_field(w, [(2, 3, 4), (19, 0, 0)], labels=lab, ctx=ctx)
  par = dijkstra3d.parental_field(w, [(2, 3, 4), (19, 0, 0)], labels=lab, ctx=ctx)
  assert np.isfinite(dist[:19]).all() and np.isfinite(dist[19:21, :, :4]).all()
  assert np.isinf(dist[21:]).all() and not par[21:].any() and np.isinf(dist[19:21, :, 4:]).all()
  fpar = dijkstra3d.parental_field(np.asfortranarray(w), [(2, 3, 4), (19, 0, 0)], labels=np.asfortranarray(lab), ctx=ctx)
  assert check_parents(fpar, np.asfortranarray(dist), np.asfortranarray(lab),
                       np.ravel_multi_index(([2, 19], [3, 0], [4, 0]), lab.shape, order="F"), 26,
                       weights=np.asfortranarray(w))
  # C-order input: the parents index the array in its own (C) order
  src = np.ravel_multi_index(([2, 19], [3, 0], [4, 0]), lab.shape, order="C")
  flat = par.ravel()
  assert flat[src[0]] == 0 and flat[np.ravel_multi_index((2, 3, 5), lab.shape)] == src[0] + 1


@pytest.mark.parametrize("connectivity", [6, 18, 26])
def test_field_weights(ctx, connectivity):
  from igneous_b200 import dijkstra3d
  rng = np.random.default_rng(connectivity)
  lab = blobs((45, 38, 21), seed=12, labels=2, block=5)
  src = first_voxels(lab)
  w = np.asfortranarray((rng.random(lab.shape) * 100 + 1e-3).astype(np.float32))
  want, wpar = G.geodesic(lab, src, connectivity, weights=w, parents=True)
  got = dijkstra3d.distance_field(w, None, connectivity, labels=lab, source_indices=src, ctx=ctx)
  par = dijkstra3d.parental_field(w, None, connectivity, labels=lab, source_indices=src, ctx=ctx)
  assert np.array_equal(bits(got), bits(want)) and np.array_equal(par, wpar)
  assert check_parents(par, got, lab, src, connectivity, weights=w)
  # one object without labels=, float64 weights
  one = dijkstra3d.distance_field(w.astype(np.float64), (1, 2, 3), connectivity, ctx=ctx)
  s = [int(np.ravel_multi_index((1, 2, 3), lab.shape, order="F"))]
  assert np.array_equal(bits(one), bits(G.geodesic(np.ones(lab.shape, np.uint8), s, connectivity, weights=w)))
  # weights with zeros: whole stretches at one distance
  w[rng.random(lab.shape) < 0.4] = 0
  assert np.array_equal(bits(dijkstra3d.distance_field(w, None, connectivity, labels=lab, source_indices=src, ctx=ctx)),
                        bits(G.geodesic(lab, src, connectivity, weights=w)))


def test_plateau_needs_the_guard(ctx):
  """2^25 + 2 rounds back to 2^25: q = (0, 0) and r = (1, 0) sit at the same distance and each is a
  float32-exact predecessor of the other.  The guard refuses r for q (same distance, higher index), so q
  takes the voxel it was entered from and r takes q: no cycle."""
  from igneous_b200 import dijkstra3d
  lab = np.asfortranarray(np.array([[1, 1, 1], [1, 0, 0]], np.uint8))  # (x, y): shape (2, 3)
  w = np.asfortranarray(np.array([[2, 2**25 - 2, 7], [1, 0, 0]], np.float32))
  dist = dijkstra3d.distance_field(w, (0, 2), 4, labels=lab, ctx=ctx)
  assert dist[0, 1] == 2**25 - 2 and dist[0, 0] == dist[1, 0] == 2**25
  par = dijkstra3d.parental_field(w, (0, 2), 4, labels=lab, ctx=ctx)
  assert par.ravel(order="F").tolist() == [3, 1, 5, 0, 0, 0]
  assert np.array_equal(par[:, :, None], G.geodesic(lab, [4], 6, weights=w, parents=True)[1].reshape(2, 3, 1))
  assert dijkstra3d.path_from_parents(par, (1, 0)).tolist() == [[0, 2], [0, 1], [0, 0], [1, 0]]


def test_plateau_entered_from_a_higher_index_is_refused(ctx):
  from igneous_b200 import dijkstra3d, _shim
  lab = np.ones(6, np.uint8)
  w = np.zeros(6, np.float32)
  assert dijkstra3d.parental_field(w, 0, ctx=ctx).tolist() == [0, 1, 2, 3, 4, 5]
  with pytest.raises(_shim.IgneousB200Error, match="index 0 .*plateau"):  # voxel 0: its only neighbour has the higher index
    dijkstra3d.parental_field(w, 5, ctx=ctx)
  with pytest.raises(G.NoParent):
    G.geodesic(lab, [5], 6, weights=w, parents=True)
  assert (dijkstra3d.distance_field(w, 5, ctx=ctx) == 0).all()  # the distances alone are fine


def test_path_from_parents(ctx):
  from igneous_b200 import dijkstra3d
  lab = blobs((30, 26, 14), seed=21, labels=1, block=7)
  lab[:, 0, :] = 1
  lab[0, :, :] = 1
  rng = np.random.default_rng(1)
  w = (rng.random(lab.shape) + 0.5).astype(np.float32)
  for arr, ww in ((lab, np.asfortranarray(w)), (np.ascontiguousarray(lab), np.ascontiguousarray(w))):
    par = dijkstra3d.parental_field(ww, (0, 0, 0), 26, labels=arr, ctx=ctx)
    dist = dijkstra3d.distance_field(ww, (0, 0, 0), 26, labels=arr, ctx=ctx)
    target = tuple(int(v) for v in np.argwhere(np.isfinite(dist))[-1])
    path = dijkstra3d.path_from_parents(par, target)
    assert tuple(path[0]) == (0, 0, 0) and tuple(path[-1]) == target and len(path) > 3
    assert np.abs(np.diff(path, axis=0)).max() == 1
    d = np.float32(0)
    for v in path[1:]:
      d = d + w[tuple(v)]
    assert d == dist[target]


def test_label_argmax(ctx):
  from igneous_b200 import _shim
  rng = np.random.default_rng(6)
  n, K = 70001, 37
  lab = rng.integers(0, K + 3, n).astype(np.uint16)  # labels K+1, K+2 lie above max_label
  field = rng.integers(-5, 9, n).astype(np.float32)  # many ties
  field[rng.random(n) < 0.1] = np.inf
  field[rng.random(n) < 0.05] = np.nan
  field[lab == 5] = -np.inf  # a label without a finite value
  d_lab, d_field = ctx.to_device(lab), ctx.to_device(field)
  d_idx, d_val = ctx.alloc((K + 1) * 8), ctx.alloc((K + 1) * 4)
  _shim.check(ctx.lib.ign_label_argmax_dev(ctx.handle, _shim.ptr(d_lab), _shim.IGN_U16, n, _shim.ptr(d_field), K,
                                           _shim.ptr(d_idx), _shim.ptr(d_val)))
  idx, val = ctx.to_host(d_idx, (K + 1,), np.uint64), ctx.to_host(d_val, (K + 1,), np.float32)
  for l in range(K + 1):
    mine = np.flatnonzero((lab == l) & np.isfinite(field)) if l else np.zeros(0, int)
    if mine.size == 0:
      assert idx[l] == 2**64 - 1 and val[l] == -np.inf
    else:
      assert idx[l] == mine[np.argmax(field[mine])] and val[l] == field[mine].max()
  assert ctx.lib.ign_label_argmax_dev(ctx.handle, _shim.ptr(d_lab), _shim.IGN_U16, n, _shim.ptr(d_field), 2**32,
                                      _shim.ptr(d_idx), _shim.ptr(d_val)) == -3
  for b in (d_lab, d_field, d_idx, d_val):
    b.free()


def _renumbered(seg):
  flat = seg.ravel(order="F")
  ids, first = np.unique(flat, return_index=True)
  order = [i for i in np.argsort(first) if ids[i] != 0]
  table = {int(ids[i]): k + 1 for k, i in enumerate(order)}
  lut = np.zeros(len(ids), np.uint32)
  for i in order:
    lut[i] = table[int(ids[i])]
  return np.asfortranarray(lut[np.searchsorted(ids, flat)].reshape(seg.shape, order="F")), table


@pytest.mark.parametrize("anisotropy", [(1.0, 1.0, 1.0), (4.0, 4.0, 40.0)], ids=["iso", "4-4-40"])
def test_teasar_fields(ctx, oracle, anisotropy):
  from igneous_b200 import edt, teasar
  seg = oracle.synth_seg((128, 128, 64), pitch=32, num_ids=1 << 20, dtype=np.uint64)
  got = teasar.fields(seg, anisotropy, ctx=ctx)
  lab, table = _renumbered(seg)
  assert np.array_equal(got["labels"], lab) and {k: v for k, v in got["mapping"].items() if k} == table
  K = len(table)
  flat = lab.ravel(order="F")
  dbf = edt.edt(lab, anisotropy, black_border=True, ctx=ctx)
  assert np.array_equal(bits(got["dbf"]), bits(dbf))
  from_first = G.geodesic(lab, first_voxels(lab), 26, anisotropy).ravel(order="F")
  roots = np.zeros(K, np.uint64)
  for l in range(1, K + 1):
    mine = np.flatnonzero((flat == l) & np.isfinite(from_first))
    roots[l - 1] = mine[np.argmax(from_first[mine])]  # the first of equal maxima: the lowest index
  assert np.array_equal(np.ravel_multi_index(tuple(got["roots"].T), lab.shape, order="F"), roots.astype(np.int64))
  daf = G.geodesic(lab, roots, 26, anisotropy)
  assert np.array_equal(bits(got["daf"]), bits(daf))
  pdrf = geodesicref.pdrf(lab, dbf, daf)
  assert np.array_equal(bits(got["pdrf"]), bits(pdrf))
  _, parents = G.geodesic(lab, roots, 26, weights=pdrf, parents=True)
  assert np.array_equal(got["parents"], parents)
  assert check_parents(got["parents"], G.geodesic(lab, roots, 26, weights=pdrf), lab, roots, 26, weights=pdrf)
  # a distance-to-boundary field of the caller's is used as given
  again = teasar.fields(seg, anisotropy, dbf=dbf * np.float32(0.5), ctx=ctx)
  assert np.array_equal(bits(again["daf"]), bits(daf))
  assert np.array_equal(bits(again["pdrf"]), bits(geodesicref.pdrf(lab, dbf * np.float32(0.5), daf)))


def test_refusals(ctx):
  from igneous_b200 import dijkstra3d, _shim
  lab = np.ones((6, 5, 4), np.uint32, order="F")
  lab[0, 0, 0] = 0
  w = np.ones(lab.shape, np.float32, order="F")
  with pytest.raises(_shim.IgneousB200Error, match="label 0"):
    dijkstra3d.euclidean_distance_field(lab, (0, 0, 0), ctx=ctx)
  with pytest.raises(ValueError):
    dijkstra3d.euclidean_distance_field(lab, (6, 0, 0), ctx=ctx)
  with pytest.raises(_shim.IgneousB200Error, match="outside"):
    dijkstra3d.euclidean_distance_field(lab, source_indices=[lab.size], ctx=ctx)
  with pytest.raises(ValueError):  # three numbers are one voxel of a 3-D array, never three indices; and not both
    dijkstra3d.euclidean_distance_field(lab, (1, 1, 1), source_indices=[1], ctx=ctx)
  with pytest.raises(ValueError):
    dijkstra3d.euclidean_distance_field(lab, ctx=ctx)
  with pytest.raises(ValueError):
    dijkstra3d.euclidean_distance_field(lab, (1, 1), ctx=ctx)
  one = dijkstra3d.euclidean_distance_field(lab, np.array([1, 1, 1], np.uint64), connectivity=6, ctx=ctx)
  assert one[1, 1, 1] == 0 and np.count_nonzero(one == 0) == 1
  with pytest.raises(NotImplementedError):
    dijkstra3d.euclidean_distance_field(lab, (1, 1, 1), free_space_radius=3, ctx=ctx)
  with pytest.raises(NotImplementedError):
    dijkstra3d.euclidean_distance_field(lab.astype(np.float32), (1, 1, 1), ctx=ctx)
  with pytest.raises(ValueError):
    dijkstra3d.euclidean_distance_field(lab, (1, 1, 1), connectivity=7, ctx=ctx)
  with pytest.raises(ValueError):
    dijkstra3d.euclidean_distance_field(lab, (1, 1, 1), anisotropy=(1, 0, 1), ctx=ctx)
  with pytest.raises(ValueError):
    dijkstra3d.euclidean_distance_field(lab, {2: (1, 1, 1)}, ctx=ctx)
  for bad in (-1.0, np.nan, np.inf):
    w[3, 2, 1] = bad
    with pytest.raises(_shim.IgneousB200Error, match="weight"):
      dijkstra3d.distance_field(w, (1, 1, 1), labels=lab, ctx=ctx)
    with pytest.raises(_shim.IgneousB200Error, match="weight"):
      dijkstra3d.parental_field(w, (1, 1, 1), ctx=ctx)
  w[3, 2, 1] = 1
  src = np.array([1], np.uint64)
  out = np.empty(lab.shape, np.float32, order="F")
  a = (c.c_float * 3)(1, 1, 1)
  for code in (0, 5, 9):  # 5 is float32: not a label dtype
    assert ctx.lib.ign_geodesic(ctx.handle, _shim.ptr(lab), code, 6, 5, 4, 26, a, None, _shim.ptr(src), 1,
                                _shim.ptr(out), None) == -3
  assert ctx.lib.ign_geodesic(ctx.handle, _shim.ptr(lab), _shim.IGN_U32, 6, 5, 4, 8, a, None, _shim.ptr(src), 1,
                              _shim.ptr(out), None) == -2
  # the context is as usable as before
  got = dijkstra3d.distance_field(w, (1, 1, 1), 6, labels=lab, ctx=ctx)
  assert got[1, 1, 1] == 0 and got[5, 4, 3] == 4 + 3 + 2 and np.isinf(got[0, 0, 0])
  assert dijkstra3d.euclidean_distance_field(np.zeros((0, 4), np.uint8), [], connectivity=8, ctx=ctx).shape == (0, 4)


# ------------------------------------------------ sources on brick faces, edges and corners
# bricks are 32 x 8 x 8 voxels: a source never falls, so nothing but the source pass can wake the brick
# across a face it lies on, and in a one-voxel-wide object it is the only voxel joining the two bricks
@pytest.mark.parametrize("source", [31, 32, 0, 63, 33])
def test_source_on_a_brick_face_of_a_row(ctx, source):
  from igneous_b200 import dijkstra3d
  row = np.ones(64, np.uint8)
  got = dijkstra3d.euclidean_distance_field(row, source, ctx=ctx)
  assert np.array_equal(got, np.abs(np.arange(64) - source).astype(np.float32))
  par = dijkstra3d.parental_field(np.ones(64, np.float32), source, ctx=ctx)
  want = np.arange(64) + 1 + np.sign(source - np.arange(64))
  want[source] = 0
  assert np.array_equal(par, want)


@pytest.mark.parametrize("axis", [0, 1, 2])
@pytest.mark.parametrize("connectivity", [6, 18, 26])
def test_source_on_each_face_of_a_thin_line(ctx, axis, connectivity):
  from igneous_b200 import dijkstra3d
  shape = [5, 5, 5]
  shape[axis] = 70
  brick = (32, 8, 8)[axis]
  lab = np.zeros(shape, np.uint16, order="F")
  line = [2, 2, 2]
  line[axis] = slice(None)
  lab[tuple(line)] = 7
  for at in (brick - 1, brick, 2 * brick - 1, 2 * brick):
    v = [2, 2, 2]
    v[axis] = at
    s = [int(np.ravel_multi_index(v, shape, order="F"))]
    want, wpar = G.geodesic(lab, s, connectivity, (4, 4, 40), parents=True)
    assert np.isfinite(want[lab != 0]).all()
    got = dijkstra3d.euclidean_distance_field(lab, tuple(v), (4, 4, 40), connectivity, ctx=ctx)
    assert np.array_equal(bits(got), bits(want))
    w = np.ones(shape, np.float32, order="F")
    assert np.array_equal(dijkstra3d.parental_field(w, tuple(v), connectivity, labels=lab, ctx=ctx),
                          G.geodesic(lab, s, connectivity, weights=w, parents=True)[1])


def _staircase(shape, connectivity):
  """a one-voxel-wide path from the origin towards the far corner: the full diagonal at connectivity 26,
  (x, y) then z steps at 18, single-axis steps at 6; it crosses brick faces, edges and corners"""
  lab = np.zeros(shape, np.uint8, order="F")
  v, path, k = [0, 0, 0], [(0, 0, 0)], 0
  while True:
    if connectivity == 26:
      step = [1, 1, 1]
    elif connectivity == 18:
      step = [[1, 1, 0], [0, 1, 1], [1, 0, 1]][k % 3]
    else:
      step = [[1, 0, 0], [0, 1, 0], [0, 0, 1]][k % 3]
    k += 1
    v = [a + b for a, b in zip(v, step)]
    if any(a >= n for a, n in zip(v, shape)):
      break
    path.append(tuple(v))
  for p in path:
    lab[p] = 1
  return lab, path


@pytest.mark.parametrize("connectivity", [6, 18, 26])
def test_sources_along_a_diagonal_through_brick_corners(ctx, connectivity):
  from igneous_b200 import dijkstra3d
  shape = (40, 40, 40)
  lab, path = _staircase(shape, connectivity)
  on_corner = [p for p in path if p[0] % 32 in (0, 31) or p[1] % 8 in (0, 7) or p[2] % 8 in (0, 7)]
  assert len(on_corner) >= 8
  rng = np.random.default_rng(connectivity)
  w = np.asfortranarray((rng.random(shape) + 0.25).astype(np.float32))
  for v in on_corner:
    s = [int(np.ravel_multi_index(v, shape, order="F"))]
    want = G.geodesic(lab, s, connectivity, (1.1, 0.7, 3.3))
    assert np.isfinite(want[lab != 0]).all()  # the path is connected under this connectivity
    assert np.array_equal(bits(dijkstra3d.euclidean_distance_field(lab, v, (1.1, 0.7, 3.3), connectivity, ctx=ctx)),
                          bits(want))
  # every voxel of the path its own source, and a handful of them, in one call each
  for some in (path, path[3::7]):
    s = np.ravel_multi_index(tuple(np.array(some).T), shape, order="F")
    wd, wp = G.geodesic(lab, s, connectivity, weights=w, parents=True)
    assert np.array_equal(bits(dijkstra3d.distance_field(w, some, connectivity, labels=lab, ctx=ctx)), bits(wd))
    assert np.array_equal(dijkstra3d.parental_field(w, some, connectivity, labels=lab, ctx=ctx), wp)


def test_several_sources_of_one_label_in_different_bricks(ctx):
  from igneous_b200 import dijkstra3d
  lab = blobs((97, 41, 23), seed=17, labels=2, block=6)
  rng = np.random.default_rng(5)
  nz = np.flatnonzero(lab.ravel(order="F"))
  src = np.unique(rng.choice(nz, 40))
  # and voxels on brick faces wherever the labels have them
  x, y, z = np.unravel_index(nz, lab.shape, order="F")
  faces = nz[(x % 32 == 31) & (y % 8 == 0) | (z % 8 == 7) & (x % 32 == 0)]
  src = np.unique(np.concatenate([src, faces[::97]]))
  for connectivity in (6, 26):
    want, wpar = G.geodesic(lab, src, connectivity, (4, 4, 40), parents=True)
    got = dijkstra3d.euclidean_distance_field(lab, None, (4, 4, 40), connectivity, source_indices=src, ctx=ctx)
    assert np.array_equal(bits(got), bits(want))


def test_teasar_fields_of_thin_objects(ctx):
  """one-voxel-wide objects whose tips (TEASAR's roots) lie on brick faces and corners"""
  from igneous_b200 import edt, teasar
  shape = (72, 24, 24)
  lab = np.zeros(shape, np.uint32, order="F")
  lab[:64, 1, 5] = 5           # tips at x = 0 and x = 63: both on x faces
  lab[5, 8:16, 9] = 6          # tips at y = 8 and y = 15
  lab[40, 20, 7:17] = 8        # tips at z = 7 and z = 16
  diag, _ = _staircase((24, 24, 24), 26)
  lab[44:68, :, :][diag != 0] = 9  # tips at brick corners
  got = teasar.fields(lab, (4, 4, 40), ctx=ctx)
  ren, table = _renumbered(lab)
  assert np.array_equal(got["labels"], ren) and len(table) == 4
  flat = ren.ravel(order="F")
  from_first = G.geodesic(ren, first_voxels(ren), 26, (4, 4, 40)).ravel(order="F")
  assert np.isfinite(from_first[flat != 0]).all()
  roots = np.zeros(4, np.uint64)
  for l in range(1, 5):
    mine = np.flatnonzero(flat == l)
    roots[l - 1] = mine[np.argmax(from_first[mine])]
  assert np.array_equal(np.ravel_multi_index(tuple(got["roots"].T), shape, order="F"), roots.astype(np.int64))
  daf = G.geodesic(ren, roots, 26, (4, 4, 40))
  assert np.isfinite(daf[ren != 0]).all() and np.array_equal(bits(got["daf"]), bits(daf))
  dbf = edt.edt(ren, (4, 4, 40), black_border=True, ctx=ctx)
  pdrf = geodesicref.pdrf(ren, dbf, daf)
  assert np.array_equal(bits(got["pdrf"]), bits(pdrf))
  assert np.array_equal(got["parents"], G.geodesic(ren, roots, 26, weights=pdrf, parents=True)[1])
  assert np.array_equal(got["parents"] != 0, (ren != 0) & (daf != 0))


# ------------------------------------------------------------ past 2^32 voxels
BIG = (4099, 1031, 1017)  # 4.298e9 voxels, element 2^32 in the last plane but one; sides not brick multiples


def test_distances_past_2_32_voxels(ctx):
  """one label filling the box, 6-connected with unit steps from the origin: d = x + y + z"""
  import torch
  from igneous_b200 import _shim
  sx, sy, sz = BIG
  n = sx * sy * sz
  assert n > 2**32
  if torch.cuda.mem_get_info()[0] < n * 5 + (4 << 30):
    pytest.skip("needs %.0f GB of free device memory" % ((n * 5 + (4 << 30)) / 1e9))
  big = _shim.Context()  # a context of its own, so that its scratch arena goes with it
  bufs = []
  try:
    lab, out, src = big.alloc(n), big.alloc(n * 4), big.alloc(8)
    bufs += [lab, out, src]
    big.memset(lab, 1, n)
    big.h2d(src, np.zeros(1, np.uint64))
    a = (c.c_float * 3)(1, 1, 1)
    _shim.check(big.lib.ign_geodesic_dev(big.handle, _shim.ptr(lab), _shim.IGN_U8, sx, sy, sz, 6, a, None,
                                         _shim.ptr(src), 1, _shim.ptr(out), None))
    big.sync()
    par = big.alloc(16)
    bufs.append(par)
    assert big.lib.ign_geodesic_dev(big.handle, _shim.ptr(lab), _shim.IGN_U8, sx, sy, sz, 6, a, None,
                                    _shim.ptr(src), 1, _shim.ptr(out), _shim.ptr(par)) == -6  # parents: < 2^32 - 1
    xs, ys = np.meshgrid(np.arange(sx), np.arange(sy), indexing="ij")
    plane = np.empty((sx, sy), np.float32, order="F")
    zb = 2**32 // (sx * sy)
    for z in sorted({0, 1, zb - 1, zb, min(zb + 1, sz - 1), sz - 1}):
      big.d2h(plane, out.offset(z * sx * sy * 4))
      big.sync()
      assert np.array_equal(plane, (xs + ys + z).astype(np.float32)), "plane z=%d" % z
  finally:
    for b in bufs:
      b.free()
    big.close()
