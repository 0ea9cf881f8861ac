"""igneous_b200.kimimaro.cross_sectional_area against the serial C checker of DESIGN.md §5i (oracle_xsection):
the normals bit for bit, contacts exactly, areas within 2^-20 relative.  Analytic boxes and lines at three
anisotropies, skeletons of capsule-tree neurites and of a pitch-16 synthetic segmentation at windows 1 and 5,
every dtype and both orders, dict / list / single input, in_place both ways, all labels at once against one
call per label, slab sections that take the large path alone and among thousands of small ones, refusals."""
import ctypes

import numpy as np
import pytest

import oracle_xsection as X
import teasarref as T
from igneous_b200 import _shim, kimimaro

pytestmark = pytest.mark.gpu

REL = 2.0 ** -20
ANISO = [(1, 1, 1), (16, 16, 40), (1.1, 0.7, 3.3)]
_UNSIGNED = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}


def _inputs(lab, skels, a):
  """concatenated voxels, edges, point labels and per-label ranges of {label: Skeleton}"""
  av = np.asarray(a, np.float64)
  unsigned = _UNSIGNED[lab.dtype.itemsize]
  vox, edges, pl, ranges, base = [], [], [], {}, 0
  for label, s in skels.items():
    v = np.rint(np.asarray(s.vertices, np.float64).reshape(-1, 3) / av).astype(np.int64)
    vox.append(v)
    edges.append(np.asarray(s.edges, np.int64).reshape(-1, 2) + base)
    pl.append(np.full(len(v), np.asarray(label).astype(lab.dtype).view(unsigned), np.uint64))
    ranges[label] = (base, base + len(v))
    base += len(v)
  return (np.concatenate(vox), np.concatenate(edges).astype(np.uint32), np.concatenate(pl), ranges)


def expected(lab, skels, a, w):
  """{label: (normals, area, contacts)} by the C checker, and the voxels its sections visited"""
  vox, edges, pl, ranges = _inputs(lab, skels, a)
  nrm = X.normals(vox, edges, a, w)
  area, cont, visited = X.sections(lab, vox, pl, nrm, a)
  return {k: (nrm[b:e], area[b:e], cont[b:e]) for k, (b, e) in ranges.items()}, visited


def device_normals(lab, skels, a, w):
  vox, edges, _, ranges = _inputs(lab, skels, a)
  vox = np.ascontiguousarray(vox)
  out = np.empty((len(vox), 3), np.float64)
  _shim.check(_shim.load().ign_cross_section_normals(len(vox), _shim.ptr(vox), len(edges), _shim.ptr(edges),
                                                     (ctypes.c_double * 3)(*a), w, _shim.ptr(out)))
  return {k: out[b:e] for k, (b, e) in ranges.items()}


def check(ctx, lab, skels, a, w, large=None):
  got = kimimaro.cross_sectional_area(lab, skels, anisotropy=a, smoothing_window=w, ctx=ctx)
  stats = list(kimimaro.last_stats)
  want, visited = expected(lab, skels, a, w)
  dn = device_normals(lab, skels, a, w)
  assert list(got) == list(skels)
  for label, (nrm, area, cont) in want.items():
    g = got[label]
    assert np.array_equal(dn[label], nrm), label
    assert g.cross_sectional_area.dtype == np.float32 and g.cross_sectional_area_contacts.dtype == np.uint8
    assert np.array_equal(g.cross_sectional_area_contacts, cont), label
    np.testing.assert_allclose(g.cross_sectional_area, area, rtol=REL, atol=0, err_msg=str(label))
  assert stats[0] == visited
  if large is not None:
    assert (stats[1] > 0) == large, stats
  return got, stats


def line(points, label, a):
  v = np.asarray(points, np.float32) * np.asarray(a, np.float32)
  e = np.array([(i, i + 1) for i in range(len(points) - 1)], np.uint32).reshape(-1, 2)
  return kimimaro.Skeleton(v, e, np.ones(len(v), np.float32), np.zeros(len(v), np.uint8), label)


@pytest.mark.parametrize("a", ANISO)
def test_analytic_boxes_and_lines(ctx, a):
  lab = np.zeros((24, 21, 19), np.uint32)
  lab[2:22, 3:18, 2:16] = 5  # a solid box away from the faces
  lab[0:10, 19, 17] = 6  # a one-voxel line
  lab[15:24, 18:21, 16:19] = 7  # a box touching x = sx - 1, y = sy - 1, z = sz - 1
  skels = {
    5: line([(x, 10, 9) for x in range(4, 20)] + [(19, 10 + k, 9 + k) for k in range(1, 5)], 5, a),
    6: line([(x, 19, 17) for x in range(10)], 6, a),
    7: line([(16, 19, z) for z in range(16, 19)], 7, a),
    8: line([(6, 10, 9), (7, 10, 9), (0, 0, 0), (3, 19, 17)], 8, a),  # voxels of labels 5, 0 and 6
  }
  got, _ = check(ctx, lab, skels, a, 1)
  assert not got[8].cross_sectional_area.any() and not got[8].cross_sectional_area_contacts.any()
  av = np.asarray(a, np.float64)
  np.testing.assert_allclose(got[5].cross_sectional_area[2:14], 15 * av[1] * 14 * av[2], rtol=REL)
  np.testing.assert_allclose(got[6].cross_sectional_area, av[1] * av[2], rtol=REL)
  assert list(got[7].cross_sectional_area_contacts) == [0b1010, 0b1010, 0b101010]
  check(ctx, lab, skels, a, 5)


@pytest.mark.parametrize("w", [1, 5])
def test_capsule_tree_skeletons(ctx, w):
  a = (16, 16, 40)
  lab = T.capsule_trees((120, 110, 60), 10, seed=3, anisotropy=a)
  skels = kimimaro.skeletonize(lab, {"scale": 1.5, "const": 50}, anisotropy=a, dust_threshold=0, ctx=ctx)
  assert sum(len(s.vertices) for s in skels.values()) > 500
  check(ctx, lab, skels, a, w)


@pytest.mark.parametrize("w", [1, 5])
def test_synthetic_segmentation_skeletons(ctx, oracle, w):
  a = (16, 16, 40)
  lab = np.asfortranarray(oracle.synth_seg((96, 80, 40), pitch=16, num_ids=40).astype(np.uint32))
  skels = kimimaro.skeletonize(lab, {"scale": 4, "const": 500}, anisotropy=a, dust_threshold=0, ctx=ctx)
  assert len(skels) > 10
  check(ctx, lab, skels, a, w)


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.uint32, np.uint64, np.int8, np.int16, np.int32,
                                   np.int64, np.bool_])
@pytest.mark.parametrize("order", ["C", "F"])
def test_dtypes_and_orders(ctx, dtype, order):
  a = (1.1, 0.7, 3.3)
  base = np.zeros((18, 15, 12), np.int64)
  base[2:16, 2:9, 2:10] = 1
  base[2:16, 10:14, 3:9] = 2
  labels = {1: -3, 2: 100} if np.dtype(dtype).kind == "i" else {1: 1, 2: 100}
  if dtype == np.bool_:
    lab = np.asarray(base == 1, order=order)
    skels = {True: line([(x, 5, 6) for x in range(3, 15)], True, a)}
  else:
    lab = np.zeros(base.shape, dtype, order=order)
    for b, v in labels.items():
      lab[base == b] = v
    skels = {labels[1]: line([(x, 5, 6) for x in range(3, 15)], labels[1], a),
             labels[2]: line([(5, 11 + k, 4 + k) for k in range(3)] + [(6 + x, 13, 6) for x in range(6)], labels[2], a)}
  check(ctx, lab, skels, a, 3)


def test_dict_list_single_and_in_place(ctx):
  a = (16, 16, 40)
  lab = np.zeros((30, 20, 12), np.uint16)
  lab[1:29, 4:12, 2:9] = 4
  lab[1:29, 14:18, 2:6] = 9
  skels = {4: line([(x, 8, 5) for x in range(2, 28)], 4, a), 9: line([(x, 16, 3) for x in range(2, 28)], 9, a)}
  before = {k: (s.vertices.copy(), s.edges.copy()) for k, s in skels.items()}
  got = kimimaro.cross_sectional_area(lab, skels, anisotropy=a, ctx=ctx)
  for k, s in skels.items():
    assert s.cross_sectional_area is None and s.cross_sectional_area_contacts is None  # input untouched
    assert got[k] is not s and np.array_equal(s.vertices, before[k][0]) and np.array_equal(s.edges, before[k][1])
    assert got[k].vertices is not s.vertices and np.array_equal(got[k].vertices, s.vertices)
  as_list = kimimaro.cross_sectional_area(lab, list(skels.values()), anisotropy=a, ctx=ctx)
  assert isinstance(as_list, list) and [s.id for s in as_list] == [4, 9]
  one = kimimaro.cross_sectional_area(lab, skels[9], anisotropy=a, ctx=ctx)
  assert isinstance(one, kimimaro.Skeleton) and one.id == 9
  for s in (as_list[1], one):
    assert np.array_equal(s.cross_sectional_area, got[9].cross_sectional_area)
    assert np.array_equal(s.cross_sectional_area_contacts, got[9].cross_sectional_area_contacts)
  res = kimimaro.cross_sectional_area(lab, skels, anisotropy=a, in_place=True, ctx=ctx)
  for k, s in skels.items():
    assert res[k] is s and np.array_equal(s.cross_sectional_area, got[k].cross_sectional_area)
  assert kimimaro.Skeleton(np.zeros((0, 3), np.float32), np.zeros((0, 2), np.uint32), None, None, 1) \
      .cross_sectional_area is None


def test_all_labels_at_once_match_one_call_per_label(ctx):
  a = (16, 16, 40)
  lab = T.capsule_trees((90, 80, 50), 8, seed=11, anisotropy=a)
  skels = kimimaro.skeletonize(lab, {"scale": 1.5, "const": 50}, anisotropy=a, dust_threshold=0, ctx=ctx)
  together = kimimaro.cross_sectional_area(lab, skels, anisotropy=a, smoothing_window=5, ctx=ctx)
  for label, s in skels.items():
    alone = kimimaro.cross_sectional_area(lab, s, anisotropy=a, smoothing_window=5, ctx=ctx)
    assert np.array_equal(alone.cross_sectional_area, together[label].cross_sectional_area)
    assert np.array_equal(alone.cross_sectional_area_contacts, together[label].cross_sectional_area_contacts)


@pytest.mark.parametrize("a", [(1, 1, 1), (16, 16, 40)])
def test_slab_sections_take_the_large_path(ctx, a):
  lab = np.ones((400, 400, 6), np.uint32, order="F")
  skels = {1: line([(200, 200, z) for z in range(6)] + [(201 + k, 200, 5) for k in range(3)], 1, a)}
  _, stats = check(ctx, lab, skels, a, 1, large=True)
  assert stats[1] >= 6
  # an oblique plane across the whole slab
  skels = {1: line([(100 + k, 100 + k, min(k, 5)) for k in range(40)], 1, a)}
  check(ctx, lab, skels, a, 3, large=True)


@pytest.mark.parametrize("shape", [(400, 200, 4), (600, 600, 4)])
def test_large_path_ctas_take_several_points(ctx, shape):
  """More large points than CTAs: each CTA clears its bitmap and takes the next point.  At 400 x 200 x 4 the
  large path runs one CTA per SM; at 600 x 600 x 4 the slots' 512 MB budget allows fewer."""
  import torch
  sms = torch.cuda.get_device_properties(ctx.device).multi_processor_count
  a = (16, 16, 40)
  lab = np.ones(shape, np.uint32, order="F")
  lab[:, :, 3] = 2
  # along x with a step in y every 50 voxels: sections of the whole y-z face, some of them oblique
  pts = [(x, shape[1] // 2 + (x // 50) % 3, 1) for x in range(1, shape[0] - 1)]
  _, stats = check(ctx, lab, {1: line(pts, 1, a)}, a, 1, large=True)
  assert stats[1] > stats[3] and stats[1] > sms, stats
  if shape[1] == 200:
    assert stats[3] == sms
  else:
    assert stats[3] == (512 << 20) // (shape[0] * shape[1] * 13) < sms


def test_one_huge_section_among_thousands_of_small(ctx):
  a = (16, 16, 40)
  lab = np.zeros((300, 300, 40), np.uint32, order="F")
  lab[:, :, 0:4] = 1  # a slab: its vertical skeleton's sections are the whole 300 x 300 layer
  skels = {1: line([(150, 150, z) for z in range(4)], 1, a)}
  for t in range(12):  # tubes along x: every section is 3 x 3
    y, z = 10 + 24 * t, 10 + 2 * (t % 10)
    lab[:, y:y + 3, z:z + 3] = 2 + t
    skels[2 + t] = line([(x, y + 1, z + 1) for x in range(1, 299)], 2 + t, a)
  got, stats = check(ctx, lab, skels, a, 1, large=True)
  assert stats[1] == 4
  assert sum(len(s.vertices) for s in skels.values()) > 3000
  np.testing.assert_allclose(got[1].cross_sectional_area, 300 * 16 * 300 * 16, rtol=REL)
  assert np.all(got[5].cross_sectional_area == np.float32(3 * 16 * 3 * 40))


def test_refusals(ctx):
  lab = np.zeros((10, 10, 10), np.uint8)
  lab[2:8, 2:8, 2:8] = 1
  s = line([(x, 5, 5) for x in range(2, 8)], 1, (1, 1, 1))
  with pytest.raises(NotImplementedError):
    kimimaro.cross_sectional_area(lab, s, fill_holes=True, ctx=ctx)
  with pytest.raises(NotImplementedError):
    kimimaro.cross_sectional_area(lab, s, repair_contacts=True, ctx=ctx)
  for bad in [(1, 1), (0, 1, 1), (1, -1, 1), (1, 1, np.nan), (1, np.inf, 1)]:
    with pytest.raises(ValueError, match="anisotropy"):
      kimimaro.cross_sectional_area(lab, s, anisotropy=bad, ctx=ctx)
  for bad in [0, -1, 1.5, True]:
    with pytest.raises(ValueError, match="smoothing_window"):
      kimimaro.cross_sectional_area(lab, s, smoothing_window=bad, ctx=ctx)
  out = line([(x, 5, 5) for x in range(2, 8)] + [(10, 5, 5)], 1, (1, 1, 1))
  with pytest.raises(ValueError, match=r"vertex 6 .* label 1 lies outside"):
    kimimaro.cross_sectional_area(lab, {1: out}, ctx=ctx)
  for bad_label in (300, -1):
    with pytest.raises(ValueError, match="dtype uint8"):
      kimimaro.cross_sectional_area(lab, {bad_label: s}, ctx=ctx)
  with pytest.raises(ValueError, match="dtype bool"):
    kimimaro.cross_sectional_area(lab.astype(bool), {2: s}, ctx=ctx)
  assert s.cross_sectional_area is None


def test_copies_keep_the_callers_dtypes(ctx):
  lab = np.zeros((10, 10, 10), np.uint8)
  lab[2:8, 2:8, 2:8] = 1
  s = kimimaro.Skeleton(np.array([(x, 5, 5) for x in range(2, 8)], np.float64),
                        np.array([(i, i + 1) for i in range(5)], np.int64), np.ones(6, np.float64),
                        np.zeros(6, np.int32), 1)
  t = line([(x, 4, 4) for x in range(2, 8)], 1, (1, 1, 1))
  got = kimimaro.cross_sectional_area(lab, [s, t], ctx=ctx)
  for old, new in zip([s, t], got):
    for f in ("vertices", "edges", "radii", "vertex_types"):
      assert getattr(new, f).dtype == getattr(old, f).dtype and np.array_equal(getattr(new, f), getattr(old, f))
  assert np.all(got[0].cross_sectional_area == 36) and np.all(got[1].cross_sectional_area == 36)
