"""ign_skeleton_merge_dev against the serial C checker (oracle_skeleton, itself checked against the numpy
restatement by test_skelmergeref.py) bit for bit, kimimaro.postprocess against the batch path, the entry's
refusals, and UnshardedSkeletonMergeTask end to end on a file:// layer after SkeletonTask."""
import ctypes
import pickle
import re

import numpy as np
import pytest

import oracle_skeleton as C
from igneous_b200 import _shim, kimimaro
from igneous_b200 import task_creation as tc
from igneous_b200._compat import Bbox, CloudFiles, CloudVolume, LocalTaskQueue
from test_skelmergeref import _S, random_batch, signed_zero_batch

pytestmark = pytest.mark.gpu


def same_as_checker(ctx, batch, crop=0, dust=0, tick=0, max_cable=None, vertex_types=True):
  _, packed = kimimaro.pack_fragments(batch, crop=crop)
  want, wtable = C.merge(packed, dust, tick, max_cable, vertex_types)
  got, table = kimimaro.merge_packed(packed, dust, tick, max_cable, vertex_types, ctx)
  assert np.array_equal(table, wtable)
  assert bytes(got[:want.size]) == bytes(want) and not got[want.size:].any()
  return table


def big_batch(seed, labels=300, scale=3.5):
  """random trees of up to 400 vertices per fragment, up to 6 fragments per label, with loops and gaps"""
  rng = np.random.default_rng(seed)
  out = {}
  for l in range(labels):
    frags = []
    for _ in range(int(rng.integers(1, 7))):
      n = int(rng.integers(1, 400))
      walk = np.cumsum(rng.integers(-1, 2, size=(n, 3)), axis=0) + rng.integers(0, 20, 3)
      v = walk.astype(np.float32) * np.float32(scale)
      e = [(i, int(rng.integers(max(0, i - 3), i))) for i in range(1, n)]
      e += [tuple(int(x) for x in rng.integers(0, n, 2)) for _ in range(int(rng.integers(0, 3)))]
      r = rng.uniform(0.5, 6.0, n).astype(np.float32)
      lo = rng.integers(-5, 40, 3) * 3
      box = Bbox(lo, lo + 60) if rng.random() < 0.5 else None
      frags.append((box, _S(v, np.array(e, np.uint32).reshape(-1, 2), r, rng.integers(0, 4, n).astype(np.uint8))))
    out[(1 << 33) + l if l % 3 == 0 else l + 1] = frags
  return out


@pytest.mark.parametrize("crop,dust,tick,max_cable", [
  (0, 0, 0, None),      # fuse and consolidate, loops and connect pieces
  (0, 40, 0, None),     # + dust
  (0, 0, 15, None),     # + ticks
  (2, 0, 0, None),      # + crop
  (0, 30, 12, 150.5),   # long labels written as fused
  (1, 30, 12, None),    # everything
])
@pytest.mark.parametrize("seed", [0, 1])
def test_device_matches_checker_small(ctx, seed, crop, dust, tick, max_cable):
  same_as_checker(ctx, random_batch(seed, labels=40), crop, dust, tick, max_cable)


@pytest.mark.parametrize("crop,dust,tick", [(0, 0, 0), (0, 200, 40), (3, 200, 40)])
def test_device_matches_checker_many_labels(ctx, crop, dust, tick):
  table = same_as_checker(ctx, big_batch(7), crop, dust, tick)
  assert (table[:, 2] > 50).any() and (table[:, 3] == table[:, 2] - 1).any()


@pytest.mark.parametrize("seed", range(3))
def test_signed_zeros_fold_and_keep_the_first_occurrence_bits(ctx, seed):
  """-0.0 and 0.0 are one position, and the written bits are those of its first occurrence"""
  batch = signed_zero_batch(seed, labels=40)
  same_as_checker(ctx, batch, dust=0, tick=0)
  got = kimimaro.merge_fragments(batch, dust_threshold=0, tick_threshold=0, ctx=ctx)
  out = np.concatenate([s.vertices for s, _ in got.values()])
  zeros = out[out == 0]
  assert np.signbit(zeros).any() and not np.signbit(zeros).all()
  assert all(len(np.unique(s.vertices + np.float32(0), axis=0)) == len(s.vertices) for s, _ in got.values())


def test_empty_results_one_and_many_fragments_without_vertex_types(ctx):
  tiny = _S(np.zeros((1, 3), np.float32), np.zeros((0, 2), np.uint32), np.ones(1, np.float32), np.zeros(1, np.uint8))
  line = _S(np.array([[0, 0, 0], [1, 0, 0]], np.float32), np.array([[0, 1]], np.uint32), np.ones(2, np.float32),
            np.ones(2, np.uint8))
  batch = {5: [(None, tiny)], (1 << 40) + 3: [(None, line)] * 4, 9: [], 12: [(None, line)]}
  table = same_as_checker(ctx, batch, dust=0.5, vertex_types=False)
  assert table[:, 2].tolist() == [0, 2, 0, 2]
  got = kimimaro.merge_fragments(batch, dust_threshold=1.5, vertex_types=False, ctx=ctx)
  assert list(got) == list(batch) and all(s.empty() for s, _ in got.values())
  assert all(bytes(b) == b"\0" * 8 for _, b in got.values())


def test_postprocess_equals_the_batch_path(ctx):
  batch = random_batch(3, labels=8)
  merged = kimimaro.merge_fragments(batch, dust_threshold=20, tick_threshold=10, ctx=ctx)
  for segid, frags in batch.items():
    fused = kimimaro.merge_fragments({segid: frags}, max_cable_length=-1.0, ctx=ctx)[segid][0]
    got = kimimaro.postprocess(fused, dust_threshold=20, tick_threshold=10, ctx=ctx)
    want = merged[segid][0]
    assert got.id == segid
    for a, b in ((got.vertices, want.vertices), (got.edges, want.edges), (got.radii, want.radii),
                 (got.vertex_types, want.vertex_types)):
      assert a.dtype == b.dtype and np.array_equal(a, b)


def raw_call(ctx, packed, capacity=None):
  lib, h, ptr = ctx.lib, ctx.handle, _shim.ptr
  L = packed["label_frag"].size - 1
  d = {k: ctx.alloc(max(v.nbytes, 8)) for k, v in packed.items()}
  for k, v in packed.items():
    ctx.h2d(d[k], np.ascontiguousarray(v))
  cap = ctypes.c_uint64(0)
  _shim.check(lib.ign_skeleton_merge_capacity(L, packed["radius"].size, packed["edges"].shape[0], ctypes.byref(cap)))
  capacity = cap.value if capacity is None else capacity
  out, table, nb = ctx.alloc(cap.value), ctx.alloc(L * 32), ctypes.c_uint64(7)
  try:
    _shim.check(lib.ign_skeleton_merge_dev(
      h, L, ptr(d["label_frag"]), packed["frag_box"].shape[0], ptr(d["frag_vert"]), ptr(d["frag_edge"]),
      ptr(d["frag_box"]), ptr(d["vertices"]), ptr(d["radius"]), ptr(d["vertex_types"]), packed["radius"].size,
      ptr(d["edges"]), packed["edges"].shape[0], 0.0, 0.0, float("inf"), 1, ptr(out), capacity, ptr(table),
      ctypes.byref(nb)))
  finally:
    for b in list(d.values()) + [out, table]:
      b.free()
  return nb.value


def test_refusals(ctx):
  _, packed = kimimaro.pack_fragments(random_batch(0, labels=3))
  assert raw_call(ctx, packed) > 0
  with pytest.raises(_shim.IgneousB200Error, match="capacity"):
    raw_call(ctx, packed, capacity=100)
  bad = dict(packed, edges=packed["edges"].copy())
  bad["edges"][1, 0] = packed["frag_vert"][1] - packed["frag_vert"][0]
  with pytest.raises(_shim.IgneousB200Error, match="edge 1 has an end outside its fragment"):
    raw_call(ctx, bad)
  bad = dict(packed, vertices=packed["vertices"].copy())
  bad["vertices"][2, 1] = np.inf
  with pytest.raises(_shim.IgneousB200Error, match="vertex 2 is not finite"):
    raw_call(ctx, bad)
  bad = dict(packed, frag_vert=packed["frag_vert"].copy())
  bad["frag_vert"][-1] += 1
  with pytest.raises(_shim.IgneousB200Error, match="ranges"):
    raw_call(ctx, bad)


# ------------------------------------------------------------------------ end to end
LABELS = (3, 42, 777, (1 << 33) + 5)


def neurites(shape):
  """tubes along x that cross every task face in x (labels 3, 42 and one above 2^32), and a capsule tree
  (label 777): a trunk along y with two branches along x, crossing faces in x and y"""
  img = np.zeros(shape, np.uint64)
  x, y, z = np.meshgrid(*[np.arange(n) for n in shape], indexing="ij")
  for cy, cz, label in ((8, 8, 3), (30, 10, 42), (50, 5, (1 << 33) + 5)):
    img[((y - cy) ** 2 + (z - cz) ** 2 <= 9)] = label
  trunk = ((x - 20) ** 2 + (z - 24) ** 2 <= 9) & (y >= 4) & (y < 60)
  b1 = ((y - 20) ** 2 + (z - 24) ** 2 <= 6) & (x >= 20) & (x < 60)
  b2 = ((y - 44) ** 2 + (z - 24) ** 2 <= 6) & (x >= 6) & (x < 20)
  img[trunk | b1 | b2] = 777
  return np.asfortranarray(img)


def fragments_by_label(path):
  vol = CloudVolume(path)
  cf = CloudFiles(vol.skeleton.path)
  out = {}
  for name in cf.list():
    m = re.search(r"(\d+):", name)
    if m:
      out.setdefault(int(m.group(1)), []).append((Bbox.from_filename(name), pickle.loads(cf.get(name))))
  return out


def test_end_to_end(ctx, tmp_path):
  path = "file://" + str(tmp_path / "seg")
  CloudVolume.from_numpy(neurites((64, 64, 32)), path, resolution=(16, 16, 40), chunk_size=(32, 32, 32),
                         layer_type="segmentation")
  tq = LocalTaskQueue()
  tq.insert(tc.create_skeletonizing_tasks(path, mip=0, shape=(32, 32, 32), teasar_params={"scale": 4, "const": 50},
                                          dust_threshold=0))
  vol = CloudVolume(path)
  cf = CloudFiles(vol.skeleton.path)
  spatial = [n for n in cf.list() if n.endswith(".spatial")]
  assert len(spatial) == 4
  frags = fragments_by_label(path)
  assert sorted(frags) == sorted(LABELS) and all(len(frags[l]) >= 2 for l in LABELS)
  kw = dict(crop=1, dust_threshold=100, tick_threshold=150)
  merged = []
  orig = tc.create_unsharded_skeleton_merge_tasks(path, magnitude=2, **kw)
  for t in orig:
    merged += list(t.execute())
  assert sorted(merged) == sorted(LABELS)  # each label exactly once across the prefixes
  want = {}
  for l in LABELS:
    ordered = sorted(frags[l], key=lambda f: "%d:%s" % (l, f[0].to_filename()))
    want[l] = ordered
  segids, packed = kimimaro.pack_fragments(want, crop=1, resolution=vol.resolution)
  buf, table = C.merge(packed, 100, 150, None, vertex_types=False)
  vol = CloudVolume(path)
  assert [a["id"] for a in vol.skeleton.meta.info["vertex_attributes"]] == ["radius"]
  for l, (_, off, nv, ne) in zip(segids, table.tolist()):
    s = vol.skeleton.get(l)
    got = buf[off:off + 8 + 16 * nv + 8 * ne]
    assert s.vertices.tobytes() == got[8:8 + 12 * nv].tobytes()
    assert s.edges.tobytes() == got[8 + 12 * nv:8 + 12 * nv + 8 * ne].tobytes()
    assert s.radii.tobytes() == got[8 + 12 * nv + 8 * ne:].tobytes()
    assert nv > 0 and ne <= nv - 1, l  # a forest
    if l != 777:
      assert ne == nv - 1, l  # a tube crossing task faces is one tree
  # without delete_fragments nothing was removed; with it only the fragments go
  assert fragments_by_label(path).keys() == frags.keys()
  LocalTaskQueue().insert(tc.create_unsharded_skeleton_merge_tasks(path, magnitude=1, delete_fragments=True, **kw))
  left = cf.list()
  assert not fragments_by_label(path)
  assert sorted(n for n in left if n.endswith(".spatial")) == sorted(spatial)
  assert {str(l) for l in LABELS} <= set(left) and "info" in left
  assert CloudVolume(path).skeleton.get(777).vertices.tobytes() == vol.skeleton.get(777).vertices.tobytes()


def test_unreadable_fragment_names_the_file(ctx, tmp_path):
  path = "file://" + str(tmp_path / "seg")
  CloudVolume.from_numpy(np.zeros((8, 8, 8), np.uint64), path, resolution=(4, 4, 40), layer_type="segmentation")
  vol = CloudVolume(path)
  vol.info["skeletons"] = "skel"
  vol.commit_info()
  CloudFiles(CloudVolume(path).skeleton.path).put("5:0-32_0-32_0-320", b"not a pickle", compress="gzip")
  with pytest.raises(ValueError, match="5:0-32_0-32_0-320"):
    next(t for t in tc.create_unsharded_skeleton_merge_tasks(path, magnitude=1) if t.prefix == 5).execute()
