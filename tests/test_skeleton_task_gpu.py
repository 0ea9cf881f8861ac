"""SkeletonTask and create_skeletonizing_tasks on the GPU, and ign_skeleton_export_dev on its own.  The
reference is igneous_b200.kimimaro.skeletonize on the same cutout (checked bit for bit against the serial
checkers by test_skeletonize_gpu.py), the vertex shift restated in numpy float64 (the vertices
fl32((double)v + corrected_offset), corrected_offset as skeleton.py:229-230 computes it), and a numpy
decoder of the precomputed format written here."""
import ctypes
import gzip
import json
import pickle

import numpy as np
import pytest

from igneous_b200 import _shim, kimimaro
from igneous_b200 import task_creation as tc
from igneous_b200 import tasks
from igneous_b200._compat import Bbox, CloudFiles, CloudVolume, LocalTaskQueue

pytestmark = pytest.mark.gpu

PARAMS = {"scale": 10, "const": 10}


def decode(blob, vertex_types=False):
  buf = np.frombuffer(blob, np.uint8)
  nv, ne = (int(v) for v in buf[:8].view(np.uint32))
  at = [8, 8 + 12 * nv, 8 + 12 * nv + 8 * ne, 8 + 16 * nv + 8 * ne]
  assert buf.size == at[3] + (nv if vertex_types else 0)
  v = buf[at[0]:at[1]].view(np.float32).reshape(nv, 3)
  e = buf[at[1]:at[2]].view(np.uint32).reshape(ne, 2)
  r = buf[at[2]:at[3]].view(np.float32)
  t = buf[at[3]:] if vertex_types else None
  return v, e, r, t


def layer(tmp_path, img, resolution=(4, 4, 40), offset=(0, 0, 0), chunk=(32, 32, 16), name="seg"):
  path = "file://" + str(tmp_path / name)
  CloudVolume.from_numpy(np.asfortranarray(img), path, resolution=resolution, voxel_offset=offset, chunk_size=chunk,
                         layer_type="segmentation")
  return path


def corrected_offset(vol, bbox, mip):
  """skeleton.py:229-230 restated in float64"""
  lo = np.asarray(bbox.minpt, np.float64)
  return ((lo - np.asarray(vol.meta.voxel_offset(mip), np.float64) + 0.5) *
          np.asarray(vol.meta.resolution(mip), np.float64) +
          np.asarray(vol.meta.voxel_offset(0), np.float64) * np.asarray(vol.meta.resolution(0), np.float64))


def expected(ctx, task):
  """{segid: (vertices, edges, radii)} of kimimaro.skeletonize on the task's cutout, moved by the offset"""
  vol = CloudVolume(task.cloudpath, mip=task.mip)
  bbox = Bbox.clamp(task.bounds, vol.bounds)
  cut = np.asfortranarray(vol.download(bbox)[..., 0])
  for ids, fn in ((task.mask_ids, lambda a, l: np.where(np.isin(a, l), 0, a)),
                  (task.object_ids, lambda a, l: np.where(np.isin(a, l), a, 0))):
    if ids:
      cut = np.asfortranarray(fn(cut, np.asarray(ids, cut.dtype)).astype(cut.dtype))
  got = kimimaro.skeletonize(cut, teasar_params=task.teasar_params, object_ids=task.object_ids,
                             anisotropy=vol.resolution, dust_threshold=task.dust_threshold,
                             fix_branching=task.fix_branching, fix_borders=task.fix_borders, ctx=ctx)
  off = corrected_offset(vol, bbox, task.mip)
  return {l: ((s.vertices.astype(np.float64) + off).astype(np.float32), s.edges, s.radii)
          for l, s in got.items()}, bbox, vol


def assert_same(v, e, r, want):
  for x, y in zip((v, e, r), want):
    assert x.dtype == y.dtype and x.shape == y.shape and np.array_equal(x, y)


def blobs(shape, seed, labels=4, block=3, dtype=np.uint64):
  rng = np.random.default_rng(seed)
  coarse = rng.integers(0, labels + 1, size=[(n + block - 1) // block for n in shape])
  return np.asfortranarray(np.kron(coarse, np.ones((block,) * 3, int))[:shape[0], :shape[1], :shape[2]].astype(dtype))


def spatial(path, name):
  return json.loads(gzip.decompress(open(path[len("file://"):] + "/" + name + ".gz", "rb").read()))


# ------------------------------------------------------------------------ the reference's known answer
@pytest.mark.parametrize("object_ids", [None, [2]])
def test_reference_known_answer(ctx, tmp_path, object_ids):
  img = np.full((128, 128, 128), 2, np.uint64)
  path = layer(tmp_path, img, chunk=(64, 64, 64))
  LocalTaskQueue().insert_all(tc.create_skeletonizing_tasks(path, mip=0, teasar_params=PARAMS, object_ids=object_ids))
  skel = CloudVolume(path).skeleton.get(2)
  assert len(skel.vertices) > 0 and len(skel.edges) == len(skel.vertices) - 1
  with pytest.raises(NotImplementedError):
    tc.create_skeletonizing_tasks(path, mip=0, cross_sectional_area=True, cross_sectional_area_smoothing_window=1)


# ------------------------------------------------------------------------ one task, blobs in the layer
def test_single_task_blobs_and_spatial_index(ctx, tmp_path):
  img = blobs((61, 47, 19), 3, labels=6)
  path = layer(tmp_path, img, offset=(3, 5, 7))
  itr = list(tc.create_skeletonizing_tasks(path, mip=0, shape=(64, 64, 32), teasar_params=PARAMS, dust_threshold=0))
  assert len(itr) == 1 and itr[0].will_postprocess is False
  itr[0].execute()
  want, bbox, vol = expected(ctx, itr[0])
  assert len(want) >= 5
  cf = CloudFiles(path)
  assert cf.list("skeletons_mip_0/") == sorted(["skeletons_mip_0/info", "skeletons_mip_0/12-256_20-208_280-1040.spatial"] +
                                               ["skeletons_mip_0/%d" % l for l in want])
  for l, w in want.items():
    v, e, r, _ = decode(cf.get("skeletons_mip_0/%d" % l))
    assert_same(v, e, r, w)
    s = vol.skeleton.get(l)
    assert_same(s.vertices, s.edges, s.radii, w)
  index = spatial(path, "skeletons_mip_0/12-256_20-208_280-1040.spatial")
  assert sorted(map(int, index)) == sorted(want)
  for l, (v, _, _) in want.items():
    assert np.array_equal(np.float32(index[str(l)]), np.concatenate([v.min(axis=0), v.max(axis=0)]))


# ------------------------------------------------------------------------ several tasks, mip 1, fragments
def tubes(shape):
  """uint64 tubes along x (radius 3) at three (y, z), two of them labelled above 2^32, and a 4 x 4 bar"""
  img = np.zeros(shape, np.uint64)
  y, z = np.meshgrid(np.arange(shape[1]), np.arange(shape[2]), indexing="ij")
  for cy, cz, label in ((8, 8, 7), (20, 10, (1 << 32) + 5), (12, 22, (1 << 64) - 1)):
    img[:, (y - cy) ** 2 + (z - cz) ** 2 <= 9] = label
  img[5:60, 26:30, 26:30] = 11  # ends inside the volume
  return img


def test_several_tasks_mip1_fragments(ctx, tmp_path):
  mip1 = tubes((64, 32, 32))
  mip0 = np.repeat(np.repeat(mip1, 2, axis=0), 2, axis=1)
  path = layer(tmp_path, mip0, resolution=(4, 4, 40), offset=(5, 7, 3))
  vol = CloudVolume(path)
  vol.add_resolution((8, 8, 40))
  vol.commit_info()
  vol1 = CloudVolume(path, mip=1)
  assert list(map(int, vol1.voxel_offset)) == [2, 3, 3]
  vol1[vol1.bounds] = mip1
  itr = list(tc.create_skeletonizing_tasks(path, mip=1, shape=(32, 32, 32), teasar_params=PARAMS, dust_threshold=0))
  assert len(itr) == 2 and all(t.will_postprocess for t in itr)
  frags = {}
  for t in itr:
    t.execute()
    want, bbox, vol = expected(ctx, t)
    name = (bbox * vol.resolution).to_filename()
    cf = CloudFiles(path)
    for l, w in want.items():
      s = pickle.loads(cf.get("skeletons_mip_1/%d:%s" % (l, name)))
      assert s.id == l
      assert_same(s.vertices, s.edges, s.radii, w)
      frags.setdefault(l, []).append(s.vertices)
  assert sorted(frags) == sorted([7, (1 << 32) + 5, (1 << 64) - 1, 11])
  # the shared plane x = 34 (mip 1) lies at physical x = (34 - 2 + 0.5) * 8 + 5 * 4
  plane = np.float32((34 - 2 + 0.5) * 8 + 5 * 4)
  for l in (7, (1 << 32) + 5, (1 << 64) - 1, 11):
    a, b = frags[l]
    on_a = {tuple(p) for p in a[a[:, 0] == plane].tolist()}
    on_b = {tuple(p) for p in b[b[:, 0] == plane].tolist()}
    assert on_a and on_a & on_b, l


# ------------------------------------------------------------------------ options
def test_options(ctx, tmp_path):
  img = blobs((40, 36, 14), 11, labels=7)
  path = layer(tmp_path, img)
  base = dict(mip=0, shape=(64, 64, 32), teasar_params=PARAMS, dust_threshold=0)
  cf = CloudFiles(path)
  # dry_run: the skeletons, nothing written but the creator's info
  t = list(tc.create_skeletonizing_tasks(path, **base))[0]
  t.dry_run = True
  got = t.execute()
  want, _, _ = expected(ctx, t)
  assert list(got) == sorted(want) and cf.list("skeletons_mip_0/") == ["skeletons_mip_0/info"]
  for l, s in got.items():
    assert_same(s.vertices, s.edges, s.radii, want[l])
  # mask_ids, object_ids, dust_threshold, fix_branching
  for kw in (dict(mask_ids=[1, 2]), dict(object_ids=[3, 5]), dict(dust_threshold=200), dict(fix_branching=False),
             dict(mask_ids=[4], object_ids=[4, 6])):
    t = list(tc.create_skeletonizing_tasks(path, **{**base, **kw}))[0]
    t.dry_run = True
    got = t.execute()
    want, _, _ = expected(ctx, t)
    assert list(got) == sorted(want), kw
    for l, s in got.items():
      assert_same(s.vertices, s.edges, s.radii, want[l])
  assert set(got) <= {6}
  # strip_integer_attributes=False: the blob carries vertex_types (zeros)
  t = list(tc.create_skeletonizing_tasks(path, **base))[0]
  t.strip_integer_attributes = False
  t.execute()
  want, _, _ = expected(ctx, t)
  for l, w in want.items():
    v, e, r, vt = decode(cf.get("skeletons_mip_0/%d" % l), vertex_types=True)
    assert_same(v, e, r, w)
    assert vt.size == v.shape[0] and not vt.any()
  # frag_path, plain directory: fragments and the index go there; a volume: under its skeleton directory
  plain = str(tmp_path / "frags")
  t = list(tc.create_skeletonizing_tasks(path, **{**base, "shape": (20, 64, 32)}, frag_path=plain))[0]
  t.execute()
  want, bbox, vol = expected(ctx, t)
  name = (bbox * vol.resolution).to_filename()
  assert sorted(CloudFiles(plain).list()) == sorted(["info", "0-80_0-144_0-560.spatial"] +
                                                    ["%d:%s" % (l, name) for l in want])
  other = layer(tmp_path, np.zeros((8, 8, 8), np.uint64), name="other")
  t = list(tc.create_skeletonizing_tasks(path, **{**base, "shape": (20, 64, 32)}, frag_path=other))[0]
  t.execute()
  assert sorted(CloudFiles(other).list("skeletons_mip_0/")) == sorted(
    ["skeletons_mip_0/info", "skeletons_mip_0/0-80_0-144_0-560.spatial"] +
    ["skeletons_mip_0/%d:%s" % (l, name) for l in want])


def test_all_zero_task(ctx, tmp_path):
  path = layer(tmp_path, np.zeros((40, 36, 14), np.uint64))
  t = list(tc.create_skeletonizing_tasks(path, mip=0, shape=(64, 64, 32), teasar_params=PARAMS))[0]
  t.execute()
  assert CloudFiles(path).list("skeletons_mip_0/") == ["skeletons_mip_0/0-160_0-144_0-560.spatial",
                                                       "skeletons_mip_0/info"]
  assert spatial(path, "skeletons_mip_0/0-160_0-144_0-560.spatial") == {}
  assert tasks.skeleton.last_phase_seconds["writes"] >= 0


# ------------------------------------------------------------------------ export edge cases
def test_every_label_a_single_voxel(ctx, tmp_path):
  img = np.zeros((64, 64, 16), np.uint64)
  n = img[::2, ::2, ::2].size
  img[::2, ::2, ::2] = (np.arange(n, dtype=np.uint64) * 7919 + (1 << 40)).reshape(32, 32, 8)
  path = layer(tmp_path, img)
  t = list(tc.create_skeletonizing_tasks(path, mip=0, shape=(64, 64, 16), teasar_params=PARAMS, dust_threshold=0))[0]
  t.execute()
  want, _, _ = expected(ctx, t)
  assert len(want) == n == 8192
  index = spatial(path, "skeletons_mip_0/0-256_0-256_0-640.spatial")
  assert len(index) == n
  cf = CloudFiles(path)
  for l in list(want)[::97]:
    v, e, r, _ = decode(cf.get("skeletons_mip_0/%d" % l))
    assert v.shape == (1, 3) and e.shape == (0, 2)
    assert_same(v, e, r, want[l])
    assert np.float32(index[str(l)]).tolist() == v[0].tolist() * 2


def test_labels_at_the_top_of_uint64(ctx, tmp_path):
  img = tubes((30, 32, 32))
  path = layer(tmp_path, img)
  t = list(tc.create_skeletonizing_tasks(path, mip=0, shape=(64, 64, 64), teasar_params=PARAMS, dust_threshold=0))[0]
  t.execute()
  want, _, _ = expected(ctx, t)
  assert sorted(want) == [7, 11, (1 << 32) + 5, (1 << 64) - 1]
  cf = CloudFiles(path)
  for l in want:
    assert_same(*decode(cf.get("skeletons_mip_0/%d" % l))[:3], want[l])
  assert ((1 << 64) - 1) in {int(k) for k in spatial(path, "skeletons_mip_0/0-120_0-128_0-1280.spatial")}


def test_skeletonize_keys_signed_order(ctx):
  lab = np.zeros((24, 12, 9), np.int16)
  lab[1:8, 2:9, 1:7] = -3
  lab[9:15, 2:9, 1:7] = 5
  lab[16:23, 2:9, 1:7] = -30000
  got = kimimaro.skeletonize(lab, anisotropy=(1, 1, 1), dust_threshold=0, fix_borders=False, ctx=ctx)
  assert list(got) == [-30000, -3, 5]
  s = got[5]
  assert s.vertices.flags.c_contiguous and s.edges.flags.c_contiguous and s.vertices.flags.writeable
  s.vertices[:] += 1  # views may be changed in place, as SkeletonTask's reference does
  assert got[5].vertices.min() >= 1


def export_raw(ctx, lab, skel, nxt, rad, K, capacity=None, vt=1, anisotropy=(1, 1, 1), offset=(0, 0, 0)):
  """ign_skeleton_export_dev on host-built input -> (n_skeletons, the capacity's bytes (0xFF where nothing was
  written), nbytes, table rows, boxes, the capacity bound)"""
  lab = np.asfortranarray(lab, np.uint32)
  skel, nxt, rad = (np.ascontiguousarray(a, dt) for a, dt in ((skel, np.uint32), (nxt, np.uint32),
                                                               (rad, np.float32)))
  bound = ctypes.c_uint64(0)
  _shim.check(ctx.lib.ign_skeleton_export_capacity(skel.size, K, ctypes.byref(bound)))
  cap = bound.value if capacity is None else capacity
  bufs = [ctx.alloc(max(a.nbytes, 8)) for a in (lab, skel, nxt, rad)]
  for b, a in zip(bufs, (lab, skel, nxt, rad)):
    if a.size:
      ctx.h2d(b, a)
  rows = max(min(K, skel.size), 1)
  out = [ctx.alloc(max(cap, 8)), ctx.alloc(rows * 32), ctx.alloc(rows * 24)]
  ctx.memset(out[0], 0xFF, max(cap, 8))
  ns, nb = ctypes.c_uint64(7), ctypes.c_uint64(7)
  try:
    _shim.check(ctx.lib.ign_skeleton_export_dev(
      ctx.handle, _shim.ptr(bufs[0]), *lab.shape, K, _shim.ptr(bufs[1]), _shim.ptr(bufs[2]), _shim.ptr(bufs[3]),
      skel.size, (ctypes.c_float * 3)(*anisotropy), (ctypes.c_double * 3)(*offset), vt, _shim.ptr(out[0]), cap,
      _shim.ptr(out[1]), _shim.ptr(out[2]), ctypes.byref(ns), ctypes.byref(nb)))
    S = int(ns.value)
    blob = np.empty(cap, np.uint8)
    table, boxes = np.empty((S, 4), np.uint64), np.empty((S, 6), np.float32)
    if cap:
      ctx.d2h(blob, out[0])
    if S:
      ctx.d2h(table, out[1])
      ctx.d2h(boxes, out[2])
    ctx.sync()
    return S, blob, int(nb.value), table, boxes, int(bound.value)
  finally:
    for b in bufs + out:
      b.free()


def two_labels():
  lab = np.zeros((6, 5, 4), np.uint32)
  lab[:3] = 1
  lab[3:] = 2
  return lab


def test_export_known_answer(ctx):
  """Two labels of three voxels each, every output checked against values worked out by hand: the vertex
  rule in numpy, the edges and radii per label, the table, the boxes and the zeroed padding."""
  lab = two_labels()
  # label 1: voxels 1 (1,0,0), 7 (1,1,0), 32 (2,0,1), rooted at 7; label 2: 3 (3,0,0), 4 (4,0,0), 10 (4,1,0),
  # rooted at 3
  skel = [1, 3, 4, 7, 10, 32]
  nxt = [7, 3, 3, 7, 4, 1]
  rad = [10, 11, 12, 13, 14, 15]
  a, off = (2.0, 3.0, 0.7), (0.25, -1.0, 10.5)
  ns, buf, nb, table, boxes, bound = export_raw(ctx, lab, skel, nxt, rad, 2, anisotropy=a, offset=off)

  def vertices(coords):
    prod = np.asarray(coords, np.float32) * np.asarray(a, np.float32)
    return (prod.astype(np.float64) + np.asarray(off, np.float64)).astype(np.float32)

  want = {1: (vertices([(1, 0, 0), (1, 1, 0), (2, 0, 1)]), [[0, 1], [0, 2]], [10, 13, 15]),
          2: (vertices([(3, 0, 0), (4, 0, 0), (4, 1, 0)]), [[0, 1], [1, 2]], [11, 12, 14])}
  size = 8 + 16 * 3 + 8 * 2 + 3  # 75 bytes, padded to 80
  assert ns == 2 and nb == 80 + size and bound == 6 * 25 + 2 * 16
  assert table.tolist() == [[1, 0, 3, 2], [2, 80, 3, 2]]
  # the padding after each blob, the last one's included, is zeros; nothing past it is written
  assert not buf[size:80].any() and not buf[nb:160].any() and (buf[160:] == 0xFF).all()
  for row, (label, o, nv, ne) in enumerate(table.tolist()):
    v, e, r, t = decode(buf[o:o + size], vertex_types=True)
    wv, we, wr = want[label]
    assert np.array_equal(v, wv) and e.tolist() == we and r.tolist() == wr and not t.any()
    assert np.array_equal(boxes[row], np.concatenate([wv.min(axis=0), wv.max(axis=0)]))
  # without vertex_types the blobs are 72 bytes, already on the 8-byte grid
  ns, buf, nb, table, _, _ = export_raw(ctx, lab, skel, nxt, rad, 2, vt=0, anisotropy=a, offset=off)
  assert table.tolist() == [[1, 0, 3, 2], [2, 72, 3, 2]] and nb == 144
  assert np.array_equal(decode(buf[72:144])[0], want[2][0])


def test_export_count_zero_capacity_and_corrupt_next(ctx):
  lab = two_labels()
  ns, _, nb, _, _, bound = export_raw(ctx, lab, [], [], [], 2)
  assert ns == 0 and nb == 0 and bound == 0
  assert kimimaro.skeletonize(np.zeros((4, 4, 4), np.uint8), ctx=ctx) == {}
  # two voxels of label 1 (x = 1, 2 at y = z = 0) and one of label 2 (x = 3): a valid tree per label
  skel, rad = [1, 2, 3], [1, 2, 3]
  ns, _, _, _, _, bound = export_raw(ctx, lab, skel, [2, 2, 3], rad, 2)
  assert ns == 2 and bound == 3 * 25 + 2 * 16
  with pytest.raises(_shim.IgneousB200Error, match="capacity"):
    export_raw(ctx, lab, skel, [2, 2, 3], rad, 2, capacity=bound - 1)
  # next(2) = 3 crosses from label 1 to label 2: refused, naming voxel 2
  with pytest.raises(_shim.IgneousB200Error, match="linear index 2 has its next voxel on another label"):
    export_raw(ctx, lab, skel, [2, 3, 3], rad, 2)
  # a next voxel off the skeleton
  with pytest.raises(_shim.IgneousB200Error, match="linear index 1 has a next voxel that is not a skeleton voxel"):
    export_raw(ctx, lab, skel, [0, 2, 3], rad, 2)
  # a skeleton voxel above max_label (here 1)
  with pytest.raises(_shim.IgneousB200Error, match="linear index 3 lies on label 0 or above max_label"):
    export_raw(ctx, lab, skel, [2, 2, 3], rad, 1)
  # many voxels above max_label: more label runs than the call has rows for, refused before any is formed
  many = np.asfortranarray(np.arange(120, dtype=np.uint32).reshape(6, 5, 4, order="F") + 1)
  with pytest.raises(_shim.IgneousB200Error, match="linear index 2 lies on label 0 or above max_label"):
    export_raw(ctx, many, np.arange(0, 120, 2), np.arange(0, 120, 2), np.ones(60), 1)
  # a skeleton voxel outside the volume (120 voxels) that another voxel's next points to
  with pytest.raises(_shim.IgneousB200Error, match="linear index 500 lies outside the volume"):
    export_raw(ctx, lab, [1, 2, 500], [500, 2, 500], [1, 1, 1], 2)
