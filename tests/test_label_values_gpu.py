"""GPU: label kernels at adversarial label values, against the plain references of
tests/labelref.py (numpy, scipy and the Neuroglancer spec; no code shared with oracle/).

- compressed_segmentation: tables shared by content, never by hash alone (blocks {0,1} and
  {1,64}; CCL / renumber output, whose small consecutive ids give many similar tables; and
  IGN_CSEG_HASH_BITS=k, which keeps k bits of the hash so that collisions are the rule);
- 2^64-1 is an ordinary uint64 label for mask / remap / renumber / unique and the Mesher;
- uint64 labels that differ only in the high word, and the maximum of every dtype, through
  CCL, dust, mode pooling, the fastremap kernels, the codec and the Mesher;
- the fused CCL task body (cc3d.ccl_task) at threshold, rail and label-offset edges."""
import ctypes as c

import numpy as np
import pytest

from labelref import (U64_MAX, blob_volume, ccl6, ccl_task, check_block_mode, countless2x2, cseg_decode_spec,
                      dust, label_sets, order_preserving_relabel)

pytestmark = pytest.mark.gpu

M = np.uint64(U64_MAX)


# ------------------------------------------------------------------ compressed_segmentation
def _cseg_check(oracle, v, bs=(8, 8, 8)):
  from igneous_b200 import codecs
  v = np.asfortranarray(v)
  got = np.frombuffer(codecs.cseg_encode(v, bs), dtype=np.uint32)
  want = oracle.cseg_encode(v, bs)
  assert len(got) == len(want) and np.array_equal(got, want), (v.shape, v.dtype, bs)
  assert np.array_equal(cseg_decode_spec(got, v.shape, v.dtype, bs)[..., 0], v), (v.shape, bs)
  assert np.array_equal(codecs.cseg_decode(got.tobytes(), v.shape, v.dtype, bs)[..., 0], v), (v.shape, bs)


def _collision_pair(dtype):
  v = np.zeros((16, 8, 8), dtype=dtype, order="F")
  v[0:8, :, :4] = 1        # block 0: {0, 1}
  v[8:16] = 1
  v[8:16, :, 4:] = 64      # block 1: {1, 64}
  return v


def _same_ends(dtype):
  """blocks {1,2,5}, {1,3,5}, {1,2,5}, {1,3,5}, {1,2,4,5}: tables of more than two values with
  equal size and ends, told apart only by their middle values; blocks 2 and 3 share the tables
  of blocks 0 and 1"""
  v = np.full((40, 8, 8), 1, dtype=dtype, order="F")
  for i, mid in enumerate(((2,), (3,), (2,), (3,), (2, 4))):
    v[8 * i:8 * i + 8, :, 4:] = 5
    for j, m in enumerate(mid):
      v[8 * i:8 * i + 8, j, 0] = m
  return v


@pytest.mark.parametrize("dtype", [np.uint32, np.uint64])
def test_cseg_blocks_with_colliding_tables(ctx, oracle, dtype):
  v = _collision_pair(dtype)
  _cseg_check(oracle, v)
  # more pairs of the same kind, side by side in one chunk
  w = np.zeros((48, 8, 8), dtype=dtype, order="F")
  for i, (a, b) in enumerate(((0, 1), (1, 64), (0, 2), (1, 67), (1, 2), (3, 389))):
    w[8 * i:8 * i + 8] = a
    w[8 * i:8 * i + 4, :4] = b
  _cseg_check(oracle, w)
  _cseg_check(oracle, _same_ends(dtype))


def _realistic(ctx, oracle, shape, dtype):
  from igneous_b200 import cc3d, fastremap
  seg = oracle.synth_seg(shape, pitch=16, num_ids=1 << 20)
  cc = cc3d.connected_components(seg, connectivity=6, out_dtype=np.uint64)
  ren, _ = fastremap.renumber(seg)
  return [np.asfortranarray(cc.astype(dtype)), np.asfortranarray(ren.astype(dtype))]


REALISTIC = [((64, 64, 64), bs) for bs in ((8, 8, 8), (4, 4, 4), (8, 4, 2))] + \
            [((256, 256, 64), bs) for bs in ((8, 8, 8), (4, 4, 4), (8, 4, 2))]


@pytest.mark.parametrize("dtype", [np.uint32, np.uint64])
@pytest.mark.parametrize("shape,bs", REALISTIC)
def test_cseg_ccl_and_renumber_output(ctx, oracle, shape, bs, dtype):
  for v in _realistic(ctx, oracle, shape, dtype):
    _cseg_check(oracle, v, bs)


@pytest.mark.parametrize("bits", ["0", "1", "8"])
def test_cseg_forced_hash_collisions(ctx, oracle, monkeypatch, bits):
  """IGN_CSEG_HASH_BITS=k keeps k bits of the table hash: almost every table collides, and the
  stream must still be the oracle's (tables shared only between identical label sets)."""
  from test_cseg_gpu import _vols
  monkeypatch.setenv("IGN_CSEG_HASH_BITS", bits)
  for dtype in (np.uint32, np.uint64):
    for v in _vols(oracle, dtype) + [_collision_pair(dtype), _same_ends(dtype)]:
      _cseg_check(oracle, v)
    for shape, bs in REALISTIC:
      for v in _realistic(ctx, oracle, shape, dtype):
        _cseg_check(oracle, v, bs)
  monkeypatch.delenv("IGN_CSEG_HASH_BITS")


def test_downsample_task_cseg_small_consecutive_ids(ctx, oracle, tmp_path):
  """DownsampleTask writing compressed_segmentation mips of a renumbered (1..K) volume: the
  mips read back equal the oracle's pooling."""
  import igneous_b200.task_creation as tc
  from igneous_b200 import fastremap
  from igneous_b200._compat import CloudVolume, LocalTaskQueue
  seg, _ = fastremap.renumber(oracle.synth_seg((256, 256, 64), pitch=16, num_ids=1 << 20))
  seg = np.asfortranarray(seg.astype(np.uint32))[..., np.newaxis]
  path = "file://" + str(tmp_path / "layer")
  CloudVolume.from_numpy(seg, vol_path=path, resolution=(1, 1, 1), voxel_offset=(0, 0, 0), chunk_size=(64, 64, 64),
                         layer_type="segmentation", max_mip=0)
  LocalTaskQueue(parallel=1).insert_all(tc.create_downsampling_tasks(
    path, mip=0, num_mips=2, encoding="compressed_segmentation", compress="gzip"))
  cv = CloudVolume(path)
  want = oracle.downsample_segmentation(seg, (2, 2, 1, 1), num_mips=2)
  for m in (1, 2):
    cv.mip = m
    assert np.array_equal(cv[cv.meta.bounds(m)], want[m - 1]), m


# ------------------------------------------------------------------ 2^64-1 as a label
def _with_max(rng, shape=(30, 20, 10)):
  v = rng.integers(0, 6, size=shape).astype(np.uint64)
  v[v == 5] = M
  v[v == 4] = np.uint64(1 << 40)
  return np.asfortranarray(v)


def test_mask_and_mask_except_with_u64_max(ctx):
  from igneous_b200 import fastremap
  rng = np.random.default_rng(20)
  v = _with_max(rng)
  for labels in ([1, 2], [U64_MAX], [U64_MAX, 2], [1 << 40, U64_MAX, 0]):
    inl = np.isin(v, np.array(labels, dtype=np.uint64))
    assert np.array_equal(fastremap.mask(v, labels), np.where(inl, 0, v)), labels
    assert np.array_equal(fastremap.mask_except(v, labels), np.where(inl, v, 0)), labels
    assert np.array_equal(fastremap.mask(v, labels, value=7), np.where(inl, 7, v).astype(np.uint64)), labels
  # 2^64-1 in the list only
  w = np.asfortranarray(rng.integers(0, 4, size=(9, 8, 7)).astype(np.uint64))
  assert np.array_equal(fastremap.mask(w, [U64_MAX]), w)
  assert np.array_equal(fastremap.mask_except(w, [U64_MAX]), np.zeros_like(w))


def test_remap_with_u64_max(ctx):
  from igneous_b200 import fastremap
  rng = np.random.default_rng(21)
  v = _with_max(rng)
  full = {0: 0, 1: 10, 2: 20, 3: 30, 1 << 40: U64_MAX, U64_MAX: 5}
  want = np.vectorize(lambda x: full[int(x)], otypes=[np.uint64])(v)
  assert np.array_equal(fastremap.remap(v, full), want)
  absent = {k: x for k, x in full.items() if k != U64_MAX}
  with pytest.raises(KeyError) as e:
    fastremap.remap(v, absent)
  assert str(U64_MAX) in str(e.value)
  kept = np.vectorize(lambda x: absent.get(int(x), int(x)), otypes=[np.uint64])(v)
  assert np.array_equal(fastremap.remap(v, absent, preserve_missing_labels=True), kept)
  # a key of 2^64-1 must not take a slot of another key
  many = {int(k): int(k) + 1 for k in range(5000)}
  many[U64_MAX] = 3
  w = np.asfortranarray(np.concatenate([np.arange(5000, dtype=np.uint64), [M]]).reshape(-1, 1, 1))
  assert np.array_equal(fastremap.remap(w, many).ravel(), np.array([many[int(x)] for x in w.ravel()], dtype=np.uint64))


def _first_appearance(v):
  flat = v.ravel(order="K")
  u, idx = np.unique(flat, return_index=True)
  order = u[np.argsort(idx)]
  return [int(x) for x in order if x != 0]


@pytest.mark.parametrize("order", ["F", "C"])
def test_renumber_and_unique_with_u64_max(ctx, order):
  from igneous_b200 import fastremap
  rng = np.random.default_rng(22)
  v = _with_max(rng)
  v = np.asfortranarray(v) if order == "F" else np.ascontiguousarray(v)
  got, mapping = fastremap.renumber(v)
  seq = _first_appearance(v)
  want_map = {x: i + 1 for i, x in enumerate(seq)}
  want_map[0] = 0
  assert mapping == want_map
  assert np.array_equal(got, np.vectorize(lambda x: want_map[int(x)])(v))
  u, cnt = fastremap.unique(v, return_counts=True)
  wu, wc = np.unique(v, return_counts=True)
  assert np.array_equal(u, wu) and np.array_equal(cnt.astype(np.int64), wc)
  only = np.full((5, 4, 3), M)
  assert np.array_equal(fastremap.unique(only), [M])
  assert fastremap.renumber(only)[1] == {U64_MAX: 1}


# ------------------------------------------------------------------ Mesher
def _mesh_all(vol, simplify):
  from igneous_b200 import zmesh
  m = zmesh.Mesher((4, 5, 6))
  m.mesh(vol)
  kw = dict(reduction_factor=10, max_error=40) if simplify else {}
  return m.ids(), {i: m.get(i, voxel_centered=True, **kw) for i in m.ids()}


def _check_mesher_relabel_invariant(vol):
  """metamorphic: meshing is blind to label values, so every label's mesh equals the mesh of
  its image under an order-preserving injective relabelling to 1..K"""
  rel, mapping = order_preserving_relabel(vol)
  for simplify in (False, True):
    ids, meshes = _mesh_all(vol, simplify)
    rids, rmeshes = _mesh_all(rel, simplify)
    want_ids = sorted(k for k in mapping)
    assert sorted(ids) == want_ids and sorted(rids) == sorted(mapping.values())
    for lab in ids:
      a, b = meshes[lab], rmeshes[mapping[lab]]
      assert len(a.faces) > 0
      assert np.array_equal(a.vertices, b.vertices) and np.array_equal(a.faces, b.faces), (hex(lab), simplify)


def test_mesher_with_u64_max(ctx):
  rng = np.random.default_rng(23)
  vol = blob_volume(rng, (33, 30, 20), [U64_MAX, 1 << 40, 7, U64_MAX - 1], np.uint64, p_bg=0.05)
  _check_mesher_relabel_invariant(vol)


# ------------------------------------------------------------------ high words and dtype maxima
def _cases():
  out = []
  for dt in (np.uint8, np.uint16, np.uint32, np.uint64):
    for name in label_sets(dt):
      out.append(pytest.param(dt, name, id="%s-%s" % (np.dtype(dt).name, name)))
  return out


def _vol(dtype, name, shape=(40, 37, 21), seed=30, p_bg=0.25):
  rng = np.random.default_rng(seed)
  return blob_volume(rng, shape, label_sets(dtype)[name], dtype, p_bg=p_bg)


@pytest.mark.parametrize("dtype,name", _cases())
def test_ccl_and_dust_label_values(ctx, monkeypatch, dtype, name):
  from igneous_b200 import _shim, cc3d
  for shape in ((40, 37, 21), (64, 32, 16)):  # unaligned and 16-byte aligned rows
    v = _vol(dtype, name, shape)
    want, wn = ccl6(v)
    assert wn > len(label_sets(dtype)[name])
    for no_tma in (False, True):
      if no_tma:
        monkeypatch.setenv("IGN_CCL_NO_TMA", "1")
      else:
        monkeypatch.delenv("IGN_CCL_NO_TMA", raising=False)
      got, n = cc3d.connected_components(v, connectivity=6, out_dtype=np.uint64, return_N=True)
      assert n == wn and np.array_equal(got, want), (shape, no_tma)
      d_in = ctx.to_device(v)
      d_out = ctx.alloc(v.size * 4)
      try:
        nn = c.c_uint64(0)
        _shim.check(ctx.lib.ign_ccl6_volume_dev(ctx.handle, _shim.ptr(d_in), _shim.dtype_code(dtype), shape[0],
                                                shape[1], shape[2], _shim.ptr(d_out), _shim.IGN_U32, c.byref(nn)))
        assert nn.value == wn and np.array_equal(ctx.to_host(d_out, shape, np.uint32), want.astype(np.uint32))
      finally:
        d_in.free()
        d_out.free()
      for t in (3, 40):
        assert np.array_equal(cc3d.dust(v, t, connectivity=6), dust(v, t)), (shape, no_tma, t)
  monkeypatch.delenv("IGN_CCL_NO_TMA", raising=False)


@pytest.mark.parametrize("dtype,name", _cases())
def test_mode_pooling_label_values(ctx, oracle, dtype, name):
  from igneous_b200 import tinybrain
  for shape, mips in (((64, 48, 4), 3), ((48, 40, 3), 2)):   # fused; generic (rows not a multiple of 16)
    v = _vol(dtype, name, shape, p_bg=0.1)
    got = tinybrain.downsample_segmentation(v, (2, 2, 1), num_mips=mips)
    cur = v
    for m in range(mips):
      cur = countless2x2(cur)
      assert got[m].dtype == v.dtype and np.array_equal(got[m], cur), (shape, m)
    generic = tinybrain._select(v, (2, 2, 1), mips, tinybrain._OP_MODE, None)
    for g, w in zip(generic, got):
      assert np.array_equal(g, w), shape
  v = _vol(dtype, name, (20, 12, 8), p_bg=0.1)
  got = tinybrain.downsample_segmentation(v, (2, 2, 2), num_mips=2)
  assert check_block_mode(v, got[0], (2, 2, 2)) == 10 * 6 * 4
  check_block_mode(got[0], got[1], (2, 2, 2))
  want = oracle.downsample_segmentation(v, (2, 2, 2), num_mips=2)
  for g, w in zip(got, want):
    assert np.array_equal(g, w)


@pytest.mark.parametrize("dtype,name", _cases())
def test_fastremap_label_values(ctx, dtype, name):
  from igneous_b200 import fastremap
  v = _vol(dtype, name)
  vals = label_sets(dtype)[name]
  got, mapping = fastremap.renumber(v)
  seq = _first_appearance(v)
  want_map = {x: i + 1 for i, x in enumerate(seq)}
  want_map[0] = 0
  assert mapping == want_map
  assert np.array_equal(got, np.vectorize(lambda x: want_map[int(x)])(v))
  u, cnt = fastremap.unique(v, return_counts=True)
  wu, wc = np.unique(v, return_counts=True)
  assert u.dtype == v.dtype and np.array_equal(u, wu) and np.array_equal(cnt.astype(np.int64), wc)
  table = {int(x): int(vals[(i + 1) % len(vals)]) for i, x in enumerate(wu)}
  want = np.vectorize(lambda x: table[int(x)], otypes=[np.uint64])(v).astype(dtype)
  assert np.array_equal(fastremap.remap(v, table), want)
  some = vals[::2]
  inl = np.isin(v, np.array(some, dtype=np.uint64).astype(dtype))
  assert np.array_equal(fastremap.mask(v, some), np.where(inl, 0, v))
  assert np.array_equal(fastremap.mask_except(v, some), np.where(inl, v, 0))


@pytest.mark.parametrize("dtype,name", [p for p in _cases() if p.values[0] in (np.uint32, np.uint64)])
def test_cseg_label_values(ctx, oracle, dtype, name):
  v = _vol(dtype, name, p_bg=0.1)
  for bs in ((8, 8, 8), (4, 4, 4), (8, 4, 2)):
    _cseg_check(oracle, v, bs)


@pytest.mark.parametrize("dtype,name", _cases())
def test_mesher_label_values(ctx, dtype, name):
  v = _vol(dtype, name, (33, 30, 20), p_bg=0.05)
  _check_mesher_relabel_invariant(v)


# ------------------------------------------------------------------ fused CCL task body
def _task_check(ctx, img, shape, gte=None, lte=None, dust_threshold=0, label_offset=0):
  from igneous_b200 import cc3d
  want, wn = ccl_task(img, shape, gte, lte, dust_threshold, label_offset)
  got, n = cc3d.ccl_task(img, shape, threshold_gte=gte, threshold_lte=lte, dust_threshold=dust_threshold,
                         label_offset=label_offset)
  assert n == wn and got.dtype == np.uint64 and np.array_equal(got, want), (img.dtype, shape, gte, lte, label_offset)
  return wn


def _rail_shapes(s):
  sx, sy, sz = s
  return [(sx, sy, sz),                   # every rail outside the volume
          (sx - 1, sy - 1, sz - 1),       # rails on the last planes (a task reads shape + 1)
          (sx - 7, sy // 2, sz - 3),      # rails inside
          (sx - 1, sy + 4, sz - 1)]       # one coordinate outside: only the x-z rail applies


@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.uint32, np.uint64])
@pytest.mark.parametrize("no_tma", [False, True])
def test_ccl_task_thresholds_rails_offsets(ctx, monkeypatch, dtype, no_tma):
  from igneous_b200 import cc3d
  if no_tma:
    monkeypatch.setenv("IGN_CCL_NO_TMA", "1")
  else:
    monkeypatch.delenv("IGN_CCL_NO_TMA", raising=False)
  rng = np.random.default_rng(40)
  for s in ((64, 32, 16), (37, 29, 17)):    # 16-byte aligned rows and unaligned ones
    img = np.asfortranarray(rng.integers(0, 8, size=s).astype(dtype))
    seen = 0
    for shape in _rail_shapes(s):
      for gte, lte in ((3, None), (None, 3), (3, 5), (5, 5), (4.5, None), (None, 2.5), (6, 2)):
        for off in (0, (1 << 63) - 5):
          seen += _task_check(ctx, img, shape, gte, lte, label_offset=off)
      _task_check(ctx, img, shape, 2, 6, dust_threshold=5, label_offset=1 << 40)
    assert seen > 0
    # gte > lte is empty
    got, n = cc3d.ccl_task(img, s, threshold_gte=6, threshold_lte=2)
    assert n == 0 and not got.any()
    # raw labels (no threshold), with rails, dust and an offset
    lab = blob_volume(rng, s, label_sets(dtype)["max"], dtype, p_bg=0.2)
    for shape in _rail_shapes(s):
      _task_check(ctx, lab, shape, dust_threshold=4, label_offset=(1 << 63) + 1)
  monkeypatch.delenv("IGN_CCL_NO_TMA", raising=False)


def test_ccl_task_uint64_thresholds_above_2_53(ctx):
  """(double)raw is inexact above 2^53: 2^60 - 1 would round up to 2^60 and pass gte=2^60.
  Integer images are compared with exact integer bounds."""
  from igneous_b200 import cc3d
  rng = np.random.default_rng(41)
  base = 1 << 60
  steps = np.array([-2, -1, 0, 1, 2, 255, 256, 257], dtype=np.int64)
  img = np.asfortranarray((np.uint64(base) + rng.choice(steps, size=(40, 24, 12)).astype(np.uint64)))
  s = img.shape
  for gte, lte in ((base, None), (None, base), (base, base + 256), (base + 256, None), (base - 128, base + 256),
                   (base, base)):
    assert _task_check(ctx, img, s, gte, lte) > 0, (gte, lte)
  with pytest.raises(NotImplementedError):
    cc3d.ccl_task(img, s, threshold_gte=base + 1)
  with pytest.raises(NotImplementedError):
    cc3d.ccl_task(img, s, threshold_lte=np.uint64(base - 1))


@pytest.mark.parametrize("no_tma", [False, True])
def test_ccl_task_float32_thresholds(ctx, monkeypatch, no_tma):
  """float32 images compare in float32, as numpy compares a float32 array with a Python float:
  thresholds 0.1 and 1/3 are not float32 values, and the image holds float32(t) and both of
  its neighbours."""
  if no_tma:
    monkeypatch.setenv("IGN_CCL_NO_TMA", "1")
  else:
    monkeypatch.delenv("IGN_CCL_NO_TMA", raising=False)
  rng = np.random.default_rng(42)
  vals = [0.0, 1.0, 0.5]
  for t in (0.1, 1 / 3, 0.7):
    f = np.float32(t)
    vals += [np.nextafter(f, np.float32(0)), f, np.nextafter(f, np.float32(1))]
  vals = np.array(vals, dtype=np.float32)
  for s in ((64, 32, 16), (37, 29, 17)):
    img = np.asfortranarray(vals[rng.integers(0, len(vals), size=s)])
    for gte, lte in ((0.1, None), (None, 0.1), (1 / 3, None), (None, 1 / 3), (0.1, 1 / 3), (0.7, None),
                     (None, 0.7), (float(np.float32(0.1)), float(np.float32(1 / 3)))):
      for shape in _rail_shapes(s)[:3]:
        assert _task_check(ctx, img, shape, gte, lte, label_offset=7) > 0, (gte, lte)
  monkeypatch.delenv("IGN_CCL_NO_TMA", raising=False)
