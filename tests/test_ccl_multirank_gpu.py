"""The multi-rank CCL merge on one device.  ign_ccl6_sharded_dev is ign_ccl6_volume_begin_dev, one
all-gather of the ranks' plane records and ign_ccl6_volume_finish_gathered_dev.  Here N ranks are
emulated on one GPU: slab r of a whole volume on the device is a pointer offset into it, its plane
record is record r of one buffer (the layout of the all-gather's result), and the slabs are finished
r = N-1 .. 0 into the matching slabs of one output.  The stitched output must equal a whole-volume
CCL bit for bit (same numbering), on every rank with the same global count.  The task-file path
(begin, ign_ccl6_link_dev per boundary, host ign_ccl6_solve, finish with a table) is checked the
same way."""
import ctypes as c

import numpy as np
import pytest

from labelref import U64_MAX, blob_volume, ccl6

pytestmark = pytest.mark.gpu

IGN_ERR_INVALID, IGN_ERR_OVERFLOW = -2, -6
DTYPES = [np.uint8, np.uint16, np.uint32, np.uint64]


class Ranks:
  """N ranks of a z-split volume, emulated on one device."""

  def __init__(self, ctx, vol, heights):
    from igneous_b200 import _shim, multigpu
    self.ctx, self.lib, self.vol = ctx, ctx.lib, np.asfortranarray(vol)
    self.sx, self.sy, sz = vol.shape
    assert sum(heights) == sz and min(heights) >= 1
    self.heights = [int(h) for h in heights]
    self.z0 = [int(z) for z in np.cumsum([0] + self.heights[:-1])]
    self.N = len(heights)
    self.np = self.sx * self.sy
    self.rec = multigpu.plane_record_bytes(self.np)
    self.code = _shim.dtype_code(vol.dtype)
    self.d_in = ctx.to_device(self.vol)
    self.d_rec = ctx.alloc(self.rec * self.N)
    self.vols = []  # ign_ccl_volume handles in begin order; None once consumed
    self.n_local = []

  def record(self, r):
    return self.d_rec.ptr + r * self.rec

  def planes(self, r):
    """(first values, first labels, last values, last labels) addresses of record r"""
    fv = self.record(r) + 256
    lv = fv + 8 * self.np
    fl = lv + 8 * self.np
    return fv, fl, lv, fl + 4 * self.np

  def begin(self):
    from igneous_b200 import _shim
    for r, h in enumerate(self.heights):
      v, n = c.c_void_p(), c.c_uint64(0)
      src = self.d_in.ptr + self.np * self.z0[r] * self.vol.itemsize
      _shim.check(self.lib.ign_ccl6_volume_begin_dev(self.ctx.handle, src, self.code, self.sx, self.sy, h,
                                                     *self.planes(r), c.byref(v), c.byref(n)))
      self.vols.append(v)
      self.n_local.append(int(n.value))
      self.ctx.h2d(self.record(r), np.array([n.value], dtype=np.uint64))
    self.ctx.sync()
    return self

  def out_slab(self, d_out, r, out_dtype):
    return d_out.ptr + self.np * self.z0[r] * np.dtype(out_dtype).itemsize

  def finish_gathered(self, r, d_out, out_dtype, nranks=None, rank=None, records=True):
    """ign_ccl6_volume_finish_gathered_dev on the volume of slab r -> (status, n_global)"""
    from igneous_b200 import _shim
    n = c.c_uint64(0)
    innermost = self.vols[r] is [v for v in self.vols if v is not None][-1]
    st = self.lib.ign_ccl6_volume_finish_gathered_dev(self.vols[r], self.d_rec.ptr if records else None,
                                                      self.N if nranks is None else nranks, r if rank is None else rank,
                                                      self.out_slab(d_out, r, out_dtype), _shim.dtype_code(out_dtype),
                                                      c.byref(n))
    if innermost:  # consumed, also on failure; a volume ended out of order is left open
      self.vols[r] = None
    return st, int(n.value)

  def run(self, out_dtype):
    """begin every slab, finish r = N-1 .. 0 -> (stitched labels, statuses, n_global per rank)"""
    self.begin()
    d_out = self.ctx.alloc(self.vol.size * np.dtype(out_dtype).itemsize)
    res = [self.finish_gathered(r, d_out, out_dtype) for r in reversed(range(self.N))][::-1]
    got = self.ctx.to_host(d_out, self.vol.shape, out_dtype)
    return got, [s for s, _ in res], [n for _, n in res]

  def close(self):
    for r in reversed(range(len(self.vols))):
      if self.vols[r] is not None:
        assert self.lib.ign_ccl6_volume_abort(self.vols[r]) == 0
        self.vols[r] = None


def merged(ctx, vol, heights, out_dtype=np.uint32):
  rk = Ranks(ctx, vol, heights)
  try:
    got, st, ns = rk.run(out_dtype)
  finally:
    rk.close()
  return got, st, ns


def check_merge(ctx, oracle, vol, heights, out_dtype=np.uint32, independent=False):
  want, n_want = oracle.connected_components(vol, return_N=True)
  got, st, ns = merged(ctx, vol, heights, out_dtype)
  assert st == [0] * len(heights), st
  assert ns == [n_want] * len(heights), (ns, n_want)
  assert got.dtype == np.dtype(out_dtype)
  assert np.array_equal(got, want.astype(out_dtype))
  if independent:
    ref, n_ref = ccl6(vol)
    assert n_ref == n_want and np.array_equal(got, ref.astype(out_dtype))
  return got, n_want


def random_heights(rng, n):
  h = rng.integers(1, 8, size=n)
  h[rng.integers(n)] = 1
  return [int(v) for v in h]


def values_for(dtype, k=3):
  if np.dtype(dtype) == np.uint64:
    return [(j << 32) | 7 for j in range(1, k + 1)]  # equal low words
  return list(range(1, k + 1))


def draw_path(vol, pts, value):
  """6-connected polyline through pts: x, then y, then z, one voxel at a time"""
  p = list(pts[0])
  vol[tuple(p)] = value
  for q in pts[1:]:
    for ax in range(3):
      while p[ax] != q[ax]:
        p[ax] += 1 if q[ax] > p[ax] else -1
        vol[tuple(p)] = value


# ------------------------------------------------------------------ random slabs
@pytest.mark.parametrize("nranks", [2, 3, 8])
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("kind", ["blobs", "synth"])
@pytest.mark.parametrize("plane", [(64, 24), (45, 19)])
def test_random_slabs_match_whole_volume(ctx, oracle, nranks, dtype, kind, plane):
  """(64, 24): 16-byte row pitches, TMA mask fill and vector expansion on every slab; (45, 19): slab
  offsets and row pitches that are not 16-byte aligned, cooperative fill and scalar expansion."""
  rng = np.random.default_rng(1000 * nranks + 10 * np.dtype(dtype).itemsize + len(kind) + plane[0])
  heights = random_heights(rng, nranks)
  shape = plane + (sum(heights),)
  if kind == "blobs":
    vol = blob_volume(rng, shape, values_for(dtype), dtype, p_bg=0.25)
  else:
    base = (1 << 40) if np.dtype(dtype) == np.uint64 else 0
    vol = oracle.synth_seg(shape, pitch=8, num_ids=7, seed=nranks, dtype=dtype, id_base=base)
  out_dtype = {2: np.uint16, 3: np.uint32, 8: np.uint64}[nranks]
  check_merge(ctx, oracle, vol, heights, out_dtype, independent=(nranks == 3))


# ------------------------------------------------------- components that span ranks
def test_helix_crosses_every_boundary_several_times(ctx, oracle):
  heights = [3, 5, 1, 4, 2, 6, 3]
  sx, sy, sz = 150, 20, sum(heights)
  rng = np.random.default_rng(3)
  vol = blob_volume(rng, (sx, sy, sz), [1, 2, 3], np.uint32, p_bg=0.5)
  # axis along x: z swings over the whole volume, so every boundary is crossed twice per turn
  t = np.arange(0, sx, 2)
  ys = np.rint(10 + 2 * np.cos(2 * np.pi * t / 37)).astype(int)
  zs = np.rint((sz - 1) / 2 * (1 + np.sin(2 * np.pi * t / 37))).astype(int)
  draw_path(vol, list(zip(t, ys, zs)), 9)
  helix = vol == 9
  cuts = np.cumsum(heights)[:-1]
  for z in cuts:  # path steps from plane z-1 into plane z at least 4 times per boundary
    assert (helix[:, :, z - 1] & helix[:, :, z]).sum() >= 4, z
  got, n = check_merge(ctx, oracle, vol, heights, np.uint32)
  assert len(np.unique(got[helix])) == 1


def test_u_shapes_join_only_through_other_ranks(ctx, oracle):
  """Two pieces of rank r that join only in rank r+1 or r+2, and two pieces of rank r+1 that join
  only in rank r: the unions start from ids of either side.  Every shape is one component, all of
  the same label, kept apart by empty rows."""
  heights = [4, 3, 2, 5, 3]
  z0 = np.cumsum([0] + heights[:-1])
  top = [int(z0[r] + heights[r] - 1) for r in range(len(heights))]
  shapes = []
  for r in range(len(heights) - 1):
    shapes.append([(2, top[r] - 1), (2, z0[r + 1]), (20, z0[r + 1]), (20, top[r] - 1)])       # U into r+1
    shapes.append([(3, z0[r + 1] + 1), (3, top[r]), (17, top[r]), (17, z0[r + 1] + 1)])      # inverted U into r
    if r + 2 < len(heights):
      shapes.append([(5, z0[r]), (5, z0[r + 2]), (25, z0[r + 2]), (25, z0[r])])                # U through r+1 into r+2
  sx, sy, sz = 30, 2 * len(shapes) + 1, sum(heights)
  for dtype in (np.uint16, np.uint64):
    value = 40000 if dtype == np.uint16 else U64_MAX
    vol = np.zeros((sx, sy, sz), dtype=dtype, order="F")
    for k, s in enumerate(shapes):
      draw_path(vol, [(x, 2 * k + 1, int(z)) for x, z in s], value)
    got, n = check_merge(ctx, oracle, vol, heights, np.uint32, independent=True)
    assert n == len(shapes)


def test_one_label_filling_the_volume(ctx, oracle):
  rng = np.random.default_rng(11)
  heights = random_heights(rng, 8)
  for dtype in DTYPES:
    vol = np.full((33, 17, sum(heights)), np.iinfo(dtype).max, dtype=dtype, order="F")
    got, n = check_merge(ctx, oracle, vol, heights, np.uint16)
    assert n == 1 and (got == 1).all()


# ------------------------------------------------------------ empty and thin slabs
@pytest.mark.parametrize("fill", ["full", "blobs"])
def test_empty_slabs_and_a_thin_empty_slab_cut_links(ctx, oracle, fill):
  """Slabs 0 and 7 (the ends), 4 (middle) and 2 (height 1, between two non-empty slabs) are all zero:
  begin writes zero planes for them and no label may link across them."""
  heights = [2, 3, 1, 4, 2, 1, 3, 2]
  z0 = np.cumsum([0] + heights[:-1])
  shape = (40, 12, sum(heights))
  rng = np.random.default_rng(5)
  if fill == "full":
    vol = np.full(shape, 3, dtype=np.uint16, order="F")
  else:
    vol = blob_volume(rng, shape, [1, 2], np.uint16, p_bg=0.1)
  for r in (0, 2, 4, 7):
    vol[:, :, z0[r]:z0[r] + heights[r]] = 0
  got, n = check_merge(ctx, oracle, vol, heights, np.uint32, independent=True)
  if fill == "full":
    assert n == 3  # slab 1, slab 3, slabs 5-6


# ----------------------------------------------------------------- u64 label values
def test_u64_values_equal_in_low_word_do_not_link(ctx, oracle):
  heights = [3, 2, 3]
  vol = np.zeros((32, 8, 8), dtype=np.uint64, order="F")
  vol[:, :, 0:3] = (1 << 32) | 5
  vol[:, :, 3:5] = (2 << 32) | 5           # same low word as its neighbours: three components
  vol[:, :, 5:8] = (3 << 32) | 5
  vol[0:8, 0:4, :] = 1 << 32               # low word 0, one column through every boundary
  vol[10:16, 0:4, 0:3] = 1 << 32           # ... and pieces that face a different high word
  vol[10:16, 0:4, 3:5] = 2 << 32
  got, n = check_merge(ctx, oracle, vol, heights, np.uint64, independent=True)
  assert n == 6


def test_u64_max_label_across_boundaries(ctx, oracle):
  heights = [1, 4, 2, 1, 3]
  rng = np.random.default_rng(8)
  vol = blob_volume(rng, (24, 10, sum(heights)), [U64_MAX, U64_MAX - 1, U64_MAX ^ (1 << 32), 1], np.uint64,
                    p_bg=0.2)
  vol[3:7, 2, :] = U64_MAX  # through every boundary
  got, n = check_merge(ctx, oracle, vol, heights, np.uint32, independent=True)
  assert len(np.unique(got[3:7, 2, :])) == 1


# ------------------------------------------------------------------- u16 output
def test_u16_output_bounded_by_the_global_count(ctx, oracle):
  """8 ranks of height 2 over 128 x 128 distinct z-columns: 131,072 provisional ids (every column
  counted once per rank) but 16,384 components, which fit uint16."""
  from igneous_b200 import cc3d
  col = (np.arange(128 * 128, dtype=np.uint32) + 1).reshape(128, 128, order="F")
  vol = np.asfortranarray(np.repeat(col[:, :, None], 16, axis=2))
  got, n = check_merge(ctx, oracle, vol, [2] * 8, np.uint16)
  assert n == 128 * 128
  whole, n_whole = cc3d.connected_components(vol, connectivity=6, out_dtype=np.uint16, return_N=True)
  assert n_whole == n and np.array_equal(got, whole)


def test_u16_output_overflow_raises_on_every_rank(ctx):
  """65,536 components do not fit uint16: every rank fails with IGN_ERR_OVERFLOW (the empty top slab
  too), as the whole-volume call does."""
  from igneous_b200 import _shim, cc3d
  col = (np.arange(256 * 256, dtype=np.uint32) + 1).reshape(256, 256, order="F")
  vol = np.zeros((256, 256, 5), dtype=np.uint32, order="F")
  vol[:, :, :4] = col[:, :, None]
  with pytest.raises(_shim.IgneousB200Error) as e:
    cc3d.connected_components(vol, connectivity=6, out_dtype=np.uint16)
  assert e.value.status == IGN_ERR_OVERFLOW
  got, st, ns = merged(ctx, vol, [2, 2, 1], np.uint16)
  assert st == [IGN_ERR_OVERFLOW] * 3
  got, st, ns = merged(ctx, vol, [2, 2, 1], np.uint32)
  assert st == [0] * 3 and ns == [65536] * 3


# ---------------------------------------------------------------- task-file path
def host_planes(ctx, rk, r):
  out = []
  for p, dt in zip(rk.planes(r), (np.uint64, np.uint32, np.uint64, np.uint32)):
    a = np.empty(rk.np, dtype=dt)
    ctx.d2h(a, p)
    out.append(a)
  ctx.sync()
  return out  # first values, first labels, last values, last labels


def link_dev(ctx, rk, b, off, capacity):
  """ign_ccl6_link_dev between the last plane of slab b and the first of slab b+1"""
  from igneous_b200 import _shim
  va, la = rk.planes(b)[2:]
  vb, lb = rk.planes(b + 1)[:2]
  pairs = np.full((max(capacity, 1) + 4, 2), 0xABABABABABABABAB, dtype=np.uint64)
  n = c.c_uint64(0)
  _shim.check(ctx.lib.ign_ccl6_link_dev(ctx.handle, va, la, int(off[b]), vb, lb, int(off[b + 1]), rk.np,
                                        _shim.ptr(pairs), capacity, c.byref(n)))
  return pairs, int(n.value)


@pytest.mark.parametrize("dtype", [np.uint8, np.uint64])
def test_task_file_path_matches_whole_volume(ctx, oracle, dtype):
  from igneous_b200 import _shim, multigpu
  rng = np.random.default_rng(17)
  heights = [3, 1, 4, 2, 5]
  vol = blob_volume(rng, (45, 19, sum(heights)), values_for(dtype), dtype, p_bg=0.2)
  want, n_want = oracle.connected_components(vol, return_N=True)
  rk = Ranks(ctx, vol, heights).begin()
  try:
    off = np.concatenate([[0], np.cumsum(rk.n_local)]).astype(np.uint64)
    planes = [host_planes(ctx, rk, r) for r in range(rk.N)]
    for r in range(rk.N):  # begin's planes hold the slab's first and last z-plane values
      z_first, z_last = rk.z0[r], rk.z0[r] + heights[r] - 1
      assert np.array_equal(planes[r][0], vol[:, :, z_first].ravel(order="F").astype(np.uint64))
      assert np.array_equal(planes[r][2], vol[:, :, z_last].ravel(order="F").astype(np.uint64))
      assert np.array_equal(planes[r][1] != 0, planes[r][0] != 0)
    all_pairs = []
    for b in range(rk.N - 1):
      pairs, n = link_dev(ctx, rk, b, off, rk.np)
      want_pairs = multigpu.link_planes_numpy(planes[b][2], planes[b][3], off[b], planes[b + 1][0],
                                              planes[b + 1][1], off[b + 1])
      assert n >= len(want_pairs) > 0
      assert np.array_equal(np.unique(pairs[:n], axis=0), want_pairs)
      assert (pairs[n:] == 0xABABABABABABABAB).all()
      all_pairs.append(pairs[:n])
      # a smaller capacity still reports every pair and copies only `capacity` of them
      cap = n // 2
      part, n2 = link_dev(ctx, rk, b, off, cap)
      assert n2 == n
      assert (part[cap:] == 0xABABABABABABABAB).all()
      hit = (part[:cap, None, :] == want_pairs[None, :, :]).all(axis=2).any(axis=1)
      assert hit.all()
    lut, n_global = multigpu.solve_pairs(np.concatenate(all_pairs), int(off[-1]))
    assert n_global == n_want
    d_out = ctx.alloc(vol.size * 4)
    for r in reversed(range(rk.N)):
      table = np.concatenate([[0], lut[int(off[r]) + 1:int(off[r + 1]) + 1]]).astype(np.uint32)
      st = ctx.lib.ign_ccl6_volume_finish_dev(rk.vols[r], _shim.ptr(table), n_global, rk.out_slab(d_out, r, np.uint32),
                                              _shim.IGN_U32)
      rk.vols[r] = None
      _shim.check(st)
    got = ctx.to_host(d_out, vol.shape, np.uint32)
  finally:
    rk.close()
  assert np.array_equal(got, want.astype(np.uint32))


# ---------------------------------------------------------------- argument checks
def test_finish_gathered_rejects_bad_arguments(ctx, oracle):
  """Each bad argument is refused with IGN_ERR_INVALID before any kernel runs; the volume is consumed
  (except when volumes end out of order) and the next merge is unaffected."""
  vol = np.zeros((16, 8, 6), dtype=np.uint32, order="F")
  vol[0:4, :, 0:3] = 1
  vol[8:12, :, 0:3] = 2   # slab 0: two components, slab 1: one
  vol[:, 0:2, 3:6] = 1
  heights = [3, 3]
  bad = [dict(nranks=0), dict(nranks=-1), dict(rank=-1), dict(rank=2), dict(nranks=1, rank=1),
         dict(records=False)]
  for kw in bad:
    rk = Ranks(ctx, vol, heights).begin()
    d_out = ctx.alloc(vol.size * 4)
    try:
      before = ctx.launch_count()
      st, _ = rk.finish_gathered(1, d_out, np.uint32, **kw)
      assert st == IGN_ERR_INVALID, kw
      assert ctx.launch_count() == before, kw
      assert rk.vols[1] is None
    finally:
      rk.close()
  # record `rank` whose n_local is not the volume's: the caller passed the wrong rank
  rk = Ranks(ctx, vol, heights).begin()
  try:
    assert rk.n_local == [2, 1]
    st, _ = rk.finish_gathered(1, ctx.alloc(vol.size * 4), np.uint32, rank=0)
    assert st == IGN_ERR_INVALID
  finally:
    rk.close()
  # volumes must end in reverse order of begin: slab 0 is not the innermost
  rk = Ranks(ctx, vol, heights).begin()
  try:
    st, _ = rk.finish_gathered(0, ctx.alloc(vol.size * 4), np.uint32)
    assert st == IGN_ERR_INVALID and rk.vols[0] is not None
  finally:
    rk.close()
  check_merge(ctx, oracle, vol, heights)
