"""Volume kernels past 2^32 voxels, where a 32-bit counter, index or scan would wrap silently.

The references are analytic or plain numpy / scipy on a small grid, never the oracle on a whole
volume:
- block volumes v(x, y, z) = G[x // bx, y // by, z // bz] for a small seeded grid G: their
  6-connected components are the components of G (scipy.ndimage.label per value), numbered by
  their first block in Fortran raster order, whose corner is the component's first voxel -- so
  this is cc3d's numbering -- and their bounding boxes are the blocks' boxes scaled and clipped;
- volumes whose run count, component sizes or triangle count follow from their pattern.

Every test runs in a context of its own, so that the scratch arena of one 17 GB call is released
before the next test, and reads its results back one z-slab at a time.  The helpers are checked
against the oracle and scipy at small shapes without a GPU."""
import ctypes as c

import numpy as np
import pytest
import scipy.ndimage

IGN_ERR_OVERFLOW = -6
IGN_U8, IGN_U16, IGN_U32, IGN_U64 = 1, 2, 3, 4
BLOCK = (37, 29, 23)  # runs do not line up with 32-voxel mask words or CCL tiles
BIG_TMA = (4096, 1024, 1025)   # 2^32 + 2^22 voxels, 16-byte row pitch: TMA mask fill, k_ccl_expand4
BIG_ODD = (4099, 1031, 1017)   # row pitch not a multiple of 16 bytes: cooperative fill, k_ccl_expand1
HEADLINE = (2048, 2048, 1024)  # 2^32 voxels
SLAB_BYTES = 512 << 20


# ------------------------------------------------------------- references
def block_grid(shape, block, seed):
  """seeded grid of values 0..3 with one cell per block (the last block may be clipped)"""
  gshape = tuple(-(-s // b) for s, b in zip(shape, block))
  return np.random.default_rng(seed).integers(0, 4, size=gshape).astype(np.uint8)


def block_components(grid):
  """6-connected components of the grid, equal non-zero values connecting, numbered 1..n by their
  first cell in Fortran raster order; returns (component grid u32, n)"""
  comp = np.zeros(grid.shape, np.int64)
  n = 0
  for v in range(1, int(grid.max()) + 1):
    lab, k = scipy.ndimage.label(grid == v)  # the default structure is 6-connectivity
    comp[lab > 0] = lab[lab > 0] + n
    n += k
  ids, first = np.unique(comp.ravel(order="F"), return_index=True)
  keep = ids != 0
  lut = np.zeros(n + 1, np.uint32)
  lut[ids[keep][np.argsort(first[keep])]] = np.arange(1, n + 1, dtype=np.uint32)
  return lut[comp], n


def block_plane(grid, block, shape, bz):
  """the (sx, sy) plane of the expanded volume in block layer bz"""
  ix = np.arange(shape[0]) // block[0]
  iy = np.arange(shape[1]) // block[1]
  return grid[:, :, bz][np.ix_(ix, iy)]


def expand(grid, block, shape):
  """the whole expanded volume (small shapes only)"""
  ix, iy, iz = (np.arange(s) // b for s, b in zip(shape, block))
  return np.asfortranarray(grid[np.ix_(ix, iy, iz)])


def block_boxes(comp, n, block, shape):
  """[n, 6] u32 (min x, min y, min z, max x, max y, max z), maxima inclusive, of the expanded
  components"""
  boxes = np.zeros((n, 6), np.uint32)
  for i, sl in enumerate(scipy.ndimage.find_objects(comp, max_label=n)):
    for a in range(3):
      boxes[i, a] = sl[a].start * block[a]
      boxes[i, 3 + a] = min(sl[a].stop * block[a], shape[a]) - 1
  return boxes


def mesher_triangles(shape, width):
  """marching-cubes triangles of x-slabs `width` voxels wide alternating labels 1 and 2: every
  cube across a slab boundary gives two triangles to each label"""
  sx, sy, sz = shape
  return len(range(width, sx, width)) * (sy - 1) * (sz - 1) * 4


def test_block_reference_matches_oracle_and_scipy(oracle):
  for shape, block, seed in (((83, 61, 47), (7, 5, 3), 1), ((64, 33, 20), (8, 4, 5), 2), ((150, 100, 95), BLOCK, 3)):
    grid = block_grid(shape, block, seed)
    comp, n = block_components(grid)
    vol = expand(grid, block, shape)
    want, n_want = oracle.connected_components(vol, return_N=True)
    assert n == n_want > 1
    assert np.array_equal(expand(comp, block, shape), want)
    for bz in range(grid.shape[2]):
      z = bz * block[2]
      assert np.array_equal(block_plane(comp, block, shape, bz), want[:, :, z])
    objs = scipy.ndimage.find_objects(want.astype(np.int64))
    got = block_boxes(comp, n, block, shape)
    for i, sl in enumerate(objs):
      assert tuple(got[i, :3]) == tuple(s.start for s in sl)
      assert tuple(got[i, 3:]) == tuple(s.stop - 1 for s in sl)


def test_mesher_triangle_formula_matches_oracle(oracle):
  shape = (63, 33, 17)
  x = np.arange(shape[0])
  vol = np.asfortranarray(np.broadcast_to((1 + (x // 4) % 2).astype(np.uint8)[:, None, None], shape))
  tl, tv = oracle.marching_cubes(vol)
  assert len(tl) == mesher_triangles(shape, 4)
  # the GPU test's volume: 3T between 2^31 and 2^32 corners
  assert 2**31 < 3 * mesher_triangles((1023,) * 3, 4) < 2**32


# ---------------------------------------------------------------- plumbing
def _device_used():
  import torch
  free, total = torch.cuda.mem_get_info()
  return total - free


def report_peak(name, baseline):
  """Device memory the test holds now over what the device held before it.  A scratch arena keeps
  its high-water size after a call, so with the test's buffers still allocated this is its peak
  (device-wide: other work on the device counts too)."""
  used = _device_used() - baseline
  print("\n%s: peak device memory %.1f GB" % (name, used / 1e9))


@pytest.fixture
def big(request):
  """a context of its own (its scratch arena and pinned slabs go with it) and a list of device
  buffers freed after the test"""
  from igneous_b200 import _shim
  baseline = _device_used()
  ctx = _shim.Context()
  bufs = []
  try:
    yield ctx, bufs
    report_peak(request.node.name, baseline)
  finally:
    for b in bufs:
      b.free()
    ctx.close()


def _alloc(big, nbytes):
  ctx, bufs = big
  b = ctx.alloc(nbytes)
  bufs.append(b)
  return b


def _z_slabs(shape, itemsize):
  sx, sy, sz = shape
  step = max(1, SLAB_BYTES // (sx * sy * itemsize))
  for z0 in range(0, sz, step):
    yield z0, min(sz, z0 + step)


def _fill_planes(ctx, buf, shape, plane_of_z, dtype=np.uint8):
  """volume whose z-plane z is plane_of_z(z) (a host (sx, sy) array, the same object for
  consecutive equal planes): one upload per distinct plane, device copies for the rest"""
  sx, sy, sz = shape
  pb = sx * sy * np.dtype(dtype).itemsize
  prev, src = None, None
  for z in range(sz):
    plane = plane_of_z(z)
    if plane is prev:
      ctx.d2d(buf.offset(z * pb), src, pb)
    else:
      ctx.h2d(buf.offset(z * pb), np.asfortranarray(plane, dtype=dtype))
      prev, src = plane, buf.offset(z * pb)
  ctx.sync()


def _fill_repeated(ctx, buf, shape, plane):
  """u8 volume of one repeated z-plane, by doubling device copies"""
  sx, sy, sz = shape
  pb = sx * sy
  ctx.h2d(buf, np.asfortranarray(plane, dtype=np.uint8))
  done = 1
  while done < sz:
    k = min(done, sz - done)
    ctx.d2d(buf.offset(done * pb), buf.ptr, k * pb)
    done += k
  ctx.sync()


def _read_slab(ctx, host, buf, shape, dtype, z0, z1):
  sx, sy, _ = shape
  it = np.dtype(dtype).itemsize
  view = host[: sx * sy * (z1 - z0)]
  ctx.d2h(view, buf.offset(z0 * sx * sy * it), view.nbytes)
  ctx.sync()
  return view.reshape((sx, sy, z1 - z0), order="F")


def _histogram_u8(big, buf, n):
  ctx, _ = big
  hist = _alloc(big, 256 * 8)
  ctx.memset(hist, 0, 256 * 8)
  assert ctx.lib.ign_histogram_dev(ctx.handle, buf.ptr, IGN_U8, n, hist.ptr) == 0
  out = np.empty(256, np.uint64)
  ctx.d2h(out, hist)
  ctx.sync()
  return out


def _ccl(ctx, d_in, shape, d_out, out_dtype):
  n = c.c_uint64(0)
  rc = ctx.lib.ign_ccl6_dev(ctx.handle, d_in.ptr, IGN_U8, *shape, d_out.ptr, out_dtype, c.byref(n))
  return rc, n.value


# --------------------------------------------------------- CCL, find_objects
@pytest.mark.gpu
@pytest.mark.parametrize("shape", [BIG_TMA, BIG_ODD], ids=["4096x1024x1025", "4099x1031x1017"])
def test_ccl_and_find_objects_of_block_volumes_past_2_32(big, shape):
  ctx, _ = big
  grid = block_grid(shape, BLOCK, seed=sum(shape))
  comp, n_want = block_components(grid)
  sx, sy, sz = shape
  n = sx * sy * sz
  assert n > 2**32
  d_in = _alloc(big, n)
  d_out = _alloc(big, n * 4)
  planes = {}

  def grid_plane(z):
    bz = z // BLOCK[2]
    if bz not in planes:
      planes.clear()
      planes[bz] = block_plane(grid, BLOCK, shape, bz)
    return planes[bz]

  _fill_planes(ctx, d_in, shape, grid_plane)
  rc, n_got = _ccl(ctx, d_in, shape, d_out, IGN_U32)
  assert rc == 0, ctx.lib.ign_last_error()
  assert n_got == n_want

  host = ctx.pinned_empty((SLAB_BYTES // 4,), np.uint32)
  for z0, z1 in _z_slabs(shape, 4):
    got = _read_slab(ctx, host, d_out, shape, np.uint32, z0, z1)
    for bz in range(z0 // BLOCK[2], (z1 - 1) // BLOCK[2] + 1):
      a, b = max(z0, bz * BLOCK[2]), min(z1, (bz + 1) * BLOCK[2])
      want = block_plane(comp, BLOCK, shape, bz)
      ok = got[:, :, a - z0:b - z0] == want[:, :, None]
      if not ok.all():
        x, y, z = np.argwhere(~ok)[0]
        pytest.fail("label at (%d, %d, %d) is %d, want %d" % (x, y, a + z, got[x, y, a - z0 + z], want[x, y]))

  # the largest label, found on the device, then every component's box
  max_label = c.c_uint64(0)
  assert ctx.lib.ign_find_objects_dev(ctx.handle, d_out.ptr, IGN_U32, *shape, c.byref(max_label), None) == 0
  assert max_label.value == n_want
  d_boxes = _alloc(big, n_want * 24)
  assert ctx.lib.ign_find_objects_dev(ctx.handle, d_out.ptr, IGN_U32, *shape, c.byref(max_label), d_boxes.ptr) == 0
  boxes = np.empty((n_want, 6), np.uint32)
  ctx.d2h(boxes, d_boxes)
  ctx.sync()
  assert np.array_equal(boxes, block_boxes(comp, n_want, BLOCK, shape))


# ------------------------------------------------------- run-count refusals
def _x_pattern(shape, pattern):
  sx, sy, _ = shape
  row = np.asarray(pattern, np.uint8)[np.arange(sx) % len(pattern)]
  return np.broadcast_to(row[:, None], (sx, sy))


@pytest.mark.gpu
@pytest.mark.parametrize("shape,pattern,runs", [
  (HEADLINE, (1, 2), 2**32),                 # rbase[W] wraps to 0: looked like a volume without runs
  (HEADLINE, (1, 2, 3, 0), 3 * 2**30),       # between 2^31 and 2^32
  (BIG_TMA, (1, 2), 2**32 + 2**22),          # rbase[W] wraps to 2^22
], ids=["runs_2_32", "runs_3x2_30", "runs_2_32_plus_2_22"])
def test_ccl_refuses_2_31_runs_or_more(big, shape, pattern, runs):
  ctx, _ = big
  sx, sy, sz = shape
  n = sx * sy * sz
  assert sx % len(pattern) == 0 and n // len(pattern) * sum(1 for v in pattern if v) == runs
  d_in = _alloc(big, n)
  d_out = _alloc(big, n * 2)
  _fill_repeated(ctx, d_in, shape, _x_pattern(shape, pattern))
  ctx.memset(d_out, 0xAB, 4096)
  ctx.sync()
  rc, n_got = _ccl(ctx, d_in, shape, d_out, IGN_U16)
  assert rc == IGN_ERR_OVERFLOW, (rc, n_got)
  assert b"runs exceed" in ctx.lib.ign_last_error()
  head = np.empty(4096, np.uint8)
  ctx.d2h(head, d_out)
  ctx.sync()
  assert (head == 0xAB).all()  # nothing written
  # the same refusal for dust, the task body and the multi-volume begin
  assert ctx.lib.ign_dust_dev(ctx.handle, d_in.ptr, IGN_U8, *shape, 2) == IGN_ERR_OVERFLOW
  v = c.c_void_p()
  k = c.c_uint64(0)
  assert ctx.lib.ign_ccl6_volume_begin_dev(ctx.handle, d_in.ptr, IGN_U8, *shape, None, None, None, None, c.byref(v),
                                           c.byref(k)) == IGN_ERR_OVERFLOW
  assert not v.value


# ------------------------------------------------------------------- dust
@pytest.mark.gpu
def test_dust_keeps_a_component_of_2_32_voxels(big):
  ctx, _ = big
  sx, sy, sz = HEADLINE
  n = sx * sy * sz
  d = _alloc(big, n)
  ctx.memset(d, 1, n)
  ctx.sync()
  assert ctx.lib.ign_dust_dev(ctx.handle, d.ptr, IGN_U8, *HEADLINE, 1) == 0
  hist = _histogram_u8(big, d, n)
  assert hist[1] == n and hist.sum() == n


@pytest.mark.gpu
def test_dust_between_a_huge_component_and_small_ones(big):
  """ones everywhere (one component of 2^32 + 2^22 - 3 * 2^20 - 1001 voxels) around a 2-block of
  3 * 2^20 voxels, a 3-block of 1000 and a lone 2 at (sx - 1, 0, sz - 1); threshold 2^21 removes the
  last two.  A count modulo 2^32 (2^20 - 1001) would remove the huge component too."""
  ctx, _ = big
  shape = BIG_TMA
  sx, sy, sz = shape
  n = sx * sy * sz
  keep_box = (slice(100, 228), slice(200, 328), slice(300, 492))
  small_box = (slice(4000, 4010), slice(1000, 1010), slice(1010, 1020))
  tail_z = 1008
  want_tail = np.ones((sx, sy, sz - tail_z), np.uint8, order="F")
  want_tail[small_box[0], small_box[1], small_box[2].start - tail_z:small_box[2].stop - tail_z] = 3
  want_tail[-1, 0, -1] = 2

  d = _alloc(big, n)
  ones = np.ones((sx, sy), np.uint8)
  with_keep = ones.copy()
  with_keep[keep_box[:2]] = 2
  _fill_planes(ctx, d, shape, lambda z: with_keep if keep_box[2].start <= z < keep_box[2].stop else ones)
  ctx.h2d(d.offset(tail_z * sx * sy), want_tail)
  ctx.sync()
  assert ctx.lib.ign_dust_dev(ctx.handle, d.ptr, IGN_U8, *shape, 2**21) == 0

  hist = _histogram_u8(big, d, n)
  want = np.zeros(256, np.uint64)
  want[0] = 1001
  want[2] = 3 * 2**20
  want[1] = n - want[0] - want[2]
  assert np.array_equal(hist, want)
  want_tail[want_tail == 3] = 0
  want_tail[-1, 0, -1] = 0
  host = np.empty(want_tail.size, np.uint8)
  assert np.array_equal(_read_slab(ctx, host, d, shape, np.uint8, tail_z, sz), want_tail)
  # the kept block where it was: its z-range, re-read
  got = _read_slab(ctx, np.empty(sx * sy * 2, np.uint8), d, shape, np.uint8, keep_box[2].start, keep_box[2].start + 2)
  assert (got[keep_box[0], keep_box[1]] == 2).all() and got.sum(dtype=np.int64) == 2 * (sx * sy + 128 * 128)


@pytest.mark.gpu
def test_ccl_task_dust_threshold_2_32(big):
  """the CCLFacesTask body on one component of 2^32 + 2^22 voxels with dust threshold 2^32: kept,
  u64 labels all 1"""
  ctx, _ = big
  shape = BIG_TMA
  n = shape[0] * shape[1] * shape[2]
  d_in = _alloc(big, n)
  d_out = _alloc(big, n * 8)
  ctx.memset(d_in, 1, n)
  ctx.sync()
  k = c.c_uint64(0)
  rails = shape  # rail coordinates outside the volume: none
  assert ctx.lib.ign_ccl_task_dev(ctx.handle, d_in.ptr, IGN_U8, *shape, 0, 0, 0, 0, *rails, 2**32, 0, d_out.ptr,
                                  c.byref(k)) == 0
  assert k.value == 1
  # labels narrowed onto the input buffer, then counted
  assert ctx.lib.ign_cast_dev(ctx.handle, d_out.ptr, IGN_U64, d_in.ptr, IGN_U8, n) == 0
  hist = _histogram_u8(big, d_in, n)
  assert hist[1] == n and hist.sum() == n
  for z0, z1 in ((0, 1), (shape[2] - 1, shape[2])):  # the u64 labels themselves at both ends
    got = _read_slab(ctx, np.empty(shape[0] * shape[1], np.uint64), d_out, shape, np.uint64, z0, z1)
    assert (got == 1).all()


# ----------------------------------------------------------------- mesher
@pytest.mark.gpu
def test_mesher_refuses_more_than_2_31_corners(big):
  ctx, _ = big
  shape = (1023, 1023, 1023)
  n = shape[0] * shape[1] * shape[2]
  d = _alloc(big, n)
  x = np.arange(shape[0])
  _fill_repeated(ctx, d, shape, np.broadcast_to((1 + (x // 4) % 2).astype(np.uint8)[:, None], shape[:2]))
  m = c.c_void_p()
  rc = ctx.lib.ign_mesh_begin_dev(ctx.handle, d.ptr, IGN_U8, *shape, c.byref(m))
  assert rc == IGN_ERR_OVERFLOW, ctx.lib.ign_last_error()
  assert not m.value
  assert str(mesher_triangles(shape, 4)).encode() in ctx.lib.ign_last_error()


# ---------------------------------------------------------------- pooling
# element index 2^31 and 2^32 of BIG_TMA lie in z-planes 512 and 1024 (the last)
BOUNDARY_Z = (0, 511, 512, 1023, 1024)


def _synth_image(big, shape, seed):
  ctx, _ = big
  d = _alloc(big, shape[0] * shape[1] * shape[2])
  assert ctx.lib.ign_synth_image_dev(ctx.handle, d.ptr, *shape, 0, 0, 0, seed) == 0
  return d


def _mip_shapes(shape, factor, num_mips):
  out, s = [], tuple(shape)
  for _ in range(num_mips):
    s = tuple(-(-a // f) for a, f in zip(s, factor))
    out.append(s)
  return out


@pytest.mark.gpu
@pytest.mark.parametrize("kind,shape", [
  ("mode", BIG_TMA),               # fused k_mode_fused<u8,4>
  ("sparse_mode", BIG_TMA),        # generic path
  ("avg0", BIG_TMA), ("avg1", BIG_TMA), ("avg2", BIG_TMA),  # fused, roundings 0-2
  ("avg0", (4097, 1024, 1024)),    # odd sx: generic with accumulators
])
def test_pool_2x2x1_past_2_32_matches_oracle_on_boundary_planes(big, oracle, kind, shape):
  ctx, _ = big
  sx, sy, sz = shape
  n = sx * sy * sz
  assert n > 2**32
  num_mips = 4
  seed = 11
  d_in = _synth_image(big, shape, seed)
  shapes = _mip_shapes(shape, (2, 2, 1), num_mips)
  outs = [_alloc(big, int(np.prod(s))) for s in shapes]
  from igneous_b200 import _shim
  if kind.endswith("mode"):
    fn, flag = ctx.lib.ign_pool_mode_2x2x1_dev, int(kind == "sparse_mode")
  else:
    fn, flag = ctx.lib.ign_pool_avg_2x2x1_dev, int(kind[-1])
  assert fn(ctx.handle, d_in.ptr, IGN_U8, *shape, num_mips, flag, _shim.void_pp([o.ptr for o in outs])) == 0
  ctx.sync()
  k = 2**31 // (sx * sy)  # the plane that holds element 2^31
  zs = sorted({0, k - 1, k, k + 1, min(2**32 // (sx * sy), sz - 1), sz - 1})
  for z in zs:
    plane = oracle.synth_image((sx, sy, 1), seed=seed, offset=(0, 0, z))
    if kind.endswith("mode"):
      want = oracle.downsample_segmentation(plane, (2, 2, 1), num_mips=num_mips, sparse=bool(flag))
    else:
      want = oracle.downsample_with_averaging(plane, (2, 2, 1), num_mips=num_mips, rounding=flag)
    for m, (s, o) in enumerate(zip(shapes, outs)):
      got = _read_slab(ctx, np.empty(s[0] * s[1], np.uint8), o, s, np.uint8, z, z + 1)
      assert np.array_equal(got, want[m]), (kind, z, m)


@pytest.mark.gpu
def test_pool_2x2x1_mode_of_a_block_volume_past_2_32(big):
  """blocks of 48 x 32 x 23 voxels: every 2^m x 2^m window (m <= 4) lies in one block, so mip m is
  the grid expanded with blocks of 48 / 2^m x 32 / 2^m x 23, compared whole"""
  ctx, _ = big
  shape, block, num_mips = BIG_TMA, (48, 32, 23), 4
  grid = block_grid(shape, block, seed=5)
  d_in = _alloc(big, shape[0] * shape[1] * shape[2])
  planes = {}

  def grid_plane(z):
    bz = z // block[2]
    if bz not in planes:
      planes.clear()
      planes[bz] = block_plane(grid, block, shape, bz)
    return planes[bz]

  _fill_planes(ctx, d_in, shape, grid_plane)
  shapes = _mip_shapes(shape, (2, 2, 1), num_mips)
  outs = [_alloc(big, int(np.prod(s))) for s in shapes]
  from igneous_b200 import _shim
  assert ctx.lib.ign_pool_mode_2x2x1_dev(ctx.handle, d_in.ptr, IGN_U8, *shape, num_mips, 0,
                                         _shim.void_pp([o.ptr for o in outs])) == 0
  ctx.sync()
  for m, (s, o) in enumerate(zip(shapes, outs)):
    mblock = (block[0] >> (m + 1), block[1] >> (m + 1), block[2])
    host = np.empty(s[0] * s[1] * 64, np.uint8)
    for z0 in range(0, s[2], 64):
      z1 = min(s[2], z0 + 64)
      got = _read_slab(ctx, host, o, s, np.uint8, z0, z1)
      for z in range(z0, z1):
        assert np.array_equal(got[:, :, z - z0], block_plane(grid, mblock, s, z // block[2])), (m, z)


@pytest.mark.gpu
@pytest.mark.parametrize("op", ["min", "max", "stride", "mode"])
def test_pool_select_2x2x2_past_2_32_matches_oracle(big, oracle, op):
  ctx, _ = big
  shape, num_mips, seed = BIG_TMA, 2, 13
  sx, sy, sz = shape
  d_in = _synth_image(big, shape, seed)
  shapes = _mip_shapes(shape, (2, 2, 2), num_mips)
  outs = [_alloc(big, int(np.prod(s))) for s in shapes]
  from igneous_b200 import _shim
  code = {"min": 0, "max": 1, "stride": 2, "mode": 3}[op]
  assert ctx.lib.ign_pool_select_dev(ctx.handle, d_in.ptr, IGN_U8, *shape, 2, 2, 2, num_mips, code,
                                     _shim.void_pp([o.ptr for o in outs])) == 0
  ctx.sync()
  for z0 in (0, 508, 512, 1020, 1024):  # slabs aligned to 2^num_mips; z 1024 is a partial block
    slab = oracle.synth_image((sx, sy, min(4, sz - z0)), seed=seed, offset=(0, 0, z0))
    if op == "mode":
      want = oracle.downsample_segmentation(slab, (2, 2, 2), num_mips=num_mips)
    else:
      want = oracle.downsample_select(slab, (2, 2, 2), num_mips=num_mips, op=op)
    for m, (s, o) in enumerate(zip(shapes, outs)):
      mz0 = z0 >> (m + 1)
      w = want[m]
      got = _read_slab(ctx, np.empty(w.size, np.uint8), o, s, np.uint8, mz0, mz0 + w.shape[2])
      assert np.array_equal(got, w), (op, z0, m)


# ----------------------------------------------------------- remap family
N_REMAP = 2**32 - 2   # the most elements renumber and unique accept
PERIOD = 65521        # prime: the pattern does not repeat at 2^31 or 2^32


def _fill_periodic(ctx, buf, n, pattern):
  """buf[i] = pattern[i % len(pattern)] for i < n, by doubling device copies"""
  p = len(pattern)
  it = pattern.dtype.itemsize
  head = np.resize(pattern, p * 256)
  ctx.h2d(buf, head)
  done = head.size
  while done < n:
    k = min(done, n - done)
    ctx.d2d(buf.offset(done * it), buf.ptr, k * it)
    done += k
  ctx.sync()


def _index_slabs(n, size=1 << 24):
  return [(0, size), (2**31 - size // 2, 2**31 + size // 2), (n - size, n)]


@pytest.mark.gpu
def test_renumber_and_remap_u16_at_2_32_minus_2(big):
  ctx, _ = big
  n = N_REMAP
  rng = np.random.default_rng(17)
  pattern = rng.permutation(65536)[:PERIOD].astype(np.uint16)  # distinct values, 0 among them or not
  nz = pattern[pattern != 0]
  lut = np.zeros(65536, np.uint32)
  lut[nz] = np.arange(1, nz.size + 1, dtype=np.uint32)  # first appearance order
  d_in = _alloc(big, (n + 2) * 2)
  d_out = _alloc(big, (n + 2) * 4)
  d_uniq = _alloc(big, 65536 * 8)
  _fill_periodic(ctx, d_in, n, pattern)
  k = c.c_uint64(0)
  assert ctx.lib.ign_renumber_dev(ctx.handle, d_in.ptr, IGN_U16, n, d_out.ptr, d_uniq.ptr, 65536, c.byref(k)) == 0
  assert k.value == nz.size
  uniq = np.empty(k.value, np.uint64)
  ctx.d2h(uniq, d_uniq)
  ctx.sync()
  assert np.array_equal(uniq, nz.astype(np.uint64))
  for a, b in _index_slabs(n):
    got = np.empty(b - a, np.uint32)
    ctx.d2h(got, d_out.offset(a * 4))
    ctx.sync()
    assert np.array_equal(got, lut[pattern[np.arange(a, b) % PERIOD]]), (a, b)

  # n = 2^32 - 1 is refused before any launch
  before = ctx.launch_count()
  assert ctx.lib.ign_renumber_dev(ctx.handle, d_in.ptr, IGN_U16, n + 1, d_out.ptr, d_uniq.ptr, 65536,
                                  c.byref(k)) == IGN_ERR_OVERFLOW
  assert ctx.launch_count() == before

  # remap every value in place (no value is missing)
  keys = np.unique(pattern).astype(np.uint64)
  vals = (keys * np.uint64(40503) + np.uint64(7)) % np.uint64(65536)
  table = np.zeros(65536, np.uint16)
  table[keys.astype(np.int64)] = vals.astype(np.uint16)
  assert ctx.lib.ign_remap_dev(ctx.handle, d_in.ptr, IGN_U16, n, keys.ctypes.data_as(c.c_void_p),
                               vals.ctypes.data_as(c.c_void_p), keys.size, 0) == 0
  for a, b in _index_slabs(n):
    got = np.empty(b - a, np.uint16)
    ctx.d2h(got, d_in.offset(a * 2))
    ctx.sync()
    assert np.array_equal(got, table[pattern[np.arange(a, b) % PERIOD]]), (a, b)


@pytest.mark.gpu
def test_unique_and_mask_u8_at_2_32_minus_2(big):
  ctx, _ = big
  n = N_REMAP
  p = 251
  pattern = np.random.default_rng(19).permutation(256)[:p].astype(np.uint8)
  host = np.resize(pattern, n + 1)  # one more element for the refusal
  counts_of = np.full(p, n // p, np.uint64)
  counts_of[: n % p] += 1
  order = np.argsort(pattern)
  uniq = np.zeros(256, np.uint64)
  counts = np.zeros(256, np.uint64)
  k = c.c_uint64(0)
  assert ctx.lib.ign_unique(ctx.handle, host.ctypes.data_as(c.c_void_p), IGN_U8, n, uniq.ctypes.data_as(c.c_void_p),
                            counts.ctypes.data_as(c.c_void_p), 256, c.byref(k)) == 0
  assert k.value == p
  assert np.array_equal(uniq[:p], pattern[order].astype(np.uint64))
  assert np.array_equal(counts[:p], counts_of[order])
  before = ctx.launch_count()
  assert ctx.lib.ign_unique(ctx.handle, host.ctypes.data_as(c.c_void_p), IGN_U8, n + 1, uniq.ctypes.data_as(c.c_void_p),
                            counts.ctypes.data_as(c.c_void_p), 256, c.byref(k)) == IGN_ERR_OVERFLOW
  assert ctx.launch_count() == before

  labels = pattern[::3].astype(np.uint64)
  assert ctx.lib.ign_mask(ctx.handle, host.ctypes.data_as(c.c_void_p), IGN_U8, n, labels.ctypes.data_as(c.c_void_p),
                          labels.size, 0, 255) == 0
  masked = np.where(np.isin(pattern, pattern[::3]), np.uint8(255), pattern)
  step = p * (1 << 20)
  tile = np.tile(masked, step // p)
  for a in range(0, n, step):
    b = min(n, a + step)
    assert np.array_equal(host[a:b], tile[:b - a]), a  # a is a multiple of p
  assert host[n] == pattern[n % p]  # past n: untouched


# --------------------------------------------------------------- contrast
@pytest.mark.gpu
def test_contrast_stretch_u8_past_2_32_matches_contrastref(big):
  import contrastref
  ctx, _ = big
  shape, seed = BIG_TMA, 23
  sx, sy, sz = shape
  z = np.arange(sz)
  lower = (z % 50).astype(np.uint32)
  upper = (200 + z % 55).astype(np.uint32)
  upper[z % 97 == 0] = lower[z % 97 == 0]  # slices left as they are
  d_in = _synth_image(big, shape, seed)
  d_out = _alloc(big, sx * sy * sz)
  assert ctx.lib.ign_contrast_stretch_dev(ctx.handle, d_in.ptr, IGN_U8, *shape, 1, lower.ctypes.data_as(c.c_void_p),
                                          upper.ctypes.data_as(c.c_void_p), 3, 250, d_out.ptr, IGN_U8) == 0
  ctx.sync()
  for zz in BOUNDARY_Z + (970,):  # 970 = 97 * 10: a slice left as it is
    plane = oracle_image(shape, seed, zz)
    want = contrastref.stretch(plane, [(int(lower[zz]), int(upper[zz]))], 255, 3, 250, np.uint8)
    got = _read_slab(ctx, np.empty(sx * sy, np.uint8), d_out, shape, np.uint8, zz, zz + 1)
    assert np.array_equal(got, want), zz


def oracle_image(shape, seed, z):
  from oracle import oracle as O
  return O.synth_image((shape[0], shape[1], 1), seed=seed, offset=(0, 0, z))


@pytest.mark.gpu
def test_quantize_past_2_32_matches_contrastref(big):
  import contrastref
  ctx, _ = big
  shape = BIG_TMA
  sx, sy, sz = shape
  n = sx * sy * sz
  i = np.arange(sx * sy)
  base = ((i % 1283).astype(np.float32) / np.float32(1000.0) - np.float32(0.1)).reshape((sx, sy), order="F")
  base.ravel(order="F")[::997] = np.nan
  plane_of = lambda z: base + np.float32(z) * np.float32(1e-4)  # every plane its own values
  d_in = _alloc(big, n * 4)
  d_out = _alloc(big, n)
  _fill_planes(ctx, d_in, shape, plane_of, dtype=np.float32)
  assert ctx.lib.ign_quantize_dev(ctx.handle, d_in.ptr, n, d_out.ptr) == 0
  ctx.sync()
  for z in BOUNDARY_Z:
    want = contrastref.quantize(plane_of(z)[:, :, None])[:, :, :, 0]
    got = _read_slab(ctx, np.empty(sx * sy, np.uint8), d_out, shape, np.uint8, z, z + 1)
    assert np.array_equal(got, want), z


# ------------------------------------------------------- the headline step
def _box(ctx, dptr, dtype, shape, origin, size):
  from igneous_b200 import _shim
  d = ctx.alloc(int(np.prod(size)) * np.dtype(dtype).itemsize)
  try:
    assert ctx.lib.ign_copy_box_dev(ctx.handle, dptr.ptr, _shim.dtype_code(dtype), *shape, *origin, *size,
                                    d.ptr) == 0
    return ctx.to_host(d, size, dtype)
  finally:
    d.free()


@pytest.mark.gpu
def test_headline_step_past_the_origin(oracle):
  """one step of the benchmark's workload (2048x2048x1024 u32, pitch 64, 2^20 ids, 256^3 mesh tasks,
  simplification 100, 8 mesh streams), checked at the far corner and, for CCL, over the whole volume"""
  from igneous_b200 import _shim, pipeline, zmesh
  baseline = _device_used()
  ctx = _shim.Context()
  pipe = pipeline.VolumePipeline(ctx, HEADLINE, np.uint32, num_mips=2, mesh_shape=(256, 256, 256),
                                 resolution=(16, 16, 40), pitch=64, num_ids=1 << 20, seed=0,
                                 simplification_factor=100, mesh_streams=8)
  try:
    pipe.synth()
    pipe.step(timers=False)
    ctx.sync()
    report_peak("test_headline_step_past_the_origin", baseline)
    sx, sy, sz = HEADLINE

    # mips and the input on the far-corner sub-box, bit for bit
    size = (256, 256, 64)
    origin = (sx - 256, sy - 256, sz - 64)
    seg = oracle.synth_seg(size, pitch=64, num_ids=1 << 20, seed=0, offset=origin, dtype=np.uint32)
    assert np.array_equal(_box(ctx, pipe.d_in, np.uint32, HEADLINE, origin, size), seg)
    for m, w in enumerate(oracle.downsample_segmentation(seg, (2, 2, 1), num_mips=2)):
      o = (origin[0] >> (m + 1), origin[1] >> (m + 1), origin[2])
      assert np.array_equal(_box(ctx, pipe.d_mips[m], np.uint32, pipe.mip_shapes[m], o, w.shape), w), m

    # CCL on the same sub-box: each oracle component carries one label, each label one input id
    cc = _box(ctx, pipe.d_cc, np.uint32, HEADLINE, origin, size).astype(np.uint64)
    loc = oracle.connected_components(seg).astype(np.uint64)
    assert np.array_equal(cc == 0, seg == 0)
    pairs = np.unique(np.stack([loc.ravel(), cc.ravel()], axis=1), axis=0)
    pairs = pairs[pairs[:, 0] != 0]
    assert len(np.unique(pairs[:, 0])) == len(pairs)

    # CCL over the whole volume, by z-slab, one plane carried across slabs
    ncomp = pipe.n_components
    assert ncomp > 0
    value_of = np.zeros(ncomp + 1, np.uint64)
    seen = np.zeros(ncomp + 1, bool)
    host_l = ctx.pinned_empty((SLAB_BYTES // 4,), np.uint32)
    host_v = ctx.pinned_empty((SLAB_BYTES // 4,), np.uint32)
    prev_l = prev_v = None
    run_max = 0
    largest = 0
    for z0, z1 in _z_slabs(HEADLINE, 4):
      lab = _read_slab(ctx, host_l, pipe.d_cc, HEADLINE, np.uint32, z0, z1)
      val = _read_slab(ctx, host_v, pipe.d_in, HEADLINE, np.uint32, z0, z1)
      assert np.array_equal(lab == 0, val == 0), z0
      for a in (0, 1, 2):  # equal non-zero 6-neighbours have equal labels
        sl0 = [slice(None)] * 3
        sl1 = [slice(None)] * 3
        sl0[a], sl1[a] = slice(None, -1), slice(1, None)
        v0, v1 = val[tuple(sl0)], val[tuple(sl1)]
        same = (v0 == v1) & (v0 != 0)
        assert not (same & (lab[tuple(sl0)] != lab[tuple(sl1)])).any(), (z0, a)
      if prev_l is not None:
        same = (prev_v == val[:, :, 0]) & (prev_v != 0)
        assert not (same & (prev_l != lab[:, :, 0])).any(), z0
      # each label one input value: checked at the heads of x-runs of a label, and along the runs
      flat_l = lab.ravel(order="F")
      flat_v = val.ravel(order="F")
      inrun = (flat_l[1:] == flat_l[:-1])
      assert np.array_equal(flat_v[1:][inrun], flat_v[:-1][inrun]), z0
      heads = np.concatenate([[True], ~inrun]) & (flat_l != 0)
      hl, hv = flat_l[heads], flat_v[heads].astype(np.uint64)
      known = seen[hl]
      assert np.array_equal(value_of[hl[known]], hv[known]), z0
      value_of[hl] = hv
      seen[hl] = True
      assert np.array_equal(value_of[hl], hv), z0  # one value for labels first met twice in this slab
      # first appearances in raster order are 1, 2, 3, ...
      acc = np.maximum.accumulate(np.concatenate([[run_max], flat_l.astype(np.int64)]))
      assert np.diff(acc).max() <= 1, z0
      run_max = int(acc[-1])
      largest = max(largest, int(flat_l.max()))
      prev_l, prev_v = lab[:, :, -1].copy(), val[:, :, -1].copy()
    assert largest == ncomp and run_max == ncomp and seen[1:].all()

    # the step fills the card: the standalone meshers below need what the input, the labels and the
    # mesh streams' scratch arenas hold (pipe.free() skips what is released here)
    pipe.d_in.free()
    pipe.d_cc.free()
    for wctx, buf in pipe._workers:
      buf.free()
      wctx.close()
    pipe._workers = []

    # mesh: the last MeshTask against a standalone Mesher on the same cutout
    msrc, mshape = pipe.d_mips[-1], pipe.mip_shapes[-1]
    task = list(pipe.mesh_tasks())[-1]
    cut = _box(ctx, msrc, np.uint32, mshape, task[:3], task[3:])
    m = zmesh.Mesher(pipe.resolution)
    m.mesh(cut)
    nv0, nf0 = c.c_uint64(0), c.c_uint64(0)
    _shim.check(ctx.lib.ign_mesh_totals(m._handle, c.byref(nv0), c.byref(nf0)))
    ids = m.ids()
    m.get(ids[0], reduction_factor=100, max_error=40, voxel_centered=True)
    nv, nf = c.c_uint64(0), c.c_uint64(0)
    _shim.check(ctx.lib.ign_mesh_totals(m._handle, c.byref(nv), c.byref(nf)))
    assert tuple(pipe.mesh_task_counts[-1]) == (nf.value, nv.value, len(ids), nf0.value, nv0.value)

    # a 129x129x65 cutout at the far corner of the mesh mip, bit for bit against the oracle
    csize = (129, 129, 65)
    cut = _box(ctx, msrc, np.uint32, mshape, tuple(s - b for s, b in zip(mshape, csize)), csize)
    m = zmesh.Mesher(pipe.resolution)
    m.mesh(cut)
    tl, tv = oracle.marching_cubes(cut)
    W = oracle.WeldedMeshes(tl, tv)
    assert sorted(m.ids()) == W.ids()
    ref, _ = oracle.simplify_welded(W, pipe.resolution, 100, 40.0, True)
    for lab in W.ids():
      g = m.get(lab, reduction_factor=100, max_error=40, voxel_centered=True)
      assert np.array_equal(g.vertices, ref[lab][0]) and np.array_equal(g.faces, ref[lab][1]), lab
  finally:
    pipe.free()
    ctx.close()
