"""CCL on rows of 2048 to 131,072 voxels, the longest row check_ccl_dims accepts.  The tile pass
k_ccl_tiles resolves TY x TY rows per CTA and halves TY from 8 while the tile's mask words exceed
TB_WMAX, so rows past 2048 voxels take flatter tiles (TY 4, 2, 1) and, at TY = 1, every row is a tile
face for k_ccl_merge.  The shape table below restates the host's dispatch rules and asserts that it
reaches every tile height, both mask kernels (paired or not), both mask fills (TMA or cooperative),
both word splits (shifts or divisions) and both expansions (vector or scalar), with partial tiles and
with tiles on both sides of the shared-memory run limit."""
import ctypes as c

import numpy as np
import pytest

from labelref import ccl6

TB_WMAX = 4096   # mask words of one tile
TB_RCAP = 8192   # runs of one tile resolved in shared memory
MT_BX = 128      # voxels along x of one mask tile
MAX_SX = TB_WMAX * 32
IGN_ERR_OVERFLOW = -6


def dispatch(sx, itemsize):
  """What ccl_structure / write_labels select for rows of sx voxels (16-byte aligned buffers)."""
  wpr = (sx + 31) // 32
  ty = 8
  while ty > 1 and wpr * ty * ty > TB_WMAX:
    ty //= 2
  return dict(TY=ty,
              pair=wpr % 8 == 0 and sx % MT_BX == 0 and sx // MT_BX >= 16,
              tma=(sx * itemsize) % 16 == 0,
              shift=(wpr & (wpr - 1)) == 0,
              vector=sx % 4 == 0)


# sx, sy, sz, input dtype: sy and sz are not multiples of TY (partial tiles) and span 2+ tiles
SHAPES = [
  (2048, 11, 9, np.uint32),     # TY 8, paired mask kernel chosen by the row length
  (2049, 7, 5, np.uint8),       # TY 4, row pitch not 16-byte aligned, scalar expansion
  (2176, 5, 7, np.uint16),      # TY 4, 17 mask tiles per row: no pairs
  (4096, 7, 6, np.uint32),      # TY 4, shift split
  (8192, 5, 5, np.uint64),      # TY 4, shift split
  (8224, 5, 3, np.uint32),      # TY 2, divisions, no pairs
  (16384, 3, 5, np.uint16),     # TY 2, shift split
  (32768, 5, 3, np.uint8),      # TY 2, shift split
  (32800, 3, 5, np.uint32),     # TY 1
  (65536, 1, 7, np.uint16),     # TY 1, one row per plane: z faces only
  (131072, 3, 5, np.uint32),    # TY 1, the longest accepted row
]
CONTENTS = ["runs", "snakes", "noise", "blobs"]


def _ids(dtype, lab):
  """small ids 0..k -> dtype; u64 ids get distinct high words over one low word"""
  lab = np.asarray(lab, dtype=np.uint64)
  if np.dtype(dtype) == np.uint64:
    lab = np.where(lab == 0, 0, lab * np.uint64((1 << 32) + 7))
  return np.asfortranarray(lab.astype(dtype))


def volume(sx, sy, sz, dtype, content):
  rng = np.random.default_rng(sx + 7 * sy + 13 * sz + 101 * CONTENTS.index(content))
  shape = (sx, sy, sz)
  if content == "noise":  # dense: every tile exceeds TB_RCAP and unites in global memory
    lab = rng.integers(0, 3, size=shape)
  elif content == "runs":  # a few long x-runs per row, overlapping their neighbours'
    lab = np.zeros(shape, dtype=np.int64)
    for y in range(sy):
      for z in range(sz):
        cuts = np.sort(rng.choice(np.arange(1, sx), size=7, replace=False))
        vals = rng.integers(0, 3, size=8)
        lab[:, y, z] = np.repeat(vals, np.diff(np.concatenate([[0], cuts, [sx]])))
  elif content == "blobs":  # 64 x 1 x 1 blocks of 3 labels: short chains across many tile faces
    small = rng.integers(0, 4, size=((sx + 63) // 64, sy, sz))
    lab = np.repeat(small, 64, axis=0)[:sx]
  else:  # snakes: one-voxel paths that step to a neighbouring row every `seg` voxels along x,
    # walking the (y, z) rows back and forth, so each crosses y and z tile faces many times
    lab = np.zeros(shape, dtype=np.int64)
    cells = [(y if z % 2 == 0 else sy - 1 - y, z) for z in range(sz) for y in range(sy)]
    period = max(2 * len(cells) - 2, 1)
    cell_y, cell_z = np.array(cells).T
    x = np.arange(sx)
    for value, seg in ((1, 37), (2, 53)):
      k = (x // seg) % period
      k = np.where(k < len(cells), k, period - k)
      cy, cz = cell_y[k], cell_z[k]
      lab[x, cy, cz] = value
      lab[x[1:], cy[:-1], cz[:-1]] = value  # the step: (x-1, row) - (x, row) - (x, next row)
  return _ids(dtype, lab)


def runs_per_tile(vol, ty):
  """runs (maximal x-segments of one non-zero value) in each TY x TY tile of rows"""
  v = vol
  start = (v != 0) & np.concatenate([np.ones((1,) + v.shape[1:], bool), v[1:] != v[:-1]], axis=0)
  per_row = start.sum(axis=0)  # [sy, sz]
  sy, sz = per_row.shape
  ny, nz = -(-sy // ty), -(-sz // ty)
  pad = np.zeros((ny * ty, nz * ty), dtype=np.int64)
  pad[:sy, :sz] = per_row
  return pad.reshape(ny, ty, nz, ty).sum(axis=(1, 3))


def test_shape_table_covers_every_dispatch():
  seen = {k: set() for k in ("TY", "pair", "tma", "shift", "vector")}
  for sx, sy, sz, dtype in SHAPES:
    d = dispatch(sx, np.dtype(dtype).itemsize)
    for k, v in d.items():
      seen[k].add(v)
    assert sy % d["TY"] != 0 or sz % d["TY"] != 0 or d["TY"] == 1, (sx, sy, sz)
    assert -(-sy // d["TY"]) * -(-sz // d["TY"]) > 1, (sx, sy, sz)  # tile faces to merge
    assert sx * sy * sz * np.dtype(dtype).itemsize <= 16 << 20
  assert seen["TY"] == {8, 4, 2, 1}
  for k in ("pair", "tma", "shift", "vector"):
    assert seen[k] == {False, True}, k
  assert max(sx for sx, *_ in SHAPES) == MAX_SX
  assert dispatch(2048, 4)["pair"] and not dispatch(2176, 2)["pair"]


def test_contents_reach_both_sides_of_the_tile_run_limit():
  for sx, sy, sz, dtype in SHAPES:
    ty = dispatch(sx, np.dtype(dtype).itemsize)["TY"]
    most = {content: runs_per_tile(volume(sx, sy, sz, dtype, content), ty).max() for content in CONTENTS}
    assert most["noise"] > TB_RCAP, (sx, most)
    assert most["runs"] <= TB_RCAP and most["snakes"] <= TB_RCAP, (sx, most)


@pytest.mark.gpu
@pytest.mark.parametrize("content", CONTENTS)
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "x".join(str(v) for v in s[:3]) + "-" + np.dtype(s[3]).name)
def test_long_rows_match_oracle(ctx, oracle, shape, content):
  from igneous_b200 import cc3d
  sx, sy, sz, dtype = shape
  vol = volume(sx, sy, sz, dtype, content)
  want, n_want = oracle.connected_components(vol, return_N=True)
  for out_dtype in (np.uint32, np.uint64):
    got, n = cc3d.connected_components(vol, connectivity=6, out_dtype=out_dtype, return_N=True)
    assert n == n_want and got.dtype == np.dtype(out_dtype)
    assert np.array_equal(got, want.astype(out_dtype))
  if content == "runs":  # one independent check per shape (every TY)
    ref, n_ref = ccl6(vol)
    assert n_ref == n_want and np.array_equal(want, ref)
  threshold = 64
  assert np.array_equal(cc3d.dust(vol, threshold, connectivity=6, in_place=False), oracle.dust(vol, threshold))


@pytest.mark.gpu
def test_rows_past_the_limit_are_rejected_before_any_launch(ctx):
  from igneous_b200 import _shim
  sx = MAX_SX + 1
  d_in = ctx.alloc(sx * 2)
  d_out = ctx.alloc(sx * 8)
  ctx.memset(d_in, 1, sx * 2)
  ctx.sync()
  dims = (sx, 1, 1)
  n = c.c_uint64(0)
  before = ctx.launch_count()
  assert ctx.lib.ign_ccl6_dev(ctx.handle, _shim.ptr(d_in), _shim.IGN_U16, *dims, _shim.ptr(d_out), _shim.IGN_U32,
                              c.byref(n)) == IGN_ERR_OVERFLOW
  assert ctx.lib.ign_dust_dev(ctx.handle, _shim.ptr(d_in), _shim.IGN_U16, *dims, 5) == IGN_ERR_OVERFLOW
  v = c.c_void_p()
  assert ctx.lib.ign_ccl6_volume_begin_dev(ctx.handle, _shim.ptr(d_in), _shim.IGN_U16, *dims, None, None, None, None,
                                           c.byref(v), c.byref(n)) == IGN_ERR_OVERFLOW
  assert not v.value
  assert ctx.launch_count() == before
  # the longest accepted row on the same buffers
  assert ctx.lib.ign_ccl6_dev(ctx.handle, _shim.ptr(d_in), _shim.IGN_U16, MAX_SX, 1, 1, _shim.ptr(d_out), _shim.IGN_U32,
                              c.byref(n)) == 0
  assert n.value == 1
  got = np.empty(MAX_SX, dtype=np.uint32)
  ctx.d2h(got, d_out)
  ctx.sync()
  assert (got == 1).all()
