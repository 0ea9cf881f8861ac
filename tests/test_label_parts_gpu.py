"""ign_label_parts_dev against scipy.ndimage.label: the parts of each label under 6-, 18- and 26-connectivity,
renumbered by first voxel in F order, parts below the dust threshold dropped, with each kept part's voxel
count and box.  All four label dtypes with labels at the top of their range, shapes off the 32-voxel row
segments, extent-1 planes and single rows, labels touching diagonally, checkerboards, one label filling a
volume of long rows, each output alone and together, a short capacity, and refusals."""
import ctypes

import numpy as np
import pytest
from scipy import ndimage

from igneous_b200 import _shim

pytestmark = pytest.mark.gpu

DTYPES = [np.uint8, np.uint16, np.uint32, np.uint64]
RANK = {6: 1, 18: 2, 26: 3}


def expected(lab, connectivity, dust=0):
  """(parts, rows): parts[x, y, z] = the kept part 1..n, rows = {count, min x, y, z, max x, y, z} per kept part"""
  structure = ndimage.generate_binary_structure(3, RANK[connectivity])
  every = np.zeros(lab.shape, np.int64)
  for v in np.unique(lab):
    if v:
      part, k = ndimage.label(lab == v, structure=structure)
      every[part > 0] = part[part > 0] + every.max()
  ids, first = np.unique(every.ravel(order="F"), return_index=True)
  sizes = np.bincount(every.ravel())
  kept = [i for _, i in sorted(zip(first, ids)) if i and sizes[i] >= dust]
  table = np.zeros(every.max() + 1, np.uint32)
  table[kept] = np.arange(1, len(kept) + 1)
  parts = table[every]
  rows = [[int(sizes[i])] + [s.start for s in box] + [s.stop - 1 for s in box]
          for i, box in zip(kept, ndimage.find_objects(parts))]
  return parts, rows


def run(ctx, lab, connectivity, dust=0, parts=True, rows=True, capacity=None):
  """(*n, parts or None, the rows array of `capacity` rows or None)"""
  lab = np.asfortranarray(lab)
  d_lab = ctx.to_device(lab)
  d_parts = ctx.alloc(lab.size * 4) if parts else None
  cap = (lab.size if capacity is None else capacity) if rows else 0
  h_rows = np.full((max(cap, 1), 7), 0xA5A5A5A5, np.uint32) if rows else None
  n = ctypes.c_uint64(12345)
  _shim.check(ctx.lib.ign_label_parts_dev(ctx.handle, _shim.ptr(d_lab), _shim.dtype_code(lab.dtype), *lab.shape,
                                          connectivity, dust, _shim.ptr(d_parts) if parts else None,
                                          _shim.ptr(h_rows) if rows else None, cap, ctypes.byref(n)))
  got = ctx.to_host(d_parts, lab.shape, np.uint32) if parts else None
  ctx.sync()
  return int(n.value), got, h_rows


def check(ctx, lab, connectivity, dust=0):
  want_parts, want_rows = expected(lab, connectivity, dust)
  n, parts, rows = run(ctx, lab, connectivity, dust)
  assert n == len(want_rows)
  assert np.array_equal(parts, want_parts)
  assert rows[:n].tolist() == want_rows
  return n


def top_labels(dtype, shape, seed, k=3, background=0.4):
  """labels 0 and the k largest values of dtype (2^64 - 1 and below for uint64)"""
  rng = np.random.default_rng(seed)
  top = np.iinfo(dtype).max
  values = np.array([0] + [top - i for i in range(k)], dtype=dtype)
  p = [background] + [(1 - background) / k] * k
  return values[rng.choice(len(values), size=shape, p=p)]


@pytest.mark.parametrize("connectivity", [6, 18, 26])
@pytest.mark.parametrize("dtype", DTYPES)
def test_random_labels(ctx, dtype, connectivity):
  lab = top_labels(dtype, (37, 29, 11), seed=connectivity)
  assert check(ctx, lab, connectivity) > 100
  check(ctx, lab, connectivity, dust=4)


@pytest.mark.parametrize("connectivity", [6, 18, 26])
@pytest.mark.parametrize("shape", [(1, 45, 38), (45, 1, 38), (45, 38, 1), (70, 1, 1), (1, 70, 1), (1, 1, 70)])
def test_planes_and_rows(ctx, shape, connectivity):
  """extent-1 planes (18 is 8-connected there, as the border targets use it) and single rows"""
  lab = top_labels(np.uint32, shape, seed=sum(shape), k=2, background=0.3)
  assert check(ctx, lab, connectivity) > 1
  check(ctx, lab, connectivity, dust=3)


@pytest.mark.parametrize("connectivity", [6, 18, 26])
def test_diagonal_contacts(ctx, connectivity):
  """different labels never join; one label joins across an edge at 18 and 26, across a corner at 26 only"""
  lab = np.zeros((12, 10, 6), np.uint16)
  lab[1, 1, 1], lab[2, 2, 2] = 5, 7  # corner contact, two labels
  lab[5, 1, 1], lab[6, 2, 1] = 5, 7  # edge contact, two labels
  lab[1, 6, 1], lab[2, 7, 2] = 9, 9  # corner contact, one label
  lab[5, 6, 1], lab[6, 7, 1] = 9, 9  # edge contact, one label
  assert check(ctx, lab, connectivity) == {6: 8, 18: 7, 26: 6}[connectivity]


@pytest.mark.parametrize("connectivity", [6, 18, 26])
def test_checkerboards(ctx, connectivity):
  x, y, z = np.indices((33, 20, 7))
  parity = ((x + y + z) % 2 == 0).astype(np.uint8)  # neighbours across edges: one part at 18 and 26
  n = check(ctx, parity, connectivity)
  assert n == (1 if connectivity > 6 else parity.sum())
  corners = ((x % 2 == y % 2) & (y % 2 == z % 2)).astype(np.uint8)  # neighbours across corners only
  n = check(ctx, corners, connectivity)
  assert n == (1 if connectivity == 26 else corners.sum())
  two = np.where(parity, 3, 4).astype(np.uint32)  # every voxel set: as many parts as voxels at 6
  assert check(ctx, two, connectivity) == (2 if connectivity > 6 else two.size)


@pytest.mark.parametrize("connectivity", [6, 18, 26])
@pytest.mark.parametrize("shape", [(70001, 7, 3), (4099, 40, 9)])
def test_one_label_fills_long_rows(ctx, shape, connectivity):
  lab = np.full(shape, 2 ** 32 - 1, np.uint32)
  n, parts, rows = run(ctx, lab, connectivity)
  assert n == 1 and (parts == 1).all()
  assert rows[0].tolist() == [lab.size, 0, 0, 0, shape[0] - 1, shape[1] - 1, shape[2] - 1]
  n, parts, rows = run(ctx, lab, connectivity, dust=lab.size + 1)
  assert n == 0 and not parts.any()


def test_outputs_alone_together_and_short(ctx):
  lab = top_labels(np.uint16, (50, 33, 17), seed=7)
  for dust in (0, 1, 5):
    want_parts, want_rows = expected(lab, 26, dust)
    k = len(want_rows)
    assert k > 10
    n, parts, rows = run(ctx, lab, 26, dust)
    assert n == k and np.array_equal(parts, want_parts) and rows[:n].tolist() == want_rows
    n, parts, rows = run(ctx, lab, 26, dust, rows=False)
    assert n == k and np.array_equal(parts, want_parts) and rows is None
    n, parts, rows = run(ctx, lab, 26, dust, parts=False)
    assert n == k and parts is None and rows[:n].tolist() == want_rows
    n, _, rows = run(ctx, lab, 26, dust, parts=False, capacity=k)
    assert n == k and rows.tolist() == want_rows
    n, _, rows = run(ctx, lab, 26, dust, parts=False, capacity=k - 1)
    assert n == k and (rows == 0xA5A5A5A5).all()  # too short: untouched, the count still set
    n, _, _ = run(ctx, lab, 26, dust, parts=False, rows=False)
    assert n == k


def test_no_parts(ctx):
  n, parts, rows = run(ctx, np.zeros((40, 3, 5), np.uint64), 26)
  assert n == 0 and not parts.any() and (rows == 0xA5A5A5A5).all()


def _status(ctx, shape, dtype, connectivity, capacity=0, count=True):
  n = ctypes.c_uint64(7)
  s = ctx.lib.ign_label_parts_dev(ctx.handle, None, dtype, *shape, connectivity, 0, None, None, capacity,
                                  ctypes.byref(n) if count else None)
  return s, n.value, ctx.lib.ign_last_error().decode()


def test_refusals(ctx):
  """null buffers throughout: every refusal comes before anything is allocated or read"""
  U8, F32 = _shim.IGN_U8, _shim.IGN_F32
  assert _status(ctx, (0, 5, 5), U8, 26)[:2] == (0, 0)  # an empty volume needs no buffer
  for conn in (4, 0, 8, 27):
    s, n, msg = _status(ctx, (4, 4, 4), U8, conn)
    assert s == -2 and n == 0 and "connectivity %d" % conn in msg
  for dtype in (F32, 0, 9):
    s, n, msg = _status(ctx, (4, 4, 4), dtype, 26)
    assert s == -3 and n == 0 and "unsupported label dtype %d" % dtype in msg
  for shape in [(65535, 65537, 1), (1 << 16, 1 << 16, 1), (1 << 32, 1, 1), (1 << 31, 1 << 31, 1 << 31)]:
    s, n, msg = _status(ctx, shape, U8, 26)
    assert s == -3 and n == 0 and ("32-bit voxel indices" in msg or "2^32 or more" in msg), (shape, msg)
  s, n, msg = _status(ctx, (65535, 65537, 1), U8, 26)
  assert "32-bit voxel indices" in msg
  s, _, msg = _status(ctx, (4, 4, 4), U8, 26)
  assert s == -2 and "null buffer" in msg
  s, _, msg = _status(ctx, (4, 4, 4), U8, 26, count=False)
  assert s == -2 and "null count" in msg
