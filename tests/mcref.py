"""Plain numpy restatement of the mesher's marching cubes and weld order, for the GPU tests.

Triangles are ordered by (dense label, cube raster index, t), vertices are the unique
(dense label, z2, y2, x2) points of the half-voxel lattice, and faces index the vertices of their
own label.  Dense labels are numbered in order of first appearance, x fastest."""
import os
import re

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# Bourke's corner numbering: corner k -> (dx, dy, dz)
CORNERS = np.array([(0, 0, 0), (1, 0, 0), (1, 1, 0), (0, 1, 0), (0, 0, 1), (1, 0, 1), (1, 1, 1), (0, 1, 1)])
# edge -> midpoint on the half-voxel lattice of the cube (the device's c_edge_mid)
EDGE_MID = np.array([(1, 0, 0), (2, 1, 0), (1, 2, 0), (0, 1, 0), (1, 0, 2), (2, 1, 2), (1, 2, 2), (0, 1, 2),
                     (0, 0, 1), (2, 0, 1), (2, 2, 1), (0, 2, 1)])


def edge_corners():
  """The two corners of each edge, derived from its midpoint: a midpoint coordinate of 1 spans the
  axis, 0 and 2 sit at corner offsets 0 and 1."""
  out = []
  for mid in EDGE_MID:
    ends = [tuple(0 if m == 0 else 1 if m == 2 else s for m, s in zip(mid, (side,) * 3)) for side in (0, 1)]
    out.append(tuple(int(np.flatnonzero((CORNERS == e).all(1))[0]) for e in ends))
  return out


def mc_tables():
  """(tri[256][16], ntri[256]) parsed from igneous_b200/csrc/mc_table.h."""
  text = open(os.path.join(ROOT, "igneous_b200", "csrc", "mc_table.h")).read()

  def block(name):
    body = text[text.index(name):]
    body = body[body.index("=") + 1:body.index(";")]
    return np.array([int(v) for v in re.findall(r"-?\d+", body)])

  return block("mc_tri_table").reshape(256, 16), block("mc_tri_count")


def mesh(data):
  """Dense ids, per-label offsets, vertices (half-voxel coordinates, (x2, y2, z2)) and local faces
  of a Fortran-order (sx, sy, sz) label volume."""
  tri, ntri = mc_tables()
  flat = np.asarray(data).ravel(order="F")
  uniq, first = np.unique(flat, return_index=True)
  order = np.argsort(first)
  ids = uniq[order]
  dense_of = np.empty(len(uniq), dtype=np.int64)
  dense_of[order] = np.arange(len(uniq))
  dense = dense_of[np.searchsorted(uniq, flat)]
  zero = np.flatnonzero(ids == 0)
  # label value 0 is background: it has no dense id of its own
  if len(zero):
    z0 = zero[0]
    ids = np.delete(ids, z0)
    dense = np.where(dense == z0, 0, np.where(dense > z0, dense, dense + 1))
  else:
    dense = dense + 1
  K = len(ids)
  sx, sy, sz = data.shape
  lab = dense.reshape(sz, sy, sx)  # [z, y, x]
  cx, cy, cz = sx - 1, sy - 1, sz - 1
  c = np.stack([lab[dz:dz + cz, dy:dy + cy, dx:dx + cx].ravel() for dx, dy, dz in CORNERS])
  cube = np.arange(cx * cy * cz, dtype=np.int64)
  L_all, cube_all, case_all = [], [], []
  for k in range(8):
    L = c[k]
    keep = L != 0
    for j in range(k):
      keep &= c[j] != L
    case = sum((c[j] == L).astype(np.int64) << j for j in range(8))
    L_all.append(L[keep]); cube_all.append(cube[keep]); case_all.append(case[keep])
  L = np.concatenate(L_all); cb = np.concatenate(cube_all); cs = np.concatenate(case_all)
  n = ntri[cs]
  L = np.repeat(L, n); cb = np.repeat(cb, n); cs = np.repeat(cs, n)
  t = np.arange(len(L)) - np.repeat(np.cumsum(n) - n, n)
  o = np.lexsort((t, cb, L))
  L, cb, cs, t = L[o], cb[o], cs[o], t[o]
  T = len(L)
  x, y, z = cb % cx, (cb // cx) % cy, cb // (cx * cy)
  keys = np.empty((T, 3), dtype=np.int64)
  for v in range(3):
    e = tri[cs, 3 * t + (2 - v)]
    mid = EDGE_MID[e]
    x2, y2, z2 = 2 * x + mid[:, 0], 2 * y + mid[:, 1], 2 * z + mid[:, 2]
    keys[:, v] = (L << 33) | (z2 << 22) | (y2 << 11) | x2
  ukeys, inv = np.unique(keys.ravel(), return_inverse=True)
  vlab = ukeys >> 33
  tri_off = np.searchsorted(L, np.arange(K + 2))
  vert_off = np.searchsorted(vlab, np.arange(K + 2))
  faces = inv.reshape(T, 3) - vert_off[L][:, None]
  verts = np.stack([ukeys & 2047, (ukeys >> 11) & 2047, (ukeys >> 22) & 2047], 1)
  return ids, tri_off, vert_off, verts, faces
