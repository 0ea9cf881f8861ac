"""The cross-sectional area rule of DESIGN.md §5i restated in numpy / scipy -- a checker that shares no code
with oracle_xsection/xsection_oracle.c.

Normals: scipy's breadth-first search gives the hop distances; each vertex's path is found by walking down
from it, child by child, to the shallowest leaf of its subtree.  Sections: the cut test over the whole array
at once, scipy.ndimage.label with 26-connectivity for the part through the vertex's voxel, and each voxel's
area as the polygon where the plane crosses its box: the plane's crossings of the box's twelve edges, sorted
by angle about their centroid, summed by the shoelace formula."""
import numpy as np
from scipy import ndimage
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import shortest_path


def _hops(graph, src):
  return shortest_path(graph, unweighted=True, indices=src, directed=False)


def normals(voxels, edges, anisotropy, window):
  """float64 (V, 3): the normal of every vertex by the rule of §5i"""
  vox = np.asarray(voxels, np.int64).reshape(-1, 3)
  V = len(vox)
  e = np.asarray(edges, np.int64).reshape(-1, 2)
  e = e[e[:, 0] != e[:, 1]]
  a = np.asarray(anisotropy, np.float64)
  out = np.zeros((V, 3), np.float64)
  if V == 0:
    return out
  graph = coo_matrix((np.ones(len(e)), (e[:, 0], e[:, 1])), shape=(V, V)).tocsr()
  nbrs = [[] for _ in range(V)]
  for u, w in e.tolist():
    nbrs[u].append(w)
    nbrs[w].append(u)
  seen = np.zeros(V, bool)
  for s in range(V):
    if seen[s]:
      continue
    hs = _hops(graph, s)
    comp = np.nonzero(np.isfinite(hs))[0]
    seen[comp] = True
    if len(comp) == 1:
      continue
    far = hs[comp].max()
    r = int(comp[hs[comp] == far].min())
    depth = _hops(graph, r)
    parent = {int(u): min(x for x in nbrs[u] if depth[x] == depth[u] - 1) for u in comp if u != r}
    children = {int(u): [] for u in comp}
    for u, p in parent.items():
      children[p].append(u)

    best = {}  # (depth, index) of the shallowest leaf below each vertex
    for u in sorted(comp.tolist(), key=lambda u: -depth[u]):  # children before parents
      best[u] = min(best[c] for c in children[u]) if children[u] else (depth[u], u)
    for v in comp.tolist():
      leaf = best[v][1]
      path = [leaf]
      while path[-1] != r:
        path.append(parent[path[-1]])
      steps = [vox[path[p]] - vox[path[p + 1]] for p in range(len(path) - 1)]
      steps.append(steps[-1])  # the root takes the step of its child on the path
      padded = len(steps)
      i = path.index(v)
      lo = i - window // 2
      total = np.zeros(3, np.int64)
      for j in range(lo, lo + window):
        m = j % (2 * padded)
        total += steps[m if m < padded else 2 * padded - 1 - m]
      if not total.any():
        total = steps[i]
      out[v] = total * a
  return out


def _corners():
  return np.array([[x, y, z] for z in (-1, 1) for y in (-1, 1) for x in (-1, 1)], np.float64)


# the twelve edges of a box as pairs of corner indices of _corners()
_EDGES = [(0, 1), (2, 3), (4, 5), (6, 7), (0, 2), (1, 3), (4, 6), (5, 7), (0, 4), (1, 5), (2, 6), (3, 7)]


def plane_box_area(normal, offsets, anisotropy):
  """float64 (K,): the area of {y : n.y = 0} inside the box of half-extents a/2 centred at each offset (K, 3)
  (physical units), by polygon clipping"""
  n = np.asarray(normal, np.float64)
  off = np.asarray(offsets, np.float64).reshape(-1, 3)
  half = np.asarray(anisotropy, np.float64) / 2
  corners = off[:, None, :] + _corners()[None] * half  # (K, 8, 3)
  val = corners @ n  # signed plane value at each corner
  pts = np.full((len(off), 12, 3), np.nan)
  for k, (i, j) in enumerate(_EDGES):
    vi, vj = val[:, i], val[:, j]
    cross = (vi * vj <= 0) & (vi != vj)
    t = np.where(cross, vi / np.where(vi != vj, vi - vj, 1.0), np.nan)
    pts[:, k] = corners[:, i] + t[:, None] * (corners[:, j] - corners[:, i])
  u = np.cross(n, [1.0, 0, 0] if abs(n[0]) < 0.9 * np.linalg.norm(n) else [0, 1.0, 0])
  u /= np.linalg.norm(u)
  w = np.cross(n / np.linalg.norm(n), u)
  px, py = pts @ u, pts @ w  # (K, 12), nan where an edge is not crossed
  cx, cy = np.nanmean(px, axis=1, keepdims=True), np.nanmean(py, axis=1, keepdims=True)
  ang = np.arctan2(py - cy, px - cx)
  order = np.argsort(np.where(np.isnan(ang), np.inf, ang), axis=1)
  px, py = np.take_along_axis(px, order, 1), np.take_along_axis(py, order, 1)
  px = np.where(np.isnan(px), px[:, :1], px)  # pad with the first point: the polygon closes itself
  py = np.where(np.isnan(py), py[:, :1], py)
  return 0.5 * np.abs(np.sum(px * np.roll(py, -1, 1) - np.roll(px, -1, 1) * py, axis=1))


def section(labels, voxel, label, normal, anisotropy):
  """(float64 area, contacts, boolean mask of the section) of one point by the rule of §5i"""
  lab = np.asarray(labels)
  n = np.asarray(normal, np.float64)
  a = np.asarray(anisotropy, np.float64)
  c = np.asarray(voxel, np.int64)
  if not n.any() or lab[tuple(c)] != label:
    return 0.0, 0, np.zeros(lab.shape, bool)
  g = np.indices(lab.shape)
  d = [((g[i] - c[i]) * a[i]) for i in range(3)]
  s = (n[0] * d[0] + n[1] * d[1]) + n[2] * d[2]
  h = 0.5 * ((abs(n[0]) * a[0] + abs(n[1]) * a[1]) + abs(n[2]) * a[2])
  cut = (np.abs(s) < h) & (lab == label)
  parts, _ = ndimage.label(cut, structure=np.ones((3, 3, 3), bool))
  mask = parts == parts[tuple(c)]
  q = np.argwhere(mask)
  area = float(np.sum(plane_box_area(n, (q - c) * a, a)))
  contacts = 0
  for axis in range(3):
    if q[:, axis].min() == 0:
      contacts |= 1 << (2 * axis)
    if q[:, axis].max() == lab.shape[axis] - 1:
      contacts |= 2 << (2 * axis)
  return area, contacts, mask


def sections(labels, voxels, point_labels, normals_, anisotropy):
  """(float32 area, uint8 contacts) per point"""
  out_a, out_c = [], []
  for c, l, n in zip(np.asarray(voxels).reshape(-1, 3), point_labels, np.asarray(normals_).reshape(-1, 3)):
    ar, co, _ = section(labels, c, l, n, anisotropy)
    out_a.append(ar)
    out_c.append(co)
  return np.array(out_a, np.float32), np.array(out_c, np.uint8)
