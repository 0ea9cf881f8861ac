"""The geodesic rule of DESIGN.md §5e restated with numpy and heapq (slow; small volumes only): a heap
Dijkstra whose every step is one np.float32 addition, the parent rule applied to its result, and the
TEASAR penalty field in float32.  Shares no code with oracle_geodesic/ or the kernels."""
import heapq
import itertools

import numpy as np

INF = np.float32(np.inf)


def neighbours(connectivity, anisotropy=None):
  """[((dx, dy, dz), float32 length or None)] in (dz, dy, dx) raster order, dx fastest"""
  out = []
  for dz, dy, dx in itertools.product((-1, 0, 1), repeat=3):
    if 0 < abs(dx) + abs(dy) + abs(dz) <= {6: 1, 18: 2, 26: 3}[connectivity]:
      w = None if anisotropy is None else np.float32(np.sqrt(sum(
        (float(np.float32(a)) * d) ** 2 for a, d in zip(anisotropy, (dx, dy, dz)))))
      out.append(((dx, dy, dz), w))
  return out


def geodesic(labels, sources, connectivity=26, anisotropy=(1, 1, 1), weights=None, parents=False):
  """labels: 3-D array; sources: voxel tuples.  Returns float32 dist, and uint32 parents (F-order index + 1)."""
  shape = labels.shape
  nb = neighbours(connectivity, None if weights is not None else anisotropy)
  dist = np.full(shape, INF, np.float32)
  heap = [(0.0, tuple(int(v) for v in s)) for s in sources]
  for _, s in heap:
    dist[s] = 0
  heapq.heapify(heap)

  def edges(p):
    for (d, w) in nb:
      q = tuple(a + b for a, b in zip(p, d))
      if all(0 <= c < n for c, n in zip(q, shape)) and labels[q] == labels[p] != 0:
        yield q, w

  while heap:
    d, p = heapq.heappop(heap)
    if np.float32(d) > dist[p]:
      continue
    for q, w in edges(p):
      cand = np.float32(d) + (np.float32(weights[q]) if weights is not None else w)
      if cand < dist[q]:
        dist[q] = cand
        heapq.heappush(heap, (float(cand), q))
  if not parents:
    return dist
  par = np.zeros(shape, np.uint32)
  index = lambda v: int(np.ravel_multi_index(v, shape, order="F"))
  srcs = {s for _, s in [(0, tuple(int(v) for v in s)) for s in sources]}
  for q in zip(*np.nonzero(np.isfinite(dist))):
    q = tuple(int(v) for v in q)
    if q in srcs:
      continue
    for p, w in edges(q):  # the neighbour set is symmetric; the weight is that of entering q
      step = np.float32(weights[q]) if weights is not None else w
      if dist[p] + step == dist[q] and (dist[p], index(p)) < (dist[q], index(q)):
        par[q] = index(p) + 1
        break
    else:
      raise ValueError("no parent under the rule at %r" % (q,))
  return dist, par


def pdrf(labels, dbf, daf, scale=100000, exponent=4):
  """scale * (1 - dbf / (1.01 max_l dbf))^exponent + daf / max_l daf in float32, one rounding per operation;
  0 on label 0 and where daf is +inf; the maxima over the label's finite values."""
  out = np.zeros(labels.shape, np.float32)
  for l in np.unique(labels[labels != 0]):
    m = (labels == l) & np.isfinite(daf)
    mb, ma = dbf[(labels == l) & np.isfinite(dbf)].max(), daf[m].max()
    t = np.float32(1) - dbf[m] / (np.float32(1.01) * np.float32(mb))
    p = t.copy()
    for _ in range(exponent - 1):
      p = p * t
    out[m] = np.float32(scale) * p + (daf[m] / np.float32(ma) if ma > 0 else np.float32(0))
  return out
