"""The skeleton merge and postprocess rule of DESIGN.md §5h restated with numpy, sets and sorted lists (slow;
small skeletons only).  Shares no code with oracle_skeleton/ or the kernels.

A skeleton here is a tuple (vertices (N, 3) float32, edges (E, 2) uint32, radii (N,) float32, vertex_types
(N,) uint8).  A crop box is None or (lo xyz, hi xyz) as float64; see crop_box."""
import numpy as np

f32, f64 = np.float32, np.float64


def empty():
  return (np.zeros((0, 3), f32), np.zeros((0, 2), np.uint32), np.zeros(0, f32), np.zeros(0, np.uint8))


def crop_box(lo, hi, crop, resolution):
  """the fragment box (lo, hi) shrunk by crop * resolution on every side, or None when crop <= 0 or the
  shrunk box has volume <= 0 (the fragment stays whole)"""
  if crop <= 0:
    return None
  r = np.asarray(resolution, f64) * crop
  a, b = np.asarray(lo, f64) + r, np.asarray(hi, f64) - r
  if np.prod(b - a) <= 0:
    return None
  return a, b


def crop(skel, box):
  v, e, r, t = skel
  if box is None:
    return skel
  keep = np.all((box[0] <= v.astype(f64)) & (v.astype(f64) <= box[1]), axis=1)
  new = np.cumsum(keep) - 1
  ek = keep[e[:, 0]] & keep[e[:, 1]] if len(e) else np.zeros(0, bool)
  return v[keep], new[e[ek]].astype(np.uint32).reshape(-1, 2), r[keep], t[keep]


def edge_lengths(v, e):
  """float32, (dx*dx + dy*dy) + dz*dz rounded after every operation, then sqrt"""
  if len(e) == 0:
    return np.zeros(0, f32)
  d = v[e[:, 1]] - v[e[:, 0]]
  return np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])


def cable_length(skel):
  return float(np.sum(edge_lengths(skel[0], skel[1]).astype(f64)))


def dist64(v, a, b):
  d = v[a].astype(f64) - v[b].astype(f64)
  return float(np.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]))


def consolidate(skel):
  v, e, r, t = skel
  if not np.all(np.isfinite(v)):
    raise ValueError("non-finite vertex")
  if len(v) == 0:
    return empty()
  k = v + f32(0.0)  # -0.0 -> 0.0
  order = np.lexsort((k[:, 2], k[:, 1], k[:, 0]))  # stable: the head of each run is the first occurrence
  ks = k[order]
  head = np.ones(len(v), bool)
  head[1:] = np.any(ks[1:] != ks[:-1], axis=1)
  uid = np.empty(len(v), np.int64)
  uid[order] = np.cumsum(head) - 1
  first = order[head]
  pairs = set()
  for a, b in uid[e.astype(np.int64)].tolist() if len(e) else []:
    if a != b:
      pairs.add((min(a, b), max(a, b)))
  if not pairs:
    return empty()
  pairs = sorted(pairs)
  used = sorted({x for p in pairs for x in p})
  new = {u: i for i, u in enumerate(used)}
  src = first[used]
  edges = np.array([(new[a], new[b]) for a, b in pairs], np.uint32)
  return v[src].copy(), edges, r[src].copy(), t[src].copy()


def fuse(frags, boxes):
  """crop each fragment, concatenate in the order given and consolidate"""
  parts = [crop(f, b) for f, b in zip(frags, boxes)]
  if not parts:
    return empty()
  base = np.cumsum([0] + [len(p[0]) for p in parts])
  v = np.concatenate([p[0] for p in parts]).reshape(-1, 3).astype(f32)
  e = np.concatenate([p[1].astype(np.int64) + base[i] for i, p in enumerate(parts)]).reshape(-1, 2)
  r = np.concatenate([p[2] for p in parts]).astype(f32)
  t = np.concatenate([p[3] for p in parts]).astype(np.uint8)
  return consolidate((v, e.astype(np.uint32), r, t))


class _UF:
  def __init__(self, n):
    self.p = list(range(n))

  def find(self, x):
    while self.p[x] != x:
      self.p[x] = self.p[self.p[x]]
      x = self.p[x]
    return x

  def union(self, a, b):
    a, b = self.find(a), self.find(b)
    if a == b:
      return False
    self.p[max(a, b)] = min(a, b)
    return True


def _length(v, a, b):
  return float(edge_lengths(v, np.array([[a, b]], np.int64))[0])


def _degrees(n, E):
  deg = [0] * n
  for a, b in E:
    deg[a] += 1
    deg[b] += 1
  return deg


def _components(n, E):
  uf = _UF(n)
  for a, b in E:
    uf.union(a, b)
  return [uf.find(x) for x in range(n)]


def _dust(v, E, threshold):
  comp = _components(len(v), E)
  cable = {}
  for a, b in E:
    cable[comp[a]] = cable.get(comp[a], 0.0) + _length(v, a, b)
  return {(a, b) for a, b in E if not cable[comp[a]] < threshold}


def _tree_path(n, tree, a, b):
  adj = [[] for _ in range(n)]
  for x, y in tree:
    adj[x].append(y)
    adj[y].append(x)
  prev = {a: None}
  todo = [a]
  while todo:
    x = todo.pop()
    for y in adj[x]:
      if y not in prev:
        prev[y] = x
        todo.append(y)
  path = [b]
  while path[-1] != a:
    path.append(prev[path[-1]])
  return path[::-1]


def _loops(v, E):
  n = len(v)
  E = set(E)
  while True:
    uf, tree, cyc = _UF(n), [], None
    for a, b in sorted(E):
      if not uf.union(a, b):
        cyc = (a, b)
        break
      tree.append((a, b))
    if cyc is None:
      return E
    path = _tree_path(n, tree, *cyc)
    k = len(path)
    ring = [(min(path[i], path[(i + 1) % k]), max(path[i], path[(i + 1) % k])) for i in range(k)]
    deg = _degrees(n, E)
    br = [i for i, x in enumerate(path) if deg[x] >= 3]
    if len(br) == 0:
      E -= set(ring)
    elif len(br) == 1:
      b = path[br[0]]
      far = max(path, key=lambda x: (dist64(v, b, x), -x))
      E -= set(ring)
      E.add((min(b, far), max(b, far)))
    elif len(br) == 2:
      i, j = br
      arc1 = ring[i:j]                       # path[i] .. path[j]
      arc2 = ring[j:] + ring[:i]             # path[j] .. path[k - 1], path[0] .. path[i]
      in1, in2 = path[i + 1:j], path[j + 1:] + path[:i]
      if len(arc1) != len(arc2):
        drop = arc2 if len(arc1) < len(arc2) else arc1
      else:
        drop = arc2 if min(in1) < min(in2) else arc1
      E -= set(drop)
    else:
      E.discard(max(ring, key=lambda p: (_length(v, *p), -p[0], -p[1])))


def _connect(v, r, E):
  n = len(v)
  deg = _degrees(n, E)
  alive = [x for x in range(n) if deg[x]]
  comp = _components(n, E)
  cand = []
  for i, a in enumerate(alive):
    for b in alive[i + 1:]:
      if comp[a] != comp[b]:
        d = dist64(v, a, b)
        if d < f64(r[a]) + f64(r[b]):
          cand.append((d, a, b))
  uf = _UF(n)
  for a, b in E:
    uf.union(a, b)
  E = set(E)
  for d, a, b in sorted(cand):
    if uf.union(a, b):
      E.add((a, b))
  return E


def _ticks(v, E, threshold):
  n = len(v)
  E = set(E)
  comp = _components(n, E)
  deg = _degrees(n, E)
  for c in sorted({comp[x] for x in range(n) if deg[x]}):
    while True:
      deg = _degrees(n, E)
      if not any(deg[x] >= 3 and comp[x] == c for x in range(n)):
        break
      adj = [[] for _ in range(n)]
      for a, b in E:
        adj[a].append(b)
        adj[b].append(a)
      best = None
      for leaf in range(n):
        if comp[leaf] != c or deg[leaf] != 1:
          continue
        prev, cur, length, path = None, leaf, 0.0, []
        while cur == leaf or deg[cur] < 3:
          nxt = [y for y in adj[cur] if y != prev][0]
          length += _length(v, min(cur, nxt), max(cur, nxt))
          path.append((min(cur, nxt), max(cur, nxt)))
          prev, cur = cur, nxt
        if best is None or (length, leaf) < best[:2]:
          best = (length, leaf, path)
      if not best[0] < threshold:
        break
      E -= set(best[2])
  return E


def postprocess(skel, dust_threshold=1500, tick_threshold=3000):
  v, e, r, t = consolidate(skel)
  E = {(int(a), int(b)) for a, b in e.tolist()}
  if dust_threshold > 0:
    E = _dust(v, E, dust_threshold)
  E = _loops(v, E)
  E = _connect(v, r, E)
  if tick_threshold > 0:
    E = _ticks(v, E, tick_threshold)
  return consolidate((v, np.array(sorted(E), np.uint32).reshape(-1, 2), r, t))


def merge(frags, boxes=None, dust_threshold=4000, tick_threshold=6000, max_cable_length=None):
  """one label: fuse its fragments, then postprocess unless the fused cable length exceeds max_cable_length"""
  fused = fuse(frags, boxes if boxes is not None else [None] * len(frags))
  if max_cable_length is not None and cable_length(fused) > max_cable_length:
    return fused
  return postprocess(fused, dust_threshold, tick_threshold)


def encode(skel, vertex_types=True):
  """the neuroglancer precomputed skeleton: nv, ne, vertices, edges, radius[, vertex_types]"""
  v, e, r, t = skel
  parts = [np.array([len(v), len(e)], "<u4").tobytes(), v.astype("<f4").tobytes(), e.astype("<u4").tobytes(),
           r.astype("<f4").tobytes()]
  if vertex_types:
    parts.append(t.astype(np.uint8).tobytes())
  return b"".join(parts)
