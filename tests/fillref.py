"""numpy / scipy transcription of the hole-filling rule (DESIGN.md "Hole filling"), written from
the rule's text and sharing no code with the library: components by scipy.ndimage.label per
value, contact counts by numpy, and the graph solve in plain Python (the merge rounds recompute
the whole region graph every round; the enclosure step tests every candidate separator by
removing it and searching from the outside, or on large graphs uses low-links, which the tests
check against the direct test)."""
from collections import defaultdict, deque

import numpy as np
from scipy import ndimage


def dilate(X):
  """Each 0 voxel with a non-zero voxel among its 26 in-box neighbours takes the most frequent
  non-zero neighbour label, ties to the smaller label (one Jacobi pass)."""
  X = np.asarray(X)
  pad = np.pad(X, 1)
  sx, sy, sz = X.shape
  nb = [pad[1 + dx:1 + dx + sx, 1 + dy:1 + dy + sy, 1 + dz:1 + dz + sz]
        for dz in (-1, 0, 1) for dy in (-1, 0, 1) for dx in (-1, 0, 1) if (dx, dy, dz) != (0, 0, 0)]
  idx = np.nonzero(X == 0)
  V = np.stack([n[idx] for n in nb], axis=1).astype(np.uint64)  # [M, 26]
  out = X.copy()
  if V.shape[0] == 0:
    return out
  cnt = np.zeros(V.shape, dtype=np.int64)
  for j in range(26):
    cnt += V == V[:, j:j + 1]
  cnt[V == 0] = 0
  best = cnt.max(axis=1)
  cand = np.where((cnt == best[:, None]) & (cnt > 0), V, np.uint64(np.iinfo(np.uint64).max))
  pick = cand.min(axis=1)
  has = best > 0
  out[tuple(i[has] for i in idx)] = pick[has].astype(X.dtype)
  return out


def components(X):
  """Maximal 6-connected sets of equal value, 0 included, numbered 1..N by first voxel in
  Fortran order.  Returns (int64 ids, N, value of every id [N+1])."""
  X = np.asarray(X)
  uniq, inv = np.unique(X, return_inverse=True)
  dense = inv.reshape(X.shape) + 1
  comp = np.zeros(X.shape, dtype=np.int64)
  nxt = 0
  for i, sl in enumerate(ndimage.find_objects(dense), start=1):
    if sl is None:
      continue
    lab, n = ndimage.label(dense[sl] == i)
    sub = comp[sl]
    sub[lab > 0] = lab[lab > 0] + nxt
    nxt += n
  flat = comp.ravel(order="F")
  ids, first = np.unique(flat, return_index=True)
  rank = np.zeros(nxt + 1, dtype=np.int64)
  rank[ids[np.argsort(first)]] = np.arange(1, len(ids) + 1)
  comp = rank[comp]
  value = np.zeros(len(ids) + 1, dtype=np.uint64)
  value[comp.ravel()] = X.ravel().astype(np.uint64)
  return comp, len(ids), value


def contacts(comp, axes=(0, 1, 2)):
  """{(a, b): faces} for a < b over face-adjacent voxel pairs, and {c: faces on the box
  surface} for the axes in `axes`."""
  w = defaultdict(int)
  for ax in range(3):
    if comp.shape[ax] < 2:
      continue
    a = np.take(comp, range(comp.shape[ax] - 1), axis=ax).ravel()
    b = np.take(comp, range(1, comp.shape[ax]), axis=ax).ravel()
    d = a != b
    lo, hi = np.minimum(a[d], b[d]), np.maximum(a[d], b[d])
    keys, n = np.unique(lo * (1 << 32) + hi, return_counts=True)
    for k, c in zip(keys.tolist(), n.tolist()):
      w[(k >> 32, k & 0xFFFFFFFF)] += c
  wo = defaultdict(int)
  for ax in axes:
    for side in {0, comp.shape[ax] - 1} if comp.shape[ax] > 1 else [0, 0]:
      ids, n = np.unique(np.take(comp, side, axis=ax), return_counts=True)
      for k, c in zip(ids.tolist(), n.tolist()):
        wo[k] += c
  return dict(w), dict(wo)


def merge(N, w, wo, p):
  """Merge-threshold rounds.  Returns the region root of every component [N+1]."""
  root = list(range(N + 1))

  def find(c):
    while root[c] != c:
      c = root[c]
    return c

  while True:
    W = defaultdict(int)   # region graph recomputed from the component contacts
    WO = defaultdict(int)
    for (a, b), c in w.items():
      ra, rb = find(a), find(b)
      if ra != rb:
        W[(ra, rb)] += c
        W[(rb, ra)] += c
    for a, c in wo.items():
      WO[find(a)] += c
    nbrs = defaultdict(dict)
    for (a, b), c in W.items():
      nbrs[a][b] = c
    area = {r: WO[r] + sum(nbrs[r].values()) for r in range(1, N + 1) if find(r) == r}
    target = {}
    for r in area:
      if WO[r] or not nbrs[r]:
        continue
      t = min(nbrs[r], key=lambda u: (-nbrs[r][u], u))
      if 100 * nbrs[r][t] >= (100 - p) * area[r]:
        target[r] = t
    if not target:
      return [find(c) for c in range(N + 1)]
    absorbed = []
    for r, t in target.items():
      if t not in target:
        absorbed.append((r, t))
      elif target[t] == r and (area[r], -r) < (area[t], -t):
        absorbed.append((r, t))
    if not absorbed:
      r = min(target, key=lambda u: (area[u], -u))
      absorbed.append((r, target[r]))
    for r, t in absorbed:
      root[r] = t


def _graph(edges, outside_touch):
  adj = defaultdict(set)
  for a, b in edges:
    adj[a].add(b)
    adj[b].add(a)
  for r in outside_touch:
    adj[0].add(r)
    adj[r].add(0)
  return adj


def fillers_bruteforce(regions, edges, outside_touch, value):
  """{region: filler}: S separates R when removing S leaves no path from R to the outside; the
  filler is the non-zero separator nearest the outside (breadth-first distance)."""
  adj = _graph(edges, outside_touch)

  def reach(removed):
    seen = {0}
    q = deque([0])
    while q:
      v = q.popleft()
      for u in adj[v]:
        if u != removed and u not in seen:
          seen.add(u)
          q.append(u)
    return seen

  dist = {0: 0}
  q = deque([0])
  while q:
    v = q.popleft()
    for u in adj[v]:
      if u not in dist:
        dist[u] = dist[v] + 1
        q.append(u)
  out = {}
  for s in regions:
    if value[s] == 0:
      continue
    for r in set(regions) - reach(s) - {s}:
      if r not in out or dist[s] < dist[out[r]]:
        out[r] = s
  return out


def fillers_lowlink(regions, edges, outside_touch, value):
  """The same by depth-first search from the outside with low-links: v cuts its DFS child c
  (and c's subtree) off from the outside exactly when low(c) >= disc(v)."""
  adj = {k: sorted(v) for k, v in _graph(edges, outside_touch).items()}
  disc, low, parent, order = {0: 0}, {0: 0}, {0: None}, []
  stack = [(0, iter(adj.get(0, [])))]
  while stack:
    v, it = stack[-1]
    u = next(it, None)
    if u is None:
      stack.pop()
      if parent[v] is not None:
        low[parent[v]] = min(low[parent[v]], low[v])
    elif u not in disc:
      parent[u] = v
      disc[u] = low[u] = len(disc)
      order.append(u)
      stack.append((u, iter(adj[u])))
    elif u != parent[v]:
      low[v] = min(low[v], disc[u])
  out = {}
  for c in order:
    v = parent[c]
    if v == 0:
      continue
    if v in out:
      out[c] = out[v]
    elif low[c] >= disc[v] and value[v] != 0:
      out[c] = v
  return out


BRUTE_MAX = 400  # region graphs up to this size are solved by the separator definition itself


def fill_pass(X, p, axes=(0, 1, 2)):
  """Steps 2-5 on one volume: the filled volume."""
  comp, N, value = components(X)
  w, wo = contacts(comp, axes)
  root = merge(N, w, wo, p) if p > 0 else list(range(N + 1))
  regions = sorted(set(root[1:]))
  redges = {(min(root[a], root[b]), max(root[a], root[b])) for a, b in w if root[a] != root[b]}
  touch = {root[a] for a, c in wo.items() if c}
  solver = fillers_bruteforce if len(regions) <= BRUTE_MAX else fillers_lowlink
  filler = solver(regions, redges, touch, value)
  table = np.zeros(N + 1, dtype=np.uint64)
  for c in range(1, N + 1):
    r = root[c]
    table[c] = value[filler[r]] if r in filler else (value[r] if value[r] != 0 else value[c])
  return table[comp].astype(X.dtype)


def fill_holes(X0, fix_borders=False, p=0):
  """(filled, holes) of the rule; p = 100 - merge threshold in percent."""
  X0 = np.asarray(X0)
  cur = X0.copy()
  if fix_borders:
    done = set()
    for ax in range(3):
      for idx in (0, X0.shape[ax] - 1):
        if (ax, idx) in done:
          continue
        done.add((ax, idx))
        sl = [slice(None)] * 3
        sl[ax] = idx
        plane = cur[tuple(sl)][:, :, None]   # the other two axes in x, y, z order
        cur[tuple(sl)] = fill_pass(plane, p, axes=(0, 1))[:, :, 0]
  filled = fill_pass(cur, p)
  holes = np.where((filled != X0) & (X0 != 0), X0, 0).astype(X0.dtype)
  return filled, holes


def fill_level(X, level):
  """MeshTask(fill_holes=level) on a renumbered block: (filled, holes)."""
  X0 = dilate(X) if level >= 3 else np.asarray(X)
  return fill_holes(X0, fix_borders=level >= 2, p=max(0, level - 3))


# ------------------------------------------------------------------ test volumes
def shell(X, lo, hi, label, t=2):
  """Cube [lo, hi)^3 of `label` with a hollow [lo+t, hi-t)^3 of 0."""
  X[lo:hi, lo:hi, lo:hi] = label
  X[lo + t:hi - t, lo + t:hi - t, lo + t:hi - t] = 0
  return X


def kats():
  """Hand-built volumes, name -> uint32 volume."""
  out = {}
  out["hollow_cell"] = shell(np.zeros((16, 16, 16), np.uint32), 2, 14, 3)
  X = shell(np.zeros((16, 16, 16), np.uint32), 2, 14, 3)
  X[7:9, 7:9, 7:9] = 7
  out["organelle_floating"] = X
  X = shell(np.zeros((16, 16, 16), np.uint32), 2, 14, 3)
  X[4:6, 6:9, 6:9] = 7                       # against the cavity wall at x = 3
  out["organelle_wall"] = X
  X = shell(np.zeros((16, 16, 16), np.uint32), 2, 14, 3)
  X[5:8, 6:9, 6:9] = 7
  X[8:10, 6:9, 6:9] = 8
  out["organelles_touching"] = X
  X = shell(np.zeros((24, 24, 24), np.uint32), 1, 23, 2)
  shell(X, 5, 19, 4)
  X[9:15, 9:15, 9:15] = 6
  out["nested_three"] = X
  X = np.zeros((14, 16, 16), np.uint32)      # cell cut by the x = 0 face, cavity open to it
  X[0:12, 2:14, 2:14] = 5
  X[0:10, 4:12, 4:12] = 0
  out["open_to_face"] = X
  out["threshold"] = threshold_kat()
  out["cycle2"] = cycle2_kat()
  out["triangle"] = triangle_kat()
  return out


def threshold_kat(plug=11):
  """Hollow cell against three box faces whose far wall holds a plug of another label reaching
  the outside: the cavity is not enclosed by one region, so it is filled only when the merge
  threshold lets it join the wall (after the dilation of level >= 3: at level 13, not 12)."""
  X = shell(np.zeros((24, 24, 24), np.uint32), 0, 20, 3)
  X[18:20, 4:4 + plug, 4:4 + plug] = 9
  return X


def cycle2_kat():
  """Two 1-voxel slabs A | B, each the other's largest neighbour, in a volume of unique
  single-voxel labels: at merge_threshold 0.40 both are candidates pointing at each other."""
  X = np.arange(1, 12 * 12 * 12 + 1, dtype=np.uint32).reshape((12, 12, 12), order="F") + 100
  X[2, 1:11, 1:11] = 1
  X[3, 1:11, 1:11] = 2
  return X


def triangle_kat():
  """Three bars with equal pairwise contacts: the nearest thing to a 3-cycle of candidates,
  which symmetric contact counts cannot produce (each picks the lower root on a tie)."""
  X = np.arange(1, 12 * 12 * 12 + 1, dtype=np.uint32).reshape((12, 12, 12), order="F") + 100
  X[2:4, 2:4, 1:11] = 1
  X[4:6, 2:4, 1:11] = 2
  X[2:4, 4:6, 1:11] = 3
  X[4:6, 4:6, 1:11] = 3
  return X


def random_volume(shape, seed, pitch=12):
  """Jittered-grid Voronoi segmentation with stamped solid spheres and hollow shells (holding
  a smaller sphere) of fresh labels; every fourth stamp may touch the box faces."""
  from oracle.oracle import synth_seg  # input generation only (the C build of synth_seg_np)
  rng = np.random.default_rng(seed)
  X = synth_seg(shape, pitch=pitch, num_ids=1 << 16, seed=seed).astype(np.uint32)
  nxt = int(X.max()) + 1
  for k in range(min(48, max(4, int(np.prod(shape)) // 8000))):
    r = float(rng.uniform(2.5, max(3.5, min(min(shape) / 5, 14))))
    c = [rng.integers(0, s) if k % 4 == 1 else rng.integers(min(int(r) + 1, s // 2), max(s - int(r) - 1, s // 2 + 1))
         for s in shape]
    box = tuple(slice(max(0, int(ci - r) - 1), min(s, int(ci + r) + 2)) for ci, s in zip(c, shape))
    g = np.meshgrid(*[np.arange(b.start, b.stop) for b in box], indexing="ij")
    d = np.sqrt(sum((gi - ci) ** 2 for gi, ci in zip(g, c)))
    sub = X[box]
    if k % 2:
      sub[d < r] = nxt
    else:
      sub[(d < r) & (d >= r - 1.5)] = nxt
      sub[d < r - 1.5] = 0
      sub[d < (r - 1.5) / 2] = nxt + 1
    nxt += 2
  return np.asfortranarray(X)


def single_component_labels(X):
  """Every non-zero 6-connected component gets its own label (0 stays 0)."""
  comp, _, _ = components(X)
  return np.where(X == 0, 0, comp).astype(np.uint32)


def scipy_fill(X0):
  """filled by scipy.ndimage.binary_fill_holes per label; where fills overlap, the label with
  the larger filled set wins (fills of single-component labels nest)."""
  out = np.asarray(X0).copy()
  size = np.full(out.shape, -1, dtype=np.int64)
  for L in np.unique(X0):
    if L == 0:
      continue
    m = ndimage.binary_fill_holes(X0 == L)
    n = int(m.sum())
    win = m & (n > size)
    out[win] = L
    size[win] = n
  return out
