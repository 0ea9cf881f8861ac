"""The TEASAR path loop of DESIGN.md §5f restated with heapq on top of tests/geodesicref.py (slow; small
volumes only), and the whole skeletonize rule around it: objects by scipy.ndimage.label, the fields, the
loop and the skeleton.  Shares no code with oracle_geodesic/ or the kernels; the pipeline takes the
geodesic solver and the loop as arguments so the C checkers can stand in for the restatements."""
import numpy as np
from scipy import ndimage

import edtref
import geodesicref

NONE = 0xFFFFFFFF


def _ravel(v, shape):
  return int(np.ravel_multi_index(v, shape, order="F"))


def _unravel(i, shape):
  return tuple(int(c) for c in np.unravel_index(int(i), shape, order="F"))


def loop(objects, k, anisotropy, dbf, daf, pdrf, roots, parents=None, before=(), after=(), scale=10.0, const=10.0,
         max_paths=None):
  """uint32 next (F order, NONE off the skeleton, the voxel itself at a root); arguments as the C checker"""
  shape = objects.shape
  nxt = np.full(shape, NONE, np.uint32)
  f32 = np.float32
  a = [f32(v) for v in anisotropy]
  for o in range(1, k + 1):
    mask = objects == o
    valid = mask.copy()
    lo, hi = [int(c.min()) for c in np.nonzero(mask)], [int(c.max()) for c in np.nonzero(mask)]
    root = _unravel(roots[o], shape)
    nxt[root] = roots[o]
    lab = mask.astype(np.uint8)

    def trace(t):
      D = None
      if parents is None:
        S = [tuple(int(c) for c in v) for v in zip(*np.nonzero(mask & (nxt != NONE)))]
        D = geodesicref.geodesic(lab, S, 26, weights=np.where(mask, pdrf, 0))
      q = _unravel(t, shape)
      while True:
        r = f32(f32(f32(scale) * dbf[q]) + f32(const))
        h = [int(np.floor(f32(r / ai))) for ai in a]
        box = tuple(slice(max(q[i] - h[i], lo[i]), min(q[i] + h[i], hi[i]) + 1) for i in range(3))
        valid[box] &= ~mask[box]
        if nxt[q] != NONE:
          return
        p = None
        if parents is not None:
          if parents[q]:
            p = _unravel(int(parents[q]) - 1, shape)
        else:
          for (d, _) in geodesicref.neighbours(26):
            c = tuple(x + dx for x, dx in zip(q, d))
            if all(0 <= ci < si for ci, si in zip(c, shape)) and mask[c]:
              if D[c] + pdrf[q] == D[q] and (D[c], _ravel(c, shape)) < (D[q], _ravel(q, shape)):
                p = c
                break
        if p is None:
          raise ValueError("no next voxel at %r" % (q,))
        nxt[q] = _ravel(p, shape)
        q = p

    mine = [int(t) for t in before if objects.reshape(-1, order="F")[int(t)] == o]
    for t in mine[:-1]:
      trace(t)
    paths = 0
    while max_paths is None or paths < max_paths:
      cand = np.where(valid, daf, -np.inf).reshape(-1, order="F")
      if not np.isfinite(cand.max()):
        break
      trace(int(np.argmax(cand)))  # the first of the greatest: the lowest F-order index
      paths += 1
    for t in after:
      if objects.reshape(-1, order="F")[int(t)] == o:
        trace(int(t))
  return nxt


def _crops(vol, k):
  """[(id, slices)] of ids 1..k of an integer volume, by scipy.ndimage.find_objects"""
  return [(i + 1, sl) for i, sl in enumerate(ndimage.find_objects(vol, max_label=k)) if sl is not None]


def _first_f(mask):
  """F-order index within the crop of the first True voxel (crop and volume F orders agree)"""
  return int(np.flatnonzero(mask.reshape(-1, order="F"))[0])


def parts_of(labels, structure, dust_threshold=0, keep=None):
  """ids 1..k of the connected parts (under `structure`) of each non-zero label, numbered by first voxel in
  F order, parts below dust_threshold voxels and labels not in `keep` dropped; one find_objects pass, each
  label labelled on its bounding box"""
  labels = np.asarray(labels)
  uniq, inv = np.unique(labels, return_inverse=True)
  inv = inv.reshape(labels.shape)
  if uniq[0] != 0:
    inv = inv + 1  # no background: label ids start at 1
  parts = []  # (global F index of first voxel, label id, crop slices, part mask)
  for lid, sl in _crops(inv, int(inv.max())):
    if keep is not None and uniq[lid if uniq[0] == 0 else lid - 1] not in keep:
      continue
    m = inv[sl] == lid
    cc, n = ndimage.label(m, structure=structure)
    for i in range(1, n + 1):
      pm = cc == i
      if pm.sum() < dust_threshold:
        continue
      loc = np.unravel_index(_first_f(pm), pm.shape, order="F")
      g = _ravel(tuple(int(a.start) + int(b) for a, b in zip(sl, loc)), labels.shape)
      parts.append((g, sl, pm))
  parts.sort(key=lambda t: t[0])
  out = np.zeros(labels.shape, np.uint32)
  for i, (_, sl, pm) in enumerate(parts):
    out[sl][pm] = i + 1
  return out, len(parts)


def objects_of(labels, dust_threshold=0, object_ids=None):
  """u32 ids 1..k of the 26-connected parts of each label, by first voxel in F order, dust dropped"""
  return parts_of(labels, np.ones((3, 3, 3), int), dust_threshold, object_ids)


def border_targets(obj, k, anisotropy):
  """fix_borders targets (DESIGN.md §5f): per face x = 0, x = sx - 1, y = 0, y = sy - 1, z = 0, z = sz - 1,
  the 8-connected parts of each object in the plane by first voxel, and per part its voxel of greatest
  2-D edt of the object plane (ties to the lowest plane F-order index); linear indices of the volume"""
  shape = obj.shape
  out = []
  for face in range(6):
    axis, end = face // 2, face % 2
    idx = [slice(None)] * 3
    idx[axis] = shape[axis] - 1 if end else 0
    plane = obj[tuple(idx)]
    pa = [a for i, a in enumerate(anisotropy) if i != axis]
    parts, n = parts_of(plane, np.ones((3, 3), int))
    dt = edtref.edt(plane, pa, black_border=True)
    for pid, sl in _crops(parts, n):
      v = np.where(parts[sl] == pid, dt[sl], -np.inf)
      loc = np.unravel_index(int(np.argmax(v.reshape(-1, order="F"))), v.shape, order="F")
      uv = [int(a.start) + int(b) for a, b in zip(sl, loc)]
      voxel = uv[:axis] + [int(idx[axis])] + uv[axis:]
      out.append(_ravel(tuple(voxel), shape))
  return out


def ref_geodesic(lab, sources, anisotropy=(1, 1, 1), weights=None, parents=False):
  """geodesicref.geodesic with F-order linear sources, at connectivity 26"""
  return geodesicref.geodesic(lab, [_unravel(s, lab.shape) for s in sources], 26, anisotropy, weights, parents)


def skeletonize(labels, anisotropy=(1, 1, 1), scale=10.0, const=10.0, pdrf_scale=100000, pdrf_exponent=4,
                max_paths=None, dust_threshold=0, object_ids=None, fix_branching=True, before=(), after=(),
                fix_borders=False, geodesic=ref_geodesic, run_loop=loop):
  """{label: (vertices, edges, radii)} under the rule; before / after are (x, y, z) voxels.  The fields are
  solved per object on its bounding box, so the cost is linear in the volume."""
  return skeletonize_modes(labels, anisotropy, scale, const, pdrf_scale, pdrf_exponent, max_paths, dust_threshold,
                           object_ids, (fix_branching,), before, after, fix_borders, geodesic, run_loop)[fix_branching]


def skeletonize_modes(labels, anisotropy=(1, 1, 1), scale=10.0, const=10.0, pdrf_scale=100000, pdrf_exponent=4,
                      max_paths=None, dust_threshold=0, object_ids=None, modes=(True, False), before=(), after=(),
                      fix_borders=False, geodesic=ref_geodesic, run_loop=loop):
  """{fix_branching: skeletonize(...)} for each mode of `modes`, the objects and fields computed once"""
  fix_branching = False not in modes
  labels = np.asarray(labels)
  shape = labels.shape
  obj, k = objects_of(labels, dust_threshold, object_ids)
  if k == 0:
    return {fb: {} for fb in modes}
  flat = obj.reshape(-1, order="F")
  ids = lambda pts: [_ravel(tuple(int(c) for c in p), shape) for p in pts]
  bt, at = ids(before), ids(after)
  if fix_borders:
    bt = bt + border_targets(obj, k, anisotropy)
  override = {}
  for t in bt:
    if flat[t]:
      override[int(flat[t])] = t
  dbf = edtref.edt(obj, anisotropy, black_border=True).astype(np.float32)
  daf = np.full(shape, np.inf, np.float32)
  pdrf = np.zeros(shape, np.float32)
  par = None if fix_branching else np.zeros(shape, np.uint32)
  roots = np.zeros(k + 1, np.uint64)
  for o, sl in _crops(obj, k):
    m = (obj[sl] == o).astype(np.uint8)
    cs = m.shape
    g = lambda local: _ravel(tuple(int(a.start) + int(b) for a, b in zip(sl, _unravel(local, cs))), shape)
    if o in override:
      loc = [a - int(b.start) for a, b in zip(_unravel(override[o], shape), sl)]
      root = _ravel(tuple(loc), cs)
    else:
      d = geodesic(m, [_first_f(m.astype(bool))], anisotropy)
      root = int(np.argmax(np.where(m != 0, d, -np.inf).reshape(-1, order="F")))
    roots[o] = g(root)
    a_ = geodesic(m, [root], anisotropy)
    daf[sl][m != 0] = a_[m != 0]
    pw = geodesicref.pdrf(m, dbf[sl] * (m != 0), a_, pdrf_scale, pdrf_exponent)
    pdrf[sl][m != 0] = pw[m != 0]
    if not fix_branching:
      _, pl = geodesic(m, [root], weights=pw, parents=True)
      inside = (m != 0) & (pl != 0)
      pz = np.stack(np.unravel_index(pl[inside].astype(np.int64) - 1, cs, order="F"), axis=0)
      glob = np.ravel_multi_index(tuple(pz[i] + sl[i].start for i in range(3)), shape, order="F")
      par[sl][inside] = (glob + 1).astype(np.uint32)
  out = {}
  for fb in modes:
    nxt = run_loop(obj, k, anisotropy, dbf, daf, pdrf, roots, parents=None if fb else par, before=bt, after=at,
                   scale=scale, const=const, max_paths=max_paths)
    out[fb] = assemble(labels, nxt, dbf, anisotropy)
  return out


def assemble(labels, nxt, dbf, anisotropy):
  """split the skeleton by label: one sort, no pass per label"""
  nf = nxt.reshape(-1, order="F")
  lf = np.asarray(labels).reshape(-1, order="F")
  df = dbf.reshape(-1, order="F")
  idx = np.flatnonzero(nf != NONE)
  lab = lf[idx]
  order = np.argsort(lab, kind="stable")
  idx, lab = idx[order], lab[order]
  cuts = np.flatnonzero(np.diff(lab)) + 1
  out = {}
  for part in np.split(np.arange(idx.size), cuts):
    if not part.size:
      continue
    ii = idx[part]
    nx = nf[ii].astype(np.int64)
    tree = nx != ii
    a_, b_ = np.arange(ii.size)[tree], np.searchsorted(ii, nx[tree])
    assert np.array_equal(ii[b_], nx[tree])
    e = np.sort(np.stack([a_, b_], axis=1), axis=1)
    e = e[np.lexsort((e[:, 1], e[:, 0]))]
    verts = np.stack(np.unravel_index(ii, labels.shape, order="F"), axis=1).astype(np.float32)
    out[int(lab[part[0]])] = (verts * np.asarray(anisotropy, np.float32), e.astype(np.uint32).reshape(-1, 2),
                              df[ii].astype(np.float32))
  return out


def capsule_trees(shape, trees, seed, radius=(2.5, 4.5), segments=12, length=(10, 30), anisotropy=(1, 1, 1)):
  """u32 labels 1..trees of random trees of capsules (neurite-like): each segment starts at a random earlier
  node of its tree and runs a random length in a random direction; voxels within the radius (in physical
  units / anisotropy) of a segment take the tree's label, later trees over earlier ones"""
  rng = np.random.default_rng(seed)
  shape = np.array(shape)
  a = np.asarray(anisotropy, float)
  vol = np.zeros(tuple(shape), np.uint32)
  for t in range(1, trees + 1):
    nodes = [rng.uniform(0, shape - 1)]
    r = rng.uniform(*radius)
    for _ in range(segments):
      p = nodes[rng.integers(len(nodes))]
      d = rng.normal(size=3)
      q = np.clip(p + d / np.linalg.norm(d) * rng.uniform(*length), 0, shape - 1)
      nodes.append(q)
      rv = r / a * a.min()  # the radius in voxels per axis
      lo = np.maximum(np.floor(np.minimum(p, q) - rv - 1), 0).astype(int)
      hi = np.minimum(np.ceil(np.maximum(p, q) + rv + 1), shape - 1).astype(int)
      g = np.stack(np.meshgrid(*[np.arange(l, h + 1) for l, h in zip(lo, hi)], indexing="ij"), -1).astype(float)
      u = q - p
      s = np.clip(((g - p) @ u) / max(u @ u, 1e-9), 0, 1)
      dist = np.linalg.norm(((g - p) - s[..., None] * u) * a / a.min(), axis=-1)
      sub = vol[lo[0]:hi[0] + 1, lo[1]:hi[1] + 1, lo[2]:hi[2] + 1]
      sub[dist <= r] = t
  return np.asfortranarray(vol)
