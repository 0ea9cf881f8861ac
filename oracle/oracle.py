"""CPU oracle for the igneous hot path -- TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
--impl reference legs may import this module, and only as the checker.
The product (igneous_b200/) never imports it.

Heavy loops live in igneous_oracle.c (built by oracle/Makefile); the integer
glue that the reference takes from `fastremap` is restated here in numpy.
Every function cites the reference call site it follows
(paths relative to the reference checkout, seung-lab/igneous @ 3b6e5b6).

Parity status: see the header of igneous_oracle.c and DESIGN.md.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

_SUFFIX = {np.dtype(np.uint8): "u8", np.dtype(np.uint16): "u16",
           np.dtype(np.uint32): "u32", np.dtype(np.uint64): "u64",
           np.dtype(np.float32): "f32"}


def build(force=False):
  so = os.path.join(_HERE, "liboracle.so")
  src = os.path.join(_HERE, "igneous_oracle.c")
  if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
    subprocess.check_call(["make", "-C", _HERE, "-B", "liboracle.so"],
                          stdout=subprocess.DEVNULL)
  return so


def lib():
  global _LIB
  if _LIB is None:
    _LIB = ctypes.CDLL(build())
  return _LIB


def _f3(arr):
  """3-D (or 4-D with one channel) array -> Fortran-contiguous 3-D view/copy."""
  arr = np.asarray(arr)
  if arr.ndim == 4:
    assert arr.shape[3] == 1
    arr = arr[..., 0]
  assert arr.ndim == 3
  return np.asfortranarray(arr)


def _ptr(a):
  return ctypes.c_void_p(a.ctypes.data)


# ---------------------------------------------------------------- pooling
def downsample_segmentation(img, factor=(2, 2, 1), num_mips=1, sparse=False):
  """tinybrain.downsample_segmentation as called at
  igneous/tasks/image/image.py:52-53,91 -- recursive 2x2x1 mode pooling; other
  factors of 1 or 2 per axis (2x2x2 ...) go through the block rule."""
  if tuple(int(v) for v in factor)[:3] != (2, 2, 1):
    return _block_pool(img, factor, num_mips, "mode", int(bool(sparse)))
  img = np.asarray(img)
  four_d = img.ndim == 4
  chans = [img[..., c] for c in range(img.shape[3])] if four_d else [img]
  results = [[] for _ in range(num_mips)]
  for ch in chans:
    cur = _f3(ch)
    fn = getattr(lib(), "orc_mode_pool_2x2x1_" + _SUFFIX[cur.dtype])
    for m in range(num_mips):
      sx, sy, sz = cur.shape
      out = np.zeros(((sx + 1) // 2, (sy + 1) // 2, sz), dtype=cur.dtype, order="F")
      rc = fn(_ptr(cur), ctypes.c_uint64(sx), ctypes.c_uint64(sy), ctypes.c_uint64(sz),
              _ptr(out), ctypes.c_int(int(bool(sparse))))
      assert rc == 0
      results[m].append(out)
      cur = out
  if four_d:
    return [np.asfortranarray(np.stack(r, axis=3)) for r in results]
  return [r[0] for r in results]


def downsample_with_averaging(img, factor=(2, 2, 1), num_mips=1, sparse=False,
                              rounding=0):
  """tinybrain.downsample_with_averaging as called at
  igneous/tasks/image/image.py:50-51,91 -- 2x2x1 mean, exact sums in groups
  of four mips, floor rendering (rounding=0; parity unpinned); other factors of
  1 or 2 per axis are averaged block-wise, recursively per mip."""
  if sparse:  # mean of the non-zero samples, any factor
    return _block_pool(img, factor, num_mips, "avg", int(rounding) + 3)
  if tuple(int(v) for v in factor)[:3] != (2, 2, 1):
    return _block_pool(img, factor, num_mips, "avg", int(rounding))
  img = np.asarray(img)
  four_d = img.ndim == 4
  chans = [img[..., c] for c in range(img.shape[3])] if four_d else [img]
  results = [[] for _ in range(num_mips)]
  for ch in chans:
    cur = _f3(ch)
    fn = getattr(lib(), "orc_avg_pool_2x2x1_" + _SUFFIX[cur.dtype])
    sx, sy, sz = cur.shape
    outs = []
    for m in range(num_mips):
      sx, sy = (sx + 1) // 2, (sy + 1) // 2
      outs.append(np.zeros((sx, sy, sz), dtype=cur.dtype, order="F"))
    arr = (ctypes.c_void_p * num_mips)(*[o.ctypes.data for o in outs])
    rc = fn(_ptr(cur), ctypes.c_uint64(cur.shape[0]), ctypes.c_uint64(cur.shape[1]),
            ctypes.c_uint64(cur.shape[2]), ctypes.c_int(num_mips), arr,
            ctypes.c_int(rounding))
    assert rc == 0
    for m in range(num_mips):
      results[m].append(outs[m])
  if four_d:
    return [np.asfortranarray(np.stack(r, axis=3)) for r in results]
  return [r[0] for r in results]


def _block_pool(img, factor, num_mips, kind, flag):
  """orc_block_mode_* / orc_block_avg_* applied recursively, per channel."""
  f = tuple(int(v) for v in factor)[:3]
  img = np.asarray(img)
  four_d = img.ndim == 4
  chans = [img[..., c] for c in range(img.shape[3])] if four_d else [img]
  results = [[] for _ in range(num_mips)]
  for ch in chans:
    cur = _f3(ch)
    suffix = "f32" if cur.dtype == np.float32 else _SUFFIX[cur.dtype]
    if kind == "mode" and cur.dtype == np.float32:
      cur, suffix = cur.view(np.uint32), "u32"
    fn = getattr(lib(), "orc_block_%s_%s" % (kind, suffix))
    for m in range(num_mips):
      sx, sy, sz = cur.shape
      out = np.zeros(tuple((s + ff - 1) // ff for s, ff in zip(cur.shape, f)), dtype=cur.dtype, order="F")
      rc = fn(_ptr(cur), ctypes.c_uint64(sx), ctypes.c_uint64(sy), ctypes.c_uint64(sz),
              ctypes.c_uint32(f[0]), ctypes.c_uint32(f[1]), ctypes.c_uint32(f[2]), ctypes.c_int(flag), _ptr(out))
      assert rc == 0
      results[m].append(out.view(ch.dtype) if ch.dtype == np.float32 else out)
      cur = out
  if four_d:
    return [np.asfortranarray(np.stack(r, axis=3)) for r in results]
  return [r[0] for r in results]


def downsample_select(img, factor, num_mips=1, op="min"):
  """tinybrain.downsample_with_{min,max}_pooling / _striding
  (igneous/tasks/image/image.py:46-49,55): block min / max / first sample; partial
  edge blocks reduce over the samples that exist."""
  f = tuple(int(v) for v in factor)[:3]
  cur = np.asarray(img)
  outs = []
  for _ in range(num_mips):
    if op == "stride":
      cur = cur[::f[0], ::f[1], ::f[2]]
    else:
      big, fn = (np.iinfo(cur.dtype).max if cur.dtype.kind in "ui" else np.inf), (np.minimum if op == "min" else np.maximum)
      fill = big if op == "min" else (np.iinfo(cur.dtype).min if cur.dtype.kind in "ui" else -np.inf)
      pad = [(0, (-s) % ff) for s, ff in zip(cur.shape[:3], f)] + [(0, 0)] * (cur.ndim - 3)
      p = np.pad(cur, pad, constant_values=fill)
      acc = None
      for dx in range(f[0]):
        for dy in range(f[1]):
          for dz in range(f[2]):
            part = p[dx::f[0], dy::f[1], dz::f[2]]
            acc = part if acc is None else fn(acc, part)
      cur = acc
    cur = np.asfortranarray(cur)
    outs.append(cur)
  return outs


# -------------------------------------------------------------------- CCL
def connected_components(labels, connectivity=6, out_dtype=np.uint64, return_N=False):
  """cc3d.connected_components(labels, connectivity=6, out_dtype=np.uint64)
  as called at igneous/tasks/image/ccl.py:173,235-238,339-342."""
  assert connectivity == 6
  labels = np.asarray(labels)
  if labels.dtype == bool:
    labels = labels.view(np.uint8)
  cur = _f3(labels)
  fn = getattr(lib(), "orc_ccl6_" + _SUFFIX[cur.dtype])
  out = np.zeros(cur.shape, dtype=np.uint64, order="F")
  n = ctypes.c_uint64(0)
  rc = fn(_ptr(cur), ctypes.c_uint64(cur.shape[0]), ctypes.c_uint64(cur.shape[1]),
          ctypes.c_uint64(cur.shape[2]), _ptr(out), ctypes.byref(n))
  assert rc == 0
  out = out.astype(out_dtype, copy=False)
  return (out, int(n.value)) if return_N else out


def dust(labels, threshold, connectivity=6, in_place=False):
  """cc3d.dust(labels, threshold=, connectivity=6, in_place=True)
  (igneous/tasks/image/ccl.py:169-172): zero every connected component with
  fewer than `threshold` voxels (semantic pinned by
  test/test_ccl_tasks.py:113,192-198)."""
  labels = np.asarray(labels)
  out = labels if in_place else labels.copy(order="F")
  if threshold <= 0:
    return out
  cc, n = connected_components(labels, connectivity, return_N=True)
  counts = np.bincount(cc.ravel(order="K"), minlength=n + 1)
  small = counts < threshold
  small[0] = False
  view = out.view(np.uint8) if out.dtype == bool else out
  view[small[cc]] = 0
  return out


# ------------------------------------------------------- fastremap glue
def renumber(arr, start=1, preserve_zero=True):
  """fastremap.renumber(data, in_place=True) (igneous/tasks/mesh/mesh.py:206):
  relabel to 1..K in order of first appearance in memory (Fortran) order,
  0 preserved; returns (renumbered, {old: new}).  Output dtype is the
  smallest unsigned type that holds K."""
  a = np.asarray(arr)
  flat = a.ravel(order="F")
  uniq, first = np.unique(flat, return_index=True)
  order = np.argsort(first, kind="stable")
  mapping = {}
  nxt = start
  for u in uniq[order]:
    if preserve_zero and u == 0:
      mapping[0] = 0
      continue
    mapping[int(u)] = nxt
    nxt += 1
  lut_keys = np.array(list(mapping.keys()), dtype=flat.dtype)
  lut_vals = np.array(list(mapping.values()), dtype=np.uint64)
  srt = np.argsort(lut_keys)
  pos = np.searchsorted(lut_keys[srt], flat)
  out = lut_vals[srt][pos]
  out = out.astype(fit_dtype(np.uint64, nxt - 1 if nxt > start else 0))
  return out.reshape(a.shape, order="F"), mapping


def fit_dtype(dtype, value):
  """fastremap.fit_dtype (igneous/task_creation/image.py:1832)."""
  for dt in (np.uint8, np.uint16, np.uint32, np.uint64):
    if value <= np.iinfo(dt).max:
      return np.dtype(dt)
  raise ValueError(value)


def remap(arr, table, preserve_missing_labels=False):
  """fastremap.remap(cc_labels, mapping, in_place=True)
  (igneous/tasks/image/ccl.py:346); KeyError on a missing label."""
  a = np.asarray(arr)
  keys = np.array(list(table.keys()), dtype=np.uint64)
  vals = np.array(list(table.values()), dtype=np.uint64)
  srt = np.argsort(keys)
  keys, vals = keys[srt], vals[srt]
  order = "F" if (a.flags.f_contiguous and not a.flags.c_contiguous) else "C"
  flat = a.ravel(order=order).astype(np.uint64)
  pos = np.clip(np.searchsorted(keys, flat), 0, max(len(keys) - 1, 0))
  hit = keys[pos] == flat if len(keys) else np.zeros(flat.shape, bool)
  if not hit.all():
    if not preserve_missing_labels:
      raise KeyError(int(flat[~hit][0]))
    out = np.where(hit, vals[pos], flat)
  else:
    out = vals[pos]
  return out.astype(a.dtype).reshape(a.shape, order=order)


def unique(arr, return_counts=False):
  """fastremap.unique (igneous/tasks/mesh/mesh.py:318)."""
  return np.unique(np.asarray(arr), return_counts=return_counts)


def mask(arr, labels, value=0):
  """fastremap.mask (igneous/tasks/mesh/mesh.py:204,320)."""
  a = np.asarray(arr).copy(order="K")
  a[np.isin(a, np.asarray(list(labels), dtype=a.dtype))] = value
  return a


def mask_except(arr, labels, value=0):
  """fastremap.mask_except (igneous/tasks/mesh/mesh.py:201,368)."""
  a = np.asarray(arr).copy(order="K")
  a[~np.isin(a, np.asarray(list(labels), dtype=a.dtype))] = value
  return a


def inverse_component_map(parents, components):
  """fastremap.inverse_component_map(cur_i, prev_i)
  (igneous/tasks/image/ccl.py:280): {parent: sorted unique component ids}."""
  p = np.asarray(parents).ravel(order="K").astype(np.uint64)
  c = np.asarray(components).ravel(order="K").astype(np.uint64)
  pairs = np.unique(np.stack([p, c], axis=1), axis=0)
  out = {}
  for a, b in pairs:
    out.setdefault(int(a), []).append(int(b))
  return out


# ------------------------------------------------------------------- mesh
def marching_cubes(labels, flip=True):
  """zmesh.Mesher.mesh(data) (igneous/tasks/mesh/mesh.py:245): returns
  (tri_label u64[T], tri_verts u32[T,3,3]) in half-voxel integer units.
  flip=True reverses the table winding so that triangles are counter-clockwise
  seen from outside the label (outward normals; parity unpinned)."""
  cur = _f3(labels)
  fn = getattr(lib(), "orc_marching_cubes_" + _SUFFIX[cur.dtype])
  n = ctypes.c_uint64(0)
  args = (_ptr(cur), ctypes.c_uint64(cur.shape[0]), ctypes.c_uint64(cur.shape[1]),
          ctypes.c_uint64(cur.shape[2]), ctypes.byref(n))
  assert fn(*args, None, None, ctypes.c_int(int(flip))) == 0
  T = int(n.value)
  tl = np.zeros(T, dtype=np.uint64)
  tv = np.zeros((T, 3, 3), dtype=np.uint32)
  if T:
    assert fn(*args, _ptr(tl), _ptr(tv), ctypes.c_int(int(flip))) == 0
  return tl, tv


class WeldedMeshes:
  """All labels of one marching-cubes run welded at once (oracle of
  Mesher.get with reduction_factor=0, igneous/tasks/mesh/mesh.py:376-381)."""

  def __init__(self, tl, tv):
    T = len(tl)
    self.tri_order = np.zeros(T, dtype=np.uint64)
    ulabel = np.zeros(3 * T, dtype=np.uint64)
    uxyz = np.zeros((3 * T, 3), dtype=np.uint32)
    faces = np.zeros((T, 3), dtype=np.uint32)
    n = ctypes.c_uint64(0)
    tl = np.ascontiguousarray(tl, dtype=np.uint64)
    tv = np.ascontiguousarray(tv, dtype=np.uint32)
    rc = lib().orc_weld(_ptr(tl), _ptr(tv), ctypes.c_uint64(T), _ptr(self.tri_order), _ptr(ulabel),
                        _ptr(uxyz), _ptr(faces), ctypes.byref(n))
    assert rc == 0
    U = int(n.value)
    self.ulabel, self.uxyz, self.faces = ulabel[:U], uxyz[:U], faces
    self.tlabel = tl[self.tri_order.astype(np.int64)] if T else tl
    self.labels = np.unique(self.tlabel)
    self.v0 = np.searchsorted(self.ulabel, self.labels, side="left")
    self.v1 = np.searchsorted(self.ulabel, self.labels, side="right")
    self.f0 = np.searchsorted(self.tlabel, self.labels, side="left")
    self.f1 = np.searchsorted(self.tlabel, self.labels, side="right")

  def ids(self):
    return [int(l) for l in self.labels]

  def get(self, label, resolution=(1, 1, 1), voxel_centered=True):
    j = int(np.searchsorted(self.labels, np.uint64(label)))
    if j >= len(self.labels) or self.labels[j] != label:
      raise KeyError(label)
    xyz = self.uxyz[self.v0[j]:self.v1[j]].astype(np.float32)
    verts = xyz * np.float32(0.5)
    if voxel_centered:
      verts = verts + np.float32(0.5)
    verts = verts * np.asarray(resolution, dtype=np.float32)
    faces = self.faces[self.f0[j]:self.f1[j]] - np.uint32(self.v0[j])
    return verts.astype(np.float32), faces.astype(np.uint32)


def simplify_welded(W, resolution=(1, 1, 1), reduction_factor=100, max_error=40.0,
                    voxel_centered=True, max_rounds=400):
  """Mesher.get(id, reduction_factor, max_error, voxel_centered) for every label of a
  WeldedMeshes (igneous/tasks/mesh/mesh.py:376-381): round-based quadric edge
  collapse (see orc_simplify; parity with zmesh unpinned).  Returns
  ({label: (vertices f32, faces u32)}, rounds)."""
  U, T = len(W.ulabel), len(W.faces)
  res = np.asarray(resolution, dtype=np.float64)
  pos = np.ascontiguousarray(W.uxyz.astype(np.float64) * 0.5 * res)
  faces = np.ascontiguousarray(W.faces.astype(np.uint32))
  dense = np.searchsorted(W.labels, W.tlabel).astype(np.uint32) + np.uint32(1)
  K = len(W.labels)
  nf = (W.f1 - W.f0).astype(np.uint64)
  target = np.zeros(K + 1, dtype=np.uint32)
  target[1:] = (nf // np.uint64(max(int(reduction_factor), 1))).astype(np.uint32)
  valive = np.zeros(max(U, 1), dtype=np.uint8)
  falive = np.zeros(max(T, 1), dtype=np.uint8)
  rounds = ctypes.c_int(0)
  tri_off = np.zeros(K + 1, dtype=np.uint32)
  tri_off[1:] = W.f0.astype(np.uint32)
  rc = lib().orc_simplify(ctypes.c_uint64(U), ctypes.c_uint64(T), _ptr(pos), _ptr(faces), _ptr(dense),
                          ctypes.c_uint32(K), _ptr(target), _ptr(tri_off), ctypes.c_double(float(max_error) ** 2),
                          ctypes.c_int(max_rounds), _ptr(valive), _ptr(falive), ctypes.byref(rounds))
  assert rc == 0
  out = {}
  shift = (np.float32(0.5) * np.asarray(resolution, dtype=np.float32)) if voxel_centered else np.zeros(3, np.float32)
  newid = np.cumsum(valive[:U].astype(np.int64)) - 1
  for j, lab in enumerate(W.labels):
    v0, v1, f0, f1 = int(W.v0[j]), int(W.v1[j]), int(W.f0[j]), int(W.f1[j])
    va = valive[v0:v1].astype(bool)
    fa = falive[f0:f1].astype(bool)
    verts = pos[v0:v1][va].astype(np.float32) + shift
    base = newid[v0] - (1 if valive[v0] else 0) + 1 if v1 > v0 else 0
    f = faces[f0:f1][fa].astype(np.int64)
    f = (newid[f] - base).astype(np.uint32)
    out[int(lab)] = (verts.astype(np.float32), f)
  return out, int(rounds.value)


def pack_vertex(v):
  """(x,y,z) half-voxel integer coords -> sortable 63-bit key (z major)."""
  v = np.asarray(v, dtype=np.uint64)
  return (v[..., 2] << np.uint64(42)) | (v[..., 1] << np.uint64(21)) | v[..., 0]


def mesh_for_label(tl, tv, label, resolution=(1, 1, 1), voxel_centered=True):
  """Mesher.get(id, reduction_factor=0, voxel_centered=...) without
  simplification (igneous/tasks/mesh/mesh.py:377-382): weld the label's
  triangle soup.  Vertices are ordered by packed (z,y,x) key, faces keep
  emission order.  Returns (vertices f32 [N,3], faces u32 [M,3])."""
  sel = tv[tl == label]
  keys = pack_vertex(sel)  # [M,3]
  uniq, inv = np.unique(keys.ravel(), return_inverse=True)
  faces = inv.reshape(-1, 3).astype(np.uint32)
  x = (uniq & np.uint64((1 << 21) - 1)).astype(np.float32)
  y = ((uniq >> np.uint64(21)) & np.uint64((1 << 21) - 1)).astype(np.float32)
  z = (uniq >> np.uint64(42)).astype(np.float32)
  res = np.asarray(resolution, dtype=np.float32)
  verts = np.stack([x, y, z], axis=1) * np.float32(0.5)
  if voxel_centered:
    verts = verts + np.float32(0.5)
  verts = verts * res
  return verts.astype(np.float32), faces


def canonicalise_mesh(vertices, faces, decimals=None):
  """Order-independent form: vertices sorted lexicographically (z,y,x), faces
  re-indexed, rotated to start at their smallest index (winding kept) and
  sorted.  Two meshes with the same geometry + topology compare equal."""
  v = np.asarray(vertices, dtype=np.float64)
  f = np.asarray(faces, dtype=np.int64)
  key = np.round(v, decimals) if decimals is not None else v
  order = np.lexsort((key[:, 0], key[:, 1], key[:, 2]))
  inv = np.empty(len(order), dtype=np.int64)
  inv[order] = np.arange(len(order))
  f = inv[f]
  k = np.argmin(f, axis=1)
  f = np.stack([f[np.arange(len(f)), (k + i) % 3] for i in range(3)], axis=1)
  f = f[np.lexsort((f[:, 2], f[:, 1], f[:, 0]))]
  return v[order], f


# ------------------------------------------------------ synthetic volumes
def _mix64(z):
  z = (z + np.uint64(0x9E3779B97F4A7C15)).astype(np.uint64)
  z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
  z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
  return z ^ (z >> np.uint64(31))


def cell_hash(seed, cx, cy, cz):
  """splitmix64 of (seed, cell) -- identical to csrc/synth.cu."""
  with np.errstate(over="ignore"):
    h = _mix64(np.uint64(seed) + np.asarray(cx, dtype=np.int64).astype(np.uint64) * np.uint64(0x100000001B3))
    h = _mix64(h ^ np.asarray(cy, dtype=np.int64).astype(np.uint64) * np.uint64(0xC2B2AE3D27D4EB4F))
    h = _mix64(h ^ np.asarray(cz, dtype=np.int64).astype(np.uint64) * np.uint64(0x165667B19E3779F9))
  return h


def synth_seg_np(shape, pitch=16, num_ids=1 << 20, seed=0, offset=(0, 0, 0),
              dtype=np.uint32, id_base=0):
  """numpy statement of synth_seg (slow; used to cross-check the C version).
  Jittered-grid Voronoi segmentation with membranes (SURVEY.md 8(d)),
  bit-identical to ign_synth_seg (igneous_b200/csrc/synth.cu).

  One seed point per pitch^3 cell at a hashed offset.  The 27 surrounding
  cells are scanned in (dz,dy,dx) order keeping the smallest (d1, id1) and the
  second smallest (d2) squared integer distance with strict '<' updates.
  label = 0 if d2 - d1 < 2*pitch (membrane, ~1 voxel either side of the
  bisector plane) else id1, with id = id_base + 1 + mix64(h) % num_ids."""
  sx, sy, sz = shape
  X, Y, Z = np.meshgrid(np.arange(sx, dtype=np.int64) + offset[0],
                        np.arange(sy, dtype=np.int64) + offset[1],
                        np.arange(sz, dtype=np.int64) + offset[2], indexing="ij")
  cx, cy, cz = X // pitch, Y // pitch, Z // pitch
  big = np.iinfo(np.int64).max
  d1 = np.full(shape, big, dtype=np.int64)
  d2 = np.full(shape, big, dtype=np.int64)
  id1 = np.zeros(shape, dtype=np.uint64)
  m16 = np.uint64(0xFFFF)
  for dz in (-1, 0, 1):
    for dy in (-1, 0, 1):
      for dx in (-1, 0, 1):
        ccx, ccy, ccz = cx + dx, cy + dy, cz + dz
        h = cell_hash(seed, ccx, ccy, ccz)
        px = ccx * pitch + ((h & m16) % np.uint64(pitch)).astype(np.int64)
        py = ccy * pitch + (((h >> np.uint64(16)) & m16) % np.uint64(pitch)).astype(np.int64)
        pz = ccz * pitch + (((h >> np.uint64(32)) & m16) % np.uint64(pitch)).astype(np.int64)
        cid = np.uint64(id_base) + np.uint64(1) + _mix64(h) % np.uint64(num_ids)
        d = (X - px) ** 2 + (Y - py) ** 2 + (Z - pz) ** 2
        closer = d < d1
        d2 = np.where(closer, d1, np.where(d < d2, d, d2))
        id1 = np.where(closer, cid, id1)
        d1 = np.where(closer, d, d1)
  out = np.where((d2 - d1) < 2 * pitch, np.uint64(0), id1)
  return np.asfortranarray(out.astype(dtype))


def synth_image(shape, seed=0, offset=(0, 0, 0)):
  """Uniform hash bytes 0..254 (mirrors test/layer_harness.py:36
  np.random.randint(255)); bit-identical to ign_synth_image."""
  sx, sy, sz = shape
  X, Y, Z = np.meshgrid(np.arange(sx, dtype=np.int64) + offset[0],
                        np.arange(sy, dtype=np.int64) + offset[1],
                        np.arange(sz, dtype=np.int64) + offset[2], indexing="ij")
  h = cell_hash(seed, X, Y, Z)
  return np.asfortranarray(((h >> np.uint64(11)) % np.uint64(255)).astype(np.uint8))


def synth_seg(shape, pitch=16, num_ids=1 << 20, seed=0, offset=(0, 0, 0),
              dtype=np.uint32, id_base=0):
  """C version of synth_seg_np (same integer hash, bit identical)."""
  sx, sy, sz = (int(v) for v in shape)
  out = np.zeros((sx, sy, sz), dtype=np.uint64, order="F")
  rc = lib().orc_synth_seg_u64(_ptr(out), ctypes.c_uint64(sx), ctypes.c_uint64(sy), ctypes.c_uint64(sz),
                               ctypes.c_int64(offset[0]), ctypes.c_int64(offset[1]),
                               ctypes.c_int64(offset[2]), ctypes.c_int(pitch), ctypes.c_uint64(num_ids),
                               ctypes.c_uint64(seed), ctypes.c_uint64(id_base))
  assert rc == 0
  return np.asfortranarray(out.astype(dtype))


def synth_tiled(shape, seed):
  """Bench chunk for the CPU reference arm: a distinct region of the bench
  dataset per (seed), generated by the C synthesiser."""
  return synth_seg(shape, pitch=64, num_ids=1 << 20, seed=0,
                   offset=(0, 0, (seed % 100000) * shape[2]))


# ------------------------------------------------- compressed_segmentation codec
def cseg_encode(labels, block_size=(8, 8, 8)):
  """Precomputed `compressed_segmentation` encoding of a [x,y,z,(c)] uint32 / uint64 chunk
  (SURVEY 8(f) row 1; what CloudVolume does on the host before uploading a segmentation
  chunk).  Returns the file as a uint32 array."""
  arr = np.asarray(labels)
  if arr.ndim == 3:
    arr = arr[..., np.newaxis]
  assert arr.ndim == 4 and arr.dtype in (np.uint32, np.uint64)
  arr = np.asfortranarray(arr)
  fn = getattr(lib(), "orc_cseg_encode_" + _SUFFIX[arr.dtype])
  fn.restype = ctypes.c_int64
  args = (_ptr(arr), ctypes.c_uint64(arr.shape[0]), ctypes.c_uint64(arr.shape[1]), ctypes.c_uint64(arr.shape[2]),
          ctypes.c_uint64(arr.shape[3]), ctypes.c_uint32(block_size[0]), ctypes.c_uint32(block_size[1]),
          ctypes.c_uint32(block_size[2]))
  need = fn(*args, None, ctypes.c_uint64(0))
  assert need > 0
  out = np.zeros(need, dtype=np.uint32)
  got = fn(*args, _ptr(out), ctypes.c_uint64(need))
  assert got == need
  return out


def cseg_decode(words, shape, dtype, block_size=(8, 8, 8)):
  """Inverse of cseg_encode (accepts any conforming stream): returns the [x,y,z,c] chunk."""
  words = np.ascontiguousarray(words, dtype=np.uint32)
  shape = tuple(int(s) for s in shape)
  if len(shape) == 3:
    shape = shape + (1,)
  out = np.zeros(shape, dtype=dtype, order="F")
  fn = getattr(lib(), "orc_cseg_decode_" + _SUFFIX[np.dtype(dtype)])
  rc = fn(_ptr(words), ctypes.c_uint64(len(words)), ctypes.c_uint64(shape[0]), ctypes.c_uint64(shape[1]),
          ctypes.c_uint64(shape[2]), ctypes.c_uint64(shape[3]), ctypes.c_uint32(block_size[0]),
          ctypes.c_uint32(block_size[1]), ctypes.c_uint32(block_size[2]), _ptr(out))
  if rc != 0:
    raise ValueError("malformed compressed_segmentation stream")
  return out
