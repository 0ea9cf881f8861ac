"""Drop-in for `kimimaro.skeletonize`: TEASAR skeletons of every object of a chunk at once, on H100.

Reference call site (seung-lab/igneous):
  igneous/tasks/skeleton.py:54, :312   SkeletonTask -> kimimaro.skeletonize(all_labels, teasar_params, ...)

The rule is DESIGN.md §5f (kimimaro parity is unpinned offline).  Objects are the 26-connected parts of
each label; each gets the fields of `teasar.fields`, then every object traces its k-th path in the same
round: the target is the valid voxel farthest from the root, the path runs to the skeleton built so far,
and every path voxel invalidates a box of half-extents floor((scale * DBF + const) / anisotropy) around it.
Objects, fields, the loop and the compaction of the skeleton run in libigneous_b200
(igneous_b200/csrc/geodesic.cu), and so does the split of the compacted skeleton into one neuroglancer
precomputed skeleton per label (igneous_b200/csrc/skeleton.cu, DESIGN.md §5g): the host copies the packed
blobs back once and every Skeleton's arrays are views into them.  export_skeletons is the same call with a
vertex offset, the blobs and the bounding boxes, for SkeletonTask.  postprocess and merge_fragments run
the merge stage (igneous_b200/csrc/skelmerge.cu, DESIGN.md §5h).  cross_sectional_area measures the section of
each label across its skeleton at every vertex (igneous_b200/csrc/xsection.cu, DESIGN.md §5i).  There is no
CPU fallback.
"""
import ctypes
import time

import numpy as np

from . import _shim
from .teasar import device_fields

__all__ = ["skeletonize", "export_skeletons", "postprocess", "merge_fragments", "cross_sectional_area", "Skeleton",
           "DEFAULT_TEASAR_PARAMS"]

# seconds per phase of the last call, each ending where the host already waits for the device (diagnostic)
last_phase_seconds = {}
# cross_sectional_area's last call: voxels of every section, vertices whose section outgrew the one-warp path,
# voxels that path visited in them, and CTAs the large path ran with (diagnostic)
last_stats = [0, 0, 0, 0]

_UNSIGNED = {1: np.uint8, 2: np.uint16, 4: np.uint32, 8: np.uint64}

# kimimaro's defaults as recalled (unpinned); soma_* are read only to refuse soma mode
DEFAULT_TEASAR_PARAMS = {
  "scale": 10, "const": 10, "pdrf_scale": 100000, "pdrf_exponent": 4, "soma_acceptance_threshold": 3500,
  "soma_detection_threshold": 750, "soma_invalidation_const": 300, "soma_invalidation_scale": 2, "max_paths": None,
}


class Skeleton:
  """One label's skeleton: vertices (N, 3) float32 in physical units, edges (E, 2) uint32, radii (N,)
  float32, vertex_types (N,) uint8 and the label as id.  cross_sectional_area (N,) float32 and
  cross_sectional_area_contacts (N,) uint8 are None until cross_sectional_area sets them."""

  cross_sectional_area = None
  cross_sectional_area_contacts = None

  def __init__(self, vertices, edges, radii, vertex_types, id):
    self.vertices, self.edges, self.radii, self.vertex_types, self.id = vertices, edges, radii, vertex_types, id

  def empty(self):
    return self.vertices.shape[0] == 0

  def __repr__(self):
    return "Skeleton(id=%r, vertices=%d, edges=%d)" % (self.id, self.vertices.shape[0], self.edges.shape[0])


# the vertex attributes of the blobs the device writes: radius, then vertex_types when asked
ATTRIBUTES = [{"id": "radius", "data_type": "float32", "num_components": 1},
              {"id": "vertex_types", "data_type": "uint8", "num_components": 1}]


def split_blobs(buf, rows, ids, attributes):
  """([Skeleton], [blob]), one of each per row, of the neuroglancer precomputed skeletons in buf (a uint8
  array).  rows: (byte offset, nv, ne) of each blob; ids: each Skeleton's id; attributes: the info's
  vertex_attributes ({id, data_type, num_components}) in the order they follow the edges.  A blob is
  uint32 nv, ne, float32 vertices[nv][3], uint32 edges[ne][2], then each attribute's values for every vertex
  (DESIGN.md §5g).  A Skeleton's radii and vertex_types are the attributes of those ids, zeros when absent.
  Every array is a view into buf; the zeros are views into one array per missing attribute.  ValueError when
  a blob runs past the end of buf."""
  rows = np.asarray(rows, np.int64).reshape(-1, 3)
  off, nv, ne = rows[:, 0], rows[:, 1], rows[:, 2]

  def cut(dt, start, count):  # per row, count values of dt from byte start
    s = np.dtype(dt).itemsize
    if (start % s).any():  # after an attribute of a smaller type
      return [buf[a:a + s * n].view(dt) for a, n in zip(start.tolist(), count.tolist())]
    typed = buf[:buf.size // s * s].view(dt)
    return [typed[a:a + n] for a, n in zip((start // s).tolist(), count.tolist())]

  def shaped(col, c):
    return col if c == 1 else [v.reshape(-1, c) for v in col]

  attrs = [(a["id"], np.dtype(a["data_type"]), int(a.get("num_components", 1))) for a in attributes]
  starts = [off + 8, off + 8 + 12 * nv, off + 8 + 12 * nv + 8 * ne]  # vertices, edges, each attribute
  for _, dt, c in attrs:
    starts.append(starts[-1] + c * dt.itemsize * nv)
  end = starts.pop()
  if (end > buf.size).any():
    g = int(np.argmax(end > buf.size))
    raise ValueError("skeleton %r: its blob ends at byte %d, past the %d bytes of its buffer" % (ids[g], end[g],
                                                                                               buf.size))
  values = {k: shaped(cut(dt, at, c * nv), c) for (k, dt, c), at in zip(attrs, starts[2:])}
  for k, dt in (("radius", np.float32), ("vertex_types", np.uint8)):
    if k not in values:
      zeros = np.zeros(int(nv.sum()), dt)
      values[k] = [zeros[a:a + n] for a, n in zip((np.cumsum(nv) - nv).tolist(), nv.tolist())]
  vertices, edges = shaped(cut(np.float32, starts[0], 3 * nv), 3), shaped(cut(np.uint32, starts[1], 2 * ne), 2)
  skeletons = list(map(Skeleton, vertices, edges, values["radius"], values["vertex_types"], ids))
  return skeletons, [buf[a:b] for a, b in zip(off.tolist(), end.tolist())]


def _targets(points, arr, what):
  """linear F-order indices of voxels (x, y, z) of the caller's array; ValueError on background"""
  pts = np.asarray(points, dtype=np.int64).reshape(-1, 3) if len(points) else np.zeros((0, 3), np.int64)
  if pts.size and (pts.min() < 0 or np.any(pts >= np.array(arr.shape))):
    raise ValueError("kimimaro.skeletonize: a target of %s lies outside the volume of shape %r" % (what, arr.shape))
  for p in pts:
    if arr[tuple(p)] == 0:
      raise ValueError("kimimaro.skeletonize: the target %r of %s lies on background" % (tuple(int(c) for c in p),
                                                                                          what))
  return np.ascontiguousarray(np.ravel_multi_index(tuple(pts.T), arr.shape, order="F"), dtype=np.uint64)


def skeletonize(all_labels, teasar_params=DEFAULT_TEASAR_PARAMS, object_ids=None, anisotropy=(1, 1, 1),
                dust_threshold=1000, progress=False, fix_branching=True, in_place=False, fix_borders=True,
                parallel=1, parallel_chunk_size=100, extra_targets_before=[], extra_targets_after=[],
                fill_holes=False, fix_avocados=False, voxel_graph=None, ctx=None):
  """{label: Skeleton} of every label of a 3-D array with an object of at least dust_threshold voxels,
  in ascending label order.  `progress`, `parallel`, `parallel_chunk_size` and `in_place` are accepted and
  ignored.  fill_holes, fix_avocados, voxel_graph and soma mode (an object whose largest DBF exceeds
  soma_detection_threshold) raise NotImplementedError.  last_phase_seconds holds the host-clock time of
  each phase of the last call.  A Skeleton's arrays are writable views into one buffer of the call."""
  return export_skeletons(all_labels, teasar_params=teasar_params, object_ids=object_ids, anisotropy=anisotropy,
                          dust_threshold=dust_threshold, fix_branching=fix_branching, fix_borders=fix_borders,
                          extra_targets_before=extra_targets_before, extra_targets_after=extra_targets_after,
                          fill_holes=fill_holes, fix_avocados=fix_avocados, voxel_graph=voxel_graph, ctx=ctx)[0]


def export_skeletons(all_labels, offset=(0.0, 0.0, 0.0), vertex_types=True, teasar_params=DEFAULT_TEASAR_PARAMS,
                     object_ids=None, anisotropy=(1, 1, 1), dust_threshold=1000, fix_branching=True,
                     fix_borders=True, extra_targets_before=[], extra_targets_after=[], fill_holes=False,
                     fix_avocados=False, voxel_graph=None, ctx=None):
  """skeletonize with every vertex moved by `offset` (float64, added as numpy adds it to float32 vertices:
  fl32((double)v + offset)), encoded on the device.  Returns three dicts keyed alike, in ascending label
  order: {label: Skeleton}, {label: uint8 array of its neuroglancer precomputed skeleton (vertices, edges,
  radius, and vertex_types when `vertex_types`)}, {label: float32 (6,) min xyz, max xyz of its vertices}.
  Every array is a view into one host buffer."""
  if fill_holes or fix_avocados or voxel_graph is not None:
    raise NotImplementedError("igneous_b200 kimimaro.skeletonize: fill_holes, fix_avocados and voxel_graph are "
                              "not supported")
  arr = np.asarray(all_labels)
  if arr.ndim != 3:
    raise ValueError("kimimaro.skeletonize: expected a 3-D label array, got shape %r" % (arr.shape,))
  if not (arr.dtype == np.bool_ or arr.dtype.kind in "iu"):
    raise NotImplementedError("igneous_b200 kimimaro.skeletonize: label dtype %s is not supported" % arr.dtype)
  p = dict(DEFAULT_TEASAR_PARAMS)
  p.update(teasar_params or {})
  scale, const = float(p["scale"]), float(p["const"])
  if not (np.isfinite(scale) and scale >= 0 and np.isfinite(const) and const >= 0):
    raise ValueError("kimimaro.skeletonize: scale %r and const %r must be finite and >= 0" % (p["scale"], p["const"]))
  if int(p["pdrf_exponent"]) != p["pdrf_exponent"]:
    raise NotImplementedError("igneous_b200 kimimaro.skeletonize: pdrf_exponent must be a whole number")
  max_paths = (1 << 64) - 1 if p["max_paths"] is None else int(p["max_paths"])
  a = tuple(float(v) for v in anisotropy)
  if len(a) != 3 or not all(np.isfinite(v) and v > 0 for v in a):
    raise ValueError("kimimaro.skeletonize: anisotropy %r must be three positive finite values" % (anisotropy,))
  # the kernels take an F-order volume; linear indices below are F-order indices of the caller's axes
  vol = np.asfortranarray(arr.view(_UNSIGNED[arr.dtype.itemsize]))
  n = vol.size
  before = _targets(extra_targets_before, arr, "extra_targets_before")
  after = _targets(extra_targets_after, arr, "extra_targets_after")
  shift = tuple(float(v) for v in offset)
  if len(shift) != 3 or not all(np.isfinite(shift)):
    raise ValueError("kimimaro.export_skeletons: offset %r must be three finite values" % (offset,))
  if n == 0:
    return {}, {}, {}
  ctx = ctx or _shim.default_context()
  lib, h, ptr = ctx.lib, ctx.handle, _shim.ptr
  ca = (ctypes.c_float * 3)(*a)
  bufs = []

  def alloc(nbytes):
    bufs.append(ctx.alloc(max(int(nbytes), 8)))
    return bufs[-1]

  try:
    last_phase_seconds.clear()
    t0 = time.perf_counter()

    def phase(name):
      nonlocal t0
      t = time.perf_counter()
      last_phase_seconds[name] = t - t0
      t0 = t

    raw = alloc(vol.nbytes)
    ctx.h2d(raw, vol)
    lab = alloc(n * 4)
    k = ctypes.c_uint64(0)
    _shim.check(lib.ign_renumber_dev(h, ptr(raw), _shim.dtype_code(vol.dtype), n, ptr(lab), None, 0,
                                     ctypes.byref(k)))
    K = int(k.value)
    orig = np.empty(K, np.uint64)
    if K:
      # the original label of each renumbered one: renumber again into a table of K entries
      uniq = alloc(K * 8)
      _shim.check(lib.ign_renumber_dev(h, ptr(raw), _shim.dtype_code(vol.dtype), n, ptr(lab), ptr(uniq), K,
                                       ctypes.byref(k)))
      ctx.d2h(orig, uniq)
      ctx.sync()
    if K and object_ids is not None:
      wanted = np.asarray(list(object_ids)).astype(arr.dtype).view(_UNSIGNED[arr.dtype.itemsize]).astype(np.uint64)
      drop = np.ascontiguousarray(np.nonzero(~np.isin(orig, wanted))[0] + 1, dtype=np.uint64)
      if drop.size:
        _shim.check(lib.ign_remap_dev(h, ptr(lab), _shim.IGN_U32, n, ptr(drop), ptr(np.zeros_like(drop)),
                                      drop.size, 1))
    obj = alloc(n * 4)
    m = ctypes.c_uint64(0)
    _shim.check(lib.ign_label_parts_dev(h, ptr(lab), _shim.IGN_U32, *vol.shape, 26, int(dust_threshold), ptr(obj),
                                        None, 0, ctypes.byref(m)))
    M = int(m.value)
    phase("upload_objects")
    if M == 0:
      return {}, {}, {}
    if fix_borders:
      # kimimaro's order: the caller's before-targets, then the border targets
      cap = 2 * (vol.shape[1] * vol.shape[2] + vol.shape[0] * vol.shape[2] + vol.shape[0] * vol.shape[1])
      d_border, nb = alloc(cap * 8), ctypes.c_uint64(0)
      _shim.check(lib.ign_teasar_border_targets_dev(h, ptr(obj), *vol.shape, M, ca, ptr(d_border), cap,
                                                    ctypes.byref(nb)))
      border = np.empty(int(nb.value), np.uint64)
      if border.size:
        ctx.d2h(border, d_border, border.nbytes)
        ctx.sync()
      before = np.concatenate([before, border])
      phase("border_targets")
    d_before, d_after = alloc(before.nbytes), alloc(after.nbytes)
    if before.size:
      ctx.h2d(d_before, before)
    if after.size:
      ctx.h2d(d_after, after)
    d = device_fields(ctx, obj, M, vol.shape, ca, p["pdrf_scale"], p["pdrf_exponent"], alloc,
                      before=(d_before, before.size), parents=not fix_branching)
    roots, dbf_max = np.empty(M + 1, np.uint64), np.empty(M + 1, np.float32)
    ctx.d2h(roots, d["roots"])
    ctx.d2h(dbf_max, d["dbf_max"])
    ctx.sync()
    phase("fields")
    soma = np.nonzero(dbf_max[1:] > float(p["soma_detection_threshold"]))[0]
    if soma.size:
      o = int(soma[0]) + 1
      label = arr.reshape(-1, order="F")[int(roots[o])]
      raise NotImplementedError("igneous_b200 kimimaro.skeletonize: label %d has an object whose largest distance "
                                "to the boundary, %g, exceeds soma_detection_threshold %g; soma mode is not "
                                "supported" % (int(label), float(dbf_max[o]), float(p["soma_detection_threshold"])))
    skel, nxt, rad = alloc(n * 4), alloc(n * 4), alloc(n * 4)
    count = ctypes.c_uint64(0)
    _shim.check(lib.ign_teasar_paths_dev(
      h, ptr(obj), *vol.shape, M, ca, ptr(d["dbf"]), ptr(d["daf"]), ptr(d["pdrf"]),
      ptr(d["dist"]) if fix_branching else None, None if fix_branching else ptr(d["parents"]), ptr(d["roots"]),
      ptr(d_before), before.size, ptr(d_after), after.size, scale, const, max_paths, ptr(skel), ptr(nxt), ptr(rad),
      ctypes.byref(count)))
    ctx.sync()
    phase("loop")
    buf, table, boxes = _export(ctx, lab, vol.shape, K, skel, nxt, rad, int(count.value), ca, shift, vertex_types,
                                alloc)
  finally:
    for b in bufs:
      b.free()
  out = _views(buf, table, boxes, orig, arr.dtype, vertex_types)
  phase("assembly")
  return out


def _export(ctx, lab, shape, K, skel, nxt, rad, count, ca, offset, vertex_types, alloc):
  """ign_skeleton_export_dev on the loop's output -> (packed blobs, table rows, boxes), copied back once"""
  lib, h, ptr = ctx.lib, ctx.handle, _shim.ptr
  cap = ctypes.c_uint64(0)
  _shim.check(lib.ign_skeleton_export_capacity(count, K, ctypes.byref(cap)))
  rows = min(K, count)
  d_buf, d_table, d_boxes = alloc(cap.value), alloc(rows * 32), alloc(rows * 24)
  ns, nb = ctypes.c_uint64(0), ctypes.c_uint64(0)
  _shim.check(lib.ign_skeleton_export_dev(h, ptr(lab), *shape, K, ptr(skel), ptr(nxt), ptr(rad), count, ca,
                                          (ctypes.c_double * 3)(*offset), int(bool(vertex_types)), ptr(d_buf),
                                          cap.value, ptr(d_table), ptr(d_boxes), ctypes.byref(ns), ctypes.byref(nb)))
  S, B = int(ns.value), int(nb.value)
  buf = np.empty((B + 7) // 8 * 8, np.uint8)  # whole words, so that typed views of the buffer exist
  buf[B:] = 0
  table, boxes = np.empty((S, 4), np.uint64), np.empty((S, 6), np.float32)
  if S:
    ctx.d2h(buf, d_buf, B)
    ctx.d2h(table, d_table)
    ctx.d2h(boxes, d_boxes)
    ctx.sync()
  return buf, table, boxes


def _views(buf, table, boxes, orig, dtype, vertex_types):
  """split the packed blobs into {label: Skeleton}, {label: blob}, {label: box}, in ascending label order of
  the caller's dtype; every array is a view into buf (or, without vertex_types, into one zero array)"""
  unsigned = _UNSIGNED[np.dtype(dtype).itemsize]
  values = orig[table[:, 0].astype(np.int64) - 1].astype(unsigned).view(dtype)
  order = np.argsort(values, kind="stable")
  keys = (values.astype(np.uint8) if values.dtype == np.bool_ else values)[order].tolist()
  skeletons, blobs = split_blobs(buf, table[order, 1:], keys, ATTRIBUTES[:2 if vertex_types else 1])
  return dict(zip(keys, skeletons)), dict(zip(keys, blobs)), dict(zip(keys, boxes[order]))


def crop_box(bbox, crop, resolution):
  """The crop box of a fragment whose physical box is `bbox` (a Bbox, from its file name): shrunk by
  crop * resolution on every side, float64 (min xyz, max xyz); None when crop <= 0 or the shrunk box has
  volume <= 0, and then the fragment is kept whole (DESIGN.md §5h)."""
  if crop <= 0:
    return None
  r = np.asarray(resolution, np.float64)[:3] * crop
  lo, hi = np.asarray(bbox.minpt, np.float64) + r, np.asarray(bbox.maxpt, np.float64) - r
  if np.prod(hi - lo) <= 0:
    return None
  return np.concatenate([lo, hi])


def pack_fragments(fragments, crop=0, resolution=(1, 1, 1)):
  """(segids, packed arrays) of {segid: [(bbox, Skeleton), ...]} in the layout of ign_skeleton_merge_dev: the
  labels in the dict's order, each label's fragments in the order given.  bbox None keeps a fragment whole."""
  segids = list(fragments)
  whole = np.array([-np.inf] * 3 + [np.inf] * 3)
  label_frag, frag_vert, frag_edge, boxes = [0], [0], [0], []
  verts, radii, types, edges = [], [], [], []
  for segid in segids:
    for bbox, s in fragments[segid]:
      v = np.asarray(s.vertices, np.float32).reshape(-1, 3)
      e = np.asarray(s.edges).reshape(-1, 2)
      if e.size and (e.min() < 0 or e.max() > 0xFFFFFFFF):
        raise ValueError("skeleton merge: label %d has an edge index outside uint32" % segid)
      box = None if bbox is None else crop_box(bbox, crop, resolution)
      boxes.append(whole if box is None else box)
      verts.append(v)
      radii.append(np.asarray(s.radii, np.float32).reshape(-1) if s.radii is not None else np.zeros(len(v), np.float32))
      types.append(np.asarray(s.vertex_types, np.uint8).reshape(-1) if s.vertex_types is not None
                   else np.zeros(len(v), np.uint8))
      if radii[-1].size != len(v) or types[-1].size != len(v):
        raise ValueError("skeleton merge: label %d has a fragment whose radii or vertex_types do not match its "
                         "%d vertices" % (segid, len(v)))
      edges.append(e.astype(np.uint32))
      frag_vert.append(frag_vert[-1] + len(v))
      frag_edge.append(frag_edge[-1] + len(e))
    label_frag.append(len(boxes))
  cat = lambda parts, shape, dt: np.ascontiguousarray(np.concatenate(parts).reshape(shape) if parts
                                                      else np.zeros((0,) + shape[1:], dt), dtype=dt)
  return segids, {
    "label_frag": np.array(label_frag, np.uint64), "frag_vert": np.array(frag_vert, np.uint64),
    "frag_edge": np.array(frag_edge, np.uint64), "frag_box": cat(boxes, (-1, 6), np.float64),
    "vertices": cat(verts, (-1, 3), np.float32), "radius": cat(radii, (-1,), np.float32),
    "vertex_types": cat(types, (-1,), np.uint8), "edges": cat(edges, (-1, 2), np.uint32),
  }


def merge_packed(packed, dust_threshold=4000, tick_threshold=6000, max_cable_length=None, vertex_types=True,
                 ctx=None):
  """ign_skeleton_merge_dev on packed arrays: (bytes buffer, uint64 table (L, 4) of (label row, byte offset,
  nv, ne)), uploaded once and copied back once"""
  L = packed["label_frag"].size - 1
  V, E, F = packed["radius"].size, packed["edges"].shape[0], packed["frag_box"].shape[0]
  mc = float("inf") if max_cable_length is None else float(max_cable_length)
  if L == 0:
    return np.zeros(0, np.uint8), np.zeros((0, 4), np.uint64)
  ctx = ctx or _shim.default_context()
  lib, h, ptr = ctx.lib, ctx.handle, _shim.ptr
  cap = ctypes.c_uint64(0)
  _shim.check(lib.ign_skeleton_merge_capacity(L, V, E, ctypes.byref(cap)))
  names = ("label_frag", "frag_vert", "frag_edge", "frag_box", "vertices", "radius", "vertex_types", "edges")
  bufs = []
  try:
    d = {}
    for k in names:
      bufs.append(ctx.alloc(max(packed[k].nbytes, 8)))
      d[k] = bufs[-1]
      if packed[k].nbytes:
        ctx.h2d(d[k], packed[k])
    bufs.append(ctx.alloc(max(int(cap.value), 8)))
    d_buf = bufs[-1]
    bufs.append(ctx.alloc(L * 32))
    d_table = bufs[-1]
    nb = ctypes.c_uint64(0)
    _shim.check(lib.ign_skeleton_merge_dev(
      h, L, ptr(d["label_frag"]), F, ptr(d["frag_vert"]), ptr(d["frag_edge"]), ptr(d["frag_box"]),
      ptr(d["vertices"]), ptr(d["radius"]), ptr(d["vertex_types"]), V, ptr(d["edges"]), E, float(dust_threshold),
      float(tick_threshold), mc, int(bool(vertex_types)), ptr(d_buf), cap.value, ptr(d_table), ctypes.byref(nb)))
    B = int(nb.value)
    buf = np.zeros((B + 7) // 8 * 8, np.uint8)  # whole words, so that typed views of the buffer exist
    table = np.empty((L, 4), np.uint64)
    ctx.d2h(buf, d_buf, B)
    ctx.d2h(table, d_table)
    ctx.sync()
  finally:
    for b in bufs:
      b.free()
  return buf, table


def merge_fragments(fragments, crop=0, resolution=(1, 1, 1), dust_threshold=4000, tick_threshold=6000,
                    max_cable_length=None, vertex_types=True, ctx=None):
  """UnshardedSkeletonMergeTask's fuse and postprocess for many labels in one device call (DESIGN.md §5h).
  fragments: {segid: [(bbox, Skeleton), ...]}, each label's fragments in ascending file name order; bbox is
  the fragment's physical Bbox (None: never cropped).  Returns {segid: (Skeleton, blob)} in the same order,
  the blob its neuroglancer precomputed skeleton (radius, then vertex_types when `vertex_types`); every array
  is a view into one host buffer."""
  segids, packed = pack_fragments(fragments, crop, resolution)
  buf, table = merge_packed(packed, dust_threshold, tick_threshold, max_cable_length, vertex_types, ctx)
  skeletons, blobs = split_blobs(buf, table[:, 1:], segids, ATTRIBUTES[:2 if vertex_types else 1])
  return dict(zip(segids, zip(skeletons, blobs)))


def postprocess(skeleton, dust_threshold=1500, tick_threshold=3000, ctx=None):
  """Drop-in for kimimaro.postprocess: consolidate, remove dust, break loops, connect nearby pieces and trim
  ticks (DESIGN.md §5h), on the device through the batched entry point.  Returns a new Skeleton."""
  segid = skeleton.id
  return merge_fragments({segid: [(None, skeleton)]}, dust_threshold=dust_threshold, tick_threshold=tick_threshold,
                         ctx=ctx)[segid][0]


def cross_sectional_area(all_labels, skeletons, anisotropy=(1, 1, 1), smoothing_window=1, progress=False,
                         in_place=False, fill_holes=False, repair_contacts=False, ctx=None):
  """Drop-in for kimimaro.cross_sectional_area (DESIGN.md §5i): at every vertex of every skeleton, the area
  (float32, physical units squared) of the section of its label through the vertex's voxel across the skeleton's
  smoothed direction there, and the faces of the array that section touches (uint8: bit 0 x = 0, 1 x = sx - 1,
  2 y = 0, 3 y = sy - 1, 4 z = 0, 5 z = sz - 1), as cross_sectional_area and cross_sectional_area_contacts.
  skeletons: {label: Skeleton}, a list of Skeletons or one Skeleton (the label is its id); the result has the
  same shape, the caller's objects when in_place, else new Skeletons with copies of the arrays in their own
  dtypes.  A label the array's dtype cannot hold raises ValueError.  `progress` is
  accepted and ignored; fill_holes and repair_contacts raise NotImplementedError.  last_phase_seconds holds
  the host-clock time of each phase of the last call."""
  if fill_holes or repair_contacts:
    raise NotImplementedError("igneous_b200 kimimaro.cross_sectional_area: fill_holes and repair_contacts are not "
                              "supported")
  arr = np.asarray(all_labels)
  if arr.ndim != 3:
    raise ValueError("kimimaro.cross_sectional_area: expected a 3-D label array, got shape %r" % (arr.shape,))
  if not (arr.dtype == np.bool_ or arr.dtype.kind in "iu"):
    raise NotImplementedError("igneous_b200 kimimaro.cross_sectional_area: label dtype %s is not supported"
                              % arr.dtype)
  a = tuple(float(v) for v in anisotropy)
  if len(a) != 3 or not all(np.isfinite(v) and v > 0 for v in a):
    raise ValueError("kimimaro.cross_sectional_area: anisotropy %r must be three positive finite values"
                     % (anisotropy,))
  w = smoothing_window
  if isinstance(w, (bool, np.bool_)) or not isinstance(w, (int, np.integer)) or w < 1:
    raise ValueError("kimimaro.cross_sectional_area: smoothing_window %r must be an integer >= 1" % (w,))
  last_phase_seconds.clear()
  last_stats[:] = [0, 0, 0, 0]
  t0 = time.perf_counter()

  def phase(name):
    nonlocal t0
    t = time.perf_counter()
    last_phase_seconds[name] = t - t0
    t0 = t

  if isinstance(skeletons, Skeleton):
    items = [(skeletons.id, skeletons)]
  elif isinstance(skeletons, dict):
    items = list(skeletons.items())
  else:
    items = [(s.id, s) for s in skeletons]
  verts = [np.asarray(s.vertices).reshape(-1, 3) for _, s in items]
  edges = [np.asarray(s.edges).reshape(-1, 2) for _, s in items]
  counts = np.array([len(v) for v in verts], np.int64)
  bounds = np.concatenate([[0], np.cumsum(counts)])
  V = int(bounds[-1])
  vall = np.concatenate(verts).astype(np.float64) if V else np.zeros((0, 3))
  c = np.rint(vall / np.array(a, np.float64))
  shape = np.array(arr.shape, np.int64)
  bad = np.nonzero(~np.all(np.isfinite(c) & (c >= 0) & (c < shape), axis=1))[0]
  if bad.size:
    k = int(np.searchsorted(bounds, bad[0], side="right")) - 1
    raise ValueError("kimimaro.cross_sectional_area: vertex %d %r of label %r lies outside the array of shape %r"
                     % (int(bad[0] - bounds[k]), tuple(float(x) for x in vall[bad[0]]), items[k][0], arr.shape))
  ecounts = np.array([len(e) for e in edges], np.int64)
  eall = np.concatenate(edges).astype(np.int64) if ecounts.sum() else np.zeros((0, 2), np.int64)
  local_max = np.repeat(counts, ecounts)
  wrong = np.nonzero((eall.min(axis=1) < 0) | (eall.max(axis=1) >= local_max))[0] if eall.size else []
  if len(wrong):
    k = int(np.searchsorted(np.cumsum(ecounts), wrong[0], side="right"))
    raise ValueError("kimimaro.cross_sectional_area: label %r has an edge index outside its %d vertices"
                     % (items[k][0], counts[k]))
  vox = np.ascontiguousarray(c, dtype=np.int64)
  edg = np.ascontiguousarray(eall + np.repeat(bounds[:-1], ecounts)[:, None], dtype=np.uint32)
  unsigned = _UNSIGNED[arr.dtype.itemsize]
  # a label outside the array's dtype would wrap onto another label: refuse it
  lo, hi = (0, 1) if arr.dtype == np.bool_ else (int(np.iinfo(arr.dtype).min), int(np.iinfo(arr.dtype).max))
  keys = []
  for label, _ in items:
    if not isinstance(label, (bool, int, np.bool_, np.integer)) or not lo <= int(label) <= hi:
      raise ValueError("kimimaro.cross_sectional_area: label %r is not an integer the array's dtype %s holds"
                       % (label, arr.dtype))
    keys.append(int(label))
  values = np.array(keys, np.int64 if lo < 0 else np.uint64).astype(arr.dtype).view(unsigned).astype(np.uint64)
  lab = np.ascontiguousarray(np.repeat(values, counts))
  if not in_place:
    def copied(parts):
      """copies of the caller's arrays in their own dtypes: views into one buffer when they share a dtype"""
      arrays = [None if p is None else np.asarray(p) for p in parts]
      kinds = {(p.dtype, p.shape[1:]) for p in arrays if p is not None and p.ndim}
      if not arrays or len(kinds) != 1 or any(p is None or not p.ndim for p in arrays):
        return [None if p is None else np.array(p, copy=True) for p in arrays]
      ends = np.cumsum([len(p) for p in arrays])
      flat = np.concatenate(arrays)
      return [flat[e - len(p):e] for p, e in zip(arrays, ends)]
    cv, ce, cr, ct = (copied([getattr(s, f) for _, s in items]) for f in ("vertices", "edges", "radii", "vertex_types"))
    items = [(label, Skeleton(v, e, r, t, s.id)) for (label, s), v, e, r, t in zip(items, cv, ce, cr, ct)]
  area, contacts = np.zeros(V, np.float32), np.zeros(V, np.uint8)
  if V:
    ctx = ctx or _shim.default_context()
    lib, h, ptr = ctx.lib, ctx.handle, _shim.ptr
    vol = np.asfortranarray(arr.view(unsigned))
    ca = (ctypes.c_double * 3)(*a)
    bufs = []
    try:
      bufs.append(ctx.alloc(vol.nbytes))
      d_vol = bufs[-1]
      ctx.h2d(d_vol, vol)
      ctx.sync()
      phase("upload")
      normals = np.empty((V, 3), np.float64)
      _shim.check(lib.ign_cross_section_normals(V, ptr(vox), edg.shape[0], ptr(edg), ca, int(w), ptr(normals)))
      phase("normals")
      lin = np.ascontiguousarray(vox[:, 0] + shape[0] * (vox[:, 1] + shape[1] * vox[:, 2]), dtype=np.uint64)
      d = []
      for host in (lin, lab, normals):
        bufs.append(ctx.alloc(host.nbytes))
        d.append(bufs[-1])
        ctx.h2d(d[-1], host)
      bufs.append(ctx.alloc(V * 4))
      d_area = bufs[-1]
      bufs.append(ctx.alloc(V))
      d_contacts = bufs[-1]
      stats = (ctypes.c_uint64 * 4)()
      _shim.check(lib.ign_cross_section_dev(h, ptr(d_vol), _shim.dtype_code(vol.dtype), *vol.shape, ptr(d[0]),
                                            ptr(d[1]), ptr(d[2]), V, ca, ptr(d_area), ptr(d_contacts), stats))
      phase("sections")
      ctx.d2h(area, d_area)
      ctx.d2h(contacts, d_contacts)
      ctx.sync()
      last_stats[:] = [int(x) for x in stats]
    finally:
      for b in bufs:
        b.free()
  for (label, s), b, e in zip(items, bounds[:-1], bounds[1:]):
    s.cross_sectional_area = area[b:e]  # views into one array per call
    s.cross_sectional_area_contacts = contacts[b:e]
  if V:
    phase("copy_back")
  if isinstance(skeletons, Skeleton):
    return items[0][1]
  if isinstance(skeletons, dict):
    return dict(items)
  return [s for _, s in items]
