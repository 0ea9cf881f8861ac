"""Drop-in for the `fastremap` calls on the igneous hot path, running on H100.

Reference call sites (seung-lab/igneous):
  igneous/tasks/mesh/mesh.py:201      fastremap.mask_except(data, object_ids, in_place=True)
  igneous/tasks/mesh/mesh.py:204      fastremap.mask(data, exclude_object_ids, in_place=True)
  igneous/tasks/mesh/mesh.py:206      fastremap.renumber(data, in_place=True)
  igneous/tasks/mesh/mesh.py:318-320  fastremap.unique(data, return_counts=True) / mask
  igneous/tasks/mesh/mesh.py:368-369  fastremap.mask_except / remap
  igneous/tasks/image/ccl.py:280      fastremap.inverse_component_map(cur_i, prev_i)
  igneous/tasks/image/ccl.py:283      fastremap.unique(adj_labels)
  igneous/tasks/image/ccl.py:346      fastremap.remap(cc_labels, mapping, in_place=True)
  igneous/task_creation/image.py:1832 fastremap.fit_dtype(np.uint64, max_label)
"""
import ctypes

import numpy as np

from . import _shim

__all__ = ["renumber", "remap", "unique", "mask", "mask_except",
           "inverse_component_map", "fit_dtype"]


def fit_dtype(dtype, value, exotics=False):
  """Smallest unsigned integer dtype that holds `value`."""
  value = int(value)
  for dt in (np.uint8, np.uint16, np.uint32, np.uint64):
    if 0 <= value <= np.iinfo(dt).max:
      return np.dtype(dt)
  raise ValueError("Unable to find a dtype for %r" % (value,))


def _order(a):
  return "F" if (a.flags.f_contiguous and not a.flags.c_contiguous) else "C"


def _contig(arr):
  """array -> (contiguous array in its own memory order, order)"""
  a = np.asarray(arr)
  if not (a.flags.c_contiguous or a.flags.f_contiguous):
    a = np.ascontiguousarray(a)
  return a, _order(a)


def _u64(values):
  return np.ascontiguousarray(np.asarray(list(values) if not isinstance(values, np.ndarray) else values,
                                         dtype=np.uint64))


def renumber(arr, start=1, preserve_zero=True, in_place=False, ctx=None):
  """Relabel to start..start+K-1 in order of first appearance in memory order;
  0 is preserved.  Returns (renumbered array of the smallest fitting unsigned
  dtype, {old: new})."""
  if start != 1 or not preserve_zero:
    raise NotImplementedError("igneous_b200.fastremap.renumber: only start=1, preserve_zero=True")
  a, order = _contig(arr)
  if a.dtype == np.bool_:
    a = a.view(np.uint8)
  n = a.size
  out = np.zeros(n, dtype=np.uint32)
  k = ctypes.c_uint64(0)
  uniq = np.zeros(max(n, 1), dtype=np.uint64)
  if n:
    ctx = ctx or _shim.default_context()
    _shim.check(ctx.lib.ign_renumber(ctx.handle, _shim.ptr(a), _shim.dtype_code(a.dtype), n, _shim.ptr(out),
                                     _shim.ptr(uniq), uniq.size, ctypes.byref(k)))
  K = int(k.value)
  mapping = {int(u): i + 1 for i, u in enumerate(uniq[:K])}
  if n and (out == 0).any():
    mapping[0] = 0
  res = out.astype(fit_dtype(np.uint64, K), copy=False).reshape(a.shape, order=order)
  return res, mapping


def remap(arr, table, preserve_missing_labels=False, in_place=False, ctx=None):
  """arr[i] = table[arr[i]]; KeyError on a label missing from the table unless
  preserve_missing_labels."""
  src = np.asarray(arr)
  a, order = _contig(src)
  work = a if (in_place and a is src) else a.copy(order=order)
  if work.size:
    keys = _u64(table.keys())
    vals = _u64(table.values())
    ctx = ctx or _shim.default_context()
    _shim.check(ctx.lib.ign_remap(ctx.handle, _shim.ptr(work), _shim.dtype_code(work.dtype), work.size,
                                  _shim.ptr(keys), _shim.ptr(vals), len(keys), bool(preserve_missing_labels)))
  if in_place and work is not src:
    src[...] = work.reshape(src.shape, order=order)
    return src
  return work


def unique(arr, return_counts=False, ctx=None):
  """Sorted unique labels (and their voxel counts)."""
  a, _ = _contig(arr)
  if a.dtype == np.bool_:
    a = a.view(np.uint8)
  n = a.size
  if n == 0:
    e = np.zeros(0, dtype=a.dtype)
    return (e, np.zeros(0, dtype=np.uint64)) if return_counts else e
  ctx = ctx or _shim.default_context()
  code = _shim.dtype_code(a.dtype)
  k = ctypes.c_uint64(0)
  _shim.check(ctx.lib.ign_unique(ctx.handle, _shim.ptr(a), code, n, None, None, 0, ctypes.byref(k)))
  K = int(k.value)
  uniq = np.zeros(K, dtype=np.uint64)
  counts = np.zeros(K, dtype=np.uint64)
  _shim.check(ctx.lib.ign_unique(ctx.handle, _shim.ptr(a), code, n, _shim.ptr(uniq),
                                 _shim.ptr(counts), K, ctypes.byref(k)))
  uniq = uniq.astype(a.dtype)
  return (uniq, counts) if return_counts else uniq


def _mask(arr, labels, in_place, value, except_, ctx):
  src = np.asarray(arr)
  a, order = _contig(src)
  work = a if (in_place and a is src) else a.copy(order=order)
  if work.size:
    lab = _u64(labels)
    ctx = ctx or _shim.default_context()
    _shim.check(ctx.lib.ign_mask(ctx.handle, _shim.ptr(work), _shim.dtype_code(work.dtype), work.size,
                                 _shim.ptr(lab), len(lab), bool(except_), int(value)))
  if in_place and work is not src:
    src[...] = work.reshape(src.shape, order=order)
    return src
  return work


def mask(arr, labels, in_place=False, value=0, ctx=None):
  """Set every voxel whose label is in `labels` to `value`."""
  return _mask(arr, labels, in_place, value, False, ctx)


def mask_except(arr, labels, in_place=False, value=0, ctx=None):
  """Set every voxel whose label is NOT in `labels` to `value`."""
  return _mask(arr, labels, in_place, value, True, ctx)


def inverse_component_map(parent_labels, component_labels, ctx=None):
  """{parent label: sorted unique component labels seen at the same positions}."""
  p = np.ascontiguousarray(np.asarray(parent_labels)).ravel()
  c = np.ascontiguousarray(np.asarray(component_labels)).ravel()
  if p.size != c.size:
    raise ValueError("parent and component label arrays must have the same size")
  if p.size == 0:
    return {}
  dt = np.promote_types(p.dtype, c.dtype)
  if dt.kind not in "ub":
    dt = np.dtype(np.uint64)
  p = np.ascontiguousarray(p.astype(dt, copy=False))
  c = np.ascontiguousarray(c.astype(dt, copy=False))
  ctx = ctx or _shim.default_context()
  pairs = np.zeros((p.size, 2), dtype=np.uint64)
  n_pairs = ctypes.c_uint64(p.size)
  _shim.check(ctx.lib.ign_inverse_component_map(ctx.handle, _shim.ptr(p), _shim.ptr(c), _shim.dtype_code(dt), p.size,
                                                _shim.ptr(pairs), ctypes.byref(n_pairs)))
  out = {}
  for a, b in pairs[:int(n_pairs.value)]:
    out.setdefault(int(a), []).append(int(b))
  return out
