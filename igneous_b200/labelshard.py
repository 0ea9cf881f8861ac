"""Hashed label shards on the GPU (igneous_b200/csrc/labelshard.cu, DESIGN.md §5l): the shard and minishard
of every label of a layer, and the skeletons of one shard re-encoded without their integer attributes and,
for raw data, assembled into the shard file on the device.  There is no CPU fallback."""
import ctypes

import numpy as np

from . import _shim


def shard_hash(labels, preshift_bits, minishard_bits, shard_bits, ctx=None):
  """ign_shard_hash_dev on a host array of labels -> (labels sorted by (shard, minishard, label), the location
  (shard << minishard_bits) | minishard of each, run starts (one per shard present, then len(labels)), the
  shard of each run)"""
  labels = np.ascontiguousarray(labels, dtype=np.uint64).ravel()
  n = labels.size
  ctx = ctx or _shim.default_context()
  lib, ptr = ctx.lib, _shim.ptr
  runs = min(n, 1 << min(int(shard_bits), 40))
  bufs = [ctx.alloc(max(8 * n, 8)) for _ in range(3)] + [ctx.alloc(8 * (runs + 1)), ctx.alloc(max(8 * runs, 8))]
  try:
    d_in, d_lab, d_loc, d_start, d_shard = bufs
    if n:
      ctx.h2d(d_in, labels)
    nr = ctypes.c_uint64(0)
    _shim.check(lib.ign_shard_hash_dev(ctx.handle, ptr(d_in), n, int(preshift_bits), int(minishard_bits),
                                       int(shard_bits), ptr(d_lab), ptr(d_loc), ptr(d_start), ptr(d_shard),
                                       ctypes.byref(nr)))
    k = int(nr.value)
    out_lab, out_loc = np.empty(n, np.uint64), np.empty(n, np.uint64)
    starts, shards = np.empty(k + 1, np.uint64), np.empty(k, np.uint64)
    for arr, buf in ((out_lab, d_lab), (out_loc, d_loc), (starts, d_start), (shards, d_shard)):
      if arr.size:
        ctx.d2h(arr, buf)
    ctx.sync()
  finally:
    for b in bufs:
      b.free()
  return out_lab, out_loc, starts, shards


def attribute_table(attributes, keep=("float32", "float64")):
  """HOST uint32 [n][2] of ign_skeleton_restrip_dev: (bytes per vertex, keep) of each vertex attribute"""
  rows = [(np.dtype(a["data_type"]).itemsize * int(a.get("num_components", 1)), a["data_type"] in keep)
          for a in attributes]
  return np.array(rows, dtype=np.uint32).reshape(-1, 2)


def restrip(blobs, attributes, locations=None, labels=None, minishard_bits=0, ctx=None):
  """The precomputed skeleton blobs (bytes, in (minishard, label) order) without their integer attributes, in
  one device pass.  attributes: the source's vertex_attributes.  Without locations -> (uint8 array of the
  re-encoded blobs back to back, their n + 1 offsets).  With locations and labels (uint64, one per blob) ->
  the whole raw shard file as bytes, assembled on the device and copied back once.  A blob that does not
  match its header and the attributes raises ValueError naming its row."""
  n = len(blobs)
  attrs = attribute_table(attributes)
  offs = np.zeros(n + 1, np.uint64)
  np.cumsum([len(b) for b in blobs], out=offs[1:])
  total = int(offs[-1])
  index_len = 16 << int(minishard_bits) if locations is not None else 0
  capacity = index_len + total + (24 * n if locations is not None else 0)
  ctx = ctx or _shim.default_context()
  lib, ptr = ctx.lib, _shim.ptr
  bufs = [ctx.alloc(max(total, 8)), ctx.alloc(8 * (n + 1)), ctx.alloc(8 * (n + 1)), ctx.alloc(max(capacity, 8))]
  try:
    d_in, d_off, d_out_off, d_out = bufs
    if total:
      ctx.h2d(d_in, np.frombuffer(b"".join(blobs), np.uint8))
    ctx.h2d(d_off, offs)
    nb = ctypes.c_uint64(0)
    try:
      _shim.check(lib.ign_skeleton_restrip_dev(ctx.handle, ptr(d_in), ptr(d_off), n, ptr(attrs), len(attrs),
                                               d_out.offset(index_len), capacity - index_len, ptr(d_out_off),
                                               ctypes.byref(nb)))
    except _shim.IgneousB200Error as e:
      if e.status == -2:
        raise ValueError(str(e)) from e
      raise
    if locations is None:
      out, out_offs = np.empty(max(int(nb.value), 1), np.uint8), np.empty(n + 1, np.uint64)
      ctx.d2h(out, d_out, int(nb.value))
      ctx.d2h(out_offs, d_out_off)
      ctx.sync()
      return out[:int(nb.value)], out_offs
    d_loc, d_lab = ctx.alloc(max(8 * n, 8)), ctx.alloc(max(8 * n, 8))
    bufs += [d_loc, d_lab]
    if n:
      ctx.h2d(d_loc, np.ascontiguousarray(locations, dtype=np.uint64))
      ctx.h2d(d_lab, np.ascontiguousarray(labels, dtype=np.uint64))
    _shim.check(lib.ign_shard_assemble_dev(ctx.handle, ptr(d_loc), ptr(d_lab), ptr(d_out_off), n,
                                           int(minishard_bits), ptr(d_out), capacity, ctypes.byref(nb)))
    shard = np.empty(int(nb.value), np.uint8)
    ctx.d2h(shard, d_out)
    ctx.sync()
    return shard.tobytes()
  finally:
    for b in bufs:
      b.free()
