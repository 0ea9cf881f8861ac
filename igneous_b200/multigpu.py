"""Multi-GPU CCL: one process per GPU, every rank holds one z-slab of the
dataset (rank r above rank r-1), and ONE all-gather of the ranks' outer planes
replaces the face / equivalence / relabel files of
igneous/tasks/image/ccl.py:177-194, :245-294 and :358-420.

  1. each rank resolves its own volume and exposes its first and last z-plane
     as (voxel value, volume-local id);
  2. all ranks all-gather [n_local | first plane | last plane]  (NCCL over
     NVLink / NVSwitch; ~48 MB per rank for 2048^2 planes);
  3. every rank links the N-1 rank boundaries straight into a union-find over the
     dataset-wide provisional ids (k_ccl_link_union), solves it (smaller id wins,
     final ids by ascending minimum) and expands its slab once -- all on the device,
     inside ign_ccl6_sharded_dev.  solve_global / solve_pairs / link_planes_numpy
     below are the host statement of the same steps (CPU tests, world_size-2 gloo).
The result is bit-identical to one whole-volume cc3d call on the stacked
dataset.  Downsampling and meshing need no communication (replicas).
"""
import ctypes as c

import numpy as np

from . import _shim


def plane_record_bytes(n_plane):
  """[n_local u64 (padded to 256 B) | first values u64 | last values u64 | first ids u32 | last ids u32]"""
  return 256 + 2 * n_plane * 8 + 2 * n_plane * 4


def solve_global(n_locals, link_boundary, solve):
  """Host orchestration shared by the GPU path and the CPU (gloo) tests.

  n_locals[r]      components of rank r's volume
  link_boundary(r, off_lo, off_hi) -> uint64 [k,2] equivalence pairs between the last
                   plane of rank r and the first plane of rank r+1, already offset
  solve(pairs, total) -> (lut uint32 [total+1], n_global)
  Returns (offsets per rank, lut, n_global)."""
  offs = np.concatenate([[0], np.cumsum(np.asarray(n_locals, dtype=np.uint64))]).astype(np.uint64)
  pairs = [np.zeros((0, 2), dtype=np.uint64)]
  for r in range(len(n_locals) - 1):
    pairs.append(np.asarray(link_boundary(r, int(offs[r]), int(offs[r + 1])), dtype=np.uint64).reshape(-1, 2))
  pairs = np.ascontiguousarray(np.concatenate(pairs))
  lut, n_global = solve(pairs, int(offs[-1]))
  return offs, lut, n_global


def solve_pairs(pairs, total):
  """ign_ccl6_solve: host union-find, smaller id wins, final ids by ascending minimum."""
  lib = _shim.load()
  lut = np.zeros(total + 1, dtype=np.uint32)
  n = c.c_uint64(0)
  pairs = np.ascontiguousarray(pairs, dtype=np.uint64)
  _shim.check(lib.ign_ccl6_solve(_shim.ptr(pairs) if len(pairs) else None, len(pairs), total, _shim.ptr(lut),
                                 c.byref(n)))
  return lut, int(n.value)


def link_planes_numpy(va, la, off_a, vb, lb, off_b):
  """numpy statement of k_ccl_link (CPU tests): pairs where both planes hold the
  same non-zero value at the same (x,y)."""
  va, vb = np.asarray(va).ravel(), np.asarray(vb).ravel()
  m = (va != 0) & (va == vb)
  a = np.asarray(la).ravel()[m].astype(np.uint64) + np.uint64(off_a)
  b = np.asarray(lb).ravel()[m].astype(np.uint64) + np.uint64(off_b)
  if len(a) == 0:
    return np.zeros((0, 2), dtype=np.uint64)
  return np.unique(np.stack([a, b], axis=1), axis=0)


class Group:
  """NCCL communicator of the C library + the orchestration above."""

  def __init__(self, ctx, rank, world, dist=None, unique_id=None):
    self.ctx, self.rank, self.world = ctx, rank, world
    self.lib = ctx.lib
    if unique_id is None:
      uid = (c.c_uint8 * 128)()
      if rank == 0:
        _shim.check(self.lib.ign_group_unique_id(uid))
      box = [bytes(uid)]
      if dist is None:
        raise ValueError("Group needs torch.distributed (to broadcast the NCCL id) or an explicit unique_id")
      dist.broadcast_object_list(box, src=0)
      unique_id = box[0]
    buf = (c.c_uint8 * 128).from_buffer_copy(unique_id)
    h = c.c_void_p()
    _shim.check(self.lib.ign_group_init(ctx.handle, rank, world, buf, c.byref(h)))
    self.handle = h
    self._bufs = None

  def close(self):
    if self.handle is not None:
      self.lib.ign_group_destroy(self.handle)
      self.handle = None

  def _buffers(self, n_plane):
    rec = plane_record_bytes(n_plane)
    if self._bufs is None or self._bufs[0] != rec:
      self._bufs = (rec, self.ctx.alloc(rec), self.ctx.alloc(rec * self.world))
    return self._bufs

  def ccl_sharded(self, pipe, _unused=None):
    """CCL of pipe.d_in (this rank's slab) -> pipe.d_cc with dataset-wide ids; returns the
    global number of components.  One C call (ign_ccl6_sharded_dev): local CCL, ONE NCCL
    all-gather of the boundary planes, then linking, the replicated union-find and the
    relabelling on the device of every rank."""
    sx, sy, sz = pipe.shape
    n = c.c_uint64(0)
    _shim.check(self.lib.ign_ccl6_sharded_dev(
      self.handle, _shim.ptr(pipe.d_in), pipe.code, sx, sy, sz,
      _shim.ptr(pipe.d_cc), _shim.dtype_code(pipe.ccl_out_dtype), c.byref(n)))
    return int(n.value)
