"""Drop-in for the `fastmorph` calls of MeshTask(fill_holes=N), running on H100.

Reference call sites (seung-lab/igneous):
  igneous/tasks/mesh/mesh.py:211-218  fastmorph.dilate(data, mode=fastmorph.Mode.multilabel,
                                        background_only=True, parallel=1)
  igneous/tasks/mesh/mesh.py:220-228  fastmorph.fill_holes_v2(data, return_crackle=True,
                                        fix_borders=(fill_level >= 2), merge_threshold=..., parallel=1)

fastmorph itself is not available offline, so these compute the rule stated in DESIGN.md
"Hole filling" (parity with fastmorph is unpinned).  fill_holes_v2 returns numpy arrays:
there is no crackle codec here, so return_crackle=True is refused.
"""
import enum

import numpy as np

from . import _shim

__all__ = ["Mode", "dilate", "fill_holes_v2"]


class Mode(enum.Enum):
  multilabel = 0
  grey = 1


def _volume(labels, what):
  arr = np.asarray(labels)
  if arr.dtype == np.bool_:
    arr = arr.view(np.uint8)
  _shim.require_unsigned(arr.dtype, what)
  if arr.dtype.kind != "u":
    raise NotImplementedError("igneous_b200 %s: unsupported dtype %s" % (what, arr.dtype))
  if arr.ndim == 2:
    arr = arr[:, :, np.newaxis]
  if arr.ndim != 3:
    raise ValueError("%s expects a 2- or 3-D array, got shape %r" % (what, arr.shape))
  return np.asfortranarray(arr)


def dilate(labels, mode=Mode.multilabel, background_only=True, parallel=1, ctx=None):
  """One multilabel dilation step of the background: every 0 voxel with a non-zero voxel among
  its 26 neighbours takes their most frequent non-zero label (ties to the smaller label)."""
  if mode != Mode.multilabel:
    raise NotImplementedError("igneous_b200.fastmorph.dilate: only mode=Mode.multilabel")
  if not background_only:
    raise NotImplementedError("igneous_b200.fastmorph.dilate: only background_only=True")
  arr = _volume(labels, "fastmorph.dilate")
  out = np.empty_like(arr, order="F")
  if arr.size:
    ctx = ctx or _shim.default_context()
    sx, sy, sz = arr.shape
    _shim.check(ctx.lib.ign_dilate_multilabel(ctx.handle, _shim.ptr(arr), _shim.dtype_code(arr.dtype), sx, sy, sz,
                                              _shim.ptr(out)))
  return out.reshape(np.shape(labels)) if np.ndim(labels) == 2 else out


def merge_threshold_pct(merge_threshold):
  """merge_threshold in [0, 1] as a whole percentage; anything finer is refused, because the
  rule compares contact counts exactly in integers."""
  pct = round(float(merge_threshold) * 100)
  if not (0 <= pct <= 100) or abs(float(merge_threshold) * 100 - pct) > 1e-6:
    raise ValueError("merge_threshold must be a whole percentage in [0, 1], got %r" % (merge_threshold,))
  return int(pct)


def fill_holes_v2(labels, return_crackle=False, fix_borders=False, merge_threshold=1.0, parallel=1, ctx=None):
  """(filled, holes): every region enclosed by a non-zero region takes the label of the
  enclosing region nearest the outside; holes keeps the input where it was overwritten."""
  if return_crackle:
    raise NotImplementedError("igneous_b200.fastmorph.fill_holes_v2: return_crackle=True "
                              "(there is no crackle codec here)")
  pct = merge_threshold_pct(merge_threshold)
  arr = _volume(labels, "fastmorph.fill_holes_v2")
  filled = np.empty_like(arr, order="F")
  holes = np.empty_like(arr, order="F")
  if arr.size:
    ctx = ctx or _shim.default_context()
    sx, sy, sz = arr.shape
    _shim.check(ctx.lib.ign_fill_holes(ctx.handle, _shim.ptr(arr), _shim.dtype_code(arr.dtype), sx, sy, sz,
                                       bool(fix_borders), pct, _shim.ptr(filled), _shim.ptr(holes)))
  if np.ndim(labels) == 2:
    return filled.reshape(np.shape(labels)), holes.reshape(np.shape(labels))
  return filled, holes
