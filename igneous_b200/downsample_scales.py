"""Host-side scale arithmetic of the downsample path (pure Python, no kernels).

Mirrors the functions of igneous/downsample_scales.py that sit on the hot path:
  compute_factors        :135-172   how many mips one task produces
  axis_to_factor         :174-182
  compute_scales         :184-212
  create_downsample_scales :214-244 adds the new scales to the info file
  downsample_shape_from_memory_target :280-358 the task shape of a transfer
"""
import copy
import math

import numpy as np

from ._compat import CloudVolume, Vec, min2


def axis_to_factor(axis):
  table = {"x": (1, 2, 2), "y": (2, 1, 2), "z": (2, 2, 1)}
  if axis not in table:
    raise ValueError("Axis not supported: " + str(axis))
  return table[axis]


def compute_factors(ds_shape, factor, chunk_size, volume_size):
  """[factor] * N where N is the number of downsamples the least tolerant
  pooled axis allows for this task shape (float32 arithmetic and the +1e-4
  guard as in the reference; a partial last level is allowed only when the
  whole volume is already smaller than a chunk)."""
  pooled = [i for i, f in enumerate(factor) if f != 1]
  if not pooled:
    return []
  grid = np.array([ds_shape[i] for i in pooled], dtype=np.float32) / \
      np.array([chunk_size[i] for i in pooled], dtype=np.float32)
  fdiv = np.array([factor[i] for i in pooled], dtype=np.float32)
  eps = 0.0001
  n_float = float(np.min(np.log(grid) / np.log(fdiv) + np.float32(eps)))
  if n_float < eps:
    return []
  dsvol = np.array(volume_size, dtype=np.float64) / (np.array(factor, dtype=np.float64) ** int(math.ceil(n_float)))
  small = all(dsvol[i] < chunk_size[i] for i in pooled)
  n = int(n_float)
  if small and (n_float - n) > 0.05:
    n += 1
  return [tuple(factor)] * n


def _precision(x):
  s = repr(float(x))
  return len(s.split(".")[1].rstrip("0")) if "." in s else 0


def compute_scales(vol, mip, shape, axis, factor, chunk_size=None):
  shape = min2(vol.meta.volume_size(mip), shape)
  underlying = (mip + 1) if (mip + 1) in vol.available_mips else mip
  cs = np.asarray(chunk_size, dtype=np.float32) if chunk_size else \
      np.asarray(vol.meta.chunk_size(underlying), dtype=np.float32)
  if factor is None:
    factor = axis_to_factor(axis)
  factors = compute_factors(shape, factor, cs, vol.meta.volume_size(mip))
  base = [float(r) for r in vol.meta.resolution(mip)]
  prec = max(_precision(r) for r in base)
  scales, cur = [], base
  for f in factors:
    cur = [c * ff for c, ff in zip(cur, f)]
    scales.append([int(c) if prec == 0 else round(c, prec) for c in cur])
  return scales


def create_downsample_scales(layer_path, mip, ds_shape, axis="z", preserve_chunk_size=False,
                             chunk_size=None, encoding=None, factor=None, max_mips=None):
  vol = CloudVolume(layer_path, mip)
  resolutions = compute_scales(vol, mip, ds_shape, axis, factor, chunk_size)
  if max_mips is not None:
    resolutions = resolutions[:max_mips]
  if not resolutions:
    print("WARNING: No scales generated.")
  for res in resolutions:
    vol.meta.add_resolution(res, encoding=encoding, chunk_size=chunk_size)
  if chunk_size is None:
    src = mip if (preserve_chunk_size or not resolutions) else mip + 1
    new_cs = vol.scales[src]["chunk_sizes"]
  else:
    new_cs = [list(chunk_size)]
  for i in range(mip + 1, mip + len(resolutions) + 1):
    vol.scales[i]["chunk_sizes"] = new_cs
  vol.commit_info()
  return vol


def add_scales(layer_path, mip, num_mips, preserve_chunk_size=True, chunk_size=None, encoding=None, factor=None):
  """igneous/downsample_scales.py:246-278: append exactly `num_mips` scales above `mip`
  (no memory-driven truncation; used by the sharded downsample creator)."""
  vol = CloudVolume(layer_path, mip=mip)
  if factor is None:
    factor = (2, 2, 1)
  for _ in range(num_mips):
    res = [r * f for r, f in zip(vol.meta.resolution(mip), factor)]
    vol.meta.add_resolution(res, encoding=encoding, chunk_size=chunk_size)
    if chunk_size is None:
      new_cs = vol.scales[mip if preserve_chunk_size else mip + 1]["chunk_sizes"]
    else:
      new_cs = [list(chunk_size)]
    if encoding is None:
      encoding = vol.scales[mip]["encoding"]
    vol.scales[mip + 1]["chunk_sizes"] = copy.deepcopy(new_cs)
    mip += 1
    vol.mip = mip
  return vol


def downsample_shape_from_memory_target(data_width, cx, cy, cz, factor, byte_target, max_mips=float("inf")):
  """The task shape (whole chunks of cx x cy x cz voxels of `data_width` bytes) that yields the most
  downsamples while the task's image and its pyramid stay within `byte_target` bytes.

  factor (2,2,1): the pyramid adds a third, so the image may hold V = 3/4 * target / (w * cz) voxels
    per z-slab one chunk thick.  That budget is shared between x and y so that each axis's extent is
    its chunk size raised to one common power e: cx^e * cy^e = V.  Each axis then takes chunk * 2^k,
    k the integer part of log2(c^e / c), at most max_mips; z stays one chunk.
  factor (2,2,2): the same with V = 7/8 * target / w shared by x, y and z (cx^e * cy^e * cz^e = V).
    Non-square chunks thus get different doubling counts per axis.
  factor (1,1,1): no pyramid; a single chunk-thick slab of about byte_target bytes that is as square
    as whole chunks allow: n = floor(sqrt(target / (w*cx*cy*cz))) chunks in x, floor(n*cx/cy) in y.
  Example: uint64, 128 x 128 x 64 chunks, 3 GB, (2,2,1) -> 2048 x 2048 x 64 (2.9 GB with its pyramid)."""
  factor = tuple(int(f) for f in factor)
  if byte_target <= 0:
    raise ValueError("Unable to pick a shape for a byte budget <= 0. Got: %r" % (byte_target,))
  if cx * cy * cz <= 0:
    raise ValueError("Chunk size must have a positive integer volume. Got: <%r,%r,%r>" % (cx, cy, cz))
  chunk = (int(cx), int(cy), int(cz))
  if factor == (1, 1, 1):
    n = int(math.sqrt(byte_target / (float(data_width) * cx * cy * cz)))
    out = Vec(n * cx, int(n * cx / cy) * cy, cz)
  elif factor in ((2, 2, 1), (2, 2, 2)):
    pooled = 2 if factor == (2, 2, 1) else 3
    budget = 3.0 / 4.0 * byte_target / data_width / cz if pooled == 2 else 7.0 / 8.0 * byte_target / data_width
    prod = float(np.prod(chunk[:pooled]))
    ks = []
    for c in chunk[:pooled]:
      if prod == 1:  # the common power is undefined: an even split
        k = int(math.log2(budget ** (1.0 / pooled)))
      else:
        e = math.log(budget) / math.log(prod)
        k = int(math.log2((c ** e) / c))
      ks.append(int(min(k, max_mips)))
    out = Vec(*[c * 2.0 ** k for c, k in zip(chunk[:pooled], ks)] + ([cz] if pooled == 2 else []))
  else:
    raise ValueError("Only the factors (1,1,1), (2,2,1) and (2,2,2) are supported. Got: %r" % (factor,))
  out = out.astype(int)
  if np.any(np.asarray(out) < np.asarray(chunk)):
    raise ValueError("Too little memory allocated to create a valid task. Got: %r Predicted Shape: %r "
                     "Minimum Shape: %r" % (byte_target, list(out), list(chunk)))
  return out
