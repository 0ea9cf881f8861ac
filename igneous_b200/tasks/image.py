"""DownsampleTask / TransferTask with the pooling done on the GPU, and the other image tasks.

Same names, arguments and side effects as igneous/tasks/image/image.py:
  downsample_method_to_fn :37-55, downsample_and_upload :57-100,
  TransferTask :434-516, DownsampleTask :518-549, ImageShardTransferTask :595-670.
  ImageShardDownsampleTask :672-843, CountVoxelsTask :845-880.
  DeleteTask :103-122, BlackoutTask :124-135, TouchTask :137-143.
  QuantizeTask :145-162, CLAHETask :164-209, ContrastNormalizationTask :211-343,
  LuminanceLevelsTask :345-432 (per-voxel work in igneous_b200.contrast).
Only the library behind `fn(image, factors[0], num_mips=...)` (:91) changes:
igneous_b200.tinybrain instead of the CPU tinybrain wheel.
"""
import json
import math
import os
import random
from collections import defaultdict
from collections.abc import Sequence
from functools import partial

import numpy as np

from .. import contrast, downsample_scales, fastremap, sharding, shards, tinybrain
from .._compat import CloudVolume, CloudFiles, Bbox, EmptyVolumeException, Vec, min2, queueable, RegisteredTask
from ..storage import DeviceCutout
from ..types import DownsampleMethods


def downsample_method_to_fn(method, sparse, vol):
  if method == DownsampleMethods.AUTO:
    method = {"image": DownsampleMethods.AVERAGE_POOLING,
              "segmentation": DownsampleMethods.MODE_POOLING}.get(vol.layer_type, DownsampleMethods.STRIDING)
  if method == DownsampleMethods.AVERAGE_POOLING:
    return partial(tinybrain.downsample_with_averaging, sparse=sparse)
  if method == DownsampleMethods.MODE_POOLING:
    return partial(tinybrain.downsample_segmentation, sparse=sparse)
  if method == DownsampleMethods.MIN_POOLING:
    return tinybrain.downsample_with_min_pooling
  if method == DownsampleMethods.MAX_POOLING:
    return tinybrain.downsample_with_max_pooling
  return tinybrain.downsample_with_striding


def _method_kind(method, vol):
  """the pooling rule downsample_method_to_fn picks, by name (tinybrain.downsample_dev)"""
  if method == DownsampleMethods.AUTO:
    method = {"image": DownsampleMethods.AVERAGE_POOLING,
              "segmentation": DownsampleMethods.MODE_POOLING}.get(vol.layer_type, DownsampleMethods.STRIDING)
  return {DownsampleMethods.AVERAGE_POOLING: "average", DownsampleMethods.MODE_POOLING: "mode",
          DownsampleMethods.MIN_POOLING: "min", DownsampleMethods.MAX_POOLING: "max"}.get(method, "striding")


def downsample_and_upload(image, bounds, vol, ds_shape, mip=0, axis="z", skip_first=False,
                          sparse=False, factor=None, max_mips=None, method=DownsampleMethods.AUTO):
  """Write `image` (a host array or a DeviceCutout) at `bounds` and its pyramid above it.  The image
  goes to the device once; the mips are pooled, cut and encoded there (tinybrain.downsample_dev,
  the layer's upload_dev)."""
  ds_shape = min2(vol.meta.volume_size(mip), Vec(*ds_shape[:3]))
  underlying = (mip + 1) if (mip + 1) in vol.available_mips else mip
  chunk = np.asarray(vol.meta.chunk_size(underlying), dtype=np.float32)
  if factor is None:
    factor = downsample_scales.axis_to_factor(axis)
  factors = downsample_scales.compute_factors(ds_shape, factor, chunk, vol.meta.volume_size(mip))
  if max_mips is not None:
    factors = factors[:max_mips]
  vol.mip = mip
  if not isinstance(image, DeviceCutout) and not (skip_first and not factors):
    image = DeviceCutout.from_host(image)  # pooled in its own dtype, converted to the layer's on upload
  if not skip_first:
    vol.upload_dev(bounds, image, mip=mip)
  if not factors:
    return
  # <- the kernel call (image.py:91)
  mips = tinybrain.downsample_dev(image, _method_kind(method, vol), factors[0], len(factors), sparse=bool(sparse))
  box = bounds.clone()
  for f3, mipped in zip(factors, mips):
    vol.mip += 1
    box //= f3
    box.maxpt = box.minpt + Vec(*mipped.shape[:3])
    vol.upload_dev(box, mipped, mip=vol.mip)


@queueable
def TransferTask(src_path, dest_path, mip, shape, offset, translate=(0, 0, 0), fill_missing=False,
                 skip_first=False, skip_downsamples=False, delete_black_uploads=False,
                 background_color=0, sparse=False, axis="z", agglomerate=False, timestamp=None,
                 compress="gzip", factor=None, max_mips=None, stop_layer=None,
                 downsample_method=DownsampleMethods.AUTO, use_https_for_source=False):
  shape, offset, translate = Vec(*shape), Vec(*offset), Vec(*translate)
  src = CloudVolume(src_path, fill_missing=bool(fill_missing), mip=mip, bounded=False)
  dest = CloudVolume(dest_path, fill_missing=bool(fill_missing), mip=mip,
                     delete_black_uploads=bool(delete_black_uploads),
                     background_color=background_color, compress=compress)
  dst_box = Bbox.clamp(Bbox(offset, shape + offset), dest.meta.bounds(mip))
  if skip_downsamples and _same_chunks(src, dest, mip) and dest._sharding(mip) is None and not np.any(translate):
    # the files are copied as they are (image.py:483-496)
    src.image.transfer_to(dest_path, dst_box, mip, compress=compress)
    return
  image = src.download_dev(dst_box - translate)
  if skip_downsamples:
    dest.upload_dev(dst_box, image, mip=mip)
    return
  downsample_and_upload(image, dst_box, dest, shape, mip=mip, skip_first=bool(skip_first),
                        sparse=bool(sparse), axis=axis, factor=factor, max_mips=max_mips,
                        method=downsample_method)


def _same_chunks(src, dest, mip):
  """Can dest's chunk files at `mip` be src's files as they are?  The reference asks for the same
  chunk size and dtype; the stand-in copies files without decoding them, so it also asks for the same
  encoding (and its parameters), channel count and scale bounds: chunk names and the extent of the
  edge chunks follow each scale's own bounds, so a cropped destination needs its chunks re-cut."""
  a, b = src.scales[mip], dest.scales[mip]
  keys = ("encoding", "compressed_segmentation_block_size", "jpeg_quality")
  return (np.array_equal(src.meta.chunk_size(mip), dest.meta.chunk_size(mip)) and src.dtype == dest.dtype
          and src.num_channels == dest.num_channels and all(a.get(k) == b.get(k) for k in keys)
          and src.meta.bounds(mip) == dest.meta.bounds(mip))


@queueable
def ImageShardTransferTask(src_path, dst_path, shape, offset, mip=0, fill_missing=False, translate=(0, 0, 0),
                           agglomerate=False, timestamp=None, stop_layer=None, use_https_for_source=False):
  """One shard of a sharded copy of a layer at `mip`, without downsamples (image.py:595-670).  The
  box is expanded to whole chunks; when it needs no translation and the two scales have the same
  chunk grid and encoding, the source's encoded chunks go into the shard as they are, otherwise the cutout is built on the device
  and its chunks encoded there.  The shard file is written once."""
  if agglomerate or timestamp is not None or stop_layer is not None:
    raise NotImplementedError("ImageShardTransferTask: agglomerate / timestamp / stop_layer need a graphene source")
  shape, offset, translate = Vec(*shape), Vec(*offset), Vec(*translate)
  mip = int(mip)
  src = CloudVolume(src_path, fill_missing=bool(fill_missing), mip=mip, bounded=False)
  dst = CloudVolume(dst_path, fill_missing=bool(fill_missing), mip=mip, compress=None)
  dst_box = Bbox.clamp(Bbox(offset, offset + shape), dst.meta.bounds(mip))
  dst_box = dst_box.expand_to_chunk_size(dst.meta.chunk_size(mip), offset=dst.meta.voxel_offset(mip))
  src_box = dst_box - translate
  if src_box == dst_box and _same_chunks(src, dst, mip):
    shard_cache, chunks = {}, {}
    for c in dst._chunks(mip, Bbox.clamp(dst_box, dst.meta.bounds(mip))):
      data = src._read_chunk(mip, c, shard_cache)
      if data is None:
        if not fill_missing:
          raise EmptyVolumeException(src._chunk_name(mip, c))
        continue
      chunks[dst._chunk_id(mip, c)] = data
    if not chunks:
      return
    filename, shard = dst.image.make_shard(chunks, dst_box, mip)
  else:
    img = src.download_dev(src_box, mip=mip)
    filename, shard = dst.image.make_shard(img, dst_box, mip)
    del img
  CloudFiles(dst.meta.join(dst.cloudpath, dst.meta.key(mip))).put(filename, shard, compress=None)


@queueable
def DownsampleTask(layer_path, mip, shape, offset, fill_missing=False, axis="z", sparse=False,
                   delete_black_uploads=False, background_color=0, dest_path=None, compress="gzip",
                   factor=None, max_mips=None, method=DownsampleMethods.AUTO):
  """2x2x1 (by default) downsample pyramid of one cutout.  As in the reference
  the `method` argument is accepted but AUTO is what runs (image.py:524,548)."""
  return TransferTask(layer_path, dest_path or layer_path, mip, shape, offset, translate=(0, 0, 0),
                      fill_missing=fill_missing, skip_first=True, skip_downsamples=False,
                      delete_black_uploads=delete_black_uploads, background_color=background_color,
                      sparse=sparse, axis=axis, compress=compress, factor=factor, max_mips=max_mips,
                      downsample_method=DownsampleMethods.AUTO)


@queueable
def ImageShardDownsampleTask(src_path, shape, offset, mip=0, fill_missing=False, sparse=False,
                             agglomerate=False, timestamp=None, factor=(2, 2, 1),
                             method=DownsampleMethods.AUTO, num_mips=1, progress=False):
  """Downsample the region under one (stack of) output shard(s) and write whole shard files
  for mips mip+1 .. mip+num_mips (image.py:672-843).

  As in the reference the region is walked in z-layers one chunk thick at the coarsest
  mip; segmentation layers are renumbered to a small dtype before pooling and mapped back
  afterwards (renumber / pooling / remap run on the GPU).  Chunks are collected per output
  shard -- keyed by the shard number their chunk id hashes to, which for the identity hash
  is the reference's (shard_x, shard_y, shard_z) box -- and every shard is written once."""
  shape, offset = Vec(*shape), Vec(*offset)
  mip, num_mips = int(mip), int(num_mips)
  factor = tuple(int(f) for f in factor)
  src = CloudVolume(src_path, fill_missing=bool(fill_missing), mip=mip, bounded=False)
  chunk_size = src.meta.chunk_size(mip)
  bbox = Bbox.clamp(Bbox(offset, offset + shape), src.meta.bounds(mip))
  bbox = bbox.expand_to_chunk_size(chunk_size, offset=src.meta.voxel_offset(mip))

  def shard_shape_at(m):
    return shards.image_shard_shape_from_spec(src.scales[m]["sharding"], src.meta.volume_size(m),
                                              src.meta.chunk_size(m))

  first = shard_shape_at(mip + 1)
  upper = offset // Vec(*factor)
  upper_box = Bbox.clamp(Bbox(upper, upper + Vec(*[int(v) for v in first])), src.meta.bounds(mip + 1))
  if upper_box.subvoxel():
    return
  fn = downsample_method_to_fn(method, sparse, src)
  renumber = src.layer_type == "segmentation"
  cz = int(chunk_size[2]) * factor[2] ** num_mips
  nz = int(math.ceil(int(bbox.size3()[2]) / cz))
  f3 = np.asarray(factor, dtype=int)
  pending = [defaultdict(dict) for _ in range(num_mips)]  # per mip: shard grid position -> {chunk id: bytes}
  zbox = bbox.clone()
  zbox.maxpt[2] = zbox.minpt[2] + cz
  for _ in range(nz):
    if renumber:
      img, mapping = src.download(zbox, agglomerate=agglomerate, timestamp=timestamp, renumber=True)
      back = {int(new): int(old) for old, new in mapping.items()}
      back[src.background_color] = src.background_color
    else:
      img = src.download(zbox, agglomerate=agglomerate, timestamp=timestamp)
    mips = fn(img, factor, num_mips=num_mips)  # <- the kernel call (image.py:764)
    del img
    for i in range(num_mips):
      m = mip + i + 1
      cutout = mips[i]
      if renumber:
        cutout = fastremap.remap(cutout.astype(src.dtype), back, preserve_missing_labels=False)
      lo = np.asarray(zbox.minpt, dtype=int) // (f3 ** (i + 1))
      box = Bbox(lo, lo + np.asarray(cutout.shape[:3], dtype=int))
      bounds_m = src.meta.bounds(m)
      if box.minpt[2] >= bounds_m.maxpt[2]:
        continue
      sshape = np.asarray(shard_shape_at(m), dtype=int)
      origin = np.asarray(src.meta.voxel_offset(m), dtype=int)
      g0 = (np.asarray(box.minpt) - origin) // sshape
      g1 = -((-(np.asarray(box.maxpt) - origin)) // sshape)
      for gz in range(int(g0[2]), int(g1[2])):
        for gy in range(int(g0[1]), int(g1[1])):
          for gx in range(int(g0[0]), int(g1[0])):
            smin = origin + np.asarray([gx, gy, gz]) * sshape
            part = Bbox.intersection(Bbox(smin, smin + sshape), box)
            if part.subvoxel():
              continue
            sl = tuple(slice(int(a - o), int(b - o)) for a, b, o in zip(part.minpt, part.maxpt, box.minpt))
            pending[i][(gx, gy, gz)].update(_shard_chunks(src, cutout[sl], part, m))
    del mips
    zbox.minpt[2] += cz
    zbox.maxpt[2] += cz
  for i in range(num_mips):
    m = mip + i + 1
    sshape = np.asarray(shard_shape_at(m), dtype=int)
    origin = np.asarray(src.meta.voxel_offset(m), dtype=int)
    base = src.meta.join(src.cloudpath, src.meta.key(m))
    done = Bbox(np.asarray(bbox.minpt, dtype=int) // (f3 ** (i + 1)), -((-np.asarray(bbox.maxpt, dtype=int)) // (f3 ** (i + 1))))
    for grid_pos, chunk_dict in pending[i].items():
      smin = origin + np.asarray(grid_pos) * sshape
      shard_box = Bbox(smin, smin + sshape)
      inside = Bbox.clamp(shard_box, src.meta.bounds(m))
      if not (np.all(inside.minpt >= done.minpt) and np.all(inside.maxpt <= done.maxpt)):
        # a coarser shard that is taller than this task (the reference would let the last task win):
        # keep the chunks other tasks already stored in it
        spec = sharding.ShardingSpecification(src.scales[m]["sharding"])
        name = spec.shard_filename(spec.locate(next(iter(chunk_dict)))[0])
        old = CloudFiles(base).get(name)
        if old is not None:
          merged = {cid: spec.read_chunk(old, cid) for cid in spec.chunk_ids(old)}
          merged.update(chunk_dict)
          chunk_dict = merged
      filename, blob = src.image.make_shard(chunk_dict, shard_box, m, progress=False)
      CloudFiles(base).put(filename, blob, compress=None)
    pending[i] = None


@queueable
def CountVoxelsTask(cloudpath, shape, offset, mip=0, fill_missing=False, agglomerate=False, timestamp=None):
  """Voxel count of every label (0 included) in the task's box, clamped to the dataset, written to
  {key}/stats/voxel_counts/{bbox}.json (image.py:845-880); the counts come from fastremap.unique
  on the GPU."""
  shape, offset = Vec(*shape), Vec(*offset)
  mip = int(mip)
  cv = CloudVolume(cloudpath, fill_missing=bool(fill_missing), mip=mip, bounded=False, progress=False)
  bbox = Bbox.clamp(Bbox(offset, offset + shape), cv.meta.bounds(mip))
  labels = cv.download(bbox, agglomerate=agglomerate, timestamp=timestamp)
  uniq, cts = fastremap.unique(labels, return_counts=True)
  voxel_counts = {str(int(segid)): int(ct) for segid, ct in zip(uniq, cts)}
  cf = CloudFiles(cloudpath)
  cf.put_json(cf.join(cv.key, "stats", "voxel_counts", "%s.json" % bbox.to_filename()), voxel_counts)


# ------------------------------------------------------------ blackout, touch, delete
# image.py:103-143: edit and check a layer in place.

def layer_value(dtype, value):
  """`value` as a scalar of the layer's dtype; a value the dtype cannot hold (out of range, a fraction for
  an integer dtype, a finite number that overflows float32) raises ValueError."""
  dt = np.dtype(dtype)
  if dt.kind in "ui":
    try:
      iv = int(value)
      exact = iv == value
    except (TypeError, ValueError, OverflowError):
      exact = False
    if not exact or not (np.iinfo(dt).min <= iv <= np.iinfo(dt).max):
      raise ValueError("%r is not a %s value" % (value, dt))
    return dt.type(iv)
  with np.errstate(over="ignore"):
    typed = dt.type(value)
  if math.isfinite(float(value)) and not np.isfinite(typed):
    raise ValueError("%r is not a %s value" % (value, dt))
  return typed


def refuse_sharded(vol, mips, what):
  if any(vol._sharding(m) is not None for m in mips):
    raise NotImplementedError("%s: sharded scales are not supported (a shard holds many chunks and would "
                              "have to be rewritten whole)" % what)


@queueable
def BlackoutTask(cloudpath, mip, shape, offset, value=0, non_aligned_writes=False):
  """Write `value` over the box, clamped to the volume at `mip` (image.py:124-135).  As in the reference
  the box is not clamped to the creator's bounds: the last task of each axis paints up to the next
  multiple of the task shape past them, or the volume's edge.  The box is filled
  on the device: a chunk-aligned box in a fresh cutout; with non_aligned_writes, a box off the chunk
  grid inside the chunk-aligned region read around it (missing chunks as 0), so the voxels of the edge
  chunks outside the box keep their values.  A value the layer's dtype cannot hold raises ValueError, a
  sharded scale NotImplementedError, and a box off the grid without non_aligned_writes the storage's
  ValueError, each before anything is written."""
  shape, offset, mip = Vec(*shape), Vec(*offset), int(mip)
  vol = CloudVolume(cloudpath, mip, non_aligned_writes=non_aligned_writes)
  bounds = Bbox.clamp(Bbox(offset, shape + offset), vol.bounds)
  value = layer_value(vol.dtype, value)
  refuse_sharded(vol, [mip], "BlackoutTask")
  region = vol._write_region(bounds, mip)
  if bounds.subvoxel():
    return
  if region == bounds:
    img = DeviceCutout.empty(tuple(int(v) for v in bounds.size3()) + (vol.num_channels,), vol.dtype)
  else:
    img = vol.download_dev(region, mip=mip, fill_missing=True)
  img.fill(bounds - region.minpt, value)
  vol.upload_dev(region, img, mip=mip)


@queueable
def TouchTask(cloudpath, mip, shape, offset):
  """Read the box, clamped to the volume at `mip`, and discard it (image.py:137-143): a missing chunk
  raises EmptyVolumeException and a corrupt one its codec's error.  The chunks are decoded on the
  device (download_dev)."""
  shape, offset, mip = Vec(*shape), Vec(*offset), int(mip)
  vol = CloudVolume(cloudpath, mip, fill_missing=False)
  bounds = Bbox.clamp(Bbox(offset, shape + offset), vol.bounds)
  vol.download_dev(bounds, mip=mip)


@queueable
def DeleteTask(layer_path, shape, offset, mip=0, num_mips=5):
  """Delete a block of a layer at every mip from `mip` to min(top mip, mip + num_mips) (image.py:103-122):
  at each the box is mapped to that mip, rounded to the nearest chunk boundaries
  (Bbox.round_to_chunk_size) and clamped to the bounds, and the chunk files inside it are deleted.
  A sharded scale in that range raises NotImplementedError before anything is deleted."""
  shape, offset, mip = Vec(*shape), Vec(*offset), int(mip)
  vol = CloudVolume(layer_path, mip=mip, max_redirects=0)
  highres_bbox = Bbox(offset, offset + shape)
  top_mip = min(vol.available_mips[-1], mip + num_mips)
  refuse_sharded(vol, range(mip, top_mip + 1), "DeleteTask")
  for mip_i in range(mip, top_mip + 1):
    vol.mip = mip_i
    bbox = vol.bbox_to_mip(highres_bbox, mip, mip_i)
    bbox = bbox.round_to_chunk_size(vol.chunk_size, offset=vol.bounds.minpt)
    bbox = Bbox.clamp(bbox, vol.bounds)
    if bbox.volume() == 0:
      continue
    vol.delete(bbox)


def _shard_chunks(vol, cutout, box, mip):
  """make_shard_chunks on a cutout whose far edges may be short of a chunk boundary: pad with the
  background colour (image.py:797-799) and let the chunker clamp to the dataset bounds."""
  cs = np.asarray(vol.meta.chunk_size(mip), dtype=int)
  off = np.asarray(vol.meta.voxel_offset(mip), dtype=int)
  want = np.ceil((np.asarray(box.maxpt) - off) / cs).astype(int) * cs + off
  pad = [(0, int(max(w - h, 0))) for w, h in zip(want, box.maxpt)]
  if any(p[1] for p in pad):
    if cutout.ndim == 4:
      pad = pad + [(0, 0)]
    cutout = np.pad(cutout, pad, mode="constant", constant_values=vol.background_color)
    box = Bbox(box.minpt, np.asarray(box.minpt) + np.asarray(cutout.shape[:3]))
  return vol.image.make_shard_chunks(cutout, box, mip)


# ------------------------------------------------------- contrast, CLAHE, quantize
# image.py:145-432: the same tasks with the per-voxel work on the GPU (igneous_b200.contrast,
# rules in DESIGN.md §5b) and the pyramids through downsample_and_upload as above.

@queueable
def QuantizeTask(source_layer_path, dest_layer_path, shape, offset, mip, fill_missing=False):
  """Channel 0 of a float32 affinity layer as uint8 trunc(v * 255), then the z pyramid
  (image.py:145-162).  Out-of-range products saturate and NaN gives 0."""
  shape, offset = Vec(*shape), Vec(*offset)
  srcvol = CloudVolume(source_layer_path, mip=mip, fill_missing=fill_missing)
  bounds = Bbox.clamp(Bbox(offset, shape + offset), srcvol.bounds)
  image = contrast.quantize(srcvol[bounds][:, :, :, :1])
  destvol = CloudVolume(dest_layer_path, mip=mip)
  downsample_and_upload(image, bounds, destvol, shape, mip=mip, axis="z")


@queueable
def CLAHETask(src, dest, mip, fill_missing, shape, offset, clip_limit=40.0, tile_grid_size=(8, 8)):
  """CLAHE of every z-slice of channel 0 (image.py:164-209).  As in the reference the box is
  enlarged by tile_grid_size[0] voxels in x and tile_grid_size[1] in y (grid counts, not tile
  sizes) and clamped to the dataset, each slice is equalised at that size, and only the task's
  own box is written (no pyramid)."""
  shape, offset = Vec(*shape), Vec(*offset)
  src_cv = CloudVolume(src, mip=mip, fill_missing=fill_missing)
  bounds = Bbox.clamp(Bbox(offset, shape + offset), src_cv.bounds)
  over = bounds.clone()
  over.minpt.x -= tile_grid_size[0]
  over.maxpt.x += tile_grid_size[0]
  over.minpt.y -= tile_grid_size[1]
  over.maxpt.y += tile_grid_size[1]
  over = Bbox.clamp(over, src_cv.bounds)
  stack = contrast.clahe(src_cv[over][..., 0], clip_limit, tile_grid_size)
  crop = tuple(slice(int(a - o), int(b - o)) for a, b, o in zip(bounds.minpt, bounds.maxpt, over.minpt))
  dest_cv = CloudVolume(dest, mip=mip)
  dest_cv[bounds] = stack[crop]


def read_levels(cf, paths):
  """{path: bytes or None} for the levels files, from CloudFiles.get of a list in either form:
  the real package's [{'path', 'content', ...}] or a {path: content} mapping."""
  got = cf.get(list(paths))
  if isinstance(got, dict):
    return {p: got.get(p) for p in paths}
  return {item["path"]: item.get("content") for item in got}


class ContrastNormalizationTask(RegisteredTask):
  """TransferTask + contrast correction from LuminanceLevelsTask's histograms (image.py:211-343).
  Each z-slice is stretched between the (lower, upper) luminance of its histogram on the GPU,
  then the pyramid is built by downsample_and_upload at bounds + translate."""

  def __init__(self, src_path, dest_path, levels_path, shape, offset, mip, clip_fraction, fill_missing,
               translate, minval, maxval):
    super().__init__(src_path, dest_path, levels_path, shape, offset, mip, clip_fraction, fill_missing,
                     translate, minval, maxval)
    self.src_path = src_path
    self.dest_path = dest_path
    self.shape = Vec(*shape)
    self.offset = Vec(*offset)
    self.fill_missing = fill_missing
    self.translate = Vec(*translate)
    self.mip = int(mip)
    if isinstance(clip_fraction, Sequence):
      assert len(clip_fraction) == 2
      self.lower_clip_fraction = float(clip_fraction[0])
      self.upper_clip_fraction = float(clip_fraction[1])
    else:
      self.lower_clip_fraction = self.upper_clip_fraction = float(clip_fraction)
    self.minval = minval
    self.maxval = maxval
    self.levels_path = levels_path if levels_path else self.src_path
    assert 0 <= self.lower_clip_fraction <= 1
    assert 0 <= self.upper_clip_fraction <= 1
    assert self.lower_clip_fraction + self.upper_clip_fraction <= 1

  def execute(self):
    srccv = CloudVolume(self.src_path, fill_missing=self.fill_missing, mip=self.mip)
    destcv = CloudVolume(self.dest_path, fill_missing=self.fill_missing, mip=self.mip)
    bounds = Bbox.clamp(Bbox(self.offset, self.shape[:3] + self.offset), srccv.bounds)
    image = srccv[bounds]
    zlevels = self.fetch_z_levels(bounds)
    image = contrast.stretch(image, zlevels, self.lower_clip_fraction, self.upper_clip_fraction,
                             minval=self.minval, maxval=self.maxval, out_dtype=destcv.dtype)
    bounds += self.translate
    downsample_and_upload(image, bounds, destcv, self.shape, mip=self.mip)

  def find_section_clamping_values(self, zlevel, lowerfract, upperfract):
    return contrast.find_section_clamping_values(zlevel, lowerfract, upperfract)

  def fetch_z_levels(self, bounds):
    cf = CloudFiles(self.levels_path)
    paths = [cf.join("levels", str(self.mip), str(z)) for z in range(int(bounds.minpt.z), int(bounds.maxpt.z))]
    got = read_levels(cf, paths)
    missing = [p for p in paths if got[p] is None]
    if missing:
      raise Exception(", ".join(missing) + " were not defined. Did you run a LuminanceLevelsTask for these slices?")
    return [np.array(json.loads(got[p].decode("utf-8"))["levels"], dtype=np.uint64) for p in paths]


class LuminanceLevelsTask(RegisteredTask):
  """Histogram of randomly sampled 2048 x 2048 x 1 patches of one slice, written to
  $levels_path/levels/$mip/$z (image.py:345-432).  All patches go to the GPU in one call."""

  def __init__(self, src_path, levels_path, shape, offset, coverage_factor, mip):
    super().__init__(src_path, levels_path, shape, offset, coverage_factor, mip)
    self.src_path = src_path
    self.shape = Vec(*shape)
    self.offset = Vec(*offset)
    self.coverage_factor = coverage_factor
    self.mip = int(mip)
    self.levels_path = levels_path
    assert 0 < coverage_factor <= 1, "Coverage Factor must be between 0 and 1"

  def execute(self):
    srccv = CloudVolume(self.src_path, mip=self.mip, fill_missing=True)
    bounds = Bbox.clamp(Bbox(self.offset, self.shape[:3] + self.offset), srccv.bounds)
    bboxes = self.select_bounding_boxes(bounds)
    if len(bboxes) == 0:
      return
    patches = [np.asarray(srccv[b]).ravel(order="F") for b in bboxes]
    levels = contrast.histogram(np.concatenate(patches))
    covered_area = sum(b.volume() for b in bboxes)
    sizes = sorted(((b.volume(), b.size3()) for b in bboxes), key=lambda x: x[0])
    output = {
      "levels": levels.tolist(),
      "patch_size": [int(v) for v in sizes[-1][1]],
      "num_patches": len(bboxes),
      "coverage_ratio": covered_area / self.shape.rectVolume(),
    }
    path = os.path.join(self.levels_path if self.levels_path else self.src_path, "levels")
    CloudFiles(path).put_json("{}/{}".format(self.mip, self.offset.z), output, cache_control="no-cache")

  def select_bounding_boxes(self, dataset_bounds):
    """Non-overlapping patches on a 2048 x 2048 grid, drawn with random.randint in the
    reference's order, so that a seeded `random` picks the same patches."""
    sample = Vec(2048, 2048, 1)
    area = self.shape.rectVolume()
    total_patches = int(math.ceil(area / (2048 * 2048)))
    n = int(math.ceil(float(total_patches) * self.coverage_factor))
    patch_indices = set()
    while len(patch_indices) < n:
      patch_indices.add(random.randint(0, total_patches - 1))
    gridx = int(math.ceil(self.shape.x / sample.x))
    bboxes = []
    for i in patch_indices:
      start = Vec(i % gridx, i // gridx, 0) * sample + self.offset
      bbox = Bbox.clamp(Bbox(start, start + sample), dataset_bounds)
      if not bbox.subvoxel():
        bboxes.append(bbox)
    return bboxes
