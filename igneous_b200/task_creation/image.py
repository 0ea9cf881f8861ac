"""create_downsampling_tasks, create_image_shard_downsample_tasks, the transfer creators, the
contrast / CLAHE / quantize creators, the three CCL task creators, create_voxel_counting_tasks, the
blackout / touch / deletion creators and compute_rois (igneous/task_creation/image.py:76-171, 170-345,
507-637, 639-770, 772-813, 815-1133, 1247-1618, 1726-1936, 1995-2058): same signatures, same info /
provenance side effects, tasks from igneous_b200.tasks."""
import copy
import math
from functools import partial, reduce
from time import strftime

import numpy as np

from .. import _shim, downsample_scales, fastremap, rois, sharding, shards, tinybrain
from .._compat import Bbox, CloudVolume, CloudFiles, InfoUnavailableError, Vec, min2
from ..tasks import (DownsampleTask, TransferTask, ImageShardTransferTask, ImageShardDownsampleTask, CCLFacesTask, CCLEquivalancesTask, RelabelCCLTask,
                     QuantizeTask, CLAHETask, ContrastNormalizationTask, LuminanceLevelsTask, CountVoxelsTask,
                     BlackoutTask, TouchTask, DeleteTask)
from ..tasks.image import layer_value, refuse_sharded
from ..types import DownsampleMethods
from .common import FinelyDividedTaskIterator, get_bounds, operator_contact

MEMORY_TARGET = int(3.5e9)


def num_mips_from_memory_target(memory_target, dtype, chunk_size, num_channels, factor):
  voxels = memory_target / np.dtype(dtype).itemsize / num_channels
  chunks = voxels // reduce(lambda a, b: a * b, chunk_size)
  total = reduce(lambda a, b: a * b, factor)
  chunks /= total / (total - 1)  # the pyramid on top of mip 0 costs 1/(f-1) more
  side = chunks ** (1.0 / math.log2(total))
  if side <= 0:
    return 1
  n = math.log2(side)
  if math.ceil(n) - n <= 0.01:
    n = int(math.ceil(n))
  return max(1, int(n))


def _log(vol, task_name, **fields):
  vol.provenance.processing.append({"method": dict(task=task_name, **fields), "by": operator_contact(),
                                    "date": strftime("%Y-%m-%d %H:%M %Z")})
  vol.commit_provenance()


def create_downsampling_tasks(layer_path, mip=0, fill_missing=False, axis="z", num_mips=None,
                              preserve_chunk_size=True, sparse=False, bounds=None, chunk_size=None,
                              encoding=None, delete_black_uploads=False, background_color=0,
                              dest_path=None, compress=None, factor=None, bounds_mip=0,
                              memory_target=MEMORY_TARGET, encoding_level=None, encoding_effort=None,
                              method=DownsampleMethods.AUTO):
  vol = CloudVolume(layer_path, mip=mip)

  def task_shape(at_mip):
    nonlocal num_mips
    shape = Vec(*chunk_size) if chunk_size else Vec(*vol.meta.chunk_size(at_mip)[:3])
    f = factor if factor is not None else downsample_scales.axis_to_factor(axis)
    viable = num_mips_from_memory_target(memory_target, vol.dtype, shape, vol.num_channels, f)
    if num_mips is None:
      num_mips = viable
    if viable < num_mips:
      print("WARNING: memory limit (%d bytes) too low for %d mips at a time; %d possible."
            % (memory_target, num_mips, viable))
    return Vec(*[int(s) * int(ff) ** viable for s, ff in zip(shape, f)])

  shape = task_shape(mip)
  vol = downsample_scales.create_downsample_scales(
    layer_path, mip, shape, preserve_chunk_size=preserve_chunk_size, chunk_size=chunk_size,
    encoding=encoding, factor=factor, max_mips=num_mips)
  if encoding is not None:
    for m in range(mip + 1, min(mip + num_mips, len(vol.available_mips))):
      vol.scales[m]["encoding"] = encoding
    vol.commit_info()
  if not preserve_chunk_size or chunk_size:
    shape = task_shape(mip + 1)
  vol.mip = mip
  roi = get_bounds(vol, bounds, mip, bounds_mip=bounds_mip, chunk_size=vol.meta.chunk_size(mip))

  class DownsampleTaskIterator(FinelyDividedTaskIterator):
    def task(self, shape, offset):
      return partial(DownsampleTask, layer_path=layer_path, mip=mip, shape=shape.clone(),
                     offset=offset.clone(), axis=axis, fill_missing=fill_missing, sparse=sparse,
                     delete_black_uploads=delete_black_uploads, background_color=background_color,
                     dest_path=dest_path, compress=compress, factor=factor, max_mips=num_mips, method=method)

    def on_finish(self):
      _log(vol, "DownsampleTask", mip=mip, num_mips=num_mips, shape=[int(s) for s in shape], axis=axis,
           sparse=sparse, bounds=str(roi), chunk_size=(list(chunk_size) if chunk_size else None),
           preserve_chunk_size=preserve_chunk_size, encoding=encoding, fill_missing=bool(fill_missing),
           delete_black_uploads=bool(delete_black_uploads), background_color=background_color,
           dest_path=dest_path, compress=compress, factor=(tuple(factor) if factor else None),
           downsample_method=int(method))

  return DownsampleTaskIterator(roi, shape)


def set_encoding(cv, mip, encoding, encoding_level, encoding_effort):
  """task_creation/common.py:215-236.  `jpeg_quality` is what the device jpeg codec encodes a
  scale with (85 when absent); the jxl / png / fpzip keys are recorded, but those codecs are
  outside this implementation."""
  scale = cv.scales[mip]
  if encoding is not None:
    scale["encoding"] = encoding
    if encoding == "compressed_segmentation" and "compressed_segmentation_block_size" not in scale:
      scale["compressed_segmentation_block_size"] = (8, 8, 8)
  if encoding_level is None:
    return
  key = {"jpeg": "jpeg_quality", "jxl": "jxl_quality", "png": "png_level", "fpzip": "fpzip_precision"}.get(encoding)
  if key:
    scale[key] = int(encoding_level)
  if encoding == "jxl" and encoding_effort is not None:
    scale["jxl_effort"] = int(encoding_effort)


def create_image_shard_downsample_tasks(cloudpath, mip=0, fill_missing=False, sparse=False, chunk_size=None,
                                        encoding=None, memory_target=MEMORY_TARGET, agglomerate=False,
                                        timestamp=None, factor=(2, 2, 1), bounds=None, bounds_mip=0,
                                        encoding_level=None, encoding_effort=None,
                                        method=DownsampleMethods.AUTO, num_mips=None, truncate_scales=True):
  """Downsample an (un)sharded layer into SHARDED scales mip+1 .. mip+num_mips
  (task_creation/image.py:639-770).  One task covers the footprint of one shard of
  mip+1 scaled up by factor^num_mips."""
  if num_mips is None:
    num_mips = 3
  cv = CloudVolume(cloudpath)
  if truncate_scales:
    cv.info["scales"] = cv.info["scales"][:mip + 1]
    cv.commit_info()
  cv = downsample_scales.add_scales(cloudpath, mip, num_mips, preserve_chunk_size=True, chunk_size=chunk_size,
                                    encoding=encoding, factor=factor)
  for i in range(1, num_mips + 1):
    scale = cv.scales[mip + i]
    scale["sharding"] = sharding.create_sharded_image_info(
      dataset_size=scale["size"], chunk_size=scale["chunk_sizes"][0], encoding=scale["encoding"],
      dtype=cv.dtype, uncompressed_shard_bytesize=int(memory_target))
  cv.mip = mip
  for i in range(num_mips):
    set_encoding(cv, mip + i + 1, encoding, encoding_level, encoding_effort)
  if num_mips > 1:  # keep the top level lossless so that further levels can be built on it
    if encoding == "jxl":
      set_encoding(cv, mip + num_mips, encoding, 100, encoding_effort)
    elif encoding == "jpeg":
      set_encoding(cv, mip + num_mips, "png", 9, encoding_effort)
  cv.commit_info()
  base_shape = shards.image_shard_shape_from_spec(cv.info["scales"][mip + 1]["sharding"],
                                                  cv.meta.volume_size(mip + 1), cv.meta.chunk_size(mip + 1))
  shape = Vec(*[int(b) * int(f) ** num_mips for b, f in zip(base_shape, factor)])
  cv.mip = mip
  roi = get_bounds(cv, bounds, mip, bounds_mip=bounds_mip, chunk_size=cv.meta.chunk_size(mip + 1))

  class ImageShardDownsampleTaskIterator(FinelyDividedTaskIterator):
    def task(self, shape, offset):
      return partial(ImageShardDownsampleTask, cloudpath, shape=tuple(int(v) for v in shape),
                     offset=tuple(int(v) for v in offset), mip=int(mip), fill_missing=bool(fill_missing),
                     sparse=bool(sparse), agglomerate=bool(agglomerate), timestamp=timestamp,
                     factor=tuple(factor), method=method, num_mips=int(num_mips))

    def on_finish(self):
      cv.provenance.sources = [cloudpath]
      _log(cv, "ImageShardDownsampleTask", cloudpath=cloudpath, shape=[int(v) for v in shape],
           fill_missing=fill_missing, sparse=bool(sparse), bounds=[roi.minpt.tolist(), roi.maxpt.tolist()],
           mip=mip, agglomerate=agglomerate, timestamp=timestamp, method=int(method),
           encoding_level=encoding_level, encoding_effort=encoding_effort, num_mips=int(num_mips))

  return ImageShardDownsampleTaskIterator(roi, shape)


# ------------------------------------------------------------------------ transfer
# task_creation/image.py:507-637 and 815-1133.

# encodings the chunk codecs of this implementation cannot write
_UNSUPPORTED_ENCODINGS = ("png", "jxl", "jpegxl", "compresso", "crackle", "fpzip", "kempressed", "zfpc")


def _refuse_transfer(encoding, compress, agglomerate, timestamp, stop_layer):
  """what the transfer creators refuse, before any info file is written"""
  if agglomerate or timestamp is not None or stop_layer is not None:
    raise NotImplementedError("transfer: agglomerate / timestamp / stop_layer need a graphene source")
  if encoding is not None and str(encoding).lower() in _UNSUPPORTED_ENCODINGS:
    raise NotImplementedError("transfer: the %r chunk encoding is not implemented (raw, jpeg and "
                              "compressed_segmentation are)" % encoding)
  if compress == "br":
    raise NotImplementedError("transfer: brotli compression is not implemented (gzip is)")


def _refuse_layer_encodings(src_vol, dest_path, mip, encoding):
  """the source scale's encoding, and the destination's when it exists and `encoding` keeps it, must be
  ones the chunk codecs read and write; checked before any info file is written"""
  found = [("source", src_vol.scales[mip].get("encoding", "raw"))]
  if encoding is None:
    try:
      dest = CloudVolume(dest_path, mip=mip)
      if len(dest.scales) > mip:
        found.append(("destination", dest.scales[mip].get("encoding", "raw")))
    except InfoUnavailableError:
      pass
  for which, enc in found:
    if str(enc).lower() in _UNSUPPORTED_ENCODINGS:
      raise NotImplementedError("transfer: the %s's %r chunk encoding is not implemented (raw, jpeg and "
                                "compressed_segmentation are)" % (which, enc))


def clean_xfer_info(info):
  """Removes fields that could interfere with additional processing."""
  info.pop("mesh", None)
  info.pop("meshing", None)
  info.pop("skeletons", None)
  return info


def create_transfer_cloudvolume(src_vol, dst_cloudpath, dest_voxel_offset, mip, bounds_mip, encoding, encoding_level,
                                encoding_effort, chunk_size, truncate_scales, clean_info, cutout, bounds):
  """The destination layer of a transfer: the existing one, or a copy of the source's info (cut to
  `bounds` when `cutout`), with the voxel offset, encoding, chunk size and scale edits of the request."""
  intify = lambda lst: [int(x) for x in lst]
  bounds_resolution = np.asarray(src_vol.meta.resolution(bounds_mip), dtype=np.float64)
  try:
    dest_vol = CloudVolume(dst_cloudpath, mip=mip)
  except InfoUnavailableError:
    dest_vol = CloudVolume(dst_cloudpath, info=copy.deepcopy(src_vol.info), mip=mip)
    if cutout:
      for i in range(mip + 1):
        f = bounds_resolution / np.asarray(dest_vol.meta.resolution(i), dtype=np.float64)
        dest_vol.info["scales"][i]["voxel_offset"] = intify(np.asarray(bounds.minpt) * f)
        dest_vol.info["scales"][i]["size"] = intify(np.asarray(bounds.size3()) * f)
    dest_vol.commit_info()
  if len(dest_vol.scales) <= mip:  # cloudvolume's ScaleUnavailableError branch
    dest_vol.scales.append(copy.deepcopy(src_vol.scales[mip]))
    dest_vol.commit_info()
  if bounds is None:
    bounds = Bbox([0, 0, 0], [1, 1, 1], dtype=int)
  if dest_voxel_offset is not None:
    for i in range(mip + 1):
      f = bounds_resolution / np.asarray(dest_vol.meta.resolution(i), dtype=np.float64)
      dest_vol.info["scales"][i]["voxel_offset"] = intify((np.asarray(dest_voxel_offset) + np.asarray(bounds.minpt)) * f)
  set_encoding(dest_vol, mip, encoding, encoding_level, encoding_effort)
  if truncate_scales:
    dest_vol.info["scales"] = dest_vol.info["scales"][:mip + 1]
  dest_vol.info["scales"][mip]["chunk_sizes"] = [[int(v) for v in chunk_size]]
  if clean_info:
    dest_vol.info = clean_xfer_info(dest_vol.info)
  return dest_vol


def _select_compression_by_encoding(encoding):
  if encoding.lower() in ("raw", "compressed_segmentation", "compresso", "crackle"):
    return "gzip"
  return False


def _downsample_ratio(vol, mip):
  return Vec(*(np.asarray(vol.meta.resolution(mip), dtype=np.float64)
               / np.asarray(vol.meta.resolution(0), dtype=np.float64)).astype(int))


def create_transfer_tasks(src_layer_path, dest_layer_path, chunk_size=None, shape=None, fill_missing=False,
                          translate=None, bounds=None, mip=0, preserve_chunk_size=True, encoding=None,
                          skip_downsamples=False, delete_black_uploads=False, background_color=0, agglomerate=False,
                          timestamp=None, compress="auto", factor=None, sparse=False, dest_voxel_offset=None,
                          memory_target=MEMORY_TARGET, max_mips=5, clean_info=False, no_src_update=False,
                          bounds_mip=0, encoding_level=None, truncate_scales=True, cutout=False, stop_layer=None,
                          downsample_method=DownsampleMethods.AUTO, encoding_effort=None, use_https_for_source=False):
  """Transfer a layer to a new one, re-chunked, re-encoded, re-compressed, moved (translate,
  dest_voxel_offset) or cropped (bounds, cutout), with its downsamples unless skip_downsamples
  (task_creation/image.py:884-1133).  The task shape comes from memory_target unless `shape` is
  given.  use_https_for_source is accepted and has no effect (file:// sources)."""
  _refuse_transfer(encoding, compress, agglomerate, timestamp, stop_layer)
  src_vol = CloudVolume(src_layer_path, mip=mip)
  _refuse_layer_encodings(src_vol, dest_layer_path, mip, encoding)
  no_src_update = no_src_update or use_https_for_source
  if dest_voxel_offset:
    dest_voxel_offset = Vec(*dest_voxel_offset, dtype=int)
  if factor is None:
    factor = (2, 2, 1)
  if skip_downsamples:
    factor = (1, 1, 1)
  if not chunk_size:
    chunk_size = src_vol.info["scales"][mip]["chunk_sizes"][0]
  chunk_size = Vec(*chunk_size)
  dest_vol = create_transfer_cloudvolume(src_vol, dest_layer_path, dest_voxel_offset, mip, bounds_mip, encoding,
                                         encoding_level, encoding_effort, chunk_size, truncate_scales, clean_info,
                                         cutout, bounds)
  if compress == "auto":
    compress = _select_compression_by_encoding(dest_vol.scales[mip]["encoding"])
  if translate is None:
    translate = dest_vol.meta.voxel_offset(mip) - src_vol.meta.voxel_offset(mip)
  else:
    translate = Vec(*translate) // _downsample_ratio(src_vol, mip)
  if cutout:
    dest_vol.scales[mip].pop("sharding", None)
  dest_vol.commit_info()
  dest_cs = dest_vol.meta.chunk_size(mip)
  if shape is None:
    if memory_target is None:
      raise ValueError("Either shape or memory_target must be specified.")
    shape = downsample_scales.downsample_shape_from_memory_target(
      np.dtype(src_vol.dtype).itemsize * src_vol.num_channels, int(dest_cs[0]), int(dest_cs[1]), int(dest_cs[2]),
      factor, memory_target, max_mips)
  shape = Vec(*shape)
  if factor[2] == 1:
    shape.z = int(dest_cs[2] * max(round(shape.z / dest_cs[2]), 1))
  if not skip_downsamples:
    downsample_scales.create_downsample_scales(dest_layer_path, mip=mip, ds_shape=shape, factor=factor,
                                               preserve_chunk_size=preserve_chunk_size, encoding=encoding)
  if not cutout:
    dest_bounds = get_bounds(dest_vol, bounds, mip, bounds_mip=bounds_mip, chunk_size=chunk_size)
  else:
    dest_bounds = dest_vol.bbox_to_mip(Bbox.create(bounds), mip=bounds_mip, to_mip=mip)
    dest_bounds = Bbox.clamp(dest_bounds, dest_vol.meta.bounds(mip))

  class TransferTaskIterator(FinelyDividedTaskIterator):
    def task(self, shape, offset):
      return partial(TransferTask, src_path=src_layer_path, dest_path=dest_layer_path, shape=shape.clone(),
                     offset=offset.clone(), fill_missing=fill_missing, translate=translate, mip=mip,
                     skip_downsamples=skip_downsamples, delete_black_uploads=bool(delete_black_uploads),
                     background_color=background_color, agglomerate=agglomerate, timestamp=timestamp,
                     compress=compress, factor=factor, sparse=sparse, stop_layer=stop_layer,
                     downsample_method=int(downsample_method), use_https_for_source=use_https_for_source)

    def on_finish(self):
      job_details = {
        "method": {
          "task": "TransferTask", "src": src_layer_path, "dest": dest_layer_path,
          "shape": list(map(int, shape)), "fill_missing": fill_missing, "translate": list(map(int, translate)),
          "skip_downsamples": skip_downsamples, "delete_black_uploads": bool(delete_black_uploads),
          "background_color": background_color,
          "bounds": [dest_bounds.minpt.tolist(), dest_bounds.maxpt.tolist()],
          "mip": mip, "agglomerate": bool(agglomerate), "timestamp": timestamp, "compress": compress,
          "encoding": encoding, "memory_target": memory_target, "factor": (tuple(factor) if factor else None),
          "sparse": bool(sparse), "encoding_level": encoding_level, "encoding_effort": encoding_effort,
          "stop_layer": stop_layer, "downsample_method": int(downsample_method),
          "use_https_for_source": bool(use_https_for_source),
        },
        "by": operator_contact(),
        "date": strftime("%Y-%m-%d %H:%M %Z"),
      }
      dvol = CloudVolume(dest_layer_path)
      dvol.provenance.sources = [src_layer_path]
      dvol.provenance.processing.append(job_details)
      dvol.commit_provenance()
      if not no_src_update:
        src_vol.provenance.processing.append(job_details)
        src_vol.commit_provenance()

  return TransferTaskIterator(dest_bounds, shape)


def create_image_shard_transfer_tasks(src_layer_path, dst_layer_path, mip=0, chunk_size=None, encoding=None,
                                      bounds=None, bounds_mip=0, fill_missing=False, translate=(0, 0, 0),
                                      dest_voxel_offset=None, agglomerate=False, timestamp=None,
                                      memory_target=MEMORY_TARGET, clean_info=False, encoding_level=None,
                                      truncate_scales=True, compress="auto", cutout=False,
                                      minishard_index_encoding="gzip", stop_layer=None, encoding_effort=None,
                                      use_https_for_source=False):
  """Copy a layer at `mip` into a sharded scale, one task per shard (task_creation/image.py:507-637).
  use_https_for_source is accepted and has no effect (file:// sources)."""
  _refuse_transfer(encoding, compress, agglomerate, timestamp, stop_layer)
  if compress not in ("auto", True, "gzip", False, None):
    raise ValueError("%s can only be True or 'gzip' for sharded images." % compress)
  src_vol = CloudVolume(src_layer_path, mip=mip)
  _refuse_layer_encodings(src_vol, dst_layer_path, mip, encoding)
  if dest_voxel_offset:
    dest_voxel_offset = Vec(*dest_voxel_offset, dtype=int)
  if not chunk_size:
    chunk_size = src_vol.info["scales"][mip]["chunk_sizes"][0]
  chunk_size = Vec(*chunk_size)
  dest_vol = create_transfer_cloudvolume(src_vol, dst_layer_path, dest_voxel_offset, mip, bounds_mip, encoding,
                                         encoding_level, encoding_effort, chunk_size, truncate_scales, clean_info,
                                         cutout, bounds)
  if compress == "auto":
    compress = _select_compression_by_encoding(dest_vol.scales[mip]["encoding"])
  compress = compress in (True, "gzip")
  if translate is None:
    translate = dest_vol.meta.voxel_offset(mip) - src_vol.meta.voxel_offset(mip)
  else:
    translate = Vec(*translate) // _downsample_ratio(src_vol, mip)
  scale = dest_vol.scales[mip]
  spec = sharding.create_sharded_image_info(
    dataset_size=scale["size"], chunk_size=scale["chunk_sizes"][0], encoding=scale["encoding"], dtype=dest_vol.dtype,
    uncompressed_shard_bytesize=memory_target, data_encoding=("gzip" if compress else "raw"),
    minishard_index_encoding=minishard_index_encoding)
  scale["sharding"] = spec
  if clean_info:
    dest_vol.info = clean_xfer_info(dest_vol.info)
  dest_vol.commit_info()
  shape = shards.image_shard_shape_from_spec(spec, scale["size"], chunk_size)
  if not cutout:
    bounds = get_bounds(dest_vol, bounds, mip, bounds_mip=bounds_mip, chunk_size=chunk_size)
  else:
    bounds = dest_vol.bbox_to_mip(Bbox.create(bounds), mip=bounds_mip, to_mip=mip)
    bounds = Bbox.clamp(bounds, dest_vol.meta.bounds(mip))
  bounds = bounds.expand_to_chunk_size(shape, offset=bounds.minpt)

  class ImageShardTransferTaskIterator(FinelyDividedTaskIterator):
    def task(self, shape, offset):
      return partial(ImageShardTransferTask, src_layer_path, dst_layer_path, shape=shape, offset=offset,
                     fill_missing=fill_missing, translate=translate, mip=mip, agglomerate=agglomerate,
                     timestamp=timestamp, stop_layer=stop_layer, use_https_for_source=bool(use_https_for_source))

    def on_finish(self):
      job_details = {
        "method": {
          "task": "ImageShardTransferTask", "src": src_layer_path, "dest": dst_layer_path,
          "shape": list(map(int, shape)), "fill_missing": fill_missing, "translate": list(map(int, translate)),
          "bounds": [bounds.minpt.tolist(), bounds.maxpt.tolist()], "mip": mip,
          "encoding_level": encoding_level, "stop_layer": stop_layer, "encoding_effort": encoding_effort,
          "timestamp": timestamp, "use_https_for_source": bool(use_https_for_source),
        },
        "by": operator_contact(),
        "date": strftime("%Y-%m-%d %H:%M %Z"),
      }
      if not use_https_for_source:
        dvol = CloudVolume(dst_layer_path)
        dvol.provenance.sources = [src_layer_path]
        dvol.provenance.processing.append(job_details)
        dvol.commit_provenance()

  return ImageShardTransferTaskIterator(bounds, shape)


def _ccl_creator(task_fn, task_name, cloudpath, mip, shape, **opts):
  vol = CloudVolume(cloudpath, mip=mip)
  shape = Vec(*shape)

  class CCLTaskIterator(FinelyDividedTaskIterator):
    def task(self, shape, offset):
      return partial(task_fn, cloudpath=cloudpath, mip=mip, shape=shape.clone(), offset=offset.clone(), **opts)

    def on_finish(self):
      _log(vol, task_name, cloudpath=cloudpath, mip=mip, shape=[int(s) for s in shape], **opts)

  return CCLTaskIterator(vol.meta.bounds(mip).clone(), shape)


def create_ccl_face_tasks(cloudpath, mip, shape=(512, 512, 512), threshold_gte=None, threshold_lte=None,
                          fill_missing=False, dust_threshold=0):
  """pass 1"""
  return _ccl_creator(CCLFacesTask, "CCLFacesTask", cloudpath, mip, shape, threshold_gte=threshold_gte,
                      threshold_lte=threshold_lte, fill_missing=fill_missing, dust_threshold=dust_threshold)


def create_ccl_equivalence_tasks(cloudpath, mip, shape=(512, 512, 512), threshold_gte=None,
                                 threshold_lte=None, fill_missing=False, dust_threshold=0):
  """pass 2 (shape must match pass 1)"""
  return _ccl_creator(CCLEquivalancesTask, "CCLEquivalancesTask", cloudpath, mip, shape,
                      threshold_gte=threshold_gte, threshold_lte=threshold_lte, fill_missing=fill_missing,
                      dust_threshold=dust_threshold)


def create_ccl_relabel_tasks(src_path, dest_path, mip, shape=(512, 512, 512), chunk_size=None, encoding=None,
                             threshold_gte=None, threshold_lte=None, fill_missing=False, dust_threshold=0):
  """pass 4: the destination layer gets the smallest dtype that holds max_label"""
  src = CloudVolume(src_path, mip=mip)
  cf = CloudFiles(src_path)
  max_label = int(cf.get_json(cf.join(src.key, "ccl", "max_label.json"))[0])
  dtype = fastremap.fit_dtype(np.uint64, max_label).name
  try:
    dest = CloudVolume(dest_path, mip=mip)
  except InfoUnavailableError:
    info = copy.deepcopy(src.info)
    info["data_type"] = dtype
    info["type"] = "segmentation"
    info["scales"] = info["scales"][:mip + 1]
    scale = info["scales"][mip]
    if chunk_size:
      scale["chunk_sizes"] = [list(chunk_size)]
    if encoding:
      scale["encoding"] = encoding
    scale.pop("sharding", None)
    dest = CloudVolume(dest_path, info=info, mip=mip)
    dest.commit_info()
  shape = Vec(*shape)

  class RelabelCCLTaskIterator(FinelyDividedTaskIterator):
    def task(self, shape, offset):
      return partial(RelabelCCLTask, src_path=src_path, dest_path=dest_path, mip=mip, shape=shape.clone(),
                     offset=offset.clone(), threshold_gte=threshold_gte, threshold_lte=threshold_lte,
                     fill_missing=fill_missing, dust_threshold=dust_threshold)

    def on_finish(self):
      _log(dest, "RelabelCCLTask", src_path=src_path, dest_path=dest_path, mip=mip,
           shape=[int(s) for s in shape], threshold_gte=threshold_gte, threshold_lte=threshold_lte,
           fill_missing=bool(fill_missing), dust_threshold=dust_threshold)

  return RelabelCCLTaskIterator(src.meta.bounds(mip).clone(), shape)


# ------------------------------------------------------- contrast, CLAHE, quantize
# task_creation/image.py:1247-1618: same signatures, destination info, scales, task grids and
# provenance as the reference; the tasks are those of igneous_b200.tasks.

def _new_dest(src_vol, dest_path, mip):
  """The destination layer, or (when it has no info yet) the source's info cut to scales[:mip+1]."""
  try:
    dvol = CloudVolume(dest_path, mip=mip)
  except InfoUnavailableError:
    dvol = CloudVolume(dest_path, mip=mip, info=copy.deepcopy(src_vol.info))
    dvol.info["scales"] = dvol.info["scales"][:mip + 1]
    dvol.commit_info()
  dvol.meta.unlock_mips(mip)
  return dvol


def _default_image_task_shape(chunk_size, bounds):
  """(2048, 2048, chunk_z) shrunk to whole chunks, then clamped to [1, bounds size] per axis
  (Bbox.shrink_to_chunk_size + Vec.clamp of the reference)."""
  cs = np.asarray(chunk_size[:3], dtype=int)
  want = np.asarray([2048, 2048, int(cs[2])], dtype=int)
  shrunk = (want // cs) * cs
  return Vec(*np.maximum(np.minimum(shrunk, np.asarray(bounds.size3(), dtype=int)), 1))


def create_contrast_normalization_tasks(src_path, dest_path, levels_path=None, shape=None, mip=0, clip_fraction=0.01,
                                        fill_missing=False, translate=(0, 0, 0), minval=None, maxval=None,
                                        bounds=None, bounds_mip=0):
  """Stretch every slice between its LuminanceLevelsTask (lower, upper) levels into dest_path and
  build its downsamples (task_creation/image.py:1247-1324)."""
  srcvol = CloudVolume(src_path, mip=mip)
  dvol = _new_dest(srcvol, dest_path, mip)
  if bounds is None:
    bounds = srcvol.meta.bounds(mip).clone()
  if shape is None:
    shape = _default_image_task_shape(dvol.meta.chunk_size(mip), bounds)
  shape = Vec(*shape)
  downsample_scales.create_downsample_scales(dest_path, mip=mip, ds_shape=shape, preserve_chunk_size=True)
  dvol.refresh_info()
  # as in the reference, bounds (default: the source's bounds at `mip`) are read at bounds_mip
  bounds = get_bounds(srcvol, bounds, mip, bounds_mip=bounds_mip)

  class ContrastNormalizationTaskIterator(FinelyDividedTaskIterator):
    def task(self, shape, offset):
      return ContrastNormalizationTask(src_path=src_path, dest_path=dest_path, levels_path=levels_path,
                                       shape=shape.clone(), offset=offset.clone(), clip_fraction=clip_fraction,
                                       mip=mip, fill_missing=fill_missing, translate=translate, minval=minval,
                                       maxval=maxval)

    def on_finish(self):
      _log(dvol, "ContrastNormalizationTask", src_path=src_path, dest_path=dest_path,
           shape=[int(v) for v in shape], clip_fraction=clip_fraction, mip=mip,
           translate=[int(v) for v in translate], minval=minval, maxval=maxval,
           bounds=[[int(v) for v in bounds.minpt], [int(v) for v in bounds.maxpt]])

  return ContrastNormalizationTaskIterator(bounds, shape)


def create_luminance_levels_tasks(layer_path, levels_path=None, coverage_factor=0.01, shape=None, offset=None, mip=0,
                                  bounds_mip=0, bounds=None):
  """One LuminanceLevelsTask per slice, writing $levels_path/levels/$mip/$z
  (task_creation/image.py:1326-1426).  As in the reference the slices run over the inclusive
  range(minpt.z, maxpt.z + 1): the last task clamps to an empty box and writes nothing, and
  len() counts the slices without it.  `shape` is ignored: a task covers the whole (x, y) extent
  of the bounds."""
  if shape is not None or offset is not None:
    print("Create Luminance Levels Tasks: Deprecation Notice: "
          "shape and offset parameters are deprecated in favor of the bounds argument.")
  vol = CloudVolume(layer_path, mip=mip)
  if bounds is None:
    bounds = vol.meta.bounds(mip).clone()
  bounds = get_bounds(vol, bounds, mip, bounds_mip=bounds_mip)
  shape = Vec(*bounds.size3())
  shape.z = 1
  offset = Vec(*(bounds.minpt if offset is None or len(offset) == 0 else offset))
  if str(layer_path).startswith("boss://"):
    raise NotImplementedError("create_luminance_levels_tasks: boss:// layers are not supported")

  class LuminanceLevelsTaskIterator:
    def __len__(self):
      return int(bounds.maxpt.z - bounds.minpt.z)

    def __iter__(self):
      for z in range(int(bounds.minpt.z), int(bounds.maxpt.z) + 1):
        zoffset = offset.clone()
        zoffset.z = z
        yield LuminanceLevelsTask(src_path=layer_path, levels_path=levels_path, shape=shape.clone(),
                                  offset=zoffset, coverage_factor=coverage_factor, mip=mip)
      if levels_path:
        try:
          pvol = CloudVolume(levels_path)
        except InfoUnavailableError:
          pvol = CloudVolume(levels_path, info=vol.info)
      else:
        pvol = CloudVolume(layer_path, mip=mip)
      _log(pvol, "LuminanceLevelsTask", src=layer_path, levels_path=levels_path, shape=[int(v) for v in shape],
           offset=[int(v) for v in offset], bounds=[[int(v) for v in bounds.minpt], [int(v) for v in bounds.maxpt]],
           coverage_factor=coverage_factor, mip=mip)

  return LuminanceLevelsTaskIterator()


def create_clahe_tasks(src, dest, shape=None, mip=0, fill_missing=False, bounds=None, bounds_mip=0,
                       clip_limit=40.0, tile_grid_size=(8, 8)):
  """CLAHE (contrast limited adaptive histogram equalization) of every slice of src into dest
  (task_creation/image.py:1428-1508).  The tasks write mip `mip` only."""
  srcvol = CloudVolume(src, mip=mip)
  dvol = _new_dest(srcvol, dest, mip)
  if bounds is None:
    bounds = srcvol.meta.bounds(mip).clone()
  if shape is None:
    shape = _default_image_task_shape(dvol.meta.chunk_size(mip), bounds)
  shape = Vec(*shape)
  downsample_scales.create_downsample_scales(dest, mip=mip, ds_shape=shape, preserve_chunk_size=True)
  dvol.refresh_info()
  bounds = get_bounds(srcvol, bounds, mip, bounds_mip=bounds_mip)

  class CLAHETaskIterator(FinelyDividedTaskIterator):
    def task(self, shape, offset):
      return partial(CLAHETask, src=src, dest=dest, shape=shape.clone(), offset=offset.clone(), mip=mip,
                     fill_missing=fill_missing, clip_limit=clip_limit, tile_grid_size=tile_grid_size)

    def on_finish(self):
      _log(dvol, "CLAHETask", src=src, dest=dest, shape=[int(v) for v in shape], clip_limit=clip_limit,
           tile_grid_size=tile_grid_size, mip=mip,
           bounds=[[int(v) for v in bounds.minpt], [int(v) for v in bounds.maxpt]])

  return CLAHETaskIterator(bounds, shape)


def create_quantized_affinity_info(src_layer, dest_layer, shape, mip, chunk_size, encoding):
  """The source's info as a 1-channel uint8 image, scales[:mip+1], each with `chunk_size` and
  `encoding` (task_creation/image.py:1546-1560)."""
  info = copy.deepcopy(CloudVolume(src_layer).info)
  info["num_channels"] = 1
  info["data_type"] = "uint8"
  info["type"] = "image"
  info["scales"] = info["scales"][:mip + 1]
  for i in range(mip + 1):
    info["scales"][i]["encoding"] = encoding
    info["scales"][i]["chunk_sizes"] = [list(chunk_size)]
  return info


def create_quantize_tasks(src_layer, dest_layer, shape, mip=0, fill_missing=False, chunk_size=(128, 128, 64),
                          encoding="raw", bounds=None):
  """Quantize channel 0 of a float32 affinity layer into a uint8 image with downsamples
  (task_creation/image.py:1562-1618).  `bounds` are given at mip 0."""
  shape = Vec(*shape)
  info = create_quantized_affinity_info(src_layer, dest_layer, shape, mip, chunk_size, encoding)
  destvol = CloudVolume(dest_layer, info=info, mip=mip)
  destvol.commit_info()
  downsample_scales.create_downsample_scales(dest_layer, mip=mip, ds_shape=shape, chunk_size=chunk_size,
                                             encoding=encoding)
  if bounds is None:
    bounds = destvol.meta.bounds(mip)
  else:
    bounds = destvol.bbox_to_mip(Bbox.create(bounds), mip=0, to_mip=mip)
    bounds = bounds.expand_to_chunk_size(destvol.meta.chunk_size(mip), destvol.meta.voxel_offset(mip))

  class QuantizeTasksIterator(FinelyDividedTaskIterator):
    def task(self, shape, offset):
      return partial(QuantizeTask, source_layer_path=src_layer, dest_layer_path=dest_layer,
                     shape=[int(v) for v in shape], offset=[int(v) for v in offset], fill_missing=fill_missing,
                     mip=mip)

    def on_finish(self):
      destvol.provenance.sources = [src_layer]
      _log(destvol, "QuantizeTask", source_layer_path=src_layer, dest_layer_path=dest_layer,
           shape=[int(v) for v in shape], fill_missing=fill_missing, mip=mip)

  return QuantizeTasksIterator(bounds, shape)


def create_voxel_counting_tasks(cloudpath, mip, fill_missing=False, agglomerate=False, timestamp=None):
  """Count the voxels of every label in 512^3 tasks (clamped at the far edges) and write the JSON
  files to {key}/stats/voxel_counts/{bbox}.json (task_creation/image.py:1891-1936)."""
  vol = CloudVolume(cloudpath, max_redirects=0, mip=mip)
  shape = Vec(512, 512, 512)
  bounds = vol.bounds.clone()

  class CountVoxelsTaskIterator(FinelyDividedTaskIterator):
    def task(self, shape, offset):
      bounded_shape = min2(shape, bounds.maxpt - offset)
      return partial(CountVoxelsTask, cloudpath=cloudpath, shape=bounded_shape.clone(), offset=offset.clone(), mip=mip,
                     fill_missing=fill_missing, agglomerate=agglomerate, timestamp=timestamp)

    def on_finish(self):
      _log(CloudVolume(cloudpath, max_redirects=0), "CountVoxelsTask", cloudpath=cloudpath, mip=mip,
           shape=shape.tolist(), fill_missing=fill_missing, agglomerate=agglomerate, timestamp=timestamp)

  return CountVoxelsTaskIterator(bounds, shape)


# ------------------------------------------------------------ blackout, touch, delete, rois
# task_creation/image.py:76-171, 772-813 and 1995-2058.

def create_blackout_tasks(cloudpath, bounds, mip=0, shape=(2048, 2048, 64), value=0, non_aligned_writes=False):
  """Paint `bounds` (given at mip 0) with `value` at `mip` (task_creation/image.py:76-123).  The bounds are
  moved to `mip`, expanded to the chunk grid unless non_aligned_writes, and clamped to the mip's bounds.
  A value the dtype cannot hold raises ValueError and a sharded scale NotImplementedError, before any task.
  As in the reference, on_finish appends the provenance entry to the volume in memory and does not commit
  it: the layer's provenance file is left as it was, so a run leaves the same files as the reference's."""
  vol = CloudVolume(cloudpath, mip=mip)
  layer_value(vol.dtype, value)
  refuse_sharded(vol, [mip], "create_blackout_tasks")
  shape = Vec(*shape)
  bounds = Bbox.create(bounds)
  bounds = vol.bbox_to_mip(bounds, mip=0, to_mip=mip)
  if not non_aligned_writes:
    bounds = bounds.expand_to_chunk_size(vol.chunk_size, vol.voxel_offset)
  bounds = Bbox.clamp(bounds, vol.mip_bounds(mip))

  class BlackoutTaskIterator(FinelyDividedTaskIterator):
    def task(self, shape, offset):
      return partial(BlackoutTask, cloudpath=cloudpath, mip=mip, shape=shape.clone(), offset=offset.clone(),
                     value=value, non_aligned_writes=non_aligned_writes)

    def on_finish(self):
      vol.provenance.processing.append({
        "method": {"task": "BlackoutTask", "cloudpath": cloudpath, "mip": mip,
                   "non_aligned_writes": non_aligned_writes, "value": value, "shape": shape.tolist(),
                   "bounds": [bounds.minpt.tolist(), bounds.maxpt.tolist()]},
        "by": operator_contact(), "date": strftime("%Y-%m-%d %H:%M %Z")})

  return BlackoutTaskIterator(bounds, shape)


def create_touch_tasks(cloudpath, mip=0, shape=(2048, 2048, 64), bounds=None):
  """Read every chunk of a layer at `mip` to find missing or corrupt files (task_creation/image.py:125-171).
  As in the reference `bounds` is read at mip 0 and moved to `mip`, the default (the volume's bounds at
  `mip`) included, and each task's shape is clamped to the volume's far edge."""
  vol = CloudVolume(cloudpath, mip=mip)
  shape = Vec(*shape)
  if bounds is None:
    bounds = vol.bounds.clone()
  bounds = Bbox.create(bounds)
  bounds = vol.bbox_to_mip(bounds, mip=0, to_mip=mip)
  bounds = Bbox.clamp(bounds, vol.mip_bounds(mip))

  class TouchTaskIterator(FinelyDividedTaskIterator):
    def task(self, shape, offset):
      bounded_shape = min2(shape, vol.bounds.maxpt - offset)
      return partial(TouchTask, cloudpath=cloudpath, shape=bounded_shape.clone(), offset=offset.clone(), mip=mip)

    def on_finish(self):
      vol.provenance.processing.append({
        "method": {"task": "TouchTask", "mip": mip, "shape": shape.tolist(),
                   "bounds": [bounds.minpt.tolist(), bounds.maxpt.tolist()]},
        "by": operator_contact(), "date": strftime("%Y-%m-%d %H:%M %Z")})
      vol.commit_provenance()

  return TouchTaskIterator(bounds, shape)


def create_deletion_tasks(layer_path, mip=0, num_mips=5, shape=None, bounds=None):
  """Delete a layer's chunks from `mip` up through mip + num_mips (`igneous image rm`,
  task_creation/image.py:772-813).  The default shape is the chunk size at `mip` times 2^num_mips in x
  and y; `bounds` (a Bbox at `mip`, default its bounds) is used as given, and each task's shape is
  clamped to it.  A sharded scale in that range raises NotImplementedError before any task."""
  vol = CloudVolume(layer_path, max_redirects=0)
  refuse_sharded(vol, range(mip, min(vol.available_mips[-1], mip + num_mips) + 1), "create_deletion_tasks")
  if shape is None:
    shape = vol.meta.chunk_size(mip)[:3]
    shape.x *= 2 ** num_mips
    shape.y *= 2 ** num_mips
  else:
    shape = Vec(*shape)
  if not bounds:
    bounds = vol.mip_bounds(mip).clone()

  class DeleteTaskIterator(FinelyDividedTaskIterator):
    def task(self, shape, offset):
      bounded_shape = min2(shape, bounds.maxpt - offset)
      return partial(DeleteTask, layer_path=layer_path, shape=bounded_shape.clone(), offset=offset.clone(),
                     mip=mip, num_mips=num_mips)

    def on_finish(self):
      pvol = CloudVolume(layer_path, max_redirects=0)
      pvol.provenance.processing.append({
        "method": {"task": "DeleteTask", "mip": mip, "num_mips": num_mips, "shape": shape.tolist()},
        "by": operator_contact(), "date": strftime("%Y-%m-%d %H:%M %Z")})
      pvol.commit_provenance()

  return DeleteTaskIterator(bounds, shape)


def compute_rois(cloudpath, progress=False, suppress_faint_voxels=0, dust_threshold=10, max_axial_length=512,
                 z_step=None):
  """The bounding boxes of the non-empty parts of a layer, recorded in info["scales"][0]["rois"] and
  returned (`igneous image roi`, task_creation/image.py:1995-2058); the rules are DESIGN.md §5k's.
  The top mip is read in z slabs of z_step (default: all of z) with missing chunks as 0.  A slab whose xy
  area exceeds max_axial_length^2 is pooled by (2, 2, 1) ceil(log2(area / max_axial_length^2)) times
  (averaging, mode pooling for segmentation), thresholded (> suppress_faint_voxels) and split into
  26-connected components, those of fewer than dust_threshold voxels dropped; each box, in the order of
  its component's first voxel, is scaled by the downsample ratio (and 2^pooled mips in x and y), shifted
  by the slab's z and has 1 taken off its maximum.  All of that runs on the device and only the boxes come
  back.  Signed integer layers raise NotImplementedError before anything is read.  The reference's
  quirks are kept: the boxes are relative to the top mip's cutout in x and y (its
  voxel offset is not added), the slab's z is added at the top mip's scale after the scaling, and a top
  mip of more than 8e9 voxels prints a warning."""
  cv = CloudVolume(cloudpath, progress=progress, fill_missing=True)
  _shim.require_unsigned(cv.dtype, "compute_rois")  # the threshold kernel compares unsigned
  cv.mip = len(cv.scales) - 1  # the reference sets the top scale's resolution, which names this mip
  cv.meta.rois = None
  if cv.meta.voxels(cv.mip) > int(8e9):
    print("Warning: lowest resolution is larger than 8 gigavoxels. Consider additional downsampling.")
  bounds = cv.bounds
  if z_step is None:
    z_step = bounds.size3()[2]
  more_mips = 0
  max_size = max_axial_length ** 2
  bboxes = []
  method = "mode" if cv.layer_type == "segmentation" else "average"
  for z in range(int(bounds.minpt.z), int(bounds.maxpt.z), int(z_step)):
    upper = min(z + int(z_step), int(bounds.maxpt.z))
    slab = Bbox((bounds.minpt.x, bounds.minpt.y, z), (bounds.maxpt.x, bounds.maxpt.y, upper))
    img = rois.channel0(cv.download_dev(slab, mip=cv.mip))
    sxy = img.shape[0] * img.shape[1]
    if sxy > max_size:
      more_mips = int(np.ceil(np.log2(sxy / max_size)))
      if more_mips > 0:
        img = tinybrain.downsample_dev(img, method, (2, 2, 1), more_mips)[-1]
      else:
        more_mips = 0
    boxes = rois.component_boxes_dev(rois.threshold_dev(img, suppress_faint_voxels), dust_threshold)
    del img
    factor3 = cv.downsample_ratio
    factor3.x *= 2 ** more_mips
    factor3.y *= 2 ** more_mips
    for row in boxes:
      bbx = Bbox(row[1:4].astype(np.int64), row[4:7].astype(np.int64) + 1) * factor3
      bbx.minpt.z += z
      bbx.maxpt.z += z
      bbx.maxpt -= 1
      bboxes.append(bbx.astype(int))
  cv.scales[0]["rois"] = [bbx.to_list() for bbx in bboxes]
  cv.commit_info()
  return bboxes
