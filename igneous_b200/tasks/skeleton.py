"""SkeletonTask with TEASAR and the per-label encoding on the GPU.

Mirror of igneous/tasks/skeleton.py:54-808 for unsharded skeleton fragments: the constructor
(:54-115), execute (:117-247), upload_individuals (:772-792) and upload_spatial_index (:794-808).
kimimaro.skeletonize is replaced by igneous_b200.kimimaro.export_skeletons, which also moves every vertex
to dataset coordinates, encodes each skeleton in the precomputed format and boxes it on the device
(DESIGN.md §5g); fastremap by igneous_b200.fastremap.  The download is not renumbered on the host: the
device renumbers, and the export keys skeletons by original label.

UnshardedSkeletonMergeTask mirrors igneous/tasks/skeleton.py:810-916; its fuse and kimimaro.postprocess run on
the device (igneous_b200.kimimaro.merge_fragments, DESIGN.md §5h).  ShardedFromUnshardedSkeletonMergeTask
mirrors :1074-1130: it packs finished unsharded skeletons into one hashed shard (DESIGN.md §5l).
"""
import gzip
import os
import pickle
import re
import time
from collections import defaultdict

import numpy as np

from .. import fastremap, kimimaro, labelshard
from .._compat import CloudVolume, CloudFiles, Bbox, Vec, RegisteredTask, queueable
from ..sharding import LabelShardingSpecification, pack_shard

# seconds per phase of the last execute() in this process, host clock (diagnostic)
last_phase_seconds = {}


def refuse(who, sharded=False, dust_global=False, synapses=None, cross_sectional_area=False, fix_autapses=False,
           timestamp=None, root_ids_cloudpath=None, fix_avocados=False, fill_holes=0):
  """NotImplementedError for an option whose format or algorithm igneous_b200 does not have."""
  why = [
    (sharded, "sharded=True (the mapbuffer fragment container) is out of scope"),
    (dust_global, "dust_global=True (global voxel counts) is out of scope"),
    (synapses, "synapses (extra targets at synapse centroids) are out of scope"),
    (cross_sectional_area, "cross_sectional_area=True is out of scope"),
    (fix_autapses or timestamp is not None or root_ids_cloudpath,
     "fix_autapses, timestamp and root_ids_cloudpath (graphene volumes) are out of scope"),
    (fix_avocados, "fix_avocados=True is out of scope"),
    (fill_holes, "fill_holes > 0 is out of scope"),
  ]
  for cond, msg in why:
    if cond:
      raise NotImplementedError("igneous_b200 %s: %s (DESIGN.md §5g)" % (who, msg))


class SkeletonTask(RegisteredTask):
  """Stage 1 of skeletonization: the skeleton fragments of one chunk of segmentation.
  `progress` and `parallel` are accepted and ignored.  Soma mode is refused by the skeletonizer when a task
  meets an object whose largest distance to the boundary exceeds soma_detection_threshold."""

  def __init__(self, cloudpath, shape, offset, mip, teasar_params, will_postprocess, info=None, object_ids=None,
               mask_ids=None, fix_branching=True, fix_borders=True, fix_avocados=False, fill_holes=0,
               dust_threshold=1000, progress=False, parallel=1, fill_missing=False, sharded=False, frag_path=None,
               spatial_index=True, spatial_grid_shape=None, synapses=None, dust_global=False,
               cross_sectional_area=False, cross_sectional_area_smoothing_window=1,
               cross_sectional_area_shape_delta=150, cross_sectional_area_repair_sec_per_label=0,
               cross_sectional_area_low_memory_threshold=int(8e9), dry_run=False, strip_integer_attributes=True,
               fix_autapses=False, timestamp=None, root_ids_cloudpath=None):
    super().__init__(cloudpath, shape, offset, mip, teasar_params, will_postprocess, info, object_ids, mask_ids,
                     fix_branching, fix_borders, fix_avocados, fill_holes, dust_threshold, progress, parallel,
                     fill_missing, bool(sharded), frag_path, bool(spatial_index), spatial_grid_shape, synapses,
                     bool(dust_global), bool(cross_sectional_area), int(cross_sectional_area_smoothing_window),
                     int(cross_sectional_area_shape_delta), int(cross_sectional_area_repair_sec_per_label),
                     int(cross_sectional_area_low_memory_threshold), bool(dry_run), bool(strip_integer_attributes),
                     bool(fix_autapses), timestamp, root_ids_cloudpath)
    refuse("SkeletonTask", sharded, dust_global, synapses, cross_sectional_area, fix_autapses, timestamp,
           root_ids_cloudpath, fix_avocados, fill_holes)
    self.cloudpath, self.mip, self.info = cloudpath, int(mip), info
    self.teasar_params, self.will_postprocess = teasar_params, bool(will_postprocess)
    self.object_ids, self.mask_ids = object_ids, mask_ids
    self.fix_branching, self.fix_borders = bool(fix_branching), bool(fix_borders)
    self.dust_threshold, self.fill_missing = dust_threshold, bool(fill_missing)
    self.frag_path, self.spatial_index = frag_path, bool(spatial_index)
    self.dry_run, self.strip_integer_attributes = bool(dry_run), bool(strip_integer_attributes)
    if isinstance(self.frag_path, str):
      self.frag_path = self.frag_path.rstrip("/")
    if spatial_grid_shape is None:
      spatial_grid_shape = shape
    self.bounds = Bbox(offset, Vec(*shape) + Vec(*offset))
    self.index_bounds = Bbox(offset, Vec(*spatial_grid_shape) + Vec(*offset))

  def execute(self):
    last_phase_seconds.clear()
    t0 = time.perf_counter()
    vol = CloudVolume(self.cloudpath, mip=self.mip, bounded=True, info=self.info, fill_missing=self.fill_missing)
    bbox = Bbox.clamp(self.bounds, vol.bounds)
    index_bbox = Bbox.clamp(self.index_bounds, vol.bounds)
    path = self.fragment_path(vol)

    all_labels = vol.download(bbox)[..., 0]
    if self.mask_ids:
      all_labels = fastremap.mask(all_labels, self.mask_ids, in_place=True)
    if self.object_ids:
      all_labels = fastremap.mask_except(all_labels, self.object_ids, in_place=True)
    t1 = time.perf_counter()
    last_phase_seconds["download"] = t1 - t0

    # voxel centred (+0.5), the more accurate bounding box from mip 0 (skeleton.py:229-230), float64
    corrected_offset = (bbox.minpt.astype(np.float32) - vol.meta.voxel_offset(self.mip) + 0.5) * \
        vol.meta.resolution(self.mip)
    corrected_offset += vol.meta.voxel_offset(0) * vol.meta.resolution(0)
    corrected_offset = np.asarray(corrected_offset, dtype=np.float64)

    skeletons, blobs, boxes = kimimaro.export_skeletons(
      all_labels, offset=corrected_offset, vertex_types=not self.strip_integer_attributes,
      teasar_params=self.teasar_params, object_ids=self.object_ids, anisotropy=vol.resolution,
      dust_threshold=self.dust_threshold, fix_branching=self.fix_branching, fix_borders=self.fix_borders)
    del all_labels
    phases = dict(kimimaro.last_phase_seconds)
    t2 = time.perf_counter()
    last_phase_seconds["export"] = phases.pop("assembly", 0.0)
    last_phase_seconds["teasar"] = t2 - t1 - last_phase_seconds["export"]

    if self.dry_run:
      return skeletons
    self.upload_individuals(vol, path, bbox, skeletons, blobs)
    if self.spatial_index:
      self.upload_spatial_index(vol, path, index_bbox, boxes)
    last_phase_seconds["writes"] = time.perf_counter() - t2

  def fragment_path(self, vol):
    """skeleton.py:144-157: the layer's skeleton directory; with frag_path, the same directory under it when
    it holds a volume info (one with scales), otherwise frag_path itself."""
    path = vol.info.get("skeletons", "skeletons")
    if self.frag_path is None:
      return vol.meta.join(self.cloudpath, path)
    test_info = CloudFiles(self.frag_path).get_json("info")
    if test_info is not None and "scales" in test_info:
      return CloudFiles(self.frag_path).join(self.frag_path, path)
    return self.frag_path

  def upload_individuals(self, vol, path, bbox, skeletons, blobs):
    """Without postprocessing, each skeleton goes to the layer's skeleton directory as its precomputed blob
    (vol.skeleton.upload); with it, {segid}:{physical bbox} fragments are pickled into `path`."""
    if not self.will_postprocess:
      cf = CloudFiles(vol.skeleton.path)
      cf.puts(((str(segid), blob.tobytes()) for segid, blob in blobs.items()), compress="gzip",
              content_type="application/octet-stream", cache_control=False)
      return
    name = (bbox * vol.resolution).to_filename()
    cf = CloudFiles(path)
    cf.puts((("%d:%s" % (segid, name), pickle.dumps(skel)) for segid, skel in skeletons.items()),
            compress="gzip", content_type="application/python-pickle", cache_control=False)

  def upload_spatial_index(self, vol, path, bbox, boxes):
    """{segid: [min xyz, max xyz]} of the skeletons' vertices, from the device boxes."""
    spatial_index = {segid: [float(v) for v in box] for segid, box in boxes.items()}
    bbox = bbox.astype(vol.resolution.dtype) * vol.resolution
    precision = vol.skeleton.spatial_index.precision
    CloudFiles(path).put_json("%s.spatial" % bbox.to_filename(precision), spatial_index, compress="gzip",
                              cache_control=False)


SEGIDRE = re.compile(r"(\d+):")


class UnshardedSkeletonMergeTask(RegisteredTask):
  """Stage 2 of skeletonization (igneous/tasks/skeleton.py:810-916): fuse every fragment of the labels whose
  file names start with `prefix`, postprocess them and write one precomputed skeleton per label.  The fuse and
  kimimaro.postprocess run for the whole prefix in one device call (kimimaro.merge_fragments, DESIGN.md §5h).
  A prefix like "1" also matches labels 10, 100, ...; "1:" matches label 1 alone."""

  def __init__(self, cloudpath, prefix, crop=0, dust_threshold=4000, max_cable_length=None, tick_threshold=6000,
               delete_fragments=False):
    super().__init__(cloudpath, prefix, crop, dust_threshold, max_cable_length, tick_threshold, delete_fragments)
    self.cloudpath, self.prefix, self.crop = cloudpath, prefix, crop
    self.dust_threshold, self.tick_threshold = dust_threshold, tick_threshold
    self.max_cable_length = float(max_cable_length) if max_cable_length is not None else None
    self.delete_fragments = bool(delete_fragments)

  def execute(self):
    last_phase_seconds.clear()
    t0 = time.perf_counter()
    vol = CloudVolume(self.cloudpath)
    vol.mip = vol.skeleton.meta.mip
    cf = CloudFiles(vol.skeleton.path)
    # names without "{segid}:" are the info, the .spatial files and finished skeletons
    filenames = [name for name in cf.list(prefix=str(self.prefix)) if SEGIDRE.search(name)]
    contents = cf.get(filenames, return_dict=True)
    t1 = time.perf_counter()
    fragments = defaultdict(list)
    for name in filenames:
      try:
        skel = pickle.loads(contents[name])
      except Exception as e:
        raise ValueError("UnshardedSkeletonMergeTask: cannot unpickle the fragment %s: %s" % (name, e)) from e
      if not isinstance(skel, kimimaro.Skeleton):
        raise ValueError("UnshardedSkeletonMergeTask: the fragment %s holds a %s, not an igneous_b200 Skeleton"
                         % (name, type(skel).__name__))
      fragments[int(SEGIDRE.search(name).group(1))].append((Bbox.from_filename(name), skel))
    t2 = time.perf_counter()
    vertex_types = any(a["id"] == "vertex_types" for a in vol.skeleton.meta.info.get("vertex_attributes") or [])
    merged = kimimaro.merge_fragments(fragments, crop=self.crop, resolution=vol.resolution,
                                      dust_threshold=self.dust_threshold, tick_threshold=self.tick_threshold,
                                      max_cable_length=self.max_cable_length, vertex_types=vertex_types)
    t3 = time.perf_counter()
    cf.puts(((str(segid), blob.tobytes()) for segid, (_, blob) in merged.items()), compress="gzip",
            content_type="application/octet-stream", cache_control=False)
    if self.delete_fragments:
      cf.delete(filenames)
    last_phase_seconds.update(list=t1 - t0, unpickle=t2 - t1, merge=t3 - t2, writes=time.perf_counter() - t3)
    return merged


def _skeleton_dir(vol):
  """the skeleton directory of a volume as a comparable path (file:// resolved on disk)"""
  path = vol.skeleton.path
  if path.startswith("file://"):
    return os.path.realpath(path[len("file://"):])
  return path.rstrip("/")


def refuse_same_directory(who, cv_src, cv_dest):
  if _skeleton_dir(cv_src) == _skeleton_dir(cv_dest):
    raise ValueError("%s: the destination skeleton directory %s is the source's; pass another dest or skel_dir"
                     % (who, cv_dest.skeleton.path))


@queueable
def ShardedFromUnshardedSkeletonMergeTask(src, dest, shard_no, cache_control=False, skel_dir=None, progress=False):
  """Write shard `shard_no` of a sharded skeleton layer from the unsharded skeletons of src
  (igneous/tasks/skeleton.py:1097-1130).  The labels are `{shard_no}.labels` of the destination skeleton
  directory (written by create_sharded_skeletons_from_unsharded_tasks); each one's skeleton is read from the
  source directory, the labels are ordered on the device, and every skeleton loses its integer vertex
  attributes in one device pass (DESIGN.md §5l).  Raw data with raw minishard indices leaves the device as
  the finished shard file; otherwise the host compresses each skeleton (gzip data) and builds the indices
  (gzip indices).  An empty label list writes nothing."""
  last_phase_seconds.clear()
  t0 = time.perf_counter()
  cv_src = CloudVolume(src)
  if skel_dir is None and "skeletons" in cv_src.info:
    skel_dir = cv_src.info["skeletons"]
  cv_dest = CloudVolume(dest, skel_dir=skel_dir, progress=progress)
  refuse_same_directory("ShardedFromUnshardedSkeletonMergeTask", cv_src, cv_dest)
  sharding = cv_dest.skeleton.meta.info.get("sharding")
  if not sharding:
    raise ValueError("ShardedFromUnshardedSkeletonMergeTask: %s/info has no sharding" % cv_dest.skeleton.path)
  spec = LabelShardingSpecification(sharding)
  cf_dest = CloudFiles(cv_dest.skeleton.path)
  labels = cf_dest.get_json("%s.labels" % shard_no)
  if labels is None:
    raise FileNotFoundError("ShardedFromUnshardedSkeletonMergeTask: no %s.labels in %s"
                            % (shard_no, cv_dest.skeleton.path))
  if len(labels) == 0:
    return
  labels = np.asarray([int(l) for l in labels], dtype=np.uint64)
  if np.unique(labels).size != labels.size:
    raise ValueError("ShardedFromUnshardedSkeletonMergeTask: %s.labels lists a label twice" % shard_no)
  labels, locations, _, shards = labelshard.shard_hash(labels, spec.preshift_bits, spec.minishard_bits,
                                                       spec.shard_bits)
  if shards.size != 1 or int(shards[0]) != int(shard_no):
    wrong = int(labels[np.argmax((locations >> np.uint64(spec.minishard_bits)) != np.uint64(int(shard_no)))]) \
        if spec.minishard_bits < 64 else int(labels[0])
    raise ValueError("ShardedFromUnshardedSkeletonMergeTask: label %d of %s.labels is not in shard %s"
                     % (wrong, shard_no, shard_no))
  t1 = time.perf_counter()
  cf_src = CloudFiles(cv_src.skeleton.path)
  names = [str(l) for l in labels.tolist()]
  contents = cf_src.get(names, return_dict=True)
  blobs = []
  for name in names:
    if contents.get(name) is None:
      raise FileNotFoundError("ShardedFromUnshardedSkeletonMergeTask: label %s of %s.labels has no skeleton in %s"
                              % (name, shard_no, cv_src.skeleton.path))
    blobs.append(contents[name])
  del contents
  t2 = time.perf_counter()
  attributes = cv_src.skeleton.meta.info.get("vertex_attributes") or []
  if spec.data_encoding == "raw" and spec.minishard_index_encoding == "raw":
    data = labelshard.restrip(blobs, attributes, locations, labels, spec.minishard_bits)
    t3 = t4 = time.perf_counter()
  else:
    buf, offs = labelshard.restrip(blobs, attributes)
    t3 = time.perf_counter()
    offs = offs.tolist()
    stored = [buf[a:b].tobytes() for a, b in zip(offs[:-1], offs[1:])]
    if spec.data_encoding == "gzip":
      stored = [gzip.compress(b, compresslevel=6, mtime=0) for b in stored]
    data = pack_shard(spec.minishard_bits, spec.minishard_index_encoding,
                      locations & np.uint64((1 << spec.minishard_bits) - 1), labels, stored)
    t4 = time.perf_counter()
  cf_dest.put(spec.shard_filename(int(shard_no)), data, compress=None, content_type="application/octet-stream",
              cache_control="no-cache")
  last_phase_seconds.update(labels=t1 - t0, read=t2 - t1, device=t3 - t2, gzip=t4 - t3,
                            write=time.perf_counter() - t4)
