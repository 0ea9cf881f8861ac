"""create_skeletonizing_tasks (igneous/task_creation/skeleton.py:68-388),
create_unsharded_skeleton_merge_tasks (:535-591), create_sharded_skeletons_from_unsharded_tasks (:659-753),
create_spatial_index_skeleton_tasks (:795-867), create_skeleton_deletion_tasks (:593-657) and
create_xfer_skeleton_tasks (:756-793)."""
import copy
import re
from functools import partial
from time import strftime

import numpy as np

from .. import labelshard
from .._compat import CloudVolume, CloudFiles, Vec
from ..sharding import LabelShardingSpecification
from ..tasks import (SkeletonTask, UnshardedSkeletonMergeTask, ShardedFromUnshardedSkeletonMergeTask,
                     DeleteSkeletonFilesTask, TransferSkeletonFilesTask)
from ..tasks.skeleton import refuse, refuse_same_directory
from .common import (FinelyDividedTaskIterator, compute_shard_params_for_hashed, deletion_prefixes, operator_contact,
                     spatial_index_tasks, xfer_destination_dir, xfer_prefixes)


def create_skeletonizing_tasks(cloudpath, mip, shape=Vec(512, 512, 512), teasar_params={"scale": 10, "const": 10},
                               info=None, object_ids=None, mask_ids=None, fix_branching=True, fix_borders=True,
                               fix_avocados=False, fill_holes=0, dust_threshold=1000, progress=False, parallel=1,
                               fill_missing=False, sharded=False, frag_path=None, spatial_index=True, synapses=None,
                               num_synapses=None, dust_global=False, fix_autapses=False, cross_sectional_area=False,
                               cross_sectional_area_smoothing_window=5, timestamp=None, root_ids_cloudpath=None,
                               cross_sectional_area_repair_sec_per_label=0):
  """Tasks with one voxel of overlap on the high side in a regular grid, to be densely skeletonized
  (SkeletonTask); the fragments are merged by create_unsharded_skeleton_merge_tasks.  Records the layer's skeleton
  directory (skeletons_mip_{mip} unless it has one), the skeleton info's @type, spatial_index, mip and
  float32-only vertex_attributes, the frag_path info, and the provenance on completion.
  The options SkeletonTask refuses (sharded, dust_global, synapses, cross_sectional_area, fix_autapses /
  timestamp / root_ids_cloudpath, fix_avocados, fill_holes > 0) raise NotImplementedError here, before any
  write.  The reference narrows the grid to the mesh bounds of up to four object_ids (bounds_from_mesh);
  that needs mesh reads the storage layer here does not have, so the grid always covers the full bounds."""
  assert 0 <= fill_holes <= 103, "fill_holes must be between 0 to 103 inclusive."
  refuse("create_skeletonizing_tasks", sharded, dust_global, synapses, cross_sectional_area, fix_autapses,
         timestamp, root_ids_cloudpath, fix_avocados, fill_holes)
  shape = Vec(*shape)
  vol = CloudVolume(cloudpath, mip=mip, info=info)
  if "skeletons" not in vol.info:
    vol.info["skeletons"] = "skeletons_mip_{}".format(mip)
    vol.commit_info()

  skel_info = vol.skeleton.meta.info
  if spatial_index:
    if "spatial_index" not in skel_info or not skel_info["spatial_index"]:
      skel_info["spatial_index"] = {}
    skel_info["@type"] = "neuroglancer_skeletons"
    skel_info["spatial_index"]["resolution"] = tuple(vol.resolution.tolist())
    skel_info["spatial_index"]["chunk_size"] = tuple((shape * vol.resolution).tolist())
  skel_info["mip"] = int(mip)
  skel_info["vertex_attributes"] = [attr for attr in skel_info["vertex_attributes"]
                                    if attr["data_type"] == "float32"]
  skel_info["vertex_attributes"] = [attr for attr in skel_info["vertex_attributes"]
                                    if attr["id"] != "cross_sectional_area"]
  vol.skeleton.meta.commit_info()

  if frag_path:
    cf = CloudFiles(frag_path)
    frag_info = cf.get_json("info")
    if not frag_info:
      cf.put_json("info", vol.skeleton.meta.info)
    elif "scales" in frag_info:
      cf.put_json(cf.join(vol.info["skeletons"], "info"), vol.skeleton.meta.info)

  will_postprocess = bool(np.any(vol.bounds.size3() > shape))
  bounds = vol.bounds.clone()

  class SkeletonTaskIterator(FinelyDividedTaskIterator):
    def task(self, shape, offset):
      return SkeletonTask(
        cloudpath=cloudpath, shape=(shape + 1).clone(), offset=offset.clone(), mip=mip,
        teasar_params=teasar_params, will_postprocess=will_postprocess, info=info, object_ids=object_ids,
        mask_ids=mask_ids, fix_branching=fix_branching, fix_borders=fix_borders, fix_avocados=fix_avocados,
        dust_threshold=dust_threshold, progress=progress, parallel=parallel, fill_missing=bool(fill_missing),
        sharded=bool(sharded), frag_path=frag_path, spatial_index=bool(spatial_index),
        spatial_grid_shape=shape.clone(), synapses=None, dust_global=dust_global, fix_autapses=bool(fix_autapses),
        timestamp=timestamp, cross_sectional_area=bool(cross_sectional_area),
        cross_sectional_area_smoothing_window=int(cross_sectional_area_smoothing_window),
        root_ids_cloudpath=root_ids_cloudpath, fill_holes=fill_holes,
        cross_sectional_area_repair_sec_per_label=int(cross_sectional_area_repair_sec_per_label))

    def on_finish(self):
      vol.provenance.processing.append({
        "method": {
          "task": "SkeletonTask", "cloudpath": cloudpath, "mip": mip, "shape": shape.tolist(),
          "dust_threshold": dust_threshold, "teasar_params": teasar_params, "object_ids": object_ids,
          "mask_ids": mask_ids, "will_postprocess": will_postprocess, "fix_branching": fix_branching,
          "fix_borders": fix_borders, "fix_avocados": fix_avocados, "progress": progress, "parallel": parallel,
          "fill_missing": bool(fill_missing), "sharded": bool(sharded), "spatial_index": bool(spatial_index),
          "synapses": bool(synapses), "dust_global": bool(dust_global), "fix_autapses": bool(fix_autapses),
          "timestamp": timestamp, "cross_sectional_area": bool(cross_sectional_area),
          "cross_sectional_area_smoothing_window": int(cross_sectional_area_smoothing_window),
          "cross_sectional_area_repair_sec_per_label": int(cross_sectional_area_repair_sec_per_label),
          "root_ids_cloudpath": root_ids_cloudpath, "fill_holes": int(fill_holes),
        },
        "by": operator_contact(),
        "date": strftime("%Y-%m-%d %H:%M %Z"),
      })
      vol.commit_provenance()

  return SkeletonTaskIterator(bounds, shape)


def create_unsharded_skeleton_merge_tasks(layer_path, crop=0, magnitude=3, dust_threshold=4000, max_cable_length=None,
                                          tick_threshold=6000, delete_fragments=False):
  """UnshardedSkeletonMergeTasks over every label of the layer's skeleton fragments, split by file name
  prefix: "1:" ... "{10^(m-1) - 1}:" for the labels below 10^(m-1), then 10^(m-1) ... 10^m - 1, each of
  which also matches the longer labels that start with it.  The provenance is appended after iteration."""
  assert int(magnitude) == magnitude
  start, end = 10 ** (magnitude - 1), 10 ** magnitude

  class UnshardedSkeletonMergeTaskIterator:
    def __len__(self):
      return 10 ** magnitude

    def __iter__(self):
      for prefix in [str(p) + ":" for p in range(1, start)] + list(range(start, end)):
        yield UnshardedSkeletonMergeTask(cloudpath=layer_path, prefix=prefix, crop=crop,
                                         dust_threshold=dust_threshold, max_cable_length=max_cable_length,
                                         tick_threshold=tick_threshold, delete_fragments=delete_fragments)
      vol = CloudVolume(layer_path)
      vol.provenance.processing.append({
        "method": {
          "task": "UnshardedSkeletonMergeTask", "cloudpath": layer_path, "crop": crop,
          "dust_threshold": dust_threshold, "tick_threshold": tick_threshold, "delete_fragments": delete_fragments,
          "max_cable_length": max_cable_length,
        },
        "by": operator_contact(),
        "date": strftime("%Y-%m-%d %H:%M %Z"),
      })
      vol.commit_provenance()

  return UnshardedSkeletonMergeTaskIterator()


def create_spatial_index_skeleton_tasks(cloudpath, shape=(448, 448, 448), mip=0, fill_missing=False, compress="gzip",
                                        skel_dir=None):
  """Rebuild the spatial index of a skeleton directory (default: the layer's, else skeletons_mip_{mip}),
  or build one over a different grid than the skeleton tasks used."""
  return spatial_index_tasks(cloudpath, shape, mip, fill_missing, compress, skel_dir, "skeletons")


# a source skeleton file: the whole name is the label's digits, optionally with a compression suffix (chosen:
# the reference's re.search would also take the trailing digits of "{segid}:{bbox}" fragment names)
LABEL_FILE = re.compile(r"(\d+)(\.gz|\.br|\.zstd)?")


def create_sharded_skeletons_from_unsharded_tasks(src, dest, shard_index_bytes=2 ** 13, minishard_index_bytes=2 ** 15,
                                                  min_shards=1, minishard_index_encoding="gzip",
                                                  data_encoding="gzip", skel_dir=None):
  """ShardedFromUnshardedSkeletonMergeTasks that turn the unsharded skeletons of src into a sharded
  (murmurhash3_x86_128) skeleton layer at dest (igneous/task_creation/skeleton.py:659-753).  The destination
  skeleton info is the source's with only its float32 and float64 vertex_attributes and a `sharding` from
  compute_shard_params_for_hashed; every label is hashed on the device, each shard's labels go to a gzipped
  `{shard}.labels` JSON list in (minishard, label) order, the provenance is appended, and one task is
  returned per non-empty shard, in shard order.  A destination that is the source's skeleton directory raises
  ValueError, and a source skeleton stored with brotli or zstd NotImplementedError, before anything is
  written (DESIGN.md §5l)."""
  cv_src = CloudVolume(src)
  cv_src.mip = cv_src.skeleton.meta.mip
  cv_dest = CloudVolume(dest, skel_dir=skel_dir)
  refuse_same_directory("create_sharded_skeletons_from_unsharded_tasks", cv_src, cv_dest)
  labels = []
  for name in CloudFiles(cv_src.skeleton.path).list():
    m = LABEL_FILE.fullmatch(name)
    if m is None:
      continue
    if m.group(2) in (".br", ".zstd"):
      raise NotImplementedError("create_sharded_skeletons_from_unsharded_tasks: %s is stored with %s; only raw "
                                "and gzip skeletons are read" % (name, m.group(2)[1:]))
    if int(m.group(1)) >= 1 << 64:
      raise ValueError("create_sharded_skeletons_from_unsharded_tasks: %s is not a uint64 label" % name)
    labels.append(int(m.group(1)))

  shard_bits, minishard_bits, preshift_bits = compute_shard_params_for_hashed(
    num_labels=len(labels), shard_index_bytes=int(shard_index_bytes),
    minishard_index_bytes=int(minishard_index_bytes), min_shards=int(min_shards))
  spec = LabelShardingSpecification({
    "@type": "neuroglancer_uint64_sharded_v1", "preshift_bits": preshift_bits, "hash": "murmurhash3_x86_128",
    "minishard_bits": minishard_bits, "shard_bits": shard_bits,
    "minishard_index_encoding": minishard_index_encoding, "data_encoding": data_encoding})
  info = copy.deepcopy(cv_src.skeleton.meta.info)
  info["vertex_attributes"] = [a for a in info.get("vertex_attributes") or []
                               if a["data_type"] in ("float32", "float64")]
  info["sharding"] = spec.to_dict()
  ordered, _, starts, shards = labelshard.shard_hash(np.array(labels, dtype=np.uint64), preshift_bits,
                                                     minishard_bits, shard_bits)
  starts = starts.tolist()

  cv_dest.skeleton.meta.info = info
  cv_dest.skeleton.meta.commit_info()
  cf = CloudFiles(cv_dest.skeleton.path)
  cf.put_jsons((("%d.labels" % s, ordered[a:b].tolist()) for s, a, b in zip(shards.tolist(), starts[:-1], starts[1:])),
               compress="gzip", cache_control="no-cache")
  cv_dest.provenance.processing.append({
    "method": {
      "task": "ShardedFromUnshardedSkeletonMergeTask", "src": src, "dest": dest, "preshift_bits": preshift_bits,
      "minishard_bits": minishard_bits, "shard_bits": shard_bits, "skel_dir": skel_dir,
    },
    "by": operator_contact(),
    "date": strftime("%Y-%m-%d %H:%M %Z"),
  })
  cv_dest.commit_provenance()
  return [partial(ShardedFromUnshardedSkeletonMergeTask, src=src, dest=dest, shard_no=str(s), skel_dir=skel_dir)
          for s in shards.tolist()]


def create_skeleton_deletion_tasks(cloudpath, magnitude=2, skel_dir=None):
  """Tasks that delete the skeleton directory's files.  The directory's info is deleted here, while the
  tasks are made, and the provenance is appended.  A sharded directory gets one task over every file;
  otherwise 10^m tasks: "0", "1:" ... "{10^(m-1) - 1}:", then 10^(m-1) ... 10^m - 1 (DESIGN.md §5m lists the
  files these leave).  magnitude=0 raises ValueError before anything is deleted."""
  assert int(magnitude) == magnitude
  assert magnitude >= 0
  prefixes = deletion_prefixes("create_skeleton_deletion_tasks", magnitude)
  cv = CloudVolume(cloudpath, skel_dir=skel_dir)
  CloudFiles(cv.skeleton.meta.layerpath).delete("info")
  if cv.skeleton.meta.is_sharded():
    prefixes = [""]
  cv.provenance.processing.append({
    "method": {"task": "DeleteSkeletonFilesTask", "cloudpath": cloudpath, "skel_dir": skel_dir},
    "by": operator_contact(),
    "date": strftime("%Y-%m-%d %H:%M %Z"),
  })
  cv.commit_provenance()
  return [partial(DeleteSkeletonFilesTask, cloudpath=cloudpath, prefix=p, skel_dir=skel_dir) for p in prefixes]


def create_xfer_skeleton_tasks(src, dest, skel_dir=None, magnitude=2):
  """Tasks that copy src's skeleton files, byte for byte, to dest's skeleton directory (skel_dir, else
  dest's info['skeletons']), after writing src's skeleton info there.  The prefixes are every string of
  `magnitude` digits (hex digits for a sharded source), then every shorter one, which overlap the longer ones.
  A dest without an info file, or with neither skel_dir nor a `skeletons` in its info, raises ValueError before
  anything is written."""
  cv_src = CloudVolume(src)
  cf_dest = CloudFiles(dest)
  skel_dir = xfer_destination_dir("create_xfer_skeleton_tasks", cf_dest, skel_dir, "skeletons")
  cf_dest.put_json("%s/info" % skel_dir, cv_src.skeleton.meta.info)
  prefixes = xfer_prefixes(magnitude, cv_src.skeleton.meta.is_sharded(), "")
  return [partial(TransferSkeletonFilesTask, src=src, dest=dest, prefix=p, skel_dir=skel_dir) for p in prefixes]
