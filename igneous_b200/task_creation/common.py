"""Grid enumeration shared by the task creators
(igneous/task_creation/common.py:11-104)."""
import copy
import itertools
import os
import subprocess
from functools import partial
from time import strftime

import numpy as np

from .._compat import Bbox, CloudFiles, CloudVolume, Vec
from ..tasks import SpatialIndexTask


def operator_contact():
  try:
    return str(subprocess.check_output("git config user.email", shell=True, stderr=subprocess.DEVNULL).rstrip())
  except Exception:
    return os.environ.get("USER", "")


def get_bounds(vol, bounds, mip, bounds_mip=0, chunk_size=None):
  if bounds is None:
    return vol.meta.bounds(mip)
  bounds = vol.bbox_to_mip(Bbox.create(bounds), mip=bounds_mip, to_mip=mip)
  if chunk_size is not None:
    bounds = bounds.expand_to_chunk_size(chunk_size, vol.meta.voxel_offset(mip))
  return Bbox.clamp(bounds, vol.meta.bounds(mip))


def num_tasks(bounds, shape):
  return int(np.prod(np.ceil(np.asarray(bounds.size3(), dtype=np.float64) / np.asarray(shape))))


class FinelyDividedTaskIterator:
  """Regular grid of non-overlapping tasks, x fastest (common.py:60-104)."""

  def __init__(self, bounds, shape):
    self.bounds = bounds
    self.shape = Vec(*shape)
    self.start = 0
    self.end = num_tasks(bounds, shape)

  def __len__(self):
    return self.end - self.start

  def __getitem__(self, slc):
    itr = copy.deepcopy(self)
    itr.start = max(self.start + slc.start, self.start)
    itr.end = min(self.start + slc.stop, self.end)
    return itr

  def to_coord(self, index):
    gx, gy, _ = np.ceil(np.asarray(self.bounds.size3(), dtype=np.float64) / np.asarray(self.shape)).astype(int)
    z, rem = divmod(index, gx * gy)
    y, x = divmod(rem, gx)
    return Vec(x, y, z)

  def __iter__(self):
    for i in range(self.start, self.end):
      offset = self.to_coord(i) * self.shape + self.bounds.minpt
      yield self.task(self.shape.clone(), Vec(*offset))
    self.on_finish()

  def task(self, shape, offset):
    raise NotImplementedError()

  def on_finish(self):
    pass


def spatial_index_tasks(cloudpath, shape, mip, fill_missing, compress, subdir, kind):
  """The body the mesh and skeleton spatial-index creators share (task_creation/mesh.py:363-435,
  task_creation/skeleton.py:795-867).  kind is "mesh" or "skeletons": the info key naming the
  directory.  Sets the layer's directory if it has none, records @type / mip / chunk_size /
  spatial_index in {subdir}/info when they change, and yields one SpatialIndexTask per grid cell."""
  shape = Vec(*shape)
  vol = CloudVolume(cloudpath, mip=mip)
  if subdir is None:
    subdir = vol.info.get(kind) or ("mesh_mip_%d_err_40" % mip if kind == "mesh" else "skeletons_mip_%d" % mip)
  if kind not in vol.info:
    vol.info[kind] = subdir
    vol.commit_info()
  cf = CloudFiles(cloudpath)
  info_filename = cf.join(subdir, "info")
  info = cf.get_json(info_filename) or {}
  new_info = copy.deepcopy(info)
  new_info["@type"] = new_info.get("@type", "neuroglancer_legacy_mesh" if kind == "mesh" else "neuroglancer_skeletons")
  new_info["mip"] = new_info.get("mip", int(vol.mip))
  new_info["chunk_size"] = shape.tolist()
  new_info["spatial_index"] = {"resolution": vol.resolution.tolist(), "chunk_size": (shape * vol.resolution).tolist()}
  if new_info != info:
    cf.put_json(info_filename, new_info)
  vol = CloudVolume(cloudpath, mip=mip)  # reload the spatial index
  precision = (vol.mesh if kind == "mesh" else vol.skeleton).spatial_index.precision

  class SpatialIndexTaskIterator(FinelyDividedTaskIterator):
    def task(self, shape, offset):
      return partial(SpatialIndexTask, cloudpath=cloudpath, shape=shape, offset=offset, subdir=subdir,
                     precision=precision, mip=int(mip), fill_missing=bool(fill_missing), compress=compress)

    def on_finish(self):
      vol.provenance.processing.append({
        "method": {"task": "SpatialIndexTask", "cloudpath": vol.cloudpath, "shape": shape.tolist(), "mip": int(mip),
                   "subdir": subdir, "fill_missing": fill_missing, "compress": compress},
        "by": operator_contact(), "date": strftime("%Y-%m-%d %H:%M %Z")})
      vol.commit_provenance()

  return SpatialIndexTaskIterator(vol.bounds, shape)


def compute_shard_params_for_hashed(num_labels, shard_index_bytes=2 ** 13, minishard_index_bytes=2 ** 15, min_shards=1):
  """(shard_bits, minishard_bits, preshift_bits) for labels spread evenly by a hash
  (igneous/task_creation/common.py:140-213).  A shard index of shard_index_bytes holds
  shard_index_bytes / 16 minishards; a minishard index of minishard_index_bytes holds
  minishard_index_bytes / 24 labels.  Enough minishard and shard bits are taken for num_labels to fit:
  a full shard index once the labels fill more than one shard, then whole shards; a shard less than 55%
  used gives one shard bit back.  At least round(log2(min_shards)) shard bits are kept, taken from the
  minishard bits.  Preshift is 0: hashed labels have no locality to keep."""
  assert min_shards >= 1
  if num_labels <= 0:
    return (0, 0, 0)
  minishards_per_shard = shard_index_bytes / 16
  labels_per_minishard = minishard_index_bytes / 24
  labels_per_shard = minishards_per_shard * labels_per_minishard
  if num_labels >= labels_per_shard:
    minishard_bits = int(np.ceil(np.log2(minishards_per_shard)))
    shard_bits = int(np.ceil(np.log2(num_labels / (labels_per_minishard * 2 ** minishard_bits))))
  elif num_labels >= labels_per_minishard:
    minishard_bits, shard_bits = int(np.ceil(np.log2(num_labels / labels_per_minishard))), 0
  else:
    minishard_bits, shard_bits = 0, 0
  if num_labels / (labels_per_shard * 2 ** shard_bits) <= 0.55:
    shard_bits -= 1
  shard_bits = max(shard_bits, 0)
  want = int(np.round(np.log2(min_shards)))
  if want > shard_bits:
    minishard_bits -= want - shard_bits
    shard_bits = want
  return (int(shard_bits), int(max(minishard_bits, 0)), 0)


def deletion_prefixes(who, magnitude):
  """the prefixes of the unsharded mesh and skeleton deletions: "0" (spatial index files from 0), "1:" ...
  "{10^(m-1) - 1}:", then 10^(m-1) ... 10^m - 1.  magnitude 0 has none (the reference's range(1, 0.1)
  fails), so it raises ValueError."""
  magnitude = int(magnitude)
  if magnitude < 1:
    raise ValueError("%s: magnitude must be at least 1 (got %d)" % (who, magnitude))
  start, end = 10 ** (magnitude - 1), 10 ** magnitude
  return ["0"] + [str(p) + ":" for p in range(1, start)] + [str(p) for p in range(start, end)]


def xfer_destination_dir(who, cf_dest, subdir, key):
  """the directory a mesh or skeleton transfer writes to: subdir, else the destination info's `key`.
  ValueError when the destination has no info (its tasks could not open it) or neither names a directory."""
  info = cf_dest.get_json("info")
  if info is None:
    raise ValueError("%s: %s has no info file" % (who, cf_dest.cloudpath))
  if not subdir:
    subdir = info.get(key)
  if not subdir:
    raise ValueError("%s: pass the destination directory or give %s/info a `%s`" % (who, cf_dest.cloudpath, key))
  return subdir


def xfer_prefixes(magnitude, sharded, suffix):
  """every string of `magnitude` characters over 0-9 (and a-f when sharded), then every shorter one
  followed by `suffix`"""
  alphabet = [str(i) for i in range(10)] + (list("abcdef") if sharded else [])
  prefixes = ["".join(x) for x in itertools.product(alphabet, repeat=int(magnitude))]
  for i in range(1, int(magnitude)):
    prefixes += ["".join(x) + suffix for x in itertools.product(alphabet, repeat=i)]
  return prefixes
