"""Minimal stand-ins for cloud-volume / cloud-files / task-queue, used ONLY when
those packages cannot be imported (they are absent from the build image, see
SURVEY.md 8(b) H8).  They implement just enough of the Precomputed `file://`
layout for the task layer to run end to end in tests:

  info JSON            {data_type, num_channels, type, scales:[{key, size,
                        resolution, voxel_offset, chunk_sizes, encoding}], mesh}
  chunk files          {key}/{x0}-{x1}_{y0}-{y1}_{z0}-{z1}[.gz]   raw, Fortran order
  mesh / ccl files     plain files under the layer directory

This is not a storage engine and it is never on the compute path: when the
real packages import, `igneous_b200._compat` uses them instead.
"""
import copy
import math
import gzip
import json
import os
import re
import shutil

import numpy as np


class EmptyVolumeException(Exception):
  pass


class InfoUnavailableError(Exception):
  pass


class OutOfBoundsError(Exception):
  pass


# ------------------------------------------------------------------ geometry
class Vec(np.ndarray):
  def __new__(cls, *args, dtype=int):
    if len(args) == 1 and hasattr(args[0], "__len__"):
      args = tuple(args[0])
    return np.array(args, dtype=dtype).view(cls)

  @property
  def x(self):
    return self[0]

  @x.setter
  def x(self, v):
    self[0] = v

  @property
  def y(self):
    return self[1]

  @y.setter
  def y(self, v):
    self[1] = v

  @property
  def z(self):
    return self[2]

  @z.setter
  def z(self, v):
    self[2] = v

  def clone(self):
    return Vec(*self, dtype=self.dtype)

  def rectVolume(self):
    return int(np.prod(self))


def min2(a, b):
  return Vec(*np.minimum(a, b), dtype=np.asarray(a).dtype)


def max2(a, b):
  return Vec(*np.maximum(a, b), dtype=np.asarray(a).dtype)


class Bbox:
  def __init__(self, a, b, dtype=int):
    a, b = np.asarray(a)[:3], np.asarray(b)[:3]
    self.minpt = Vec(*np.minimum(a, b), dtype=dtype)
    self.maxpt = Vec(*np.maximum(a, b), dtype=dtype)

  @classmethod
  def create(cls, obj):
    if isinstance(obj, Bbox):
      return obj.clone()
    if isinstance(obj, (list, tuple)) and len(obj) == 3 and isinstance(obj[0], slice):
      return cls([s.start for s in obj], [s.stop for s in obj])
    raise TypeError("cannot make a Bbox from %r" % (obj,))

  @classmethod
  def from_filename(cls, name):
    """the box in a file name such as 0-64_0-64_0-32.spatial or 5:0-64_0-64_0-32 (a skeleton fragment)"""
    m = re.search(r"(-?\d+)-(-?\d+)_(-?\d+)-(-?\d+)_(-?\d+)-(-?\d+)", os.path.basename(name))
    if m is None:
      raise ValueError("no bounding box in the file name %r" % name)
    v = [int(x) for x in m.groups()]
    return cls(v[0::2], v[1::2])

  @classmethod
  def clamp(cls, box, bounds):
    box = box.clone()
    box.minpt = Vec(*np.clip(box.minpt, bounds.minpt, bounds.maxpt), dtype=box.minpt.dtype)
    box.maxpt = Vec(*np.clip(box.maxpt, bounds.minpt, bounds.maxpt), dtype=box.maxpt.dtype)
    return box

  @classmethod
  def intersection(cls, a, b):
    lo = np.maximum(a.minpt, b.minpt)
    hi = np.minimum(a.maxpt, b.maxpt)
    if np.any(hi <= lo):
      return cls((0, 0, 0), (0, 0, 0))
    return cls(lo, hi)

  def clone(self):
    return Bbox(self.minpt, self.maxpt, dtype=self.minpt.dtype)

  def size3(self):
    return Vec(*(self.maxpt - self.minpt), dtype=self.minpt.dtype)

  size = size3

  def volume(self):
    return int(np.prod(self.size3()))

  def subvoxel(self):
    return bool(np.any(self.size3() <= 0))

  empty = subvoxel

  def center(self):
    return (self.minpt + self.maxpt) / 2.0

  def to_slices(self):
    return tuple(slice(int(a), int(b)) for a, b in zip(self.minpt, self.maxpt))

  def to_list(self):
    return [v.item() if hasattr(v, "item") else v for v in list(self.minpt) + list(self.maxpt)]

  def to_filename(self, precision=None):
    def fmt(v):
      if precision:
        return ("%." + str(int(precision)) + "f") % float(v)
      return str(int(v))
    return "_".join("%s-%s" % (fmt(a), fmt(b)) for a, b in zip(self.minpt, self.maxpt))

  def astype(self, dtype):
    return Bbox(self.minpt.astype(dtype), self.maxpt.astype(dtype), dtype=dtype)

  def round_to_chunk_size(self, chunk_size, offset=(0, 0, 0)):
    """minpt and maxpt each moved to the nearest chunk boundary (cloudvolume's rule as recalled: np.round
    of the chunk count, computed in float64, so a half goes to the even multiple)"""
    cs, off = np.asarray(chunk_size, dtype=np.float64)[:3], np.asarray(offset)[:3]
    lo = np.round((self.minpt - off) / cs) * cs + off
    hi = np.round((self.maxpt - off) / cs) * cs + off
    return Bbox(lo.astype(int), hi.astype(int))

  def expand_to_chunk_size(self, chunk_size, offset=(0, 0, 0)):
    cs, off = np.asarray(chunk_size)[:3], np.asarray(offset)[:3]
    lo = np.floor((self.minpt - off) / cs) * cs + off
    hi = np.ceil((self.maxpt - off) / cs) * cs + off
    return Bbox(lo.astype(int), hi.astype(int))

  def __floordiv__(self, f):
    f = np.asarray(f)[:3]
    return Bbox(self.minpt // f, -(-self.maxpt // f))

  def __ifloordiv__(self, f):
    f = np.asarray(f)[:3]
    self.minpt = Vec(*(self.minpt // f), dtype=self.minpt.dtype)
    self.maxpt = Vec(*(-(-self.maxpt // f)), dtype=self.maxpt.dtype)
    return self

  def __mul__(self, f):
    f = np.asarray(f)[:3]
    return Bbox(self.minpt * f, self.maxpt * f, dtype=np.result_type(self.minpt.dtype, f.dtype))

  def __sub__(self, v):
    return Bbox(self.minpt - np.asarray(v)[:3], self.maxpt - np.asarray(v)[:3])

  def __add__(self, v):
    return Bbox(self.minpt + np.asarray(v)[:3], self.maxpt + np.asarray(v)[:3])

  def __eq__(self, o):
    return isinstance(o, Bbox) and np.array_equal(self.minpt, o.minpt) and np.array_equal(self.maxpt, o.maxpt)

  def __repr__(self):
    return "Bbox(%s, %s)" % (list(self.minpt), list(self.maxpt))


# ------------------------------------------------------------ device cutouts
class DeviceCutout:
  """An F-order [x, y, z, c] array in device memory: what download_dev returns and upload_dev,
  make_shard_chunks and downsample_and_upload take, so that a cutout's chunks are decoded, re-cut,
  pooled and re-encoded without passing through host memory."""

  def __init__(self, buf, shape, dtype, ctx):
    self.buf, self.shape, self.dtype, self.ctx = buf, tuple(int(v) for v in shape), np.dtype(dtype), ctx

  @classmethod
  def empty(cls, shape, dtype, ctx=None):
    from . import _shim
    ctx = ctx or _shim.default_context()
    nbytes = int(np.prod(shape)) * np.dtype(dtype).itemsize
    return cls(ctx.alloc(max(nbytes, 8)), shape, dtype, ctx)

  @classmethod
  def from_host(cls, arr, ctx=None):
    arr = np.asarray(arr)
    if arr.ndim == 3:
      arr = arr[..., np.newaxis]
    out = cls.empty(arr.shape, arr.dtype, ctx)
    if arr.size:
      out.ctx.h2d(out.buf, np.asfortranarray(arr))
    return out

  @property
  def ptr(self):
    from . import _shim
    return _shim.ptr(self.buf)

  @property
  def size(self):
    return int(np.prod(self.shape))

  @property
  def nbytes(self):
    return self.size * self.dtype.itemsize

  def fill(self, box, value):
    """Set every voxel of `box` (a Bbox relative to the cutout), every channel, to `value` on the device."""
    from . import _shim
    bits = np.asarray(value).astype(self.dtype).reshape(1).view(np.dtype("u%d" % self.dtype.itemsize))[0]
    X, Y, Z, nc = self.shape
    _shim.check(self.ctx.lib.ign_fill_box_dev(self.ctx.handle, self.ptr, _shim.dtype_code(self.dtype), X, Y, Z, nc,
                                              *(int(v) for v in box.minpt), *(int(v) for v in box.size3()),
                                              int(bits)))

  def to_host(self):
    out = np.empty(self.shape, dtype=self.dtype, order="F")
    if out.size:
      self.ctx.d2h(out, self.buf)
    self.ctx.sync()
    return out


def _packed_offsets(sizes):
  """byte offsets of buffers of the given sizes packed back to back, and the total"""
  offs = np.zeros(len(sizes) + 1, dtype=np.int64)
  np.cumsum(np.asarray(sizes, dtype=np.int64), out=offs[1:])
  return offs


def _upload_bytes(ctx, datas):
  """one H2D of byte strings packed back to back -> (device buffer, byte offsets)"""
  offs = _packed_offsets([len(d) for d in datas])
  host = np.frombuffer(b"".join(bytes(d) for d in datas), dtype=np.uint8)
  buf = ctx.alloc(max(int(offs[-1]), 8))
  if host.size:
    ctx.h2d(buf, host)
  return buf, offs


# --------------------------------------------------------------------- files
def _strip(path):
  if path.startswith("file://"):
    path = path[len("file://"):]
  elif "://" in path:
    raise NotImplementedError("the storage stand-in only implements file:// (got %s)" % path)
  return path.rstrip("/")


class CloudFiles:
  """file:// subset of cloudfiles.CloudFiles."""
  _EXT = {"gzip": ".gz", "br": ".br", None: "", False: "", "": ""}

  def __init__(self, cloudpath, progress=False, **kwargs):
    self.cloudpath = cloudpath
    self.root = _strip(cloudpath)

  def join(self, *parts):
    return "/".join(str(p).strip("/") for p in parts if str(p) != "")

  def _abs(self, key):
    return os.path.join(self.root, key)

  def put(self, key, content, compress=None, **kwargs):
    path = self._abs(key) + self._EXT.get(compress, "")
    os.makedirs(os.path.dirname(path), exist_ok=True)
    if isinstance(content, str):
      content = content.encode("utf8")
    if compress in ("gzip", "br"):  # the stand-in stores both as gzip streams
      content = gzip.compress(content, compresslevel=1)
    with open(path, "wb") as f:
      f.write(content)

  def puts(self, files, compress=None, **kwargs):
    for item in files:
      if isinstance(item, dict):
        self.put(item["path"], item["content"], compress=item.get("compress", compress))
      else:
        self.put(item[0], item[1], compress=compress)

  def put_json(self, key, obj, compress=None, **kwargs):
    self.put(key, json.dumps(obj), compress=compress)

  def put_jsons(self, files, compress=None, **kwargs):
    for key, obj in files:
      self.put_json(key, obj, compress=compress)

  def _find(self, key):
    for ext in ("", ".gz", ".br"):
      path = self._abs(key) + ext
      if os.path.isfile(path):
        return path, ext
    return None, None

  def exists(self, key):
    return self._find(key)[0] is not None

  def get(self, key, return_dict=False, **kwargs):
    if isinstance(key, (list, tuple)) or return_dict:
      keys = list(key) if isinstance(key, (list, tuple)) else [key]
      return {k: self.get(k) for k in keys}
    path, ext = self._find(key)
    if path is None:
      return None
    with open(path, "rb") as f:
      data = f.read()
    return gzip.decompress(data) if ext else data

  def get_json(self, key):
    if isinstance(key, (list, tuple)):
      return [self.get_json(k) for k in key]
    data = self.get(key)
    return None if data is None else json.loads(data.decode("utf8"))

  def list(self, prefix="", flat=False):
    base = self._abs(prefix)
    top = base if os.path.isdir(base) else os.path.dirname(base)
    out = []
    for dirpath, _, files in os.walk(top):
      for fn in files:
        full = os.path.join(dirpath, fn)
        rel = os.path.relpath(full, self.root)
        for ext in (".gz", ".br"):
          if rel.endswith(ext):
            rel = rel[:-len(ext)]
        if rel.startswith(prefix):
          out.append(rel)
    return sorted(set(out))

  def transfer_to(self, cf_dest, paths, **kwargs):
    """Copy the stored files of `paths` (keys as list() gives them) to the same keys under cf_dest, byte for
    byte: a file stored with a compression suffix keeps its suffix and its compressed stream."""
    for key in list(paths):
      path, ext = self._find(key)
      if path is None:
        continue
      dest = cf_dest._abs(key) + ext
      os.makedirs(os.path.dirname(dest), exist_ok=True)
      shutil.copyfile(path, dest)

  def delete(self, keys):
    if isinstance(keys, str):
      keys = [keys]
    for k in list(keys):
      path, _ = self._find(k)
      if path:
        os.remove(path)


# -------------------------------------------------------------------- volume
class _Provenance:
  def __init__(self):
    self.processing = []
    self.sources = []
    self.owners = []
    self.description = ""


class _SpatialIndex:
  precision = 0


class _MeshMeta:
  """cv.mesh.meta: the mesh directory's info ({dir}/info, {} when the file is absent), the directory's path
  and whether its meshes are sharded."""

  def __init__(self, cv, subdir):
    self.subdir = subdir
    self.info = cv.cf.get_json(subdir + "/info") or {}
    self.layerpath = cv.join(cv.cloudpath, subdir)

  def is_sharded(self):
    return self.info.get("sharding") is not None


class _MeshSource:
  """cv.mesh: meta and spatial_index of the mesh directory (CloudVolume(mesh_dir=...), else the layer's
  info['mesh'], else `mesh`, as recalled of cloudvolume)."""

  spatial_index = _SpatialIndex()

  def __init__(self, cv):
    self.meta = _MeshMeta(cv, cv.mesh_dir or cv.info.get("mesh", "mesh"))


# cloudvolume's default skeleton info, as recalled (unpinned): identity transform, radius then vertex_types
DEFAULT_SKELETON_INFO = {
  "@type": "neuroglancer_skeletons",
  "transform": [1, 0, 0, 0, 0, 1, 0, 0, 0, 0, 1, 0],
  "vertex_attributes": [{"id": "radius", "data_type": "float32", "num_components": 1},
                        {"id": "vertex_types", "data_type": "uint8", "num_components": 1}],
  "sharding": None,
  "spatial_index": None,
}


class _SkeletonMeta:
  """cv.skeleton.meta: the skeleton directory's info ({info['skeletons']}/info, cloudvolume's default
  when the file is absent), the directory's path, whether it is sharded, and commit_info()."""

  def __init__(self, cv, subdir):
    self._cv, self.subdir = cv, subdir
    self.info = cv.cf.get_json(subdir + "/info") or copy.deepcopy(DEFAULT_SKELETON_INFO)
    self.layerpath = cv.join(cv.cloudpath, subdir)

  def is_sharded(self):
    return self.info.get("sharding") is not None

  @property
  def mip(self):
    """the mip the skeletons were made at (the info's `mip`; 0 when absent)"""
    return int(self.info.get("mip") or 0)

  def commit_info(self):
    self._cv.cf.put_json(self.subdir + "/info", self.info)


class _SkeletonSource:
  """cv.skeleton: meta, path, spatial_index (cv.mesh's) and get(segid) of precomputed skeletons, unsharded or
  in hashed shards (the info's `sharding`)."""

  def __init__(self, cv):
    # CloudVolume(skel_dir=...), else the layer's, else cloudvolume's default directory, as recalled
    subdir = cv.skel_dir or cv.info.get("skeletons", "skeletons")
    self._cv = cv
    self.meta = _SkeletonMeta(cv, subdir)
    self.path = cv.cf.join(cv.cloudpath, subdir)
    self.spatial_index = _MeshSource.spatial_index

  def get(self, segid):
    """The skeleton {dir}/{segid} decoded per meta.info['vertex_attributes'] (a list of ids -> a list)."""
    if isinstance(segid, (list, tuple)):
      return [self.get(s) for s in segid]
    from .kimimaro import split_blobs
    if self.meta.info.get("sharding"):
      data = self._sharded(int(segid))
    else:
      data = self._cv.cf.get("%s/%d" % (self.meta.subdir, int(segid)))
    if data is None:
      raise FileNotFoundError("no skeleton %d in %s" % (int(segid), self.path))
    buf = np.frombuffer(bytearray(data), dtype=np.uint8)  # writable: the Skeleton's arrays are views into it
    nv, ne = (int(v) for v in buf[:8].view(np.uint32))
    skeletons, blobs = split_blobs(buf, [(0, nv, ne)], [int(segid)], self.meta.info.get("vertex_attributes") or [])
    if blobs[0].size != buf.size:
      raise ValueError("skeleton %d: %d bytes, the info's attributes describe %d" % (int(segid), buf.size,
                                                                                      blobs[0].size))
    return skeletons[0]

  def _sharded(self, segid):
    """the blob of segid from its shard file, or None"""
    from .sharding import LabelShardingSpecification
    spec = LabelShardingSpecification(self.meta.info["sharding"])
    shard = self._cv.cf.get("%s/%s" % (self.meta.subdir, spec.shard_filename(spec.locate(segid)[0])))
    return None if shard is None else spec.read_chunk(shard, segid)


class _Meta:
  """cv.meta: per-mip accessors (cloudvolume's PrecomputedMetadata subset)."""

  def __init__(self, cv):
    self._cv = cv

  def resolution(self, mip):
    return self._cv.resolution_at(mip)

  def chunk_size(self, mip):
    return self._cv.chunk_size_at(mip)

  def volume_size(self, mip):
    return self._cv.volume_size_at(mip)

  def voxel_offset(self, mip):
    return self._cv.voxel_offset_at(mip)

  def bounds(self, mip):
    return self._cv.bounds_at(mip)

  def voxels(self, mip):
    return self._cv.volume_size_at(mip).rectVolume()

  def add_resolution(self, *args, **kwargs):
    return self._cv.add_resolution(*args, **kwargs)

  def join(self, *parts):
    return self._cv.join(*parts)

  def key(self, mip):
    return self._cv.key_at(mip)

  def unlock_mips(self, mips):
    """Clear the write lock of the given mip(s) (in memory, as cloudvolume does until the
    next commit_info); the stand-in never sets one, so this only drops a `locked` key."""
    for m in ([mips] if np.isscalar(mips) else mips):
      if 0 <= int(m) < len(self._cv.info["scales"]):
        self._cv.info["scales"][int(m)].pop("locked", None)

  @property
  def cloudpath(self):
    return self._cv.cloudpath

  @property
  def info(self):
    return self._cv.info


class _ImageSource:
  """cv.image: the two shard builders ImageShardDownsampleTask calls
  (igneous/tasks/image/image.py:664-669,818,833) and transfer_to (image.py:483-496)."""

  def __init__(self, cv):
    self._cv = cv

  def make_shard_chunks(self, img, bbox, mip):
    """Cut `img` (occupying `bbox` at `mip`; a host array or a DeviceCutout) into the scale's chunks
    -> {chunk id: encoded bytes}, cut and encoded on the device."""
    cv = self._cv
    bbox = Bbox.create(bbox) if not isinstance(bbox, Bbox) else bbox
    spec = cv._sharding(mip)
    if spec is None:
      raise ValueError("mip %d of %s is not sharded" % (mip, cv.cloudpath))
    cs, off = cv.chunk_size_at(mip), cv.voxel_offset_at(mip)
    if np.any((np.asarray(bbox.minpt) - np.asarray(off)) % np.asarray(cs)):
      raise ValueError("shard cutout %r is not chunk aligned" % (bbox,))
    shape = img.shape if isinstance(img, DeviceCutout) else np.shape(img)
    boxes = list(cv._chunks(mip, Bbox.clamp(bbox, cv.bounds_at(mip))))
    for c in boxes:
      if np.any(np.asarray(c.maxpt) - np.asarray(bbox.minpt) > np.asarray(shape[:3])):
        raise ValueError("image %r does not cover chunk %r of %r" % (tuple(shape), c, bbox))
    files, _ = cv._chunk_files(img, [c - bbox.minpt for c in boxes], mip)
    return {cv._chunk_id(mip, c): f for c, f in zip(boxes, files)}

  def transfer_to(self, dest_path, bbox, mip, compress="gzip"):
    """Copy the chunk files under `bbox` to the same names in dest_path's layer without decoding them
    (cloudvolume's image.transfer_to).  The destination scale must have this scale's chunk grid (chunk
    size and bounds, which fix the names and extents of the files) and encoding; the files are stored
    with `compress`."""
    cv = self._cv
    dest = CloudVolume(dest_path, mip=mip)
    if dest._sharding(mip) is not None:
      raise NotImplementedError("transfer_to writes unsharded chunk files; a sharded destination takes whole shards")
    a, b = cv.scales[mip], dest.scales[mip]
    if not (np.array_equal(cv.chunk_size_at(mip), dest.chunk_size_at(mip)) and cv.bounds_at(mip) == dest.bounds_at(mip)
            and all(a.get(k) == b.get(k) for k in ("encoding", "compressed_segmentation_block_size", "jpeg_quality"))
            and cv.dtype == dest.dtype and cv.num_channels == dest.num_channels):
      raise ValueError("transfer_to copies files as they are: %s and %s differ in chunk grid or encoding at mip %d"
                       % (cv.cloudpath, dest_path, mip))
    bbox = Bbox.clamp(cv._to_bbox(bbox), cv.bounds_at(mip))
    shard_cache = {}
    for c in cv._chunks(mip, bbox):
      data = cv._read_chunk(mip, c, shard_cache)
      if data is None:
        if not cv.fill_missing:
          raise EmptyVolumeException(cv._chunk_name(mip, c))
        continue
      dest.cf.put(dest._chunk_name(mip, c), data, compress=None if cv._encoding(mip) == "jpeg" else compress)

  def make_shard(self, img, bbox, mip, progress=False):
    """-> (file name, shard bytes).  `img` is an array or a {chunk id: bytes} dict."""
    cv = self._cv
    spec = cv._sharding(mip)
    chunks = img if isinstance(img, dict) else self.make_shard_chunks(img, bbox, mip)
    if not chunks:
      raise ValueError("no chunks inside %r" % (bbox,))
    shard_no = spec.locate(next(iter(chunks)))[0]
    return spec.shard_filename(shard_no), spec.synthesize_shard(chunks)


class CloudVolume:
  """file:// Precomputed subset of cloudvolume.CloudVolume."""

  def __init__(self, cloudpath, mip=0, fill_missing=False, bounded=True, info=None, compress="gzip",
               delete_black_uploads=False, background_color=0, parallel=1, progress=False, non_aligned_writes=False,
               skel_dir=None, mesh_dir=None, **kwargs):
    self.cloudpath = cloudpath
    self.skel_dir = skel_dir
    self.mesh_dir = mesh_dir
    self.path = _strip(cloudpath)
    self.fill_missing = bool(fill_missing)
    self.bounded = bounded
    self.compress = compress
    self.delete_black_uploads = delete_black_uploads
    self.background_color = background_color
    self.non_aligned_writes = bool(non_aligned_writes)
    self.cf = CloudFiles(cloudpath)
    self.provenance = _Provenance()
    self._mesh = None
    self._skeleton = None
    if info is not None:
      self.info = copy.deepcopy(info)
    else:
      self.info = self.cf.get_json("info")
      if self.info is None:
        raise InfoUnavailableError("no info file at " + cloudpath)
    prov = self.cf.get_json("provenance")
    if prov:
      self.provenance.processing = prov.get("processing", [])
    self.mip = mip

  @property
  def meta(self):
    return _Meta(self)

  @property
  def image(self):
    return _ImageSource(self)

  @property
  def mesh(self):
    """the mesh source, read on first use (its info file and directory follow mesh_dir or info['mesh'])"""
    if self._mesh is None:
      self._mesh = _MeshSource(self)
    return self._mesh

  @property
  def skeleton(self):
    """the skeleton source, read on first use (its info file and directory follow info['skeletons'])"""
    if self._skeleton is None:
      self._skeleton = _SkeletonSource(self)
    return self._skeleton

  @classmethod
  def create_new_info(cls, num_channels, layer_type, data_type, encoding, resolution, voxel_offset,
                      volume_size, chunk_size=(64, 64, 64), mesh=None, **kwargs):
    res = [int(r) if float(r).is_integer() else float(r) for r in resolution]
    info = {"num_channels": int(num_channels), "type": layer_type, "data_type": str(np.dtype(data_type)),
            "scales": [{"encoding": encoding, "chunk_sizes": [list(map(int, chunk_size))],
                        "key": "_".join(str(r) for r in res), "resolution": res,
                        "voxel_offset": list(map(int, voxel_offset)), "size": list(map(int, volume_size))}]}
    if mesh:
      info["mesh"] = mesh
    return info

  @classmethod
  def from_numpy(cls, arr, vol_path, resolution=(4, 4, 40), voxel_offset=(0, 0, 0), chunk_size=(128, 128, 64),
                 layer_type=None, max_mip=0, encoding="raw", compress=None):
    arr = np.asarray(arr)
    if arr.ndim == 3:
      arr = arr[..., np.newaxis]
    if layer_type is None:
      layer_type = "segmentation" if arr.dtype in (np.uint16, np.uint32, np.uint64) else "image"
    info = cls.create_new_info(arr.shape[3], layer_type, arr.dtype, encoding, resolution, voxel_offset,
                               arr.shape[:3], chunk_size)
    vol = cls(vol_path, info=info, compress=compress)
    vol.commit_info()
    vol[vol.bounds] = arr
    return vol

  # ---- info accessors
  @property
  def scales(self):
    return self.info["scales"]

  @property
  def available_mips(self):
    return list(range(len(self.info["scales"])))

  @property
  def dtype(self):
    return np.dtype(self.info["data_type"])

  data_type = dtype

  @property
  def layer_type(self):
    return self.info["type"]

  @property
  def num_channels(self):
    return int(self.info["num_channels"])

  def resolution_at(self, mip):
    return Vec(*self.info["scales"][mip]["resolution"], dtype=np.float32 if any(
      not float(r).is_integer() for r in self.info["scales"][mip]["resolution"]) else int)

  def chunk_size_at(self, mip):
    return Vec(*self.info["scales"][mip]["chunk_sizes"][0])

  def volume_size_at(self, mip):
    return Vec(*self.info["scales"][mip]["size"])

  def voxel_offset_at(self, mip):
    return Vec(*self.info["scales"][mip]["voxel_offset"])

  def bounds_at(self, mip):
    off = self.voxel_offset_at(mip)
    return Bbox(off, off + self.volume_size_at(mip))

  # current-mip properties, as on cloudvolume.CloudVolume
  resolution = property(lambda self: self.resolution_at(self._mip))
  downsample_ratio = property(lambda self: Vec(*(np.asarray(self.resolution_at(self._mip), dtype=np.float64)
                                                 / np.asarray(self.resolution_at(0), dtype=np.float64)),
                                               dtype=np.float64))
  chunk_size = property(lambda self: self.chunk_size_at(self._mip))
  volume_size = property(lambda self: self.volume_size_at(self._mip))
  voxel_offset = property(lambda self: self.voxel_offset_at(self._mip))
  bounds = property(lambda self: self.bounds_at(self._mip))

  def key_at(self, mip):
    return self.info["scales"][mip]["key"]

  @property
  def key(self):
    return self.key_at(self._mip)

  def join(self, *parts):
    return "/".join(str(p).rstrip("/") for p in parts)

  def mip_bounds(self, mip):
    return self.bounds_at(mip)

  def mip_volume_size(self, mip):
    return self.volume_size_at(mip)

  def bbox_to_mip(self, bbox, mip, to_mip):
    if mip == to_mip:
      return bbox.clone()
    f = np.asarray(self.resolution_at(to_mip), dtype=np.float64) / np.asarray(self.resolution_at(mip), dtype=np.float64)
    lo = np.floor(np.asarray(bbox.minpt) / f).astype(int)
    hi = np.ceil(np.asarray(bbox.maxpt) / f).astype(int)
    return Bbox(lo, hi)

  def add_resolution(self, res, encoding=None, chunk_size=None, info=None):
    base = self.info["scales"][0]
    res = [int(r) if float(r).is_integer() else float(r) for r in res]
    factor = np.asarray(res, dtype=np.float64) / np.asarray(base["resolution"], dtype=np.float64)
    key = "_".join(str(r) for r in res)
    scale = {"encoding": encoding or base["encoding"],
             "chunk_sizes": [list(map(int, chunk_size))] if chunk_size is not None else copy.deepcopy(base["chunk_sizes"]),
             "key": key, "resolution": res,
             "voxel_offset": [int(v) for v in np.floor(np.asarray(base["voxel_offset"]) / factor)],
             "size": [int(v) for v in np.ceil(np.asarray(base["size"]) / factor)]}
    for i, s in enumerate(self.info["scales"]):
      if s["key"] == key:
        self.info["scales"][i] = scale
        return scale
    self.info["scales"].append(scale)
    self.info["scales"].sort(key=lambda s: float(np.prod(s["resolution"])))
    return scale

  # ---- mip state: cv.mip and CloudVolume properties that depend on it
  @property
  def mip(self):
    return self._mip

  @mip.setter
  def mip(self, m):
    self._mip = int(m)

  def commit_info(self):
    self.cf.put_json("info", self.info)

  def refresh_info(self):
    self.info = self.cf.get_json("info")
    return self.info

  def commit_provenance(self):
    self.cf.put_json("provenance", {"processing": self.provenance.processing, "sources": [], "owners": [],
                                    "description": ""})

  # ---- IO
  def _chunk_name(self, mip, box):
    return self.key_at(mip) + "/" + box.to_filename()

  def _chunks(self, mip, box):
    cs, off = self.chunk_size_at(mip), self.voxel_offset_at(mip)
    vb = self.bounds_at(mip)
    grid = box.expand_to_chunk_size(cs, off)
    for z in range(int(grid.minpt[2]), int(grid.maxpt[2]), int(cs[2])):
      for y in range(int(grid.minpt[1]), int(grid.maxpt[1]), int(cs[1])):
        for x in range(int(grid.minpt[0]), int(grid.maxpt[0]), int(cs[0])):
          c = Bbox.clamp(Bbox((x, y, z), (x + cs[0], y + cs[1], z + cs[2])), vb)
          if not c.subvoxel():
            yield c

  # sharded scales (neuroglancer_uint64_sharded_v1, igneous_b200.sharding)
  def _sharding(self, mip):
    spec = self.info["scales"][mip].get("sharding")
    if not spec:
      return None
    from . import sharding
    return sharding.ShardingSpecification(spec)

  def _chunk_id(self, mip, chunk_box):
    from . import sharding
    cs, off = self.chunk_size_at(mip), self.voxel_offset_at(mip)
    grid = [int(math.ceil(int(v) / int(c))) for v, c in zip(self.volume_size_at(mip), cs)]
    pt = [int((int(a) - int(o)) // int(c)) for a, o, c in zip(chunk_box.minpt, off, cs)]
    return int(sharding.compressed_morton_code(pt, grid))

  def _read_chunk(self, mip, chunk_box, shard_cache):
    spec = self._sharding(mip)
    if spec is None:
      return self.cf.get(self._chunk_name(mip, chunk_box))
    cid = self._chunk_id(mip, chunk_box)
    name = self.key_at(mip) + "/" + spec.shard_filename(spec.locate(cid)[0])
    if name not in shard_cache:
      shard_cache[name] = self.cf.get(name)
    blob = shard_cache[name]
    return None if blob is None else spec.read_chunk(blob, cid)

  # chunk codecs: `raw` is the bytes of the Fortran-order array; `compressed_segmentation` and
  # `jpeg` go through the device codecs (igneous_b200.codecs), a whole read or write per call;
  # anything else the Precomputed format knows (png, compresso, crackle, ...) is outside this stand-in
  def _encoding(self, mip):
    return self.info["scales"][mip].get("encoding", "raw")

  def _jpeg_check(self, mip):
    if self.dtype != np.uint8 or self.num_channels != 1:
      raise NotImplementedError("storage stand-in: jpeg scales hold one uint8 channel (got %s x %d)"
                                % (self.dtype, self.num_channels))

  def _cseg_block(self, mip):
    return tuple(int(v) for v in self.info["scales"][mip].get("compressed_segmentation_block_size", (8, 8, 8)))

  def _device_cutout(self, img):
    """img (a host array or a DeviceCutout) as a DeviceCutout of this layer's dtype"""
    if isinstance(img, DeviceCutout):
      if img.dtype == self.dtype:
        return img
      img = img.to_host()
    img = np.asarray(img)
    if img.ndim == 3:
      img = img[..., np.newaxis]
    return DeviceCutout.from_host(img.astype(self.dtype, copy=False))

  def _chunk_files(self, img, boxes, mip):
    """chunk files of `mip` for boxes (relative Bboxes) of a host array or DeviceCutout -> (list of
    bytes, list of all-background flags).  `raw` files of a host array are its own bytes and need no
    device; everything else is cut and encoded on the device."""
    if not isinstance(img, DeviceCutout) and self._encoding(mip) == "raw":
      return self._raw_boxes(img, boxes)
    return self._encode_boxes(self._device_cutout(img), boxes, mip)

  def _raw_boxes(self, img, boxes):
    """`raw` chunk files of boxes of a host array: the boxes' F-order bytes, which need no device"""
    img = np.asarray(img)
    if img.ndim == 3:
      img = img[..., np.newaxis]
    img = img.astype(self.dtype, copy=False)
    blocks = [np.asfortranarray(img[b.to_slices()]) for b in boxes]
    return [b.tobytes(order="F") for b in blocks], [not np.any(b != self.background_color) for b in blocks]

  def _encode_boxes(self, cutout, boxes, mip):
    """Encode boxes (Bboxes relative to the cutout) of a device cutout as chunk files of `mip`: one
    cut, one batched encode and one D2H -> (list of bytes, list of all-background flags)."""
    from . import _shim
    ctx = cutout.ctx
    enc = self._encoding(mip)
    if enc not in ("raw", "compressed_segmentation", "jpeg"):
      raise NotImplementedError("storage stand-in: chunk encoding %r is not supported" % enc)
    if enc == "jpeg":
      self._jpeg_check(mip)
    if not boxes:
      return [], []
    nc, es = cutout.shape[3], cutout.dtype.itemsize
    sizes = [np.asarray(b.size3(), dtype=np.int64) for b in boxes]
    offs = _packed_offsets([int(np.prod(z)) * nc * es for z in sizes])
    rows = np.ascontiguousarray(np.array([list(b.minpt) + list(z) + [o] for b, z, o in zip(boxes, sizes, offs[:-1])],
                                         dtype=np.uint64))
    packed = ctx.alloc(max(int(offs[-1]), 8))
    flags_dev = ctx.alloc(4 * len(boxes))
    want = np.asarray(self.background_color)
    typed = want.astype(cutout.dtype).reshape(1)
    # a background the dtype cannot hold (-1 for uint8) matches no voxel: no box is all background
    representable = bool(typed[0] == want)
    bg = typed.view(np.dtype("u%d" % es))[0]
    X, Y, Z = cutout.shape[:3]
    _shim.check(ctx.lib.ign_chunks_cut_dev(ctx.handle, cutout.ptr, _shim.dtype_code(cutout.dtype), X, Y, Z, nc,
                                           _shim.ptr(rows), len(boxes), int(bg), _shim.ptr(packed),
                                           _shim.ptr(flags_dev)))
    flags = np.empty(len(boxes), dtype=np.uint32)
    ctx.d2h(flags, flags_dev)
    shapes = np.ascontiguousarray(np.array(sizes, dtype=np.uint32).reshape(len(boxes), 3))
    if enc == "raw":
      host = np.empty(int(offs[-1]), dtype=np.uint8)
      ctx.d2h(host, packed)
      ctx.sync()
      return [host[offs[i]:offs[i + 1]].tobytes() for i in range(len(boxes))], [representable and bool(f) for f in flags]
    if enc == "compressed_segmentation":
      from . import codecs
      files = codecs.cseg_encode_batch_dev(packed, cutout.dtype, shapes, nc, self._cseg_block(mip), ctx)
      ctx.sync()
      return files, [representable and bool(f) for f in flags]
    from . import codecs
    files = codecs.jpeg_encode_batch_dev(packed, shapes, int(self.info["scales"][mip].get("jpeg_quality", 85)), ctx)
    ctx.sync()
    return files, [representable and bool(f) for f in flags]

  def _decode_into(self, cutout, pieces, mip):
    """Decode chunk files into their places in a device cutout: one H2D of the files, one batched
    decode, one place.  pieces: (chunk shape [x, y, z], file bytes, source corner in the chunk, box
    size, destination corner in the cutout)."""
    from . import _shim
    ctx = cutout.ctx
    enc = self._encoding(mip)
    if enc not in ("raw", "compressed_segmentation", "jpeg"):
      raise NotImplementedError("storage stand-in: chunk encoding %r is not supported" % enc)
    if enc == "jpeg":
      self._jpeg_check(mip)
    if not pieces:
      return
    nc, es = cutout.shape[3], cutout.dtype.itemsize
    shapes = np.ascontiguousarray(np.array([p[0] for p in pieces], dtype=np.uint32).reshape(len(pieces), 3))
    offs = _packed_offsets([int(np.prod(p[0], dtype=np.int64)) * nc * es for p in pieces])
    streams, soffs = _upload_bytes(ctx, [p[1] for p in pieces])
    if enc == "raw":
      for i, p in enumerate(pieces):
        if soffs[i + 1] - soffs[i] != offs[i + 1] - offs[i]:
          raise ValueError("raw chunk %d: %d bytes for a %r x %d chunk of %s" % (i, soffs[i + 1] - soffs[i],
                                                                               tuple(p[0]), nc, cutout.dtype))
      packed = streams
    else:
      packed = ctx.alloc(max(int(offs[-1]), 8))
      from . import codecs
      if enc == "compressed_segmentation":
        codecs.cseg_decode_batch_dev(streams, soffs, cutout.dtype, shapes, nc, self._cseg_block(mip), packed, ctx)
      else:
        codecs.jpeg_decode_batch_dev(streams, soffs, shapes, packed, ctx)
    rows = np.ascontiguousarray(np.array([list(p[0]) + [o] + list(p[2]) + list(p[3]) + list(p[4])
                                          for p, o in zip(pieces, offs[:-1])], dtype=np.uint64))
    X, Y, Z = cutout.shape[:3]
    _shim.check(ctx.lib.ign_chunks_place_dev(ctx.handle, _shim.ptr(packed), _shim.dtype_code(cutout.dtype), nc,
                                             _shim.ptr(rows), len(pieces), cutout.ptr, X, Y, Z))
    ctx.sync()

  def _to_bbox(self, key):
    if isinstance(key, Bbox):
      return key.clone()
    if isinstance(key, slice):
      key = (key,)
    if isinstance(key, tuple):
      b = self.bounds
      key = tuple(key) + (slice(None),) * (3 - len(key[:3]))
      lo = [b.minpt[i] if key[i].start is None else key[i].start for i in range(3)]
      hi = [b.maxpt[i] if key[i].stop is None else key[i].stop for i in range(3)]
      return Bbox(lo, hi)
    raise TypeError(key)

  def download(self, bbox, mip=None, renumber=False, **kwargs):
    """Cutout as an F-order [x, y, z, c] array (download_dev + one D2H).  renumber=True -> (array of
    the smallest dtype holding 1..N, {old: new}) with the relabelling done on the GPU
    (cloudvolume's download(renumber=True), image.py:745-752)."""
    if renumber:
      from . import fastremap
      img = self.download(bbox, mip=mip, **kwargs)
      small, mapping = fastremap.renumber(img, preserve_zero=True, in_place=False)
      return small, mapping
    mip = self._mip if mip is None else mip
    if self._encoding(mip) != "raw":
      return self.download_dev(bbox, mip=mip).to_host()
    # `raw` chunks are the cutout's own bytes: assembled on the host, with no device needed
    bbox, pieces = self._pieces(bbox, mip)
    out = np.zeros(tuple(int(v) for v in bbox.size3()) + (self.num_channels,), dtype=self.dtype, order="F")
    for shape, data, src, size, dst in pieces:
      chunk = np.frombuffer(data, dtype=self.dtype).reshape(tuple(shape) + (self.num_channels,), order="F")
      out[tuple(slice(d, d + z) for d, z in zip(dst, size))] = chunk[tuple(slice(a, a + z) for a, z in zip(src, size))]
    return out

  def _pieces(self, bbox, mip, fill_missing=None):
    """(bbox, the chunk files under it) for a read: (chunk shape, file bytes, corner in the chunk, box size,
    corner in the cutout) per chunk that is present; a missing chunk raises unless fill_missing (None: the
    volume's setting)"""
    fill_missing = self.fill_missing if fill_missing is None else fill_missing
    bbox = self._to_bbox(bbox)
    if self.bounded and not (np.all(bbox.minpt >= self.bounds_at(mip).minpt) and np.all(bbox.maxpt <= self.bounds_at(mip).maxpt)):
      raise OutOfBoundsError("%r is outside %r" % (bbox, self.bounds_at(mip)))
    shard_cache = {}
    pieces = []
    for c in self._chunks(mip, bbox):
      data = self._read_chunk(mip, c, shard_cache)
      inter = Bbox.intersection(c, bbox)
      if inter.subvoxel():
        continue
      if data is None:
        if not fill_missing:
          raise EmptyVolumeException(self._chunk_name(mip, c))
        continue
      pieces.append(([int(v) for v in c.size3()], data, [int(v) for v in inter.minpt - c.minpt],
                     [int(v) for v in inter.size3()], [int(v) for v in inter.minpt - bbox.minpt]))
    return bbox, pieces

  def download_dev(self, bbox, mip=None, ctx=None, fill_missing=None):
    """Cutout as a DeviceCutout: the chunk files are read (unsharded files or shard reads), sent to
    the device in one copy, decoded in one batched call and placed in one launch.  Voxels outside
    the volume, and missing chunks under fill_missing (None: the volume's setting), are 0."""
    from . import _shim
    mip = self._mip if mip is None else mip
    bbox, pieces = self._pieces(bbox, mip, fill_missing)
    ctx = ctx or _shim.default_context()
    out = DeviceCutout.empty(tuple(int(v) for v in bbox.size3()) + (self.num_channels,), self.dtype, ctx)
    ctx.memset(out.buf, 0, out.nbytes)
    self._decode_into(out, pieces, mip)
    return out

  def __getitem__(self, key):
    return self.download(key)

  def __setitem__(self, key, img):
    self.upload_dev(self._to_bbox(key), img, mip=self._mip)

  def _write_region(self, bbox, mip):
    """The chunk-aligned region a write of `bbox` at `mip` covers: bbox itself when it is chunk aligned;
    otherwise, under non_aligned_writes, bbox expanded to the chunk grid and clamped to the bounds, and
    without it a ValueError."""
    for c in self._chunks(mip, bbox):
      inter = Bbox.intersection(c, bbox)
      if inter.subvoxel() or inter == c:
        continue
      if not self.non_aligned_writes:
        raise ValueError("writes must be chunk aligned: %r vs chunk %r" % (bbox, c))
      vb = self.bounds_at(mip)
      if not (np.all(bbox.minpt >= vb.minpt) and np.all(bbox.maxpt <= vb.maxpt)):
        raise OutOfBoundsError("a non-aligned write of %r reaches outside %r" % (bbox, vb))
      return Bbox.clamp(bbox.expand_to_chunk_size(self.chunk_size_at(mip), self.voxel_offset_at(mip)), vb)
    return bbox

  def upload_dev(self, bbox, img, mip=None):
    """Write a cutout (a DeviceCutout, or a host array that is sent over first): one cut, one batched
    encode and one D2H, then one file per chunk.  Under delete_black_uploads the chunks that hold only
    background_color are deleted instead.  A box off the chunk grid raises ValueError unless
    non_aligned_writes is set; then the chunk-aligned region around it is read (missing chunks as 0),
    the cutout is placed into it on the device and the region is written."""
    mip = self._mip if mip is None else mip
    bbox = self._to_bbox(bbox)
    shape = img.shape if isinstance(img, DeviceCutout) else np.shape(img)
    if tuple(shape[:3]) != tuple(int(v) for v in bbox.size3()):
      raise ValueError("image %r does not fit %r" % (tuple(shape), bbox))
    if self._sharding(mip) is not None:
      raise NotImplementedError("writes to a sharded scale go through image.make_shard (whole shards only)")
    region = self._write_region(bbox, mip)
    if not (region == bbox):
      img, bbox = self._placed(img, bbox, region, mip), region
    boxes = [c for c in self._chunks(mip, bbox) if not Bbox.intersection(c, bbox).subvoxel()]
    files, black = self._chunk_files(img, [c - bbox.minpt for c in boxes], mip)
    # jpeg files are already entropy coded: stored without gzip, as CloudVolume stores jpeg chunks
    compress = None if self._encoding(mip) == "jpeg" else self.compress
    for c, data, bg in zip(boxes, files, black):
      name = self._chunk_name(mip, c)
      if self.delete_black_uploads and bg:
        self.cf.delete(name)
        continue
      self.cf.put(name, data, compress=compress)

  def _placed(self, img, bbox, region, mip):
    """`region` read from the layer (missing chunks as 0) with img placed at bbox, as a DeviceCutout"""
    from . import _shim
    src = self._device_cutout(img)
    out = self.download_dev(region, mip=mip, ctx=src.ctx, fill_missing=True)
    X, Y, Z, nc = out.shape
    size = [int(v) for v in bbox.size3()]
    row = np.array(size + [0, 0, 0, 0] + size + [int(v) for v in bbox.minpt - region.minpt], dtype=np.uint64)
    _shim.check(out.ctx.lib.ign_chunks_place_dev(out.ctx.handle, src.ptr, _shim.dtype_code(out.dtype), nc,
                                                 _shim.ptr(row), 1, out.ptr, X, Y, Z))
    return out

  def delete(self, bbox, mip=None):
    """Delete the chunk files at `mip` that lie wholly inside `bbox` (cloudvolume's delete)."""
    mip = self._mip if mip is None else mip
    if self._sharding(mip) is not None:
      raise NotImplementedError("deleting from a sharded scale would rewrite whole shards; only unsharded "
                                "scales are supported")
    bbox = self._to_bbox(bbox)
    self.cf.delete([self._chunk_name(mip, c) for c in self._chunks(mip, bbox) if Bbox.intersection(c, bbox) == c])


# --------------------------------------------------------------------- queue
def queueable(fn):
  return fn


class RegisteredTask:
  def __init__(self, *args, **kwargs):
    self._args, self._kwargs = args, kwargs

  def execute(self):
    raise NotImplementedError()


class LocalTaskQueue:
  """In-process immediate execution (taskqueue.LocalTaskQueue(parallel=1))."""

  def __init__(self, parallel=1, **kwargs):
    self.parallel = parallel
    self.executed = 0

  def _run(self, task):
    if hasattr(task, "execute"):
      task.execute()
    else:
      task()
    self.executed += 1

  def insert(self, tasks, **kwargs):
    if hasattr(tasks, "execute") or callable(tasks):
      tasks = [tasks]
    for t in tasks:
      self._run(t)

  insert_all = insert

  def execute(self, **kwargs):
    pass
