"""MeshTask with marching cubes + simplification on the GPU.

Mirror of igneous/tasks/mesh/mesh.py:39-464 for the unsharded `precomputed`
path (MeshTask.__init__ options :98-129, execute :140-265,
_handle_dataset_boundary :267-303, _remove_dust :313-322, _remap :357-369,
fill_holes :211-243, compute_meshes :371-383, _create_mesh_binary :432-450, uploads :399-464).
zmesh / fastremap / fastmorph are replaced by igneous_b200.zmesh / .fastremap / .fastmorph.

The manifest, transfer and deletion tasks (:624-749) only list, group, copy and delete files; they have no
device work (DESIGN.md §5m).
"""
import os
import re
from collections import defaultdict

import numpy as np

from .. import fastmorph, fastremap, zmesh
from .._compat import CloudVolume, CloudFiles, Bbox, Vec, RegisteredTask, queueable

_DEFAULTS = {
  "cache_control": None, "draco_compression_level": 1, "draco_create_metadata": False,
  "dust_threshold": None, "dust_global": False, "encoding": "precomputed", "fill_missing": False,
  "generate_manifests": False, "high_padding": 1, "low_padding": 0, "lod": 0,
  "max_simplification_error": 40, "simplification_factor": 100, "mesh_dir": None, "frag_path": None,
  "mip": 0, "object_ids": None, "exclude_object_ids": [], "parallel_download": 1, "progress": False,
  "remap_table": None, "spatial_index": False, "sharded": False, "timestamp": None,
  "agglomerate": True, "stop_layer": 2, "compress": "gzip", "closed_dataset_edges": True,
  "fill_holes": 0, "dry_run": False,
}


class MeshTask(RegisteredTask):
  def __init__(self, shape, offset, layer_path, **kwargs):
    super().__init__(shape, offset, layer_path, **kwargs)
    self.shape = Vec(*shape)
    self.offset = Vec(*offset)
    self.layer_path = layer_path
    self.options = {k: kwargs.get(k, v) for k, v in _DEFAULTS.items()}
    if self.options["encoding"] not in ("precomputed", "draco"):
      raise ValueError("Encoding {} is not supported. Options: precomputed, draco".format(self.options["encoding"]))
    if self.options["encoding"] == "draco":
      raise NotImplementedError("igneous_b200 MeshTask: draco encoding is out of scope (DESIGN.md)")
    for k in ("sharded", "dust_global"):
      if self.options[k]:
        raise NotImplementedError("igneous_b200 MeshTask: %s=True is out of scope (DESIGN.md)" % k)

  # ------------------------------------------------------------------ execute
  def execute(self):
    opt = self.options
    vol = self._volume = CloudVolume(self.layer_path, opt["mip"], bounded=False,
                                     fill_missing=opt["fill_missing"])
    mip = opt["mip"]
    self._bounds = Bbox.clamp(Bbox(self.offset, self.shape + self.offset), vol.meta.bounds(mip))
    self._mesher = zmesh.Mesher(vol.meta.resolution(mip))
    self._mesh_dir = self.get_mesh_dir()

    data_bounds = self._bounds.clone()  # marching cubes wants a 1 voxel overlap
    data_bounds.minpt = data_bounds.minpt - opt["low_padding"]
    data_bounds.maxpt = data_bounds.maxpt + opt["high_padding"]
    data = self._download(data_bounds)
    if not np.any(data):
      if opt["spatial_index"]:
        self._upload_spatial_index(self._bounds, {})
      return

    left_offset = Vec(0, 0, 0)
    if opt["closed_dataset_edges"]:
      data, left_offset = self._handle_dataset_boundary(data, data_bounds)
    data = self._remove_dust(data, opt["dust_threshold"])
    data = self._remap(data)
    if opt["object_ids"]:
      data = fastremap.mask_except(data, opt["object_ids"], in_place=True)
    if opt["exclude_object_ids"]:
      data = fastremap.mask(data, opt["exclude_object_ids"], in_place=True)
    data, renumbermap = fastremap.renumber(data, in_place=True)
    renumbermap = {v: k for k, v in renumbermap.items()}

    data = data[..., 0]
    fill_level = int(opt["fill_holes"])
    if fill_level > 0:  # mesh.py:211-243: enclosed objects keep their own meshes, their cell is solid
      if fill_level >= 3:
        data = fastmorph.dilate(data, mode=fastmorph.Mode.multilabel, background_only=True, parallel=1)
      filled, holes = fastmorph.fill_holes_v2(
        data, fix_borders=(fill_level >= 2),
        merge_threshold=(1.0 if fill_level <= 3 else (1.0 - 0.01 * (fill_level - 3))), parallel=1)
      del data
      self._mesher.mesh(filled, preserve_order=False)
      meshes = self.compute_meshes(renumbermap)
      del filled
      self._mesher.mesh(holes)
      hole_meshes = self.compute_meshes(renumbermap)
      del holes
      for segid, mesh in hole_meshes.items():
        meshes[segid] = zmesh.Mesh.concatenate(meshes[segid], mesh, id=segid) if segid in meshes else mesh
    else:
      self._mesher.mesh(data, preserve_order=False)
      del data
      meshes = self.compute_meshes(renumbermap)

    bounding_boxes = {}
    for segid, mesh in meshes.items():
      binary, bbx = self._create_mesh_binary(mesh, left_offset)
      meshes[segid] = binary
      bounding_boxes[segid] = bbx
    self._upload_individuals(meshes, opt["generate_manifests"])
    if opt["spatial_index"]:
      self._upload_spatial_index(self._bounds, bounding_boxes)

  def _download(self, bounds):
    """volume.download(bounds) with bounded=False: out-of-volume voxels read as 0."""
    vb = self._volume.meta.bounds(self.options["mip"])
    inner = Bbox.intersection(bounds, vb)
    out = np.zeros(tuple(int(v) for v in bounds.size3()) + (self._volume.num_channels,),
                   dtype=self._volume.dtype, order="F")
    if not inner.subvoxel():
      sl = tuple(slice(int(a - o), int(b - o)) for a, b, o in zip(inner.minpt, inner.maxpt, bounds.minpt))
      out[sl] = self._volume.download(inner, mip=self.options["mip"])  # mesh.py:177-182
    return out

  def _handle_dataset_boundary(self, data, bbox):
    """Zero border on every side that touches the dataset edge, so that meshes
    close there (mesh.py:267-303); returns the low-side shift it introduced."""
    vb = self._volume.meta.bounds(self.options["mip"])
    if not np.any(bbox.minpt == vb.minpt) and not np.any(bbox.maxpt == vb.maxpt):
      return data, Vec(0, 0, 0)
    lo = [int(bbox.minpt[i] == vb.minpt[i]) for i in range(3)]
    hi = [int(bbox.maxpt[i] == vb.maxpt[i]) for i in range(3)]
    shape = [data.shape[i] + lo[i] + hi[i] for i in range(3)] + [data.shape[3]]
    padded = np.zeros(shape, dtype=data.dtype, order="F")
    padded[lo[0]:lo[0] + data.shape[0], lo[1]:lo[1] + data.shape[1], lo[2]:lo[2] + data.shape[2]] = data
    return padded, Vec(*lo)

  def get_mesh_dir(self):
    if self.options["mesh_dir"] is not None:
      return self.options["mesh_dir"]
    if "mesh" in self._volume.info:
      return self._volume.info["mesh"]
    raise ValueError("The mesh destination is not present in the info file.")

  def _remove_dust(self, data, dust_threshold):
    if not dust_threshold:
      return data
    segids, counts = fastremap.unique(data, return_counts=True)
    dust = [int(s) for s, ct in zip(segids, counts) if ct < int(dust_threshold)]
    return fastremap.mask(data, dust, in_place=True)

  def _remap(self, data):
    table = self.options["remap_table"]
    if table is None:
      return data
    table = {int(k): int(v) for k, v in table.items()}
    table[0] = 0
    self.options["remap_table"] = table
    data = fastremap.mask_except(data, list(table.keys()), in_place=True)
    return fastremap.remap(data, table, in_place=True)

  def compute_meshes(self, renumbermap):
    out = {}
    for obj_id in self._mesher.ids():
      out[renumbermap[obj_id]] = self._mesher.get(
        obj_id, reduction_factor=self.options["simplification_factor"],
        max_error=self.options["max_simplification_error"], voxel_centered=True)
    return out

  def _create_mesh_binary(self, mesh, left_bound_offset):
    res = np.asarray(self._volume.meta.resolution(self.options["mip"]), dtype=np.float32)
    shift = (np.asarray(self._bounds.minpt, dtype=np.float32) - np.float32(self.options["low_padding"])
             - np.asarray(left_bound_offset, dtype=np.float32)) * res
    mesh.vertices[:] += shift.astype(np.float32)
    lo, hi = np.amin(mesh.vertices, axis=0), np.amax(mesh.vertices, axis=0)
    return mesh.to_precomputed(), [float(v) for v in lo] + [float(v) for v in hi]

  def _upload_individuals(self, binaries, generate_manifests):
    cf = CloudFiles(self.layer_path)
    lod, name = self.options["lod"], self._bounds.to_filename()
    # mesh.py:399-430: fragments carry the mesh content type and the task's cache_control,
    # manifests are stored uncompressed
    cf.puts((("%s/%s:%s:%s" % (self._mesh_dir, segid, lod, name), b) for segid, b in binaries.items()),
            compress=self.options["compress"], cache_control=self.options["cache_control"],
            content_type="model/mesh")
    if generate_manifests:
      cf.put_jsons((("%s/%s:%s" % (self._mesh_dir, segid, lod),
                     {"fragments": ["%s:%s:%s" % (segid, lod, name)]}) for segid in binaries),
                   compress=None, cache_control=self.options["cache_control"])

  def _upload_spatial_index(self, bbox, mesh_bboxes):
    cf = CloudFiles(self.layer_path)
    res = self._volume.meta.resolution(self.options["mip"])
    phys = bbox.astype(np.asarray(res).dtype) * res
    cf.put_json("%s/%s.spatial" % (self._mesh_dir, phys.to_filename(self._volume.mesh.spatial_index.precision)),
                {str(k): v for k, v in mesh_bboxes.items()}, compress=self.options["compress"],
                cache_control=False)  # mesh.py:452-464


# a fragment "{segid}:{lod}:{bbox}"; a manifest "{segid}:{lod}", the info and .spatial files never match
FRAGMENT = re.compile(r"(\d+):(\d+):")


def _manifest_dir(who, cf, mesh_dir):
  """mesh_dir, else the layer info's `mesh`; ValueError when neither names one"""
  if mesh_dir is not None:
    return mesh_dir
  info = cf.get_json("info")
  if info is None or "mesh" not in info:
    raise ValueError("%s: pass mesh_dir or give %s/info a `mesh` directory" % (who, cf.cloudpath))
  return info["mesh"]


def _put_manifests(cf, mesh_dir, lod, names):
  """{mesh_dir}/{segid}:{lod} -> {"fragments": [...]} for the names of lod's fragments, grouped by segid in
  the order they come, stored uncompressed"""
  segids = defaultdict(list)
  for name in names:
    m = FRAGMENT.search(name)
    if m is None or int(m.group(2)) != lod:
      continue
    segids[int(m.group(1))].append(name)
  cf.put_jsons(("%s/%d:%d" % (mesh_dir, segid, lod), {"fragments": frags}) for segid, frags in segids.items())


@queueable
def MeshManifestPrefixTask(layer_path, prefix, lod=0, mesh_dir=None):
  """Write the manifest of every label with a lod fragment whose name starts with `prefix` in the mesh
  directory (igneous/tasks/mesh/mesh.py:672-724).  Names are the listing's, without a storage suffix, so
  neuroglancer requests the fragments by them."""
  cf = CloudFiles(layer_path)
  mesh_dir = _manifest_dir("MeshManifestPrefixTask", cf, mesh_dir)
  names = (os.path.basename(n) for n in cf.list(prefix=cf.join(mesh_dir, prefix)))
  _put_manifests(cf, mesh_dir, int(lod), names)


@queueable
def MeshManifestFilesystemTask(layer_path, lod=0, mesh_dir=None):
  """MeshManifestPrefixTask over one scan of a file:// mesh directory (igneous/tasks/mesh/mesh.py:624-670):
  regular files only, each name without its extension (1:0:0-64_0-64_0-64.gz -> 1:0:0-64_0-64_0-64)."""
  cf = CloudFiles(layer_path)
  mesh_dir = _manifest_dir("MeshManifestFilesystemTask", cf, mesh_dir)
  path = layer_path[len("file://"):] if layer_path.startswith("file://") else layer_path
  if "://" in path:
    raise ValueError("MeshManifestFilesystemTask: %s is not a file:// path" % layer_path)
  with os.scandir(os.path.join(path, mesh_dir)) as entries:
    names = [os.path.splitext(e.name)[0] for e in entries if e.is_file()]
  _put_manifests(cf, mesh_dir, int(lod), names)


@queueable
def TransferMeshFilesTask(src, dest, prefix, mesh_dir=None):
  """Copy the stored files whose names start with `prefix` from src's mesh directory to dest's (mesh_dir,
  else dest's info), byte for byte (igneous/tasks/mesh/mesh.py:726-739)."""
  cv_src = CloudVolume(src)
  cv_dest = CloudVolume(dest, mesh_dir=mesh_dir)
  cf_src = CloudFiles(cv_src.mesh.meta.layerpath)
  cf_src.transfer_to(CloudFiles(cv_dest.mesh.meta.layerpath), paths=cf_src.list(prefix=prefix))


@queueable
def DeleteMeshFilesTask(cloudpath, prefix, mesh_dir=None):
  """Delete the files whose names start with `prefix` in the mesh directory (igneous/tasks/mesh/mesh.py:741-749)."""
  cv = CloudVolume(cloudpath, mesh_dir=mesh_dir)
  cf = CloudFiles(cv.mesh.meta.layerpath)
  cf.delete(cf.list(prefix=prefix))
