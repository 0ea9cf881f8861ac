"""create_meshing_tasks (igneous/task_creation/mesh.py:158-267), create_spatial_index_mesh_tasks (:363-435),
create_mesh_manifest_tasks (:54-89), create_mesh_deletion_tasks (:91-155) and create_xfer_meshes_tasks
(:548-588)."""
from functools import partial
from time import strftime

from .._compat import CloudVolume, CloudFiles, Vec
from ..tasks import MeshTask, MeshManifestPrefixTask, MeshManifestFilesystemTask, TransferMeshFilesTask, DeleteMeshFilesTask
from .common import (FinelyDividedTaskIterator, deletion_prefixes, operator_contact, spatial_index_tasks,
                     xfer_destination_dir, xfer_prefixes)


def create_meshing_tasks(layer_path, mip, shape=(448, 448, 448), simplification=True,
                         max_simplification_error=40.0, mesh_dir=None, cdn_cache=False,
                         dust_threshold=None, object_ids=None, progress=False, fill_missing=False,
                         encoding="precomputed", spatial_index=True, frag_path=None, sharded=False,
                         compress="gzip", closed_dataset_edges=True, dust_global=False, fill_holes=0,
                         dry_run=False, exclude_object_ids=[]):
  shape = Vec(*shape)
  assert 0 <= fill_holes <= 103, "fill_holes must be between 0 to 103 inclusive."
  vol = CloudVolume(layer_path, mip)
  if mesh_dir is None:
    mesh_dir = vol.info.get("mesh", "mesh_mip_{}_err_{}".format(mip, max_simplification_error))
  if "mesh" not in vol.info:
    vol.info["mesh"] = mesh_dir
    vol.commit_info()
  cf = CloudFiles(layer_path)
  res = vol.meta.resolution(mip)
  mesh_info = cf.get_json("{}/info".format(mesh_dir)) or {}
  mesh_info.update({"@type": "neuroglancer_legacy_mesh", "mip": int(mip), "chunk_size": [int(s) for s in shape]})
  if spatial_index:
    mesh_info["spatial_index"] = {"resolution": [float(r) for r in res],
                                  "chunk_size": [float(s * r) for s, r in zip(shape, res)]}
  cf.put_json("{}/info".format(mesh_dir), mesh_info)
  options = dict(mip=mip, simplification_factor=(100 if simplification else 0),
                 max_simplification_error=max_simplification_error, mesh_dir=mesh_dir,
                 cache_control=("" if cdn_cache else "no-cache"), dust_threshold=dust_threshold,
                 dust_global=bool(dust_global), progress=progress, object_ids=object_ids,
                 exclude_object_ids=exclude_object_ids, fill_missing=fill_missing, encoding=encoding,
                 spatial_index=spatial_index, frag_path=frag_path, sharded=sharded, compress=compress,
                 closed_dataset_edges=closed_dataset_edges, fill_holes=fill_holes, dry_run=dry_run)

  class MeshTaskIterator(FinelyDividedTaskIterator):
    def task(self, shape, offset):
      return MeshTask(shape=shape.clone(), offset=offset.clone(), layer_path=layer_path, **options)

    def on_finish(self):
      vol.provenance.processing.append({
        "method": dict(task="MeshTask", layer_path=layer_path, shape=[int(s) for s in shape],
                       simplification=simplification, **{k: v for k, v in options.items() if k != "progress"}),
        "by": operator_contact(), "date": strftime("%Y-%m-%d %H:%M %Z")})
      vol.commit_provenance()

  return MeshTaskIterator(vol.mip_bounds(mip), shape)


def create_spatial_index_mesh_tasks(cloudpath, shape=(448, 448, 448), mip=0, fill_missing=False, compress="gzip",
                                    mesh_dir=None):
  """Rebuild the spatial index of a mesh directory (default: the layer's, else mesh_mip_{mip}_err_40),
  or build one over a different grid than the mesh tasks used."""
  return spatial_index_tasks(cloudpath, shape, mip, fill_missing, compress, mesh_dir, "mesh")


def create_mesh_manifest_tasks(layer_path, magnitude=3, mesh_dir=None):
  """Tasks that write each label's legacy manifest {mesh_dir}/{segid}:0 from its fragments.  A file://
  layer gets one MeshManifestFilesystemTask; any other protocol 10^m - 1 MeshManifestPrefixTasks over the
  prefixes "1:" ... "{10^(m-1) - 1}:", then 10^(m-1) ... 10^m - 1, each of which also takes the longer labels
  that start with it (DESIGN.md §5m)."""
  assert int(magnitude) == magnitude
  assert magnitude > 0
  if "://" not in layer_path or layer_path.startswith("file://"):
    return [partial(MeshManifestFilesystemTask, layer_path=layer_path, mesh_dir=mesh_dir)]
  start, end = int(10 ** (magnitude - 1)), int(10 ** magnitude)

  class MeshManifestTaskIterator:
    def __len__(self):
      return end - 1

    def __iter__(self):
      for prefix in [str(p) + ":" for p in range(1, start)] + [str(p) for p in range(start, end)]:
        yield partial(MeshManifestPrefixTask, layer_path=layer_path, prefix=prefix, mesh_dir=mesh_dir)

  return MeshManifestTaskIterator()


def create_mesh_deletion_tasks(layer_path, magnitude=3, mesh_dir=None):
  """Tasks that delete the mesh directory's files.  The directory's info is deleted here, while the tasks
  are made, and the provenance is appended.  A sharded directory gets one task over every file; otherwise
  10^m tasks: "0", "1:" ... "{10^(m-1) - 1}:", then 10^(m-1) ... 10^m - 1 (DESIGN.md §5m lists the spatial
  index files these leave).  magnitude=0 raises ValueError before anything is deleted."""
  assert int(magnitude) == magnitude
  assert magnitude >= 0
  prefixes = deletion_prefixes("create_mesh_deletion_tasks", magnitude)
  cv = CloudVolume(layer_path, mesh_dir=mesh_dir)
  CloudFiles(cv.mesh.meta.layerpath).delete("info")
  if cv.mesh.meta.is_sharded():
    prefixes = [""]
  cv.provenance.processing.append({
    "method": {"task": "DeleteMeshFilesTask", "layer_path": layer_path, "mesh_dir": mesh_dir},
    "by": operator_contact(),
    "date": strftime("%Y-%m-%d %H:%M %Z"),
  })
  cv.commit_provenance()
  return [partial(DeleteMeshFilesTask, cloudpath=layer_path, prefix=p, mesh_dir=mesh_dir) for p in prefixes]


def create_xfer_meshes_tasks(src, dest, mesh_dir=None, magnitude=2):
  """Tasks that copy src's mesh files, byte for byte, to dest's mesh directory (mesh_dir, else dest's
  info['mesh']), after writing src's mesh info there.  The prefixes are every string of `magnitude` digits
  (hex digits for a sharded source), then every shorter one followed by ":0" (unsharded) or "." (sharded);
  DESIGN.md §5m lists the files they miss.  A dest without an info file, or with neither mesh_dir nor a
  `mesh` in its info, raises ValueError before anything is written."""
  cv_src = CloudVolume(src)
  cf_dest = CloudFiles(dest)
  mesh_dir = xfer_destination_dir("create_xfer_meshes_tasks", cf_dest, mesh_dir, "mesh")
  cf_dest.put_json("%s/info" % mesh_dir, cv_src.mesh.meta.info)
  sharded = cv_src.mesh.meta.is_sharded()
  prefixes = xfer_prefixes(magnitude, sharded, "." if sharded else ":0")
  return [partial(TransferMeshFilesTask, src=src, dest=dest, prefix=p, mesh_dir=mesh_dir) for p in prefixes]
