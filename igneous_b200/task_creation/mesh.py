"""create_meshing_tasks (igneous/task_creation/mesh.py:158-267) and
create_spatial_index_mesh_tasks (:363-435)."""
from time import strftime

from .._compat import CloudVolume, CloudFiles, Vec
from ..tasks import MeshTask
from .common import FinelyDividedTaskIterator, operator_contact, spatial_index_tasks


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
