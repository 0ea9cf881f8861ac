"""create_spatial_index_skeleton_tasks (igneous/task_creation/skeleton.py:795-867)."""
from .common import spatial_index_tasks


def create_spatial_index_skeleton_tasks(cloudpath, shape=(448, 448, 448), mip=0, fill_missing=False, compress="gzip",
                                        skel_dir=None):
  """Rebuild the spatial index of a skeleton directory (default: the layer's, else skeletons_mip_{mip}),
  or build one over a different grid than the skeleton tasks used."""
  return spatial_index_tasks(cloudpath, shape, mip, fill_missing, compress, skel_dir, "skeletons")
