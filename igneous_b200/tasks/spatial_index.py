"""SpatialIndexTask (igneous/tasks/spatial_index.py:23-75) with the renumber and the per-label
bounding boxes on the GPU (igneous_b200.fastremap, igneous_b200.spatial_index)."""
import numpy as np

from .. import spatial_index
from .._compat import CloudVolume, CloudFiles, Bbox, Vec, queueable


@queueable
def SpatialIndexTask(cloudpath, shape, offset, subdir, precision, mip=0, fill_missing=False, compress="gzip"):
  """Write {subdir}/{bounds}.spatial: {label: [x0, y0, z0, x1, y1, z1]} in physical units for every
  label in the task's box, read with one voxel of overlap on the high side as MeshTask does.
  As in the reference the label boxes are shifted by the task's `offset`, not by the clamped box."""
  cv = CloudVolume(cloudpath, mip=mip, bounded=False, fill_missing=fill_missing)
  cf = CloudFiles(cloudpath)
  bounds = Bbox.clamp(Bbox(Vec(*offset), Vec(*shape) + Vec(*offset)), cv.bounds)
  data_bounds = bounds.clone()
  data_bounds.maxpt += 1  # match typical Marching Cubes overlap
  resolution = cv.resolution

  img, remap = cv.download(data_bounds, renumber=True)
  n = max(remap.values(), default=0)
  boxes = spatial_index.bounding_boxes(img[..., 0], max_label=n) if n else np.zeros((0, 6), dtype=np.int64)
  del img
  reverse_map = {v: k for k, v in remap.items()}

  present = np.flatnonzero(boxes[:, 0] >= 0)
  phys = (boxes[present] + np.tile(np.asarray(offset, dtype=np.int64), 2)) * \
      np.tile(np.asarray(resolution, dtype=np.float32), 2)
  phys = phys.astype(resolution.dtype).tolist()
  bboxes = {str(reverse_map[int(i) + 1]): b for i, b in zip(present, phys)}

  bounds = bounds.astype(resolution.dtype) * resolution
  cf.put_json(cf.join(subdir, "%s.spatial" % bounds.to_filename(precision)), bboxes, compress=compress,
              cache_control=False)
