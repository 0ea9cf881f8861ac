"""Plain numpy / scipy statement of the distance-transform rule (DESIGN.md §5d), written from the
rule's text and sharing no code with the library.

Per label, scipy.ndimage.distance_transform_edt of the label's mask with return_indices=True gives
each voxel's nearest voxel outside the mask; the squared distance is then computed exactly in
float64 from those indices (never by squaring a sqrt) and rounded once to float32.  The mask is
cropped to the label's bounding box grown by one voxel, which is exact: a voxel q outside the
grown box is never nearer than q moved onto the box's outer layer, which is outside the mask.
With black_border the crop is padded with one layer of zeros (the shell; a pad beside a layer
that is already outside the mask is never nearer).  A label whose crop holds no zero is +inf."""
import numpy as np
from scipy import ndimage


def _aniso(anisotropy, ndim):
  return (1.0,) * ndim if anisotropy is None else tuple(float(a) for a in anisotropy)


def edtsq(labels, anisotropy=None, black_border=False):
  """float32 squared distances of the rule, any ndim"""
  L = np.asarray(labels)
  a = _aniso(anisotropy, L.ndim)
  out = np.zeros(L.shape, dtype=np.float64)
  uniq, inv = np.unique(L, return_inverse=True)
  dense = inv.reshape(L.shape) + 1
  for i, sl in enumerate(ndimage.find_objects(dense), start=1):
    if sl is None or uniq[i - 1] == 0:
      continue
    box = tuple(slice(max(0, s.start - 1), min(n, s.stop + 1)) for s, n in zip(sl, L.shape))
    mask = dense[box] == i
    pad = 1 if black_border else 0
    sub = np.pad(mask, pad) if pad else mask
    if sub.all():
      out[box][mask] = np.inf
      continue
    _, idx = ndimage.distance_transform_edt(sub, sampling=a, return_indices=True)
    grid = np.indices(sub.shape)
    d2 = np.zeros(sub.shape, dtype=np.float64)
    for ax in range(L.ndim):
      d2 += (a[ax] * (grid[ax] - idx[ax]).astype(np.float64)) ** 2
    if pad:
      d2 = d2[tuple(slice(1, -1) for _ in range(L.ndim))]
    view = out[box]
    view[mask] = d2[mask]
  return out.astype(np.float32)


def edt(labels, anisotropy=None, black_border=False):
  return np.sqrt(edtsq(labels, anisotropy, black_border))


def brute_edtsq(labels, anisotropy=None, black_border=False):
  """The rule by its definition, O(N^2) over every voxel pair (tiny volumes only)"""
  L = np.asarray(labels)
  a = np.array(_aniso(anisotropy, L.ndim))
  pts = np.indices(L.shape).reshape(L.ndim, -1).T.astype(np.float64)
  vals = L.reshape(-1)
  if black_border:  # the shell: every position one step outside the array
    full = np.indices(tuple(n + 2 for n in L.shape)).reshape(L.ndim, -1).T - 1
    outside = np.any((full < 0) | (full >= np.array(L.shape)), axis=1)
    shell = full[outside].astype(np.float64)
  else:
    shell = np.zeros((0, L.ndim))
  out = np.zeros(vals.shape, dtype=np.float64)
  for j in range(len(vals)):
    if vals[j] == 0:
      continue
    q = np.concatenate([pts[vals != vals[j]], shell])
    out[j] = np.min(np.sum((a * (q - pts[j])) ** 2, axis=1)) if len(q) else np.inf
  return out.reshape(L.shape).astype(np.float32)


def block_edtsq(coords, shape, block, anisotropy, black_border):
  """Closed form for a volume of boxes `block` voxels wide whose face-adjacent boxes always hold
  different labels and none of which is label 0: min over axes of (a_i * d_i)^2, d_i the distance
  along axis i to the nearest box face that is a boundary (a volume face only with black_border).
  coords: one integer array per axis, broadcast together."""
  best = None
  for c, n, b, a in zip(coords, shape, block, anisotropy):
    c = np.asarray(c, dtype=np.int64)
    lo = (c // b) * b                      # first voxel of the box
    hi = np.minimum(lo + b, n)             # one past its last voxel
    dl = (c - lo + 1).astype(np.float64)   # to the voxel before the box
    dh = (hi - c).astype(np.float64)       # to the voxel after it
    if not black_border:
      dl = np.where(lo == 0, np.inf, dl)
      dh = np.where(hi == n, np.inf, dh)
    d = np.minimum(dl, dh)
    v = np.where(np.isinf(d), np.inf, (a * d) ** 2)
    best = v if best is None else np.minimum(best, v)
  return best.astype(np.float32)
