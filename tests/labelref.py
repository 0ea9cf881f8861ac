"""Plain CPU references for the label kernels, written from the published definitions and
sharing no code with oracle/: a compressed_segmentation decoder from the Neuroglancer spec,
6-connected components by scipy.ndimage.label, dust from the same labelling, brute-force
mode pooling, and the label value sets the kernels must treat as ordinary labels."""
import numpy as np
from scipy import ndimage

U64_MAX = (1 << 64) - 1


def cseg_decode_spec(words, shape, dtype, block_size=(8, 8, 8)):
  """Neuroglancer `compressed_segmentation` decoder.  The file starts with one u32 offset per
  channel.  A channel holds a 2 x u32 header per block (blocks in x-fastest order): word 0 =
  lookup table offset (low 24 bits) | bits per index (high 8 bits), word 1 = offset of the
  packed indices; offsets in u32 words from the channel start.  Index i of a block (position
  x + bx*(y + by*z)) sits at bit i*bits of the packed words, little endian; table entries are
  one u32, or (low, high) u32 pairs for uint64.  Returns the [x, y, z, c] chunk."""
  words = np.asarray(words, dtype=np.uint32)
  dtype = np.dtype(dtype)
  nw = 2 if dtype == np.uint64 else 1
  shape = tuple(int(s) for s in shape)
  if len(shape) == 3:
    shape = shape + (1,)
  sx, sy, sz, sc = shape
  bx, by, bz = (int(b) for b in block_size)
  gx, gy = -(-sx // bx), -(-sy // by)
  X, Y, Z = np.meshgrid(np.arange(sx), np.arange(sy), np.arange(sz), indexing="ij")
  blk = (X // bx + gx * (Y // by + gy * (Z // bz))).astype(np.int64)
  pos = ((Z % bz) * by + (Y % by)) * bx + (X % bx)
  w64 = words.astype(np.uint64)
  out = np.zeros(shape, dtype=dtype, order="F")
  for c in range(sc):
    base = int(words[c])
    h0 = w64[base + 2 * blk]
    h1 = w64[base + 2 * blk + 1]
    bits = (h0 >> np.uint64(24)).astype(np.int64)
    assert np.isin(bits, [0, 1, 2, 4, 8, 16, 32]).all(), "bad bit width"
    toff = (h0 & np.uint64(0xFFFFFF)).astype(np.int64)
    bitpos = pos * bits
    w = np.where(bits > 0, base + h1.astype(np.int64) + bitpos // 32, 0)
    mask = np.where(bits == 32, 0xFFFFFFFF, (1 << bits) - 1).astype(np.uint64)
    idx = np.where(bits > 0, (w64[w] >> (bitpos % 32).astype(np.uint64)) & mask, 0).astype(np.int64)
    t = base + toff + idx * nw
    v = w64[t]
    if nw == 2:
      v = v | (w64[t + 1] << np.uint64(32))
    out[..., c] = v.astype(dtype)
  return out


def ccl6(labels):
  """6-connected components of every non-zero label (scipy.ndimage.label per label), numbered
  1..N by each component's first voxel in Fortran order.  Returns (uint64 ids, N)."""
  labels = np.asarray(labels)
  uniq, inv = np.unique(labels, return_inverse=True)
  dense = inv.reshape(labels.shape)  # 0 is background exactly when uniq[0] == 0
  first = 1 if uniq[0] == 0 else 0
  comp = np.zeros(labels.shape, dtype=np.int64)
  nxt = 0
  for i, sl in enumerate(ndimage.find_objects(dense + 1), start=0):
    if i < first or sl is None:
      continue
    lab, n = ndimage.label(dense[sl] == i)
    sub = comp[sl]
    sub[lab > 0] = lab[lab > 0] + nxt
    nxt += n
  flat = comp.ravel(order="F")
  ids, first_at = np.unique(flat, return_index=True)
  keep = ids != 0
  ids, first_at = ids[keep], first_at[keep]
  new = np.zeros(nxt + 1, dtype=np.uint64)
  new[ids[np.argsort(first_at)]] = np.arange(1, len(ids) + 1, dtype=np.uint64)
  return new[comp], len(ids)


def dust(labels, threshold):
  """Zero the 6-connected components of fewer than `threshold` voxels."""
  cc, _ = ccl6(labels)
  counts = np.bincount(cc.ravel().astype(np.int64))
  small = counts[cc.astype(np.int64)] < threshold
  return np.where(small & (cc != 0), 0, labels).astype(labels.dtype)


def countless2x2(img):
  """One 2x2x1 mode mip of an even-sized [x, y, z] volume by the published COUNTLESS rule,
  zero being an ordinary label: with a=(0,0), b=(1,0), c=(0,1), d=(1,1), the result is a if
  a == b or a == c, else b if b == c, else d.  Compares values only, so any dtype works."""
  a, b, c, d = img[0::2, 0::2], img[1::2, 0::2], img[0::2, 1::2], img[1::2, 1::2]
  return np.where((a == b) | (a == c), a, np.where(b == c, b, d))


def check_block_mode(img, out, factor):
  """Brute force: every output voxel is a most frequent value of its input block, and is that
  value exactly when it is the only most frequent one.  Returns the number of checked voxels."""
  fx, fy, fz = factor
  ox, oy, oz = out.shape
  for z in range(oz):
    for y in range(oy):
      for x in range(ox):
        blk = img[fx * x:fx * x + fx, fy * y:fy * y + fy, fz * z:fz * z + fz].ravel()
        vals, cnt = np.unique(blk, return_counts=True)
        top = vals[cnt == cnt.max()]
        assert out[x, y, z] in top, (x, y, z, out[x, y, z], top)
        if len(top) == 1:
          assert out[x, y, z] == top[0], (x, y, z)
  return ox * oy * oz


def label_sets(dtype):
  """Non-zero label values where narrow-word or sentinel bugs show, per dtype."""
  dtype = np.dtype(dtype)
  mx = int(np.iinfo(dtype).max)
  sets = {"max": [mx, mx - 1, 1, mx - 2, 2, 3]}
  if dtype == np.uint64:
    sets["high_word"] = [k << 32 for k in (1, 2, 3, 5, 8, 13)]              # low word 0
    sets["shared_low"] = [(k << 32) | 0xDEADBEEF for k in (1, 2, 3, 5, 8, 13)]
  return sets


def blob_volume(rng, shape, values, dtype, p_bg=0.25):
  """4^3-blocky random volume of 0 and `values`, with salt-and-pepper background."""
  small = rng.integers(0, len(values) + 1, size=tuple((s + 3) // 4 for s in shape))
  big = np.repeat(np.repeat(np.repeat(small, 4, 0), 4, 1), 4, 2)[:shape[0], :shape[1], :shape[2]]
  big[rng.random(shape) < p_bg] = 0
  table = np.array([0] + [int(v) for v in values], dtype=np.uint64)
  return np.asfortranarray(table[big].astype(dtype))


def order_preserving_relabel(labels):
  """Map the non-zero labels to 1..K keeping their order (0 stays 0): (relabelled, {old: new})."""
  uniq = np.unique(labels)
  nz = uniq[uniq != 0]
  new = np.searchsorted(nz, labels) + 1
  out = np.where(labels == 0, 0, new).astype(np.uint32)
  return np.asfortranarray(out), {int(u): i + 1 for i, u in enumerate(nz)}


def ccl_task(image, shape, threshold_gte=None, threshold_lte=None, dust_threshold=0, label_offset=0):
  """numpy transcription of the CCL task body (igneous/tasks/image/ccl.py:165-175):
  threshold_image, blackout_non_face_rails, dust, 6-connected labelling, += label_offset, then
  the background re-zeroed.  Returns (uint64 labels, N)."""
  image = np.asarray(image)
  if threshold_gte is None and threshold_lte is None:
    labels = image.copy()
  elif threshold_gte is None:
    labels = image <= threshold_lte
  elif threshold_lte is None:
    labels = image >= threshold_gte
  else:
    labels = (image >= threshold_gte) & (image <= threshold_lte)
  for slc in (np.s_[shape[0], shape[1], :], np.s_[shape[0], :, shape[2]], np.s_[:, shape[1], shape[2]]):
    try:
      labels[slc] = 0
    except IndexError:
      pass
  if dust_threshold > 0:
    labels = dust(labels, dust_threshold)
  cc, n = ccl6(labels)
  cc += np.uint64(label_offset)
  cc[labels == 0] = 0
  return cc, n
