"""compute_rois against a host restatement of its rule: the top mip in z slabs, pooled by the oracle
when a slab's xy area exceeds max_axial_length^2, thresholded, labelled 26-connected by
scipy.ndimage.label, dust dropped by np.bincount sizes, boxes from find_objects, in the order of each
component's first voxel in F order, scaled, shifted by the slab's z and with 1 taken off the maxima.
The kernels are checked against the same restatement and past 2^32 voxels."""
import math

import numpy as np
import pytest
from scipy import ndimage

pytestmark = pytest.mark.gpu


def _host_boxes(mask, dust):
  """(count, box lo, box hi exclusive) per 26-connected component of at least `dust` voxels, in the order
  of each component's first voxel in F order"""
  lab, n = ndimage.label(mask, structure=np.ones((3, 3, 3), dtype=bool))
  if n == 0:
    return []
  sizes = np.bincount(lab.ravel())
  objs = ndimage.find_objects(lab)
  ids, first = np.unique(lab.ravel(order="F"), return_index=True)
  order = [int(i) for _, i in sorted(zip(first, ids)) if i != 0]
  return [(int(sizes[l]), [s.start for s in objs[l - 1]], [s.stop for s in objs[l - 1]])
          for l in order if sizes[l] >= dust]


def _host_rois(top, segmentation, ratio, z0, z_step, suppress, dust, max_axial, oracle):
  Z = top.shape[2]
  z_step = Z if z_step is None else z_step
  max_size = max_axial ** 2
  more_mips, out = 0, []
  for z in range(z0, z0 + Z, z_step):
    img = np.asfortranarray(top[:, :, z - z0:min(z + z_step, z0 + Z) - z0])
    sxy = img.shape[0] * img.shape[1]
    if sxy > max_size:
      more_mips = int(math.ceil(math.log2(sxy / max_size)))
      pool = oracle.downsample_segmentation if segmentation else oracle.downsample_with_averaging
      img = pool(img, (2, 2, 1), num_mips=more_mips)[-1]
    f = np.array(ratio, dtype=np.float64)
    f[:2] *= 2 ** more_mips
    for _, lo, hi in _host_boxes(img > suppress, dust):
      lo, hi = np.array(lo) * f, np.array(hi) * f
      lo[2] += z
      hi[2] += z
      out.append([int(v) for v in lo] + [int(v) for v in hi - 1])
  return out


def _layer(tmp_path, top, layer, offset=(8, 0, 3), chunk=(32, 32, 8), name="vol"):
  """a two-scale layer (2x2x1) whose top mip holds `top`; mip 0 has no chunks"""
  from igneous_b200._compat import CloudVolume
  path = "file://" + str(tmp_path / name)
  size0 = (top.shape[0] * 2, top.shape[1] * 2, top.shape[2])
  vol = CloudVolume(path, info=CloudVolume.create_new_info(1, layer, top.dtype, "raw", (4, 4, 40), offset, size0,
                                                           chunk))
  vol.add_resolution((8, 8, 40))
  vol.commit_info()
  vol.mip = 1
  vol[vol.bounds] = top
  return path, int(vol.bounds.minpt.z)


def _blobs(shape, dtype, seed, n=60, faint=0):
  """random boxes of random sizes (some of a voxel or two) over faint noise"""
  rng = np.random.default_rng(seed)
  img = rng.integers(0, faint + 1, shape).astype(dtype)
  for _ in range(n):
    lo = [int(rng.integers(0, s)) for s in shape]
    ext = [int(rng.integers(1, 6)) for _ in shape]
    img[tuple(slice(a, a + e) for a, e in zip(lo, ext))] = rng.integers(faint + 1, 250)
  return np.asfortranarray(img)


def _check(path, top, segmentation, z0, oracle, **kw):
  import igneous_b200.task_creation as tc
  from igneous_b200._compat import CloudVolume
  got = tc.compute_rois(path, **kw)
  want = _host_rois(top, segmentation, (2, 2, 1), z0, kw.get("z_step"), kw.get("suppress_faint_voxels", 0),
                    kw.get("dust_threshold", 10), kw.get("max_axial_length", 512), oracle)
  assert [b.to_list() for b in got] == want
  assert CloudVolume(path).info["scales"][0]["rois"] == want
  return want


def test_image_suppress_and_dust(ctx, oracle, tmp_path):
  top = _blobs((96, 80, 24), np.uint8, 0, faint=5)
  path, z0 = _layer(tmp_path, top, "image")
  want = _check(path, top, False, z0, oracle, suppress_faint_voxels=5, dust_threshold=10)
  everything = _host_rois(top, False, (2, 2, 1), z0, None, 5, 0, 512, oracle)
  assert 0 < len(want) < len(everything)  # dust removed some, not all


def test_segmentation_z_step(ctx, oracle, tmp_path):
  top = _blobs((96, 80, 24), np.uint32, 1)
  path, z0 = _layer(tmp_path, top, "segmentation")
  assert _check(path, top, True, z0, oracle, dust_threshold=3, z_step=7)


@pytest.mark.parametrize("layer,max_axial,mips", [("image", 80, 1), ("image", 48, 2), ("segmentation", 48, 2)])
def test_pooled_slabs(ctx, oracle, tmp_path, layer, max_axial, mips):
  dtype = np.uint8 if layer == "image" else np.uint64
  top = _blobs((96, 96, 16), dtype, 2, n=120, faint=3 if layer == "image" else 0)
  assert math.ceil(math.log2(96 * 96 / max_axial ** 2)) == mips
  path, z0 = _layer(tmp_path, top, layer)
  assert _check(path, top, layer == "segmentation", z0, oracle, suppress_faint_voxels=3 if layer == "image" else 0,
                dust_threshold=2, max_axial_length=max_axial)


def test_diagonal_contact_is_one_component(ctx, oracle, tmp_path):
  top = np.zeros((40, 40, 10), dtype=np.uint8)
  top[5, 5, 2] = top[6, 6, 3] = 9  # corner contact: one 26-connected component of 2 voxels
  top[20, 20, 5] = top[21, 21, 5] = 9  # edge contact
  top[30, 10, 1] = 9  # alone
  path, z0 = _layer(tmp_path, top, "image")
  want = _check(path, top, False, z0, oracle, dust_threshold=2)
  assert want == [[10, 10, z0 + 2, 13, 13, z0 + 3], [40, 40, z0 + 5, 43, 43, z0 + 5]]


def test_empty_layer(ctx, oracle, tmp_path):
  top = np.zeros((64, 64, 8), dtype=np.uint16)
  path, z0 = _layer(tmp_path, top, "segmentation")
  assert _check(path, top, True, z0, oracle) == []


def test_mask_boxes_kernel(ctx):
  """many components, 26-connected, with their voxel counts, in one call"""
  from igneous_b200 import rois
  from igneous_b200.storage import DeviceCutout
  mask = (np.random.default_rng(3).random((300, 200, 40)) < 0.08).astype(np.uint8)
  rows = rois.component_boxes_dev(DeviceCutout.from_host(mask), 1)
  want = _host_boxes(mask, 1)
  assert len(want) > 4096
  assert rows.tolist() == [[c] + lo + [v - 1 for v in hi] for c, lo, hi in want]
  rows = rois.component_boxes_dev(DeviceCutout.from_host(mask), 4)
  assert rows.tolist() == [[c] + lo + [v - 1 for v in hi] for c, lo, hi in _host_boxes(mask, 4)]


@pytest.mark.parametrize("dtype,t", [("uint64", 2 ** 53 + 1), ("uint64", 2 ** 64 + 5), ("uint8", -1),
                                     ("uint8", 2.5), ("uint16", 300), ("float32", 0.25), ("uint8", float("nan")),
                                     ("uint16", math.inf), ("uint8", -math.inf), ("float32", 0.1),
                                     ("float32", np.float64(0.1)), ("float32", np.float64(-1e39))])
def test_threshold_kernel_is_numpys(ctx, dtype, t):
  from igneous_b200 import rois
  from igneous_b200.storage import DeviceCutout
  rng = np.random.default_rng(4)
  if dtype == "uint64":
    img = np.uint64(2 ** 53) + rng.integers(0, 4, (33, 17, 5)).astype(np.uint64)
  elif dtype == "float32":
    img = rng.standard_normal((33, 17, 5)).astype(np.float32)
    # float32(0.1) is above 0.1: greater than np.float64(0.1), not than the Python scalar 0.1
    img[:2, 0, 0] = [np.float32(0.1), np.nextafter(np.float32(0.1), np.float32(0))]
  else:
    img = rng.integers(0, 400, (33, 17, 5)).astype(dtype)
  got = rois.threshold_dev(DeviceCutout.from_host(img), t).to_host()[..., 0]
  assert np.array_equal(got, (img > t).astype(np.uint8))


def test_threshold_refuses_signed_layers(ctx):
  """the kernel compares unsigned: a negative int16 voxel would count as greater than any t >= 0"""
  from igneous_b200 import rois
  from igneous_b200.storage import DeviceCutout
  img = np.array([-5, 0, 7], dtype=np.int16).reshape(3, 1, 1)
  with pytest.raises(NotImplementedError, match="signed"):
    rois.threshold_dev(DeviceCutout.from_host(img), 1)


def test_kernels_past_2_32_voxels(ctx):
  """fill and threshold index in 64 bits; the component pass refuses a slab it cannot index"""
  from igneous_b200 import rois
  from igneous_b200._compat import Bbox
  from igneous_b200.storage import DeviceCutout
  X, Y = 65536, 65537  # 2^32 + 2^16 voxels
  cut = DeviceCutout.empty((X, Y, 1, 1), np.uint8, ctx)
  ctx.memset(cut.buf, 0, cut.nbytes)
  cut.fill(Bbox((100, Y - 1, 0), (300, Y, 1)), 9)
  mask = rois.threshold_dev(cut, 5)
  tail = np.empty(2 * X, dtype=np.uint8)
  ctx.d2h(tail, mask.buf.offset(mask.nbytes - 2 * X))
  ctx.sync()
  want = np.zeros(2 * X, dtype=np.uint8)
  want[X + 100:X + 300] = 1
  assert np.array_equal(tail, want)
  del cut
  with pytest.raises(NotImplementedError, match="32-bit voxel indices"):
    rois.component_boxes_dev(mask, 0)
