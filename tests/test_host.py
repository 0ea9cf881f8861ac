"""Host-side logic that needs no GPU."""
import ctypes as c

import numpy as np
import pytest

from igneous_b200 import _shim


def test_ccl6_solve_union_rule():
  """Host union-find: smaller id wins (ccl.py:70-73), final ids by ascending minimum."""
  lib = _shim.load()
  pairs = np.array([[5, 2], [7, 5], [3, 4], [9, 9]], dtype=np.uint64)
  lut = np.zeros(10, dtype=np.uint32)
  n = c.c_uint64(0)
  _shim.check(lib.ign_ccl6_solve(_shim.ptr(pairs), len(pairs), 9, _shim.ptr(lut), c.byref(n)))
  assert n.value == 6
  assert [int(v) for v in lut] == [0, 1, 2, 3, 3, 2, 4, 2, 5, 6]
  # out-of-range pair is rejected
  bad = np.array([[1, 11]], dtype=np.uint64)
  assert lib.ign_ccl6_solve(_shim.ptr(bad), 1, 9, _shim.ptr(lut), c.byref(n)) != 0


def test_num_mips_from_memory_target_reference_kats():
  """Known answers of the reference's own test (test/test_tasks.py:778-829)."""
  from igneous_b200.task_creation import num_mips_from_memory_target as f
  cs, ch = (128, 128, 64), 1
  assert f(0, "uint8", cs, ch, (2, 2, 1)) == 1
  assert f(100e6, "uint8", cs, ch, (2, 2, 1)) == 3
  assert f(100e6, "uint16", cs, ch, (2, 2, 1)) == 2
  assert f(100e6, "uint32", cs, ch, (2, 2, 1)) == 2
  assert f(100e6, "uint64", cs, ch, (2, 2, 1)) == 1
  assert f(3.5e9, "uint64", cs, ch, (2, 2, 1)) == 4
  assert f(12e9, "uint64", cs, ch, (2, 2, 1)) == 5
  assert f(800e6, "uint8", cs, ch, (2, 2, 2)) == 3
  assert f(500e6, "uint8", cs, ch, (2, 2, 2)) == 2
  assert f(100e6, "uint8", cs, ch, (2, 2, 2)) == 2
  assert f(50e6, "uint8", cs, ch, (2, 2, 2)) == 1


def test_compute_factors_survey_values():
  from igneous_b200 import downsample_scales as ds
  assert ds.compute_factors((128, 128, 64), (2, 2, 1), (64, 64, 64), (128, 128, 64)) == [(2, 2, 1)]  # C1
  assert len(ds.compute_factors((2048, 2048, 64), (2, 2, 1), (64, 64, 64), (2048, 2048, 64))) == 5    # C2
  assert ds.compute_factors((64, 64, 64), (2, 2, 1), (64, 64, 64), (64, 64, 64)) == []
  assert ds.axis_to_factor("z") == (2, 2, 1) and ds.axis_to_factor("x") == (1, 2, 2)


def test_threshold_image_truth_table():
  """test/test_ccl_tasks.py:82-109."""
  from igneous_b200.tasks import threshold_image
  sz = 20
  for dtype in (np.uint32, np.float32):
    image = np.arange(0, sz ** 3).reshape((sz, sz, sz), order="F").astype(dtype)
    assert np.all(threshold_image(image, None, None) == image)
    assert np.all(threshold_image(image, sz ** 3 + 1, None) == 1)
    assert np.all(threshold_image(image, None, 0) == 1)
    assert np.all(threshold_image(image, sz ** 3 + 1, 0) == 1)
    res = threshold_image(image, None, 1)
    assert res[0, 0, 0] == 0 and res.sum() == sz ** 3 - 1
    res = threshold_image(image, sz ** 3 + 1, 1)
    assert res[0, 0, 0] == 0 and res.sum() == sz ** 3 - 1


def test_task_iterator_grid_order():
  from igneous_b200.task_creation import FinelyDividedTaskIterator
  from igneous_b200._compat import Bbox

  class It(FinelyDividedTaskIterator):
    def task(self, shape, offset):
      return tuple(int(v) for v in offset)
  it = It(Bbox((0, 0, 0), (512, 512, 128)), (128, 128, 128))
  offs = list(it)
  assert len(it) == 16 and offs[0] == (0, 0, 0) and offs[1] == (128, 0, 0) and offs[4] == (0, 128, 0)


def test_storage_standin_roundtrip(tmp_path):
  from igneous_b200._compat import CloudVolume, CloudFiles, Bbox, USING_STANDINS
  rng = np.random.default_rng(0)
  data = rng.integers(0, 255, size=(100, 70, 33, 1), dtype=np.uint8)
  path = "file://" + str(tmp_path / "layer")
  cv = CloudVolume.from_numpy(data, vol_path=path, resolution=(4, 4, 40), voxel_offset=(10, 0, 5),
                              chunk_size=(64, 64, 32), layer_type="image", max_mip=0)
  cv2 = CloudVolume(path)
  assert np.array_equal(cv2[cv2.meta.bounds(0)], data)
  sub = Bbox((20, 5, 6), (90, 60, 30))
  got = cv2.download(sub)
  assert np.array_equal(got, data[10:80, 5:60, 1:25])
  cf = CloudFiles(path)
  cf.put_json("a/b.json", {"x": 1}, compress="br")
  assert cf.get_json("a/b.json") == {"x": 1} and "a/b.json" in cf.list("a/")
  assert cv2.key == "4_4_40"
  if USING_STANDINS:
    cf.delete([cv2._chunk_name(0, next(cv2._chunks(0, cv2.meta.bounds(0))))])
    import pytest
    from igneous_b200._compat import EmptyVolumeException
    with pytest.raises(EmptyVolumeException):
      cv2[cv2.meta.bounds(0)]
    assert CloudVolume(path, fill_missing=True)[cv2.meta.bounds(0)].shape == data.shape


def test_ccl_face_files_refuse_foreign_formats():
  """ADVICE r1: faces are never written under the reference's crackle names, and a crackle
  stream (or anything else foreign) is refused with a clear error instead of being mis-decoded."""
  from igneous_b200.tasks import ccl as C
  face = np.arange(12, dtype=np.uint64).reshape(3, 4)
  assert np.array_equal(C._decode_face(C._encode_face(face)), face)
  assert C.FACE_SUFFIX != ".ckl"
  with pytest.raises(C.ForeignFaceFormat, match="crackle"):
    C._decode_face(b"crkl\x00\x8a\x00" + b"\x00" * 32, "0-0-0-xy.ckl")
  with pytest.raises(C.ForeignFaceFormat):
    C._decode_face(b"\x1f\x8b garbage")


def test_signed_dtypes_refused_where_order_matters():
  """ADVICE r1: int8..int64 alias the unsigned kernels, which is exact only for equality-only
  operations; averaging, min / max pooling and thresholded CCL must refuse them loudly."""
  from igneous_b200 import tinybrain, cc3d
  img = np.full((4, 4, 2), -3, dtype=np.int16)
  for fn in (tinybrain.downsample_with_averaging, tinybrain.downsample_with_min_pooling,
             tinybrain.downsample_with_max_pooling):
    with pytest.raises(NotImplementedError, match="signed"):
      fn(img, (2, 2, 1), num_mips=1)
  with pytest.raises(NotImplementedError, match="signed"):
    cc3d.ccl_task(img, (3, 3, 1), threshold_gte=0)


def test_package_import_surface():
  """igneous/__init__.py:1-4: `from igneous import DownsampleTask, MeshTask, Mesher, ...`."""
  import igneous_b200 as ig
  from igneous_b200 import DownsampleTask, MeshTask, Mesher, LocalTaskQueue, CloudVolume, CCLFacesTask  # noqa: F401
  for name in ig.__all__:
    assert getattr(ig, name) is not None
