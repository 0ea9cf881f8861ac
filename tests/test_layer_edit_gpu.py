"""BlackoutTask, non-aligned writes and TouchTask on file:// layers.  After a blackout the whole layer must
equal a numpy restatement: the box holds the value and every other voxel keeps its value, in the edge chunks
that a non-aligned write read and rewrote too.  A jpeg chunk that was rewritten is expected to be the
re-encoding of its restated contents (the codec is lossy)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SIZE, CHUNK = (200, 180, 70), (64, 64, 32)
VALUES = {"uint8": 200, "uint16": 60000, "uint32": 2 ** 32 - 5, "uint64": 2 ** 64 - 3, "float32": -1.5}


def _data(dtype, seed=0):
  rng = np.random.default_rng(seed)
  shape = SIZE + (1,)
  if dtype == "float32":
    return rng.standard_normal(shape).astype(np.float32)
  if dtype == "uint64":  # labels near the top of the range: they do not survive a trip through float64
    return (np.uint64(2 ** 64 - 2 ** 12) + rng.integers(0, 50, shape).astype(np.uint64)).astype(np.uint64)
  return rng.integers(0, np.iinfo(dtype).max, shape, dtype=dtype, endpoint=True)


def _layer(tmp_path, data, encoding):
  from igneous_b200._compat import CloudVolume
  path = "file://" + str(tmp_path / "vol")
  layer = "segmentation" if encoding == "compressed_segmentation" else "image"
  vol = CloudVolume(path, info=CloudVolume.create_new_info(1, layer, data.dtype, encoding, (4, 4, 40), (0, 0, 0),
                                                           SIZE, CHUNK))
  vol.commit_info()
  vol[vol.bounds] = data
  return path


def _read(path):
  from igneous_b200._compat import CloudVolume
  vol = CloudVolume(path)
  return vol[vol.bounds]


def _restate(before, box, value, region, encoding):
  """`before` with `box` set to value; with jpeg, every chunk in `region` (the chunk-aligned region written)
  replaced by the decoding of its encoding"""
  from igneous_b200 import codecs
  want = before.copy()
  want[box[0][0]:box[1][0], box[0][1]:box[1][1], box[0][2]:box[1][2]] = value
  if encoding != "jpeg":
    return want
  for z in range(0, SIZE[2], CHUNK[2]):
    for y in range(0, SIZE[1], CHUNK[1]):
      for x in range(0, SIZE[0], CHUNK[0]):
        lo = (x, y, z)
        if not all(region[0][i] <= lo[i] < region[1][i] for i in range(3)):
          continue
        sl = tuple(slice(a, min(a + c, s)) for a, c, s in zip(lo, CHUNK, SIZE))
        chunk = np.asfortranarray(want[sl][..., 0])
        want[sl] = codecs.jpeg_decode(codecs.jpeg_encode(chunk, 85), chunk.shape).reshape(chunk.shape + (1,),
                                                                                          order="F")
  return want


CASES = [("raw", d) for d in VALUES] + [("jpeg", "uint8"), ("compressed_segmentation", "uint32"),
                                        ("compressed_segmentation", "uint64")]
BOXES = {  # bounds given to the creator, and its task shape
  "aligned_far_edge": (((64, 0, 32), (200, 128, 70)), (128, 128, 32)),
  # several tasks, which rewrite shared edge chunks in turn
  "non_aligned": (((10, 20, 5), (150, 170, 50)), (100, 100, 30)),
  "non_aligned_far_edge": (((130, 100, 40), (200, 180, 70)), (100, 100, 30)),
}


def _painted(bounds, shape):
  """what the tasks paint: as in the reference, each task's offset + shape clamped to the volume (not to
  the creator's bounds), so the last task of an axis reaches the next multiple of the task shape"""
  lo = np.array(bounds[0])
  hi = lo + -(-(np.array(bounds[1]) - lo) // np.array(shape)) * np.array(shape)
  return tuple(lo), tuple(np.minimum(hi, SIZE))


@pytest.mark.parametrize("encoding,dtype", CASES)
@pytest.mark.parametrize("which", list(BOXES))
def test_blackout_restated(ctx, tmp_path, encoding, dtype, which):
  import igneous_b200.task_creation as tc
  from igneous_b200._compat import Bbox, LocalTaskQueue
  data = _data(dtype)
  path = _layer(tmp_path, data, encoding)
  before = _read(path)
  bounds, shape = BOXES[which]
  aligned = which == "aligned_far_edge"
  if encoding == "jpeg":  # one task: the restatement re-encodes each rewritten chunk once
    shape = (256, 256, 128)
  value = VALUES[dtype]
  tasks = tc.create_blackout_tasks(path, Bbox(*bounds), shape=shape, value=value, non_aligned_writes=not aligned)
  LocalTaskQueue(parallel=1).insert_all(tasks)
  got = _read(path)
  box = _painted(bounds, shape)
  region = (tuple(v // c * c for v, c in zip(box[0], CHUNK)),
            tuple(min(-(-v // c) * c, s) for v, c, s in zip(box[1], CHUNK, SIZE)))
  want = _restate(before, box, np.dtype(dtype).type(value), region, encoding)
  assert got.dtype == want.dtype and np.array_equal(got, want)


@pytest.mark.parametrize("encoding,dtype", [("raw", "uint16"), ("compressed_segmentation", "uint64")])
def test_non_aligned_write(ctx, tmp_path, encoding, dtype):
  """CloudVolume(non_aligned_writes=True): the region around the box is read (a missing chunk as 0), the
  cutout placed into it and the region written; without the flag the write raises as before"""
  from igneous_b200._compat import CloudVolume
  data = _data(dtype, 1)
  path = _layer(tmp_path, data, encoding)
  vol = CloudVolume(path)
  vol.cf.delete(vol._chunk_name(0, next(iter(vol._chunks(0, vol.bounds)))))  # the chunk at the origin
  before = CloudVolume(path, fill_missing=True)[vol.bounds]
  assert not before[:64, :64, :32].any()
  lo, hi = (30, 40, 10), (170, 100, 60)
  new = _data(dtype, 2)[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]]
  with pytest.raises(ValueError, match="chunk aligned"):
    vol[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]] = new
  vol = CloudVolume(path, non_aligned_writes=True)
  vol[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]] = new
  want = before.copy()
  want[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]] = new
  assert np.array_equal(vol[vol.bounds], want)


def test_touch(ctx, tmp_path):
  import igneous_b200.task_creation as tc
  from igneous_b200._compat import CloudVolume, EmptyVolumeException, LocalTaskQueue
  path = _layer(tmp_path, _data("uint8"), "raw")
  LocalTaskQueue(parallel=1).insert_all(tc.create_touch_tasks(path, shape=(128, 128, 64)))
  vol = CloudVolume(path)
  name = vol._chunk_name(0, next(iter(vol._chunks(0, vol.bounds))))
  good = vol.cf.get(name)
  vol.cf.put(name, good[:-1], compress="gzip")  # a truncated raw chunk
  with pytest.raises(ValueError):
    LocalTaskQueue(parallel=1).insert_all(tc.create_touch_tasks(path, shape=(128, 128, 64)))
  vol.cf.delete(name)
  with pytest.raises(EmptyVolumeException):
    LocalTaskQueue(parallel=1).insert_all(tc.create_touch_tasks(path, shape=(128, 128, 64)))
