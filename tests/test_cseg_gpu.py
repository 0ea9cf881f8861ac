"""GPU parity: compressed_segmentation chunk codec on the device vs the CPU oracle
(byte-identical streams, exact round trips)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _vols(oracle, dtype):
  rng = np.random.default_rng(5)
  hi = 1 << 40 if np.dtype(dtype).itemsize == 8 else 1 << 30
  return [
    oracle.synth_seg((64, 64, 64), pitch=16, num_ids=1 << 20).astype(dtype),                # realistic labels
    np.zeros((16, 8, 8), dtype=dtype),                                                     # one value: 0 bits, one shared table
    np.full((9, 17, 5), 7, dtype=dtype),                                                   # ragged blocks
    rng.integers(0, 3, size=(33, 20, 11)).astype(dtype),                                   # 2 bits, many identical tables
    rng.integers(0, hi, size=(24, 16, 8), dtype=np.uint64).astype(dtype),                  # every voxel distinct: 16 bits
    (rng.integers(0, 300, size=(40, 40, 24)) * 1000003).astype(dtype),                     # 8 / 16 bit blocks
  ]


@pytest.mark.parametrize("dtype", [np.uint32, np.uint64])
def test_cseg_encode_is_byte_identical_to_oracle(ctx, oracle, dtype):
  from igneous_b200 import codecs
  for v in _vols(oracle, dtype):
    v = np.asfortranarray(v)
    got = np.frombuffer(codecs.cseg_encode(v), dtype=np.uint32)
    want = oracle.cseg_encode(v)
    assert len(got) == len(want), v.shape
    assert np.array_equal(got, want), v.shape
    back = codecs.cseg_decode(got.tobytes(), v.shape, dtype)
    assert np.array_equal(back[..., 0], v)
    assert np.array_equal(oracle.cseg_decode(got, v.shape, dtype)[..., 0], v)


def test_cseg_multichannel_and_block_sizes(ctx, oracle):
  from igneous_b200 import codecs
  rng = np.random.default_rng(6)
  v = np.asfortranarray(rng.integers(0, 5, size=(20, 12, 9, 2)).astype(np.uint32))
  for bs in ((8, 8, 8), (4, 4, 4), (8, 4, 2)):
    got = np.frombuffer(codecs.cseg_encode(v, bs), dtype=np.uint32)
    assert np.array_equal(got, oracle.cseg_encode(v, bs)), bs
    assert np.array_equal(codecs.cseg_decode(got.tobytes(), v.shape, np.uint32, bs), v)


def test_cseg_encode_capacity(ctx, oracle):
  """an output one word short fails and reports the words needed; the exact size takes the stream"""
  import ctypes as c
  from igneous_b200 import _shim
  v = np.asfortranarray(_vols(oracle, np.uint32)[0])
  want = oracle.cseg_encode(v)
  args = [ctx.handle, _shim.ptr(v), _shim.IGN_U32, *v.shape, 1, 8, 8, 8]
  out, n = np.zeros(len(want), np.uint32), c.c_uint64(0)
  with pytest.raises(_shim.IgneousB200Error, match="words needed"):
    _shim.check(ctx.lib.ign_cseg_encode(*args, _shim.ptr(out), len(want) - 1, c.byref(n)))
  assert n.value == len(want)
  _shim.check(ctx.lib.ign_cseg_encode(*args, _shim.ptr(out), len(want), c.byref(n)))
  assert n.value == len(want) and np.array_equal(out, want)


def test_cseg_rejects_malformed_and_unsupported(ctx):
  from igneous_b200 import codecs, _shim
  with pytest.raises(NotImplementedError):
    codecs.cseg_encode(np.zeros((8, 8, 8), dtype=np.uint8))
  with pytest.raises(_shim.IgneousB200Error):
    codecs.cseg_decode(np.array([1, 0xFF000000, 2], dtype=np.uint32).tobytes(), (8, 8, 8), np.uint32)
