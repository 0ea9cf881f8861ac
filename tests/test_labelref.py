"""CPU: the plain references of tests/labelref.py.  The Neuroglancer-spec decoder reads the
oracle's compressed_segmentation streams back to their input, including tables that the encoder
must not share between blocks with equal-looking but different label sets; the scipy labelling,
dust and the COUNTLESS rule agree with the oracle, which shares no code with them."""
import numpy as np
import pytest

from labelref import cseg_decode_spec


def _collision_pair(dtype):
  """block 0 holds {0, 1}, block 1 holds {1, 64}: tables a weak hash maps together"""
  v = np.zeros((16, 8, 8), dtype=dtype, order="F")
  v[0:8, :, :4] = 1
  v[8:16] = 1
  v[8:16, :, 4:] = 64
  return v


@pytest.mark.parametrize("dtype", [np.uint32, np.uint64])
def test_spec_decoder_reads_oracle_streams(oracle, dtype):
  rng = np.random.default_rng(12)
  vols = [_collision_pair(dtype),
          oracle.synth_seg((40, 33, 19), pitch=8, num_ids=1 << 20).astype(dtype),
          rng.integers(0, 3, size=(17, 9, 12)).astype(dtype),
          rng.integers(0, 1 << 31, size=(16, 8, 8)).astype(dtype),         # 16-bit blocks
          np.full((3, 5, 2), 7, dtype=dtype)]
  if dtype == np.uint64:
    vols.append((rng.integers(1, 6, size=(24, 16, 8)).astype(np.uint64) << np.uint64(32)))  # low words all 0
    vols.append(np.full((8, 8, 8), (1 << 64) - 1, dtype=np.uint64))
  for v in vols:
    v = np.asfortranarray(v)
    for bs in ((8, 8, 8), (4, 4, 4), (8, 4, 2)):
      words = oracle.cseg_encode(v, bs)
      assert np.array_equal(cseg_decode_spec(words, v.shape, dtype, bs)[..., 0], v), (v.shape, bs)


def test_spec_decoder_multichannel(oracle):
  rng = np.random.default_rng(13)
  v = np.asfortranarray(rng.integers(0, 5, size=(20, 12, 9, 2)).astype(np.uint32))
  words = oracle.cseg_encode(v, (4, 4, 4))
  assert np.array_equal(cseg_decode_spec(words, v.shape, np.uint32, (4, 4, 4)), v)


def test_spec_decoder_rejects_bad_bit_width():
  words = np.array([1, 3 << 24, 3, 0], dtype=np.uint32)
  with pytest.raises(AssertionError):
    cseg_decode_spec(words, (8, 8, 8), np.uint32)


@pytest.mark.parametrize("dtype", [np.uint8, np.uint64])
def test_scipy_ccl_and_dust_agree_with_oracle(oracle, dtype):
  """The scipy labelling and the oracle are written independently; they must agree."""
  from labelref import blob_volume, ccl6, dust, label_sets
  rng = np.random.default_rng(14)
  for name, vals in label_sets(dtype).items():
    v = blob_volume(rng, (33, 29, 17), vals, dtype)
    got, n = ccl6(v)
    want, wn = oracle.connected_components(v, return_N=True)
    assert n == wn and np.array_equal(got, want.astype(np.uint64)), name
    for t in (2, 30):
      assert np.array_equal(dust(v, t), oracle.dust(v, t)), (name, t)


def test_countless_rule_agrees_with_oracle(oracle):
  from labelref import countless2x2
  rng = np.random.default_rng(15)
  img = np.asfortranarray(rng.integers(0, 4, size=(48, 40, 3)).astype(np.uint32))
  want = oracle.downsample_segmentation(img, (2, 2, 1), num_mips=2)
  assert np.array_equal(countless2x2(img), want[0])
  assert np.array_equal(countless2x2(want[0]), want[1])


def test_ccl_task_transcription_on_known_cases():
  from labelref import ccl_task
  img = np.zeros((4, 3, 2), dtype=np.uint8)
  img[:, :, 0] = 5
  img[1, 1, 1] = 9
  cc, n = ccl_task(img, (4, 3, 2), threshold_gte=5)   # rails outside the volume: none applied
  assert n == 1 and (cc[:, :, 0] == 1).all() and cc[1, 1, 1] == 1 and cc[0, 0, 1] == 0
  cc, n = ccl_task(img, (4, 3, 2), threshold_gte=6)
  assert n == 1 and cc.sum() == 1 and cc[1, 1, 1] == 1
  cc, n = ccl_task(img, (3, 2, 0), threshold_gte=5, label_offset=100)
  assert cc[3, 2, 0] == 0 and cc[3, 0, 0] == 0 and cc[0, 2, 0] == 0   # the three rails through z=0
  assert cc[0, 0, 0] == 101 and cc[1, 1, 1] == 101 and n == 1
  assert ccl_task(img, (9, 9, 9), threshold_gte=6, threshold_lte=5)[1] == 0
