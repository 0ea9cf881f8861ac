"""The device jpeg codec (igneous_b200.codecs.jpeg_*) against libjpeg's recorded streams and decodes
(tests/golden/jpeg_libjpeg.npz) and against the serial restatement (oracle_jpeg) on seeded batches."""
import os

import numpy as np
import pytest

import oracle_jpeg as J
from igneous_b200 import _shim, codecs

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg_libjpeg.npz")


def golden():
  return np.load(GOLDEN)


def cases(g, prefix):
  return sorted({int(k.split("_")[1]) for k in g.files if k.startswith(prefix + "_")})


def smooth(rng, shape):
  sx, sy, sz = shape
  x = np.arange(sx)[:, None, None] / 9.0
  y = np.arange(sy)[None, :, None] / 7.0
  z = np.arange(sz)[None, None, :] / 3.0
  v = 140 + 45 * np.sin(x + 0.5 * z) * np.cos(y - 0.3 * z) - 60 * (np.abs(np.sin(0.7 * x + 0.4 * y)) < 0.12)
  return np.asfortranarray((v + rng.normal(0, 9, shape)).clip(0, 255).astype(np.uint8))


def test_encode_equals_libjpeg_bytes(ctx):
  g = golden()
  ids = cases(g, "enc")
  for i in ids:
    got = codecs.jpeg_encode(g["enc_%d_in" % i], int(g["enc_%d_quality" % i]), int(g["enc_%d_restart" % i]))
    assert got == g["enc_%d_jpeg" % i].tobytes(), i


def test_decode_equals_libjpeg_pixels(ctx):
  g = golden()
  datas = [g["enc_%d_jpeg" % i].tobytes() for i in cases(g, "enc")] + \
      [g["foreign_%d_jpeg" % i].tobytes() for i in cases(g, "foreign")]
  shapes = [g["enc_%d_in" % i].shape for i in cases(g, "enc")] + \
      [tuple(g["foreign_%d_shape" % i]) for i in cases(g, "foreign")]
  wants = [g["enc_%d_dec" % i] for i in cases(g, "enc")] + [g["foreign_%d_dec" % i] for i in cases(g, "foreign")]
  for d, s, w in zip(datas, shapes, wants):  # one stream per call
    assert np.array_equal(codecs.jpeg_decode(d, s), w)
  for got, w in zip(codecs.jpeg_decode_batch(datas, shapes), wants):  # all in one call
    assert np.array_equal(got, w)


def test_refuses_progressive_and_rgb(ctx):
  g = golden()
  for i in cases(g, "refuse"):
    with pytest.raises(NotImplementedError):
      codecs.jpeg_decode(g["refuse_%d_jpeg" % i].tobytes(), tuple(g["refuse_%d_shape" % i]))


def test_thousand_chunks_equal_the_oracle(ctx):
  rng = np.random.default_rng(11)
  chunks = [smooth(rng, (64, 64, 64)) for _ in range(4)]
  batch = [chunks[i % 4] if i % 7 else rng.integers(0, 256, (64, 64, 64), dtype=np.uint8) for i in range(1024)]
  got = codecs.jpeg_encode_batch(batch, quality=85)
  want = {}
  for i, ch in enumerate(batch):
    key = i % 4 if i % 7 else None
    w = want.get(key) if key is not None else None
    if w is None:
      w = J.encode(ch, 85)
      if key is not None:
        want[key] = w
    assert got[i] == w, i
  dec = codecs.jpeg_decode_batch(got, [(64, 64, 64)] * len(got))
  for i in (0, 1, 7, 500, 1023):
    assert np.array_equal(dec[i], J.decode(got[i], (64, 64, 64))), i


@pytest.mark.parametrize("quality,restart", [(85, None), (30, 0), (95, 3), (100, 1), (50, 13)])
def test_mixed_shapes_equal_the_oracle(ctx, quality, restart):
  rng = np.random.default_rng(quality + (restart or 0))
  shapes = [tuple(int(v) for v in rng.integers(1, 90, 3)) for _ in range(40)] + [(1, 1, 1), (64, 64, 64), (37, 23, 5)]
  chunks = [smooth(rng, s) if i % 2 else rng.integers(0, 256, s, dtype=np.uint8) for i, s in enumerate(shapes)]
  got = codecs.jpeg_encode_batch(chunks, quality=quality, restart_interval=restart)
  for ch, b in zip(chunks, got):
    assert b == J.encode(ch, quality, restart), ch.shape
  for ch, b, d in zip(chunks, got, codecs.jpeg_decode_batch(got, shapes)):
    assert np.array_equal(d, J.decode(b, ch.shape)), ch.shape


def test_batch_equals_single_calls(ctx):
  rng = np.random.default_rng(3)
  chunks = [smooth(rng, (40, 24, 6)), rng.integers(0, 256, (17, 9, 3), dtype=np.uint8), smooth(rng, (64, 64, 8))]
  batch = codecs.jpeg_encode_batch(chunks, quality=90)
  assert batch == [codecs.jpeg_encode(c, quality=90) for c in chunks]
  dec = codecs.jpeg_decode_batch(batch, [c.shape for c in chunks])
  for b, c, d in zip(batch, chunks, dec):
    assert np.array_equal(codecs.jpeg_decode(b, c.shape), d)


def test_with_and_without_restart_markers_decode_alike(ctx):
  rng = np.random.default_rng(5)
  ch = smooth(rng, (128, 128, 16))
  row = codecs.jpeg_encode(ch, restart_interval=None)
  none = codecs.jpeg_encode(ch, restart_interval=0)
  odd = codecs.jpeg_encode(ch, restart_interval=7)
  assert len(none) < len(odd) and b"\xff\xd0" in row and b"\xff\xdd" not in none
  a, b, c = codecs.jpeg_decode_batch([row, none, odd], [ch.shape] * 3)
  assert np.array_equal(a, b) and np.array_equal(a, c)
  assert np.array_equal(a, J.decode(none, ch.shape))
  # 4-D chunks with one channel round-trip in their own shape
  four = codecs.jpeg_decode(row, ch.shape + (1,))
  assert four.shape == ch.shape + (1,) and np.array_equal(four[..., 0], a)


def test_bad_streams_raise_and_the_context_keeps_working(ctx):
  g = golden()
  data = g["enc_0_jpeg"].tobytes()  # restart marker after every block row
  shape = g["enc_0_in"].shape
  with pytest.raises(_shim.IgneousB200Error):
    codecs.jpeg_decode(data[: len(data) // 2], shape)  # truncated
  bad = bytearray(data)
  i = bad.index(b"\xff\xd3")
  bad[i + 1] = 0xD5  # RST3 written as RST5
  with pytest.raises(_shim.IgneousB200Error):
    codecs.jpeg_decode(bytes(bad), shape)
  with pytest.raises(_shim.IgneousB200Error):
    codecs.jpeg_decode(data, (shape[0], shape[1], shape[2] + 1))  # dimensions differ from the chunk
  with pytest.raises(_shim.IgneousB200Error):
    codecs.jpeg_decode(b"\xff\xd8\xff\xd9", shape)  # no frame, no scan
  with pytest.raises(ValueError):
    codecs.jpeg_decode(data, (70000, 1, 1))
  with pytest.raises(NotImplementedError):
    codecs.jpeg_encode(np.zeros((8, 8, 8), np.uint16))
  with pytest.raises(NotImplementedError):
    codecs.jpeg_encode(np.zeros((8, 8, 8, 3), np.uint8))
  with pytest.raises(ValueError):
    codecs.jpeg_encode(np.zeros((8, 8, 8), np.uint8), quality=0)
  # one bad stream fails the whole call; the context then encodes and decodes correctly
  with pytest.raises(_shim.IgneousB200Error, match="stream 1"):
    codecs.jpeg_decode_batch([data, data[:200]], [shape, shape])
  assert codecs.jpeg_encode(g["enc_0_in"], 85) == data
  assert np.array_equal(codecs.jpeg_decode(data, shape), g["enc_0_dec"])
