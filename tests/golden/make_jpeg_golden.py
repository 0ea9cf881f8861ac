"""Records libjpeg's grayscale JPEG streams and decodes on seeded chunks -> jpeg_libjpeg.npz.

Run with OpenCV 4.13 and Pillow 12.2 (`python tests/golden/make_jpeg_golden.py`); both wrap
libjpeg-turbo.  A chunk [x, y, z] of uint8 is the image of width sx and height sy*sz.

  enc_*      a chunk, a quality and a restart interval (blocks; 0 = none): cv2.imencode's bytes
             and cv2.imdecode's pixels of them
  foreign_*  Pillow streams the decoder must read (optimized Huffman tables, a COM segment): the
             bytes and cv2.imdecode's pixels
  refuse_*   streams the decoder must refuse (progressive, three components)
"""
import io
import os

import cv2
import numpy as np
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))


def raster(chunk):
  sx, sy, sz = chunk.shape
  return np.ascontiguousarray(chunk.reshape((sx, sy * sz), order="F").T)


def unraster(img, shape):
  return np.asfortranarray(img.T.reshape(shape, order="F"))


def smooth(rng, shape):
  """EM-like: low-frequency membranes and cell interiors plus shot noise."""
  sx, sy, sz = shape
  x = np.arange(sx)[:, None, None] / 9.0
  y = np.arange(sy)[None, :, None] / 7.0
  z = np.arange(sz)[None, None, :] / 3.0
  v = 140 + 45 * np.sin(x + 0.5 * z) * np.cos(y - 0.3 * z) - 60 * (np.abs(np.sin(0.7 * x + 0.4 * y)) < 0.12)
  return np.asfortranarray((v + rng.normal(0, 9, shape)).clip(0, 255).astype(np.uint8))


def main():
  rng = np.random.default_rng(20261015)
  noise = lambda s: np.asfortranarray(rng.integers(0, 256, s, dtype=np.uint8))
  row = lambda s: (s[0] + 7) // 8
  enc = [  # (chunk, quality, restart interval)
    (smooth(rng, (64, 64, 8)), 85, row((64, 64, 8))),
    (smooth(rng, (64, 64, 8)), 85, 0),
    (smooth(rng, (48, 40, 4)), 30, 5),
    (smooth(rng, (48, 40, 4)), 95, row((48, 40, 4))),
    (smooth(rng, (48, 40, 4)), 100, 0),
    (noise((32, 32, 8)), 85, row((32, 32, 8))),
    (noise((32, 16, 4)), 100, 3),
    (noise((32, 16, 4)), 30, 0),
    (smooth(rng, (37, 23, 5)), 85, row((37, 23, 5))),
    (smooth(rng, (37, 23, 5)), 95, 7),
    (noise((37, 23, 5)), 85, 0),
    (noise((1, 1, 1)), 85, 1),
    (smooth(rng, (9, 3, 2)), 50, 1),
    (np.zeros((24, 16, 3), np.uint8, order="F"), 85, row((24, 16, 3))),
    (np.full((24, 16, 3), 255, np.uint8, order="F"), 85, 0),
    (np.full((13, 11, 2), 255, np.uint8, order="F"), 100, 2),
  ]
  out = {}
  for i, (chunk, q, ri) in enumerate(enc):
    ok, b = cv2.imencode(".jpg", raster(chunk), [cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_RST_INTERVAL, ri])
    assert ok
    b = b.reshape(-1)
    out["enc_%d_in" % i] = chunk
    out["enc_%d_quality" % i] = np.int64(q)
    out["enc_%d_restart" % i] = np.int64(ri)
    out["enc_%d_jpeg" % i] = b
    out["enc_%d_dec" % i] = unraster(cv2.imdecode(b, cv2.IMREAD_UNCHANGED), chunk.shape)

  foreign = [(smooth(rng, (48, 32, 4)), dict(quality=85, optimize=True)),
             (noise((37, 23, 5)), dict(quality=90, optimize=True)),
             (smooth(rng, (40, 24, 2)), dict(quality=75, comment=b"igneous_b200 golden"))]
  for i, (chunk, kw) in enumerate(foreign):
    buf = io.BytesIO()
    Image.fromarray(raster(chunk)).save(buf, "JPEG", **kw)
    b = np.frombuffer(buf.getvalue(), np.uint8)
    out["foreign_%d_jpeg" % i] = b
    out["foreign_%d_shape" % i] = np.array(chunk.shape, np.int64)
    out["foreign_%d_dec" % i] = unraster(cv2.imdecode(b, cv2.IMREAD_UNCHANGED), chunk.shape)

  prog = smooth(rng, (32, 32, 2))
  buf = io.BytesIO()
  Image.fromarray(raster(prog)).save(buf, "JPEG", quality=85, progressive=True)
  out["refuse_0_jpeg"] = np.frombuffer(buf.getvalue(), np.uint8)
  out["refuse_0_shape"] = np.array(prog.shape, np.int64)
  out["refuse_0_kind"] = np.array("progressive")
  rgb = np.stack([raster(prog)] * 3, axis=-1)
  buf = io.BytesIO()
  Image.fromarray(rgb, "RGB").save(buf, "JPEG", quality=85)
  out["refuse_1_jpeg"] = np.frombuffer(buf.getvalue(), np.uint8)
  out["refuse_1_shape"] = np.array(prog.shape, np.int64)
  out["refuse_1_kind"] = np.array("rgb")
  out["versions"] = np.array("opencv %s, pillow %s" % (cv2.__version__, Image.__version__))
  np.savez_compressed(os.path.join(HERE, "jpeg_libjpeg.npz"), **out)


if __name__ == "__main__":
  main()
