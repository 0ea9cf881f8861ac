"""The serial JPEG restatement (oracle_jpeg) against libjpeg's recorded streams and decodes
(tests/golden/jpeg_libjpeg.npz), and against OpenCV live when it imports.  No GPU."""
import os

import numpy as np
import pytest

import oracle_jpeg as J

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg_libjpeg.npz")


def golden():
  return np.load(GOLDEN)


def cases(g, prefix):
  return sorted({int(k.split("_")[1]) for k in g.files if k.startswith(prefix + "_")})


def test_golden_is_small_and_complete():
  assert os.path.getsize(GOLDEN) < 512 * 1024
  g = golden()
  assert len(cases(g, "enc")) >= 16 and len(cases(g, "foreign")) == 3 and len(cases(g, "refuse")) == 2
  qualities = {int(g["enc_%d_quality" % i]) for i in cases(g, "enc")}
  assert {30, 85, 95, 100} <= qualities


def test_oracle_encodes_every_golden_byte_for_byte():
  g = golden()
  for i in cases(g, "enc"):
    got = J.encode(g["enc_%d_in" % i], int(g["enc_%d_quality" % i]), int(g["enc_%d_restart" % i]))
    assert got == g["enc_%d_jpeg" % i].tobytes(), i


def test_oracle_decodes_every_golden_pixel_for_pixel():
  g = golden()
  for i in cases(g, "enc"):
    assert np.array_equal(J.decode(g["enc_%d_jpeg" % i].tobytes(), g["enc_%d_in" % i].shape), g["enc_%d_dec" % i]), i
  for i in cases(g, "foreign"):
    got = J.decode(g["foreign_%d_jpeg" % i].tobytes(), g["foreign_%d_shape" % i])
    assert np.array_equal(got, g["foreign_%d_dec" % i]), i


def test_oracle_refuses_progressive_and_rgb():
  g = golden()
  for i in cases(g, "refuse"):
    rc, _ = J.decode_status(g["refuse_%d_jpeg" % i].tobytes(), g["refuse_%d_shape" % i])
    assert rc == J.UNSUPPORTED, str(g["refuse_%d_kind" % i])


def test_oracle_rejects_wrong_shape_and_truncation():
  g = golden()
  data = g["enc_0_jpeg"].tobytes()
  shape = g["enc_0_in"].shape
  assert J.decode_status(data, (shape[0] + 1,) + shape[1:])[0] == J.SHAPE
  for cut in (3, 100, len(data) // 2, len(data) - 2):
    assert J.decode_status(data[:cut], shape)[0] == J.MALFORMED, cut


def test_oracle_matches_opencv_live():
  cv2 = pytest.importorskip("cv2")
  rng = np.random.default_rng(31)
  for it in range(60):
    sx, sy, sz = (int(v) for v in rng.integers(1, 80, 3))
    if it % 2:
      chunk = rng.integers(0, 256, (sx, sy, sz), dtype=np.uint8)
    else:
      x = np.add.outer(np.add.outer(np.arange(sx) / 7.0, np.arange(sy) / 5.0), np.arange(sz) / 3.0)
      chunk = (128 + 90 * np.sin(x) + rng.normal(0, 6, x.shape)).clip(0, 255).astype(np.uint8)
    chunk = np.asfortranarray(chunk)
    q = int(rng.choice([1, 10, 30, 50, 75, 85, 95, 100]))
    ri = int(rng.choice([0, 1, 5, (sx + 7) // 8]))
    img = np.ascontiguousarray(chunk.reshape((sx, sy * sz), order="F").T)
    ok, want = cv2.imencode(".jpg", img, [cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_RST_INTERVAL, ri])
    assert ok
    got = J.encode(chunk, q, ri)
    assert got == want.tobytes(), (sx, sy, sz, q, ri)
    dec = cv2.imdecode(want.reshape(-1), cv2.IMREAD_UNCHANGED)
    assert np.array_equal(J.decode(got, (sx, sy, sz)), np.asfortranarray(dec.T.reshape((sx, sy, sz), order="F")))
