"""The numpy restatement of the contrast rules (tests/contrastref.py) against literal loops,
live OpenCV and the recorded OpenCV fixtures; the host-side clamp rule of igneous_b200.contrast
against the same loop.  No GPU needed."""
import os

import numpy as np
import pytest

import contrastref as R
from igneous_b200 import contrast

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "clahe_cv2.npz")


# ------------------------------------------------------------------ clamp rule
def _loop(levels, lo, up):
  """The per-bin loop, bin by bin, with the cdf in uint64."""
  filtered = np.array(levels, dtype=np.uint64)
  filtered[0] = 0
  cdf = np.zeros(len(filtered), dtype=np.uint64)
  for i in range(len(filtered)):
    cdf[i] = (cdf[i - 1] if i else np.uint64(0)) + filtered[i]
  total = cdf[-1]
  if total == 0:
    return 0, 0
  out = []
  for f in (lo, up):
    v = 0
    for i, c in enumerate(cdf):
      if float(c) / float(total) > f:
        break
      v = i
    out.append(v)
  return tuple(out)


CLAMP_CASES = [
  (np.zeros(256, np.uint64), 0.01, 0.99),                       # all zero
  (np.eye(1, 256, 0, dtype=np.uint64)[0] * 1000, 0.01, 0.99),     # only bin 0: ignored -> (0, 0)
  (np.eye(1, 256, 77, dtype=np.uint64)[0] * 5, 0.01, 0.99),       # a single bin
  (np.array([0, 1, 1, 1, 1] + [0] * 251, np.uint64), 0.25, 0.75),  # fractions at exact cdf ties
  (np.array([0, 1, 1, 1, 1] + [0] * 251, np.uint64), 0.5, 0.5),    # lower_clip + upper_clip = 1
  (np.array([0, 1, 1, 1, 1] + [0] * 251, np.uint64), 0.0, 1.0),
  (np.array([9, 0, 3, 0, 0, 3] + [0] * 250, np.uint64), 0.5, 1.0),
]


@pytest.mark.parametrize("case", range(len(CLAMP_CASES)))
def test_clamp_rule_matches_loop(case):
  levels, lo, up = CLAMP_CASES[case]
  want = _loop(levels, lo, up)
  assert R.clamping_values(levels, lo, up) == want
  assert contrast.find_section_clamping_values(levels, lo, up) == want


def test_clamp_rule_random_histograms():
  rng = np.random.default_rng(3)
  for t in range(60):
    bins = 256 if t % 3 else 65536
    levels = np.zeros(bins, np.uint64)
    idx = rng.integers(0, bins, size=int(rng.integers(1, 40)))
    levels[idx] = rng.integers(1, 1 << 40, size=idx.size, dtype=np.uint64)
    lo = float(rng.choice([0.0, 0.01, 0.05, 0.5]))
    up = 1 - float(rng.choice([0.0, 0.01, 0.05, 0.5 if lo < 0.5 else 0.0]))
    want = R.clamping_values(levels, lo, up)
    assert contrast.find_section_clamping_values(levels, lo, up) == want
    if bins == 256:
      assert _loop(levels, lo, up) == want


def test_stretch_and_quantize_rules():
  img = np.array([[[0, 10, 11, 200]]], np.uint8).reshape(2, 2, 1)
  # lower 10, upper 200: (v - 10) * f32(255 / 190), rint, clip
  got = R.stretch(img, [(10, 200)], 255, 0, 255, np.uint8)
  scale = np.float32(255.0 / 190.0)
  want = np.clip(np.rint((img.astype(np.float32) - np.float32(10)) * scale), 0, 255).astype(np.uint8)
  assert np.array_equal(got, want)
  assert np.array_equal(R.stretch(img, [(5, 5)], 255, 0, 255, np.uint8), img)  # lower == upper: kept
  q = R.quantize(np.array([0, 1 / 255, 0.5, 1.0, 1.5, -0.2, np.nan, np.inf, -np.inf], np.float32).reshape(9, 1, 1))
  assert q.ravel().tolist() == [0, 1, 127, 255, 255, 0, 0, 255, 0]


def test_host_errors():
  with pytest.raises(NotImplementedError):
    contrast.histogram(np.zeros(4, np.float32))
  with pytest.raises(NotImplementedError):
    contrast.histogram(np.zeros(4, np.uint32))
  with pytest.raises(NotImplementedError):
    contrast.stretch(np.zeros((2, 2, 1), np.uint64), [np.zeros(2, np.uint64)], 0.01, 0.01)
  with pytest.raises(NotImplementedError):
    contrast.clahe(np.zeros((4, 4), np.float32))
  with pytest.raises(NotImplementedError):
    contrast.clahe(np.zeros((4, 4), np.uint32))
  with pytest.raises(ValueError):
    contrast.stretch(np.zeros((2, 2, 1), np.uint8), [np.zeros(256, np.uint64)], 0.01, 0.01, maxval=300)
  with pytest.raises(ValueError):
    contrast.stretch(np.zeros((2, 2, 1), np.uint16), [np.zeros(65536, np.uint64)], 0.01, 0.01, minval=-1,
                     out_dtype=np.uint16)
  with pytest.raises(ValueError):  # the default maxval (65535) does not fit uint8
    contrast.stretch(np.zeros((2, 2, 1), np.uint16), [np.zeros(65536, np.uint64)], 0.01, 0.01, out_dtype=np.uint8)


# ------------------------------------------------------------------------ CLAHE
def test_reflect101():
  assert [R.reflect101(p, 5) for p in range(5, 12)] == [3, 2, 1, 0, 1, 2, 3]
  assert [R.reflect101(p, 2) for p in range(2, 6)] == [0, 1, 0, 1]
  assert R.reflect101(7, 1) == 0


def test_clahe_geometry_pads_both_axes():
  # rows divide by 8, columns do not: the rows are padded by a whole tile count as well
  assert R.clahe_geometry(64, 61, (8, 8)) == (9, 8, True)
  assert R.clahe_geometry(64, 64, (8, 8)) == (8, 8, False)
  assert R.clahe_geometry(3, 2, (8, 8)) == (1, 1, True)


def _random_slice(rng, dt, rows, cols):
  if dt == np.uint8:
    img = rng.normal(120, 40, size=(rows, cols)).clip(0, 255).astype(dt)
  else:
    img = rng.normal(rng.integers(500, 60000), 2000, size=(rows, cols)).clip(0, 65535).astype(dt)
  if rng.random() < 0.3:
    img[: rows // 3] = 0
  return img


def test_clahe_matches_cv2():
  cv2 = pytest.importorskip("cv2")
  rng = np.random.default_rng(11)
  seen = set()
  for t in range(240):
    dt = np.uint8 if t % 2 == 0 else np.uint16
    gx, gy = int(rng.integers(1, 9)), int(rng.integers(1, 9))
    if t % 10 == 0:    # smaller than the grid
      rows, cols = int(rng.integers(1, gy + 1)), int(rng.integers(1, gx + 1))
    elif t % 10 == 1:  # divides by the grid
      rows, cols = gy * int(rng.integers(1, 40)), gx * int(rng.integers(1, 40))
    else:
      rows, cols = int(rng.integers(1, 260)), int(rng.integers(1, 260))
    clip = [0.0, 1.0, 2.5, 40.0][t % 4]
    img = _random_slice(rng, dt, rows, cols)
    want = cv2.createCLAHE(clipLimit=clip, tileGridSize=(gx, gy)).apply(img)
    got = R.clahe(img, clip, (gx, gy))
    assert np.array_equal(got, want), (dt, rows, cols, gx, gy, clip)
    seen.add((dt, rows % gy == 0 and cols % gx == 0, rows < gy or cols < gx, gx != gy, clip))
  assert len({s[1] for s in seen}) == 2 and any(s[2] for s in seen) and any(s[3] for s in seen)


def test_clahe_fixtures():
  g = np.load(GOLDEN)
  n = sum(1 for k in g.files if k.startswith("in_"))
  assert n >= 8
  for i in range(n):
    got = R.clahe(g["in_%d" % i], float(g["clip_%d" % i]), tuple(int(v) for v in g["grid_%d" % i]))
    assert np.array_equal(got, g["out_%d" % i]), i


def test_stretch_uint32_bounds_checked_in_float32():
  lv = [np.zeros(256, np.uint64)]
  img = np.zeros((2, 2, 1), np.uint8)
  with pytest.raises(ValueError):  # 4294967295 rounds to 2^32 in float32
    contrast.stretch(img, lv, 0.01, 0.01, maxval=4294967295, out_dtype=np.uint32)
  with pytest.raises(ValueError):
    contrast.stretch(img, lv, 0.01, 0.01, maxval=4294967200, out_dtype=np.uint32)
