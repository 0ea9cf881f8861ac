"""Records cv2.createCLAHE(...).apply outputs on seeded inputs -> clahe_cv2.npz.

Run with OpenCV 4.13 (`python tests/golden/make_contrast_golden.py`).  The cases include the
shapes CLAHETask produces at a dataset edge, scaled down from 2048 x 2048 to keep the file
small: a task box enlarged by the tile grid counts (8 voxels per side) and clamped, so that
the extents do not divide by the grid."""
import os

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))

# (rows, cols, dtype, clip_limit, grid)
CASES = [
  (64, 64, np.uint8, 40.0, (8, 8)),
  (264, 264, np.uint8, 40.0, (8, 8)),      # edge box: 256 + 8, clamped on one side
  (131, 264, np.uint8, 40.0, (8, 8)),      # dataset corner: clamped short in x
  (272, 125, np.uint8, 2.5, (8, 8)),
  (300, 211, np.uint16, 40.0, (8, 8)),
  (129, 259, np.uint16, 1.0, (8, 4)),
  (37, 5, np.uint8, 0.0, (3, 7)),
  (3, 2, np.uint16, 40.0, (8, 8)),         # smaller than the grid
]


def main():
  rng = np.random.default_rng(20261015)
  out = {}
  for i, (rows, cols, dt, clip, grid) in enumerate(CASES):
    if dt == np.uint8:
      img = rng.normal(120, 35, size=(rows, cols)).clip(0, 255).astype(dt)
    else:
      img = rng.normal(9000, 2500, size=(rows, cols)).clip(0, 65535).astype(dt)
    img[: rows // 5, : cols // 7] = 0  # a dark corner, as at the edge of an EM section
    out["in_%d" % i] = img
    out["out_%d" % i] = cv2.createCLAHE(clipLimit=clip, tileGridSize=grid).apply(img)
    out["clip_%d" % i] = np.float64(clip)
    out["grid_%d" % i] = np.array(grid, dtype=np.int64)
  out["cv2_version"] = np.array(cv2.__version__)
  np.savez_compressed(os.path.join(HERE, "clahe_cv2.npz"), **out)


if __name__ == "__main__":
  main()
