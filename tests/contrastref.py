"""Plain numpy restatement of the contrast rules of DESIGN.md §5b.

Written from the stated rules, independently of the library and of the code it
replaces, so that the GPU kernels can be checked bit for bit without a GPU-side
oracle:
  clamping_values  -- (lower, upper) of one z-slice's luminance histogram
  stretch          -- ContrastNormalizationTask's per-slice stretch, rint and clip
  quantize         -- QuantizeTask's float -> uint8 rule (saturating, NaN -> 0)
  clahe            -- OpenCV CLAHE::apply for one uint8 / uint16 2-D image
"""
import numpy as np

F32 = np.float32


def clamping_values(levels, lower_fract, upper_fract):
  """Per-bin loop: bin 0 is ignored, the cdf is uint64, fractions are compared in double
  with `>`; the result is the last bin whose cdf fraction does not exceed the fraction."""
  counts = [int(v) for v in levels]
  if counts:
    counts[0] = 0
  cdf, run = [], 0
  for v in counts:
    run += v
    cdf.append(run)
  total = cdf[-1] if cdf else 0
  if total == 0:
    return 0, 0

  def last_at_or_below(fract):
    out = 0
    for i, c in enumerate(cdf):
      if float(c) / float(total) > fract:
        break
      out = i
    return out

  return last_at_or_below(float(lower_fract)), last_at_or_below(float(upper_fract))


def stretch(image, bounds_per_z, maxval_t, minval, maxval, out_dtype):
  """image (x, y, z[, c]) uint8 / uint16; bounds_per_z [(lower, upper)] per z.  Each slice
  with lower != upper becomes (f32(v) - f32(lower)) * f32(maxval_t / (upper - lower)), each
  operation rounded to float32; then rint, clip to [minval, maxval] and cast."""
  img = np.asarray(image).astype(F32)
  for z, (lo, up) in enumerate(bounds_per_z):
    if lo == up:
      continue
    scale = F32(float(maxval_t) / (float(up) - float(lo)))
    img[:, :, z] = (img[:, :, z] - F32(lo)).astype(F32) * scale
  img = np.rint(img).astype(F32)
  img = np.clip(img, F32(minval), F32(maxval))
  return img.astype(out_dtype)


def quantize(image):
  """float32 (x, y, z[, c]) -> uint8 (x, y, z, 1) from channel 0: trunc(v * 255) with
  products outside [0, 256) saturated to 0 / 255 and NaN mapped to 0."""
  img = np.asarray(image, dtype=F32)
  if img.ndim == 4:
    img = img[..., :1]
  else:
    img = img[..., np.newaxis]
  p = (img * F32(255.0)).astype(F32)
  out = np.zeros(p.shape, np.uint8)
  ok = ~np.isnan(p)
  out[ok] = np.clip(np.trunc(p[ok]), 0, 255).astype(np.uint8)
  return out


# ------------------------------------------------------------------------ CLAHE
def reflect101(p, n):
  """Index p of an axis of length n under BORDER_REFLECT_101 (gfedcb|abcdefgh|gfedcba),
  repeated until it falls inside; a length-1 axis always gives 0."""
  if n == 1:
    return 0
  while p < 0 or p >= n:
    p = -p if p < 0 else 2 * (n - 1) - p
  return p


def clahe_geometry(rows, cols, grid):
  """(tile_rows, tile_cols, padded) for an image of rows x cols and grid = (tiles across
  columns, tiles across rows).  When either extent does not divide by its tile count, BOTH
  axes are padded at their far end by (tiles - extent % tiles) -- a whole tile count where
  that axis did divide -- and the tiles are cut from the padded image."""
  gx, gy = int(grid[0]), int(grid[1])
  if rows % gy == 0 and cols % gx == 0:
    return rows // gy, cols // gx, False
  return (rows + gy - rows % gy) // gy, (cols + gx - cols % gx) // gx, True


def clahe_luts(img, clip_limit, grid):
  """LUT of every tile, shape (tiles_y, tiles_x, hist_size), int64."""
  img = np.asarray(img)
  hs = 256 if img.dtype == np.uint8 else 65536
  rows, cols = img.shape
  gx, gy = int(grid[0]), int(grid[1])
  th, tw, padded = clahe_geometry(rows, cols, grid)
  if padded:
    ri = np.array([reflect101(r, rows) for r in range(th * gy)])
    ci = np.array([reflect101(c, cols) for c in range(tw * gx)])
    src = img[np.ix_(ri, ci)]
  else:
    src = img
  total = th * tw
  lim = 0
  if clip_limit > 0:
    lim = max(int(float(clip_limit) * total / hs), 1)
  scale = F32(hs - 1) / F32(total)  # float32 division
  luts = np.zeros((gy, gx, hs), np.int64)
  for ty in range(gy):
    for tx in range(gx):
      tile = src[ty * th:(ty + 1) * th, tx * tw:(tx + 1) * tw]
      hist = np.bincount(tile.ravel().astype(np.int64), minlength=hs).astype(np.int64)
      if lim > 0:
        excess = int(np.maximum(hist - lim, 0).sum())
        hist = np.minimum(hist, lim)
        batch = excess // hs
        residual = excess - batch * hs
        hist += batch
        if residual:
          step = max(hs // residual, 1)
          k = 0
          while k < hs and residual > 0:
            hist[k] += 1
            k += step
            residual -= 1
      v = np.cumsum(hist).astype(F32) * scale
      luts[ty, tx] = np.clip(np.rint(v), 0, hs - 1)
  return luts


def _axis_weights(n, tile, tiles):
  t = np.arange(n).astype(F32) * (F32(1.0) / F32(tile)) - F32(0.5)
  i1 = np.floor(t).astype(np.int64)
  a = (t - i1.astype(F32)).astype(F32)
  a1 = (F32(1.0) - a).astype(F32)
  return np.maximum(i1, 0), np.minimum(i1 + 1, tiles - 1), a, a1


def clahe(img, clip_limit=40.0, grid=(8, 8)):
  """cv2.createCLAHE(clip_limit, grid).apply(img) for a 2-D uint8 / uint16 image."""
  img = np.asarray(img)
  if img.dtype not in (np.uint8, np.uint16) or img.ndim != 2:
    raise NotImplementedError("clahe: 2-D uint8 / uint16 only")
  hs = 256 if img.dtype == np.uint8 else 65536
  rows, cols = img.shape
  gx, gy = int(grid[0]), int(grid[1])
  th, tw, _ = clahe_geometry(rows, cols, grid)
  luts = clahe_luts(img, clip_limit, grid).astype(F32)
  c1, c2, xa, xa1 = _axis_weights(cols, tw, gx)
  r1, r2, ya, ya1 = _axis_weights(rows, th, gy)
  v = img.astype(np.int64)
  # (L11 * xa1 + L12 * xa) * ya1 + (L21 * xa1 + L22 * xa) * ya, every product and sum in float32
  top = luts[r1[:, None], c1[None, :], v] * xa1[None, :] + luts[r1[:, None], c2[None, :], v] * xa[None, :]
  bot = luts[r2[:, None], c1[None, :], v] * xa1[None, :] + luts[r2[:, None], c2[None, :], v] * xa[None, :]
  res = top.astype(F32) * ya1[:, None] + bot.astype(F32) * ya[:, None]
  return np.clip(np.rint(res.astype(F32)), 0, hs - 1).astype(img.dtype)


def clahe_stack(stack, clip_limit=40.0, grid=(8, 8)):
  """Every z-slice of an (x, y, z) stack; axis 0 is OpenCV's rows."""
  stack = np.asarray(stack)
  out = np.empty_like(stack)
  for z in range(stack.shape[2]):
    out[:, :, z] = clahe(stack[:, :, z], clip_limit, grid)
  return out
