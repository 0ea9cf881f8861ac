"""Device-resident micro-benchmark of the jpeg codec (CUDA events on the ctx stream).

Batches of 64^3, 128 x 128 x 64 and 512 x 512 x 64 uint8 chunks of smooth EM-like data (about
134 M voxels per batch), quality 85.  Per batch: ign_jpeg_encode_dev and ign_jpeg_decode_dev with
a restart marker after every block row (what igneous_b200 writes), the size of the same streams
without markers, and the decode of those (one thread per stream: the fallback for foreign files);
ms, Gvox/s, bytes per voxel, and the fraction of 3.35 TB/s of the algorithmic bytes (encode: 1 B per
voxel in + the streams out; decode: the streams in + 1 B per voxel out).  Beside it, the same
chunks through OpenCV (libjpeg-turbo) on one host core when cv2 imports.  One JSON line per batch,
with the card's name, power limit and SM clocks read in the same run."""
import ctypes as c
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from igneous_b200 import _shim  # noqa: E402

PEAK = 3.35e12


def card():
  q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                     stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()
  return q[0] if q else "unknown"


def em_volume(shape, seed=0):
  rng = np.random.default_rng(seed)
  sx, sy, sz = shape
  x = (np.arange(sx, dtype=np.float32) / 11.0)[:, None, None]
  y = (np.arange(sy, dtype=np.float32) / 8.0)[None, :, None]
  z = (np.arange(sz, dtype=np.float32) / 4.0)[None, None, :]
  v = 130 + 50 * np.sin(x + 0.4 * z) * np.cos(y - 0.2 * z) - 70 * (np.abs(np.sin(0.6 * x + 0.5 * y)) < 0.1)
  v = v + rng.normal(0, 10, shape).astype(np.float32)
  return np.asfortranarray(v.clip(0, 255).astype(np.uint8))


def timed(ctx, fn, reps):
  fn()
  fn()
  ctx.sync()
  ts = []
  for _ in range(reps):
    ctx.timer_start(0)
    fn()
    ctx.timer_stop(0)
    ts.append(ctx.timer_ms(0))
  return float(np.median(ts)), float(min(ts))


def main(reps=5, host=True):
  ctx = _shim.default_context()
  lib = ctx.lib
  gpu = card()
  base = em_volume((512, 512, 64))
  for cs, n in (((64, 64, 64), 512), ((128, 128, 64), 128), ((512, 512, 64), 8)):
    gx, gy = 512 // cs[0], 512 // cs[1]
    tiles = [np.asfortranarray(base[i * cs[0]:(i + 1) * cs[0], j * cs[1]:(j + 1) * cs[1], :cs[2]])
             for j in range(gy) for i in range(gx)]
    chunks = [tiles[k % len(tiles)] for k in range(n)]
    vox = int(np.prod(cs)) * n
    packed = np.concatenate([t.reshape(-1, order="F") for t in chunks])
    shapes = np.ascontiguousarray(np.array([cs] * n, dtype=np.uint32))
    d_in, d_out, d_dec = ctx.alloc(vox), ctx.alloc(2 * vox), ctx.alloc(vox)
    ctx.h2d(d_in, packed)
    ctx.sync()
    offs = {ri: np.zeros(n + 1, np.uint64) for ri in (-1, 0)}
    need = c.c_uint64(0)

    def enc(ri):
      _shim.check(lib.ign_jpeg_encode_dev(ctx.handle, _shim.ptr(d_in), n, _shim.ptr(shapes), 85, ri, _shim.ptr(d_out),
                                          2 * vox, _shim.ptr(offs[ri]), c.byref(need)))
    rec = {"chunk": list(cs), "chunks": n, "voxels": vox, "quality": 85, "gpu": gpu, "reps": reps}
    sizes = {}
    for ri in (0, -1):  # the row-marker streams stay in d_out for the decode
      enc(ri)
      ctx.sync()
      sizes[ri] = int(need.value)
    ms, mn = timed(ctx, lambda: enc(-1), reps)
    enc_bytes = vox + sizes[-1]
    rec.update(encode_ms=round(ms, 3), encode_min_ms=round(mn, 3), encode_Gvox_s=round(vox / ms / 1e6, 2),
               encode_frac_peak=round(enc_bytes / (ms * 1e-3) / PEAK, 4),
               bytes_per_voxel=round(sizes[-1] / vox, 4), bytes_per_voxel_no_markers=round(sizes[0] / vox, 4),
               restart_marker_overhead=round(sizes[-1] / sizes[0] - 1, 4))

    def dec(ri):
      _shim.check(lib.ign_jpeg_decode_dev(ctx.handle, _shim.ptr(d_out), _shim.ptr(offs[ri]), n, _shim.ptr(shapes),
                                          _shim.ptr(d_dec)))
    ms, mn = timed(ctx, lambda: dec(-1), reps)
    dec_bytes = sizes[-1] + vox
    rec.update(decode_ms=round(ms, 3), decode_min_ms=round(mn, 3), decode_Gvox_s=round(vox / ms / 1e6, 2),
               decode_frac_peak=round(dec_bytes / (ms * 1e-3) / PEAK, 4))
    back = np.empty(vox, np.uint8)
    ctx.d2h(back, d_dec)
    ctx.sync()
    # the decode of its own streams is lossy but close: a sanity check on the measured path
    rec["decode_mean_abs_err"] = round(float(np.abs(back.astype(np.int16) - packed).mean()), 3)
    # the no-marker streams: encode them into d_out, then time the one-thread-per-stream decode
    enc(0)
    ctx.sync()
    ms0, mn0 = timed(ctx, lambda: dec(0), max(2, reps // 2))
    rec.update(decode_no_markers_ms=round(ms0, 3), decode_no_markers_Gvox_s=round(vox / ms0 / 1e6, 3))
    enc(-1)
    ctx.sync()
    if host:
      try:
        import cv2
        cv2.setNumThreads(1)
        imgs = [np.ascontiguousarray(t.reshape((cs[0], cs[1] * cs[2]), order="F").T) for t in chunks]
        t0 = time.perf_counter()
        streams = [cv2.imencode(".jpg", im, [cv2.IMWRITE_JPEG_QUALITY, 85])[1] for im in imgs]
        t1 = time.perf_counter()
        for s in streams:
          cv2.imdecode(s, cv2.IMREAD_UNCHANGED)
        t2 = time.perf_counter()
        rec.update(cv2_one_core_encode_ms=round((t1 - t0) * 1e3, 1), cv2_one_core_decode_ms=round((t2 - t1) * 1e3, 1))
      except ImportError:
        rec["cv2"] = "not installed"
    print(json.dumps(rec), flush=True)
    d_in.free(), d_out.free(), d_dec.free()


if __name__ == "__main__":
  main(host="--no-host" not in sys.argv)
