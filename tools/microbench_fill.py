"""Device-resident hole-filling micro-benchmark (CUDA events on the ctx stream).

Times ign_dilate_multilabel_dev and ign_fill_holes_dev at MeshTask fill levels 1, 2 and 4 on
the 257^3 blocks MeshTask meshes in bench.py (mip 2 of the pitch-64 uint32 Voronoi volume),
next to marching cubes + simplification of the same block.  Prints one JSON line per
measurement, with the card's name and power limit."""
import ctypes as c
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from igneous_b200 import _shim  # noqa: E402


def card():
  q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                     stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()
  return q[0] if q else "unknown"


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


def main(reps=10, blocks=2):
  ctx = _shim.default_context()
  lib = ctx.lib
  gpu = card()
  S = 257
  big = (4 * S, 4 * S, S)
  U32 = _shim.IGN_U32
  d_big = ctx.alloc(int(np.prod(big)) * 4)
  mips = [ctx.alloc(2 * S * 2 * S * S * 4), ctx.alloc(S * S * S * 4)]
  vol = ctx.alloc(S ** 3 * 4)
  filled, holes, dil = ctx.alloc(S ** 3 * 4), ctx.alloc(S ** 3 * 4), ctx.alloc(S ** 3 * 4)
  res = (c.c_float * 3)(16.0, 16.0, 40.0)
  for b in range(blocks):
    _shim.check(lib.ign_synth_seg_dev(ctx.handle, _shim.ptr(d_big), U32, big[0], big[1], big[2], 0, 0, b * S, 64,
                                      1 << 20, 0, 0))
    _shim.check(lib.ign_pool_mode_2x2x1_dev(ctx.handle, _shim.ptr(d_big), U32, big[0], big[1], big[2], 2, 0,
                                            _shim.void_pp([m.ptr for m in mips])))
    ctx.d2d(vol, mips[1], S ** 3 * 4)
    ctx.sync()
    common = {"block": b, "shape": [S, S, S], "dtype": "uint32", "gpu": gpu, "reps": reps}

    def dilate():
      _shim.check(lib.ign_dilate_multilabel_dev(ctx.handle, _shim.ptr(vol), U32, S, S, S, _shim.ptr(dil)))
    ms, mn = timed(ctx, dilate, reps)
    print(json.dumps(dict(common, op="ign_dilate_multilabel_dev", ms=round(ms, 3), min_ms=round(mn, 3))), flush=True)
    for level in (1, 2, 4):
      src = dil if level >= 3 else vol
      pct = 100 if level <= 3 else 103 - level

      def fill():
        _shim.check(lib.ign_fill_holes_dev(ctx.handle, _shim.ptr(src), U32, S, S, S, int(level >= 2), pct,
                                           _shim.ptr(filled), _shim.ptr(holes)))
      ms, mn = timed(ctx, fill, reps)
      print(json.dumps(dict(common, op="ign_fill_holes_dev", level=level, ms=round(ms, 3), min_ms=round(mn, 3))),
            flush=True)

    def mesh():
      h = c.c_void_p()
      _shim.check(lib.ign_mesh_begin_dev(ctx.handle, _shim.ptr(vol), U32, S, S, S, c.byref(h)))
      _shim.check(lib.ign_mesh_simplify(h, res, 100, 40.0))
      _shim.check(lib.ign_mesh_free(h))
    ms, mn = timed(ctx, mesh, max(3, reps // 2))
    print(json.dumps(dict(common, op="marching cubes + simplify (100, 40)", ms=round(ms, 3), min_ms=round(mn, 3))),
          flush=True)


if __name__ == "__main__":
  main()
