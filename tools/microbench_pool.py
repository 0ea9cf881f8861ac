"""Device-resident pooling micro-benchmark (CUDA events on the ctx stream)."""
import json, sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from igneous_b200 import _shim

def run(ctx, mode, dtype, shape, num_mips, reps=10):
  es = np.dtype(dtype).itemsize
  sx, sy, sz = shape
  n = sx * sy * sz
  d_in = ctx.alloc(n * es)
  code = _shim.dtype_code(dtype)
  if mode:
    _shim.check(ctx.lib.ign_synth_seg_dev(ctx.handle, _shim.ptr(d_in), code, sx, sy, sz, 0, 0, 0, 64, 1 << 20, 0, 0))
  else:
    _shim.check(ctx.lib.ign_synth_image_dev(ctx.handle, _shim.ptr(d_in), sx, sy, sz, 0, 0, 0, 0))
  outs, ob = [], 0
  x, y = sx, sy
  for m in range(num_mips):
    x, y = (x + 1) // 2, (y + 1) // 2
    outs.append(ctx.alloc(x * y * sz * es)); ob += x * y * sz * es
  pp = _shim.void_pp([o.ptr for o in outs])
  fn = ctx.lib.ign_pool_mode_2x2x1_dev if mode else ctx.lib.ign_pool_avg_2x2x1_dev
  args = (ctx.handle, _shim.ptr(d_in), code, sx, sy, sz, num_mips, 0, pp)
  for _ in range(3): _shim.check(fn(*args))
  ctx.sync()
  ts = []
  for _ in range(reps):
    ctx.timer_start(0); _shim.check(fn(*args)); ctx.timer_stop(0); ts.append(ctx.timer_ms(0))
  ms = float(np.median(ts))
  gbs = (n * es + ob) / ms / 1e6
  print(json.dumps({"kernel": "mode" if mode else "avg", "dtype": np.dtype(dtype).name, "shape": shape, "mips": num_mips, "ms": round(ms, 4), "min_ms": round(min(ts), 4), "GB/s": round(gbs, 1), "Gvox/s": round(n / ms / 1e6, 2)}))
  for o in outs: o.free()
  d_in.free()

if __name__ == "__main__":
  ctx = _shim.default_context()
  run(ctx, True, np.uint32, (2048, 2048, 256), 1)
  run(ctx, True, np.uint32, (2048, 2048, 256), 2)
  run(ctx, True, np.uint32, (2048, 2048, 256), 5)
  run(ctx, True, np.uint64, (2048, 2048, 128), 2)
  run(ctx, True, np.uint8, (2048, 2048, 512), 4)
  run(ctx, False, np.uint8, (2048, 2048, 512), 5)
  run(ctx, False, np.uint8, (512, 512, 512), 5)
  run(ctx, False, np.uint16, (2048, 2048, 256), 3)
