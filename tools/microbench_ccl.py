"""Device-resident CCL micro-benchmark (CUDA events on the ctx stream)."""
import ctypes, json, sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from igneous_b200 import _shim

def run(ctx, dtype, shape, pitch, num_ids, out_dtype=np.uint64, reps=5):
  es = np.dtype(dtype).itemsize; osz = np.dtype(out_dtype).itemsize
  sx, sy, sz = shape; n = sx * sy * sz
  d_in = ctx.alloc(n * es); d_out = ctx.alloc(n * osz)
  code = _shim.dtype_code(dtype)
  c = ctypes
  _shim.check(ctx.lib.ign_synth_seg_dev(ctx.handle, _shim.ptr(d_in), code, sx, sy, sz, 0, 0, 0, pitch, num_ids, 0, 0))
  N = c.c_uint64(0)
  args = (ctx.handle, _shim.ptr(d_in), code, sx, sy, sz, _shim.ptr(d_out), _shim.dtype_code(out_dtype), c.byref(N))
  for _ in range(2): _shim.check(ctx.lib.ign_ccl6_dev(*args))
  ctx.sync(); ts = []
  for _ in range(reps):
    ctx.timer_start(0); _shim.check(ctx.lib.ign_ccl6_dev(*args)); ctx.timer_stop(0); ts.append(ctx.timer_ms(0))
  ms = float(np.median(ts))
  print(json.dumps({"kernel": "ccl6", "in": np.dtype(dtype).name, "out": np.dtype(out_dtype).name, "shape": shape, "pitch": pitch, "N": int(N.value), "ms": round(ms, 3), "min_ms": round(min(ts), 3), "alg_GB/s": round(n * (es + osz) / ms / 1e6, 1), "Gvox/s": round(n / ms / 1e6, 2)}))
  d_in.free(); d_out.free()

if __name__ == "__main__":
  ctx = _shim.default_context()
  if len(sys.argv) > 1 and sys.argv[1] == "2048":
    from igneous_b200 import pipeline
    c = ctypes
    _shim.check(ctx.lib.ign_prof_enable(ctx.handle, 1))
    run(ctx, np.uint32, (2048, 2048, 2048), 64, 1 << 20, out_dtype=np.uint32, reps=3)
    for name, cls in pipeline.PROF_CLASSES.items():
      ms, cnt = c.c_float(0), c.c_uint64(0)
      _shim.check(ctx.lib.ign_prof_read(ctx.handle, cls, c.byref(ms), c.byref(cnt)))
      if cnt.value:
        print(name, "ms total", round(ms.value, 3), "launches", cnt.value, "ms/launch", round(ms.value / cnt.value, 4))
    sys.exit(0)
  run(ctx, np.uint32, (512, 512, 512), 64, 1 << 20)
  run(ctx, np.uint32, (513, 513, 513), 64, 1 << 20)
  run(ctx, np.uint64, (1024, 1024, 1024), 64, 4096)
  run(ctx, np.uint32, (1024, 1024, 1024), 64, 1 << 20)
  run(ctx, np.uint32, (1024, 1024, 1024), 64, 1 << 20, out_dtype=np.uint32)
  run(ctx, np.uint32, (1024, 1024, 1024), 16, 1 << 20)
  run(ctx, np.uint8, (1024, 1024, 1024), 64, 200)
  # per-kernel-class times of the last configuration (CUDA events recorded by the library)
  from igneous_b200 import pipeline
  c = ctypes
  _shim.check(ctx.lib.ign_prof_enable(ctx.handle, 1))
  run(ctx, np.uint32, (1024, 1024, 1024), 64, 1 << 20, out_dtype=np.uint32, reps=3)
  for name, cls in pipeline.PROF_CLASSES.items():
    ms, cnt = c.c_float(0), c.c_uint64(0)
    _shim.check(ctx.lib.ign_prof_read(ctx.handle, cls, c.byref(ms), c.byref(cnt)))
    if cnt.value:
      print(name, "ms total", round(ms.value, 3), "launches", cnt.value, "ms/launch", round(ms.value / cnt.value, 4))
