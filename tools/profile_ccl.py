"""One device-resident CCL call per repetition (for ncu): profile_ccl.py [size] [in dtype] [out dtype] [reps]"""
import ctypes as c, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from igneous_b200 import _shim

size = int(sys.argv[1]) if len(sys.argv) > 1 else 512
dt_in = np.dtype(sys.argv[2]) if len(sys.argv) > 2 else np.dtype(np.uint32)
dt_out = np.dtype(sys.argv[3]) if len(sys.argv) > 3 else np.dtype(np.uint32)
reps = int(sys.argv[4]) if len(sys.argv) > 4 else 2
ctx = _shim.default_context()
n = size ** 3
d_in = ctx.alloc(n * dt_in.itemsize)
d_out = ctx.alloc(n * dt_out.itemsize)
_shim.check(ctx.lib.ign_synth_seg_dev(ctx.handle, _shim.ptr(d_in), _shim.dtype_code(dt_in), size, size, size, 0, 0, 0,
                                      64, 1 << 20, 0, 0))
N = c.c_uint64(0)
for _ in range(reps):
  _shim.check(ctx.lib.ign_ccl6_dev(ctx.handle, _shim.ptr(d_in), _shim.dtype_code(dt_in), size, size, size,
                                   _shim.ptr(d_out), _shim.dtype_code(dt_out), c.byref(N)))
ctx.sync()
print("components", N.value)
