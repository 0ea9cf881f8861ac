"""Where does the streamed (host-buffer) step lose time against the resident one?  Runs the 2048^3
pipeline step in several variants in one process and prints the wall time of each."""
import ctypes as c, os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
from igneous_b200 import _shim, pipeline

S = int(sys.argv[1]) if len(sys.argv) > 1 else 2048
ctx = _shim.default_context()
pipe = pipeline.VolumePipeline(ctx, (S, S, S), np.uint32, num_mips=2, ccl_out_dtype=np.uint32,
                               simplification_factor=100, resolution=(16, 16, 40), pitch=64, num_ids=1 << 20, seed=0,
                               mesh_streams=8)
pipe.synth()
for _ in range(2):
  pipe.step()
ctx.sync()
t0 = time.perf_counter(); pipe.step(); ctx.sync(); print("resident step %.0f ms" % (1e3 * (time.perf_counter() - t0)), pipe.stage_ms())
host_in = ctx.pinned_empty(pipe.shape, np.uint32)
host = {"mips": [ctx.pinned_empty(s, np.uint32) for s in pipe.mip_shapes], "cc": ctx.pinned_empty(pipe.shape, np.uint32)}
ctx.d2h(host_in, pipe.d_in); ctx.sync()
res = (c.c_float * 3)(16.0, 16.0, 40.0)
bufs = {}
def export(task, h, nv, nf, nl, wctx):
  if nv == 0: return
  if id(wctx) not in bufs:
    bufs[id(wctx)] = (wctx.pinned_empty((1 << 22, 3), np.float32, order="C"), wctx.pinned_empty((1 << 23, 3), np.uint32, order="C"))
  bv, bf = bufs[id(wctx)]
  voff = np.zeros(nl + 1, dtype=np.uint64); foff = np.zeros(nl + 1, dtype=np.uint64)
  _shim.check(wctx.lib.ign_mesh_export(h, res, 1, _shim.ptr(bv), _shim.ptr(bf), _shim.ptr(voff), _shim.ptr(foff)))
os.environ["IGN_PIPE_TRACE"] = "1"
for name, ho, ex in (("full", host, export), ("full", host, export), ("upload only", None, None), ("upload+download", host, None),
                     ("upload+export", None, export)):
  t0 = time.perf_counter(); pipe.step_streamed(host_in, ho, ex); ctx.sync()
  print("%-18s %.0f ms" % (name, 1e3 * (time.perf_counter() - t0)), flush=True)
