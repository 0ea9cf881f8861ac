"""Per-phase device time of one MeshTask front-end at the benchmark's shape: the first 257^3 task at mip 2
of the synthetic bench volume, one mesh stream, simplification factor 100.

Phases are the kernels between the front-end's landmark kernels, in launch order (torch.profiler
with CUDA activities): renumber, count, mc_emit, tri_order, vertices, offsets, faces, simp_setup.
`begin_ms` is the host wall time of ign_mesh_begin_dev, which ends in a stream synchronise.  Bytes are
estimated from the task's counts (one read and one write per radix-sort digit pass).

usage: time_mesh_frontend.py [--root TREE] [--reps N] [--json OUT]
  --root: the source tree whose igneous_b200 is timed (default: this one), so that two builds can be
  compared in one process-per-tree sequence."""
import argparse
import ctypes as c
import json
import os
import sys
import time

ap = argparse.ArgumentParser()
ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--json", default=None)
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.root))

import numpy as np  # noqa: E402
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from igneous_b200 import _shim, pipeline  # noqa: E402

RESOLUTION, PITCH, NUM_IDS = (16, 16, 40), 64, 1 << 20  # bench.py's headline volume

# (substring of the kernel name, phase it opens); checked in order, first match wins.  k_tri_vertices
# opens the vertex phase of builds before the lattice weld, so that --root can time them too
LANDMARKS = [("k_simp_labels", None), ("k_simp_init_verts", "simp_setup"), ("k_faces", "faces"),
             ("k_fill_u32", "offsets"), ("k_tri_vertices", "vertices"), ("k_edges<true>", "vertices"),
             ("k_mc<true>", "mc_emit"), ("k_mc<false>", "count")]
PHASES = ["renumber", "count", "mc_emit", "tri_order", "vertices", "offsets", "faces", "simp_setup"]


def phase_times(events):
  """Kernel device time per phase, in launch order, from ign_mesh_begin_dev to the label launches."""
  kern = sorted((e for e in events if e.device_type == torch.autograd.DeviceType.CUDA and e.device_time > 0
                 and "memcpy" not in e.name.lower() and "memset" not in e.name.lower()),
                key=lambda e: e.time_range.start)
  out = {p: 0.0 for p in PHASES}
  phase = None
  for e in kern:
    name = e.name
    if "copy_box" in name:
      phase = "renumber"
      continue
    hit = next((p for key, p in LANDMARKS if key in name), "")
    if hit is None:  # the label launches: the front-end is over
      break
    if hit:
      phase = hit
    elif phase == "mc_emit" and "Radix" in name:
      phase = "tri_order"
    if phase:
      out[phase] += e.device_time / 1e3
  return out


def bytes_moved(n, T, U, K, new):
  """Estimated bytes per phase: one read and one write of every record per sort digit pass."""
  lb = max(1, int(K).bit_length())
  passes = lambda bits: -(-bits // 8)  # noqa: E731
  if new:
    return {"count": 2 * 4 * n, "mc_emit": 4 * n + 12 * T, "tri_order": passes(lb) * 2 * 12 * T,
            "vertices": 3 * 4 * n + 8 * U + passes(lb) * 2 * 8 * U + 8 * U + 8 * U + 4 * U,
            "faces": 12 * T + 3 * T * (4 + 8 + 8 + 4) + 12 * T,
            "simp_setup": 3 * T * 4 * 2 + 3 * T * 4 + U * 6 * 4 * 2}
  return {"count": 4 * n, "mc_emit": 4 * n + 9 * T, "tri_order": passes(33 + lb) * 2 * 9 * T,
          "vertices": 9 * T + 3 * T * 12 + passes(33 + lb) * 2 * 12 * 3 * T + 3 * T * (8 + 4) * 2
          + 3 * T * 20 + 12 * T + 8 * U,
          "faces": 3 * T * 4 * 2 + 8 * T,
          "simp_setup": 3 * T * 4 * 2 + passes(max(1, int(U).bit_length())) * 2 * 8 * 3 * T
          + 3 * T * 8 + U * 6 * 4}


def main():
  ctx = _shim.default_context()
  pipe = pipeline.VolumePipeline(ctx, (2048, 2048, 1024), np.uint32, num_mips=2, mesh_shape=(256, 256, 256),
                                 resolution=RESOLUTION, pitch=PITCH, num_ids=NUM_IDS, seed=0,
                                 simplification_factor=100, mesh_streams=1)
  pipe.synth()
  pipe.pool()
  ctx.sync()
  task = next(pipe.mesh_tasks())
  wctx, d_task = pipe._workers[0]
  lib = wctx.lib
  src = pipe.d_mips[-1]
  msx, msy, msz = pipe.mip_shapes[-1]
  x0, y0, z0, bx, by, bz = task
  res = (c.c_float * 3)(*[float(r) for r in RESOLUTION])

  def one():
    _shim.check(lib.ign_copy_box_dev(wctx.handle, _shim.ptr(src), pipe.code, msx, msy, msz, x0, y0, z0, bx, by, bz,
                                     _shim.ptr(d_task)))
    wctx.sync()
    h = c.c_void_p()
    t0 = time.perf_counter()
    _shim.check(lib.ign_mesh_begin_dev(wctx.handle, _shim.ptr(d_task), pipe.code, bx, by, bz, c.byref(h)))
    begin_ms = (time.perf_counter() - t0) * 1e3
    nv, nf, nl = c.c_uint64(0), c.c_uint64(0), c.c_uint64(0)
    _shim.check(lib.ign_mesh_totals(h, c.byref(nv), c.byref(nf)))
    _shim.check(lib.ign_mesh_num_ids(h, c.byref(nl)))
    _shim.check(lib.ign_mesh_simplify(h, res, 100, 40.0))
    wctx.sync()
    lib.ign_mesh_free(h)
    return begin_ms, int(nv.value), int(nf.value), int(nl.value)

  one()
  begin = []
  for _ in range(args.reps):
    begin.append(one()[0])
  with profile(activities=[ProfilerActivity.CUDA]) as prof:
    _, U, T, K = one()
  events = prof.events()
  phases = phase_times(events)
  lattice_weld = any("k_edges" in e.name for e in events)
  gpu = torch.cuda.get_device_name(0)
  power = None
  try:
    import subprocess
    power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True).stdout.strip()
  except OSError:
    pass
  out = {"root": os.path.abspath(args.root), "gpu": gpu, "power_limit": power, "task": list(task), "T": T, "U": U,
         "K_present": K, "lattice_weld": lattice_weld, "begin_ms": [round(b, 2) for b in begin],
         "phase_ms": {k: round(v, 3) for k, v in phases.items()},
         "frontend_kernel_ms": round(sum(phases.values()), 3)}
  out["bytes_est"] = bytes_moved(bx * by * bz, T, U, K, lattice_weld)
  print(json.dumps(out))
  if args.json:
    with open(args.json, "w") as f:
      json.dump(out, f)


if __name__ == "__main__":
  main()
