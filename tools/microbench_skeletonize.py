"""Micro-benchmark of igneous_b200.kimimaro.skeletonize (host clock around calls that end in a device
synchronise).

Workloads: uint32 synthetic segmentations (the bench's jittered-grid Voronoi generator, pitch 16, with
membranes of label 0) at 449^3 (SkeletonTask's 448^3 + 1 cutout) and 512^3 with SkeletonTask's
teasar_params scale 4, const 500; and a 449^3 volume of 120 random capsule trees (neurites, tests/teasarref.py)
with scale 1.5, const 50, where objects need many paths and rounds.  Anisotropy (16, 16, 40), dust_threshold
1000, fix_borders on, both fix_branching modes.  Per workload: median and min seconds of the whole call over
the timed reps after one warm-up, the time of each phase of the last rep (kimimaro.last_phase_seconds), the
object split alone (ign_teasar_objects_dev), and the loop's rounds, paths, box voxels visited and host
synchronisations.  The CPU baseline is the serial C checker of the loop alone (one host core) on the fields
of a 256^3 cutout, against the loop phase of the GPU call on the same cutout.  Prints one JSON line per measurement with the card's name, power
limit, SM clock and throttle reasons read before and after."""
import ctypes as c
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402

from igneous_b200 import _shim, kimimaro  # noqa: E402

U32 = _shim.IGN_U32
PARAMS = {"scale": 4, "const": 500}
NEURITE_PARAMS = {"scale": 1.5, "const": 50}  # small boxes: many paths and rounds per object
ANISO = (16, 16, 40)


def card():
  q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks_throttle_reasons.active",
                      "--format=csv,noheader"], stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()
  return q[0] if q else "unknown"


def seg(ctx, shape):
  n = int(np.prod(shape))
  raw = ctx.alloc(n * 4)
  _shim.check(ctx.lib.ign_synth_seg_dev(ctx.handle, _shim.ptr(raw), U32, *shape, 0, 0, 0, 16, 1 << 20, 0, 0))
  out = np.empty(shape, np.uint32, order="F")
  ctx.d2h(out, raw)
  ctx.sync()
  raw.free()
  return out


def timed(fn, reps):
  fn()
  ts = []
  for _ in range(reps):
    t = time.perf_counter()
    fn()
    ts.append(time.perf_counter() - t)
  return float(np.median(ts)), float(min(ts))


def objects_ms(ctx, vol, reps):
  n = vol.size
  raw, lab, obj = ctx.alloc(n * 4), ctx.alloc(n * 4), ctx.alloc(n * 4)
  ctx.h2d(raw, vol)
  k, m = c.c_uint64(0), c.c_uint64(0)
  _shim.check(ctx.lib.ign_renumber_dev(ctx.handle, _shim.ptr(raw), U32, n, _shim.ptr(lab), None, 0, c.byref(k)))

  def run():
    _shim.check(ctx.lib.ign_teasar_objects_dev(ctx.handle, _shim.ptr(lab), *vol.shape, k.value, 26, 1000,
                                               _shim.ptr(obj), c.byref(m)))
    ctx.sync()
  ms = timed(run, reps)[0] * 1e3
  for b in (raw, lab, obj):
    b.free()
  return ms, int(k.value), int(m.value)


def main(reps=3):
  import teasarref as T
  ctx = _shim.default_context()
  work = [("seg449", PARAMS, lambda: seg(ctx, (449, 449, 449))),
          ("seg512", PARAMS, lambda: seg(ctx, (512, 512, 512))),
          ("neurites449", NEURITE_PARAMS, lambda: T.capsule_trees((449, 449, 449), 120, seed=1, anisotropy=ANISO))]
  for name, params, make in work:
    vol = make()
    obj_ms, labels, objects = objects_ms(ctx, vol, reps)
    for fb in (True, False):
      before = card()
      med, mn = timed(lambda: kimimaro.skeletonize(vol, params, anisotropy=ANISO, fix_branching=fb, ctx=ctx), reps)
      phases = {k: round(v * 1e3, 1) for k, v in kimimaro.last_phase_seconds.items()}
      st = (c.c_uint64 * 4)()
      ctx.lib.ign_teasar_last_stats(st)
      print(json.dumps({"op": "skeletonize", "workload": name, "shape": list(vol.shape), "labels": labels,
                        "objects": objects, "params": params, "fix_branching": fb, "gpu_before": before,
                        "gpu_after": card(), "reps": reps, "s": round(med, 3), "min_s": round(mn, 3),
                        "phase_ms_last_rep": phases, "objects_alone_ms": round(obj_ms, 1), "rounds": int(st[0]),
                        "paths": int(st[1]), "box_voxels": int(st[2]), "host_syncs": int(st[3]),
                        "loop_ms_per_round": round(phases.get("loop", 0) / max(int(st[0]), 1), 3)}), flush=True)
  # CPU baseline: the serial C checker of the loop alone (one host core) on the fields of a 256^3 cutout
  import oracle_geodesic as G
  cut = np.asfortranarray(seg(ctx, (256, 256, 256)))
  loop_s = {}

  def timed_loop(*args, **kw):
    t = time.perf_counter()
    out = G.teasar(*args, **kw)
    loop_s[kw["parents"] is None] = time.perf_counter() - t
    return out
  ref = T.skeletonize_modes(cut, ANISO, 4.0, 500.0, dust_threshold=1000, fix_borders=True, run_loop=timed_loop,
                            geodesic=lambda lab, s, a=(1, 1, 1), weights=None, parents=False:
                            G.geodesic(lab, np.asarray(s, np.uint64), 26, a, weights, parents))
  for fb in (True, False):
    kimimaro.skeletonize(cut, PARAMS, anisotropy=ANISO, fix_branching=fb, ctx=ctx)
    kimimaro.skeletonize(cut, PARAMS, anisotropy=ANISO, fix_branching=fb, ctx=ctx)
    got = kimimaro.skeletonize(cut, PARAMS, anisotropy=ANISO, fix_branching=fb, ctx=ctx)
    same = sorted(got) == sorted(ref[fb]) and all(np.array_equal(got[l].vertices, ref[fb][l][0]) and
                                                  np.array_equal(got[l].edges, ref[fb][l][1]) for l in got)
    print(json.dumps({"op": "loop_vs_cpu", "workload": "seg256", "gpu": card(), "fix_branching": fb,
                      "cpu_loop_s": round(loop_s[fb], 3),
                      "gpu_loop_ms": round(kimimaro.last_phase_seconds["loop"] * 1e3, 2),
                      "gpu_call_ms": round(sum(kimimaro.last_phase_seconds.values()) * 1e3, 1), "labels": len(got),
                      "bit_exact": bool(same)}), flush=True)


if __name__ == "__main__":
  main()
