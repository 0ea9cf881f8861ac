"""Micro-benchmark of igneous_b200.kimimaro.cross_sectional_area (host clock around calls that end in a device
synchronise, one warm-up call first).

Workloads: the 449^3 volumes of tools/microbench_skeletonize.py -- the uint32 pitch-16 synthetic segmentation
(teasar_params scale 4, const 500) and 120 random capsule trees (scale 1.5, const 50) -- at anisotropy
(16, 16, 40), skeletonized once, then cross-sectioned at smoothing windows 1 and 5.  Per workload and window:
median and min seconds of the whole call over the timed reps, each phase of the last rep
(kimimaro.last_phase_seconds), vertices, section voxels visited, vertices on the large path, and visits per
second of the sections phase.  The CPU baseline is the serial C checker (one host core) on a 160^3 cutout of
the synthetic volume, against the GPU call on the same cutout, with the largest relative area difference.
Prints one JSON line per measurement with the card's name, power limit, SM clock and throttle reasons read
before and after."""
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np  # noqa: E402

from igneous_b200 import _shim, kimimaro  # noqa: E402
from microbench_skeletonize import ANISO, NEURITE_PARAMS, PARAMS, card, seg, timed  # noqa: E402


def main(reps=3):
  import teasarref as T
  ctx = _shim.default_context()
  work = [("seg449", PARAMS, lambda: seg(ctx, (449, 449, 449))),
          ("neurites449", NEURITE_PARAMS, lambda: T.capsule_trees((449, 449, 449), 120, seed=1, anisotropy=ANISO))]
  for name, params, make in work:
    vol = make()
    skels = kimimaro.skeletonize(vol, params, anisotropy=ANISO, ctx=ctx)
    nv = sum(len(s.vertices) for s in skels.values())
    for w in (1, 5):
      before = card()
      med, mn = timed(lambda: kimimaro.cross_sectional_area(vol, skels, anisotropy=ANISO, smoothing_window=w,
                                                            ctx=ctx), reps)
      phases = {k: round(v * 1e3, 2) for k, v in kimimaro.last_phase_seconds.items()}
      voxels, large, abandoned, ctas = kimimaro.last_stats
      print(json.dumps({"op": "cross_sectional_area", "workload": name, "shape": list(vol.shape),
                        "labels": len(skels), "vertices": nv, "window": w, "gpu_before": before,
                        "gpu_after": card(), "reps": reps, "s": round(med, 4), "min_s": round(mn, 4),
                        "phase_ms_last_rep": phases, "section_voxels": voxels, "large_vertices": large,
                        "voxels_visited_before_handoff": abandoned, "large_path_ctas": ctas,
                        "visits_per_s_sections_phase": round(voxels / max(kimimaro.last_phase_seconds["sections"],
                                                                          1e-9))}), flush=True)
  # CPU baseline: the serial C checker on a cutout, against the GPU on the same cutout
  import oracle_xsection as X
  cut = np.asfortranarray(seg(ctx, (160, 160, 160)))
  skels = kimimaro.skeletonize(cut, PARAMS, anisotropy=ANISO, ctx=ctx)
  av = np.asarray(ANISO, np.float64)
  vox = np.concatenate([np.rint(s.vertices.astype(np.float64) / av).astype(np.int64) for s in skels.values()])
  offs = np.cumsum([0] + [len(s.vertices) for s in skels.values()])
  edges = np.concatenate([s.edges.astype(np.int64) + o for s, o in zip(skels.values(), offs)]).astype(np.uint32)
  pl = np.concatenate([np.full(len(s.vertices), k, np.uint64) for k, s in skels.items()])
  for w in (1, 5):
    t = time.perf_counter()
    nrm = X.normals(vox, edges, ANISO, w)
    area, cont, visited = X.sections(cut, vox, pl, nrm, ANISO)
    cpu_s = time.perf_counter() - t
    gpu_s = timed(lambda: kimimaro.cross_sectional_area(cut, skels, anisotropy=ANISO, smoothing_window=w,
                                                        ctx=ctx), reps)[0]
    got = kimimaro.cross_sectional_area(cut, skels, anisotropy=ANISO, smoothing_window=w, ctx=ctx)
    ga = np.concatenate([s.cross_sectional_area for s in got.values()])
    gc = np.concatenate([s.cross_sectional_area_contacts for s in got.values()])
    rel = float(np.max(np.abs(ga.astype(np.float64) - area) / np.maximum(np.abs(area), 1e-30))) if len(ga) else 0.0
    print(json.dumps({"op": "cross_section_vs_cpu", "workload": "seg160", "gpu": card(), "window": w,
                      "vertices": int(len(vox)), "section_voxels": visited, "cpu_checker_s": round(cpu_s, 3),
                      "gpu_call_s": round(gpu_s, 4), "contacts_equal": bool(np.array_equal(gc, cont)),
                      "max_rel_area_diff": rel}), flush=True)


if __name__ == "__main__":
  main()
