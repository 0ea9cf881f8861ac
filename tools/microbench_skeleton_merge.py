"""Micro-benchmark of the skeleton merge stage on a file:// layer (host clock; every phase ends where the host
already waits for the device or the file system).

Workloads, anisotropy (16, 16, 40), written raw in 128^3 chunks to a layer in a temporary directory:
  voronoi   the bench's jittered-grid Voronoi segmentation (pitch 16, membranes of label 0) at 449^3
  capsules  a tree of capsule-shaped neurites (radius 3 voxels) branching across the whole volume, 449^3
SkeletonTask runs over a 2 x 2 x 2 grid (create_skeletonizing_tasks, shape 225, will_postprocess on, so each
task writes fragments), then every UnshardedSkeletonMergeTask of magnitude 1 (nine prefixes; crop 0,
dust_threshold 4000, tick_threshold 6000).  Reported per workload: labels and fragments, the merge tasks'
phases summed (list / get, unpickle, device call, writes), and for the same packed batch the device call
against the C checker (oracle_skeleton) and the numpy restatement (tests/skelmergeref.py, on at most
`--ref-labels` labels), each on one host core.
A third workload, `large`, times one device call on a single neuron-like label without any task: a random
tree of `--large` vertices (steps of 40 nm, a branch every ~100 vertices, radius 200 nm) cut into 8 fragments by
vertex order, the cuts alternately sharing their end vertex and leaving a 60 nm gap that connect pieces must
bridge.  The C checker runs on it up to `--checker-max` vertices (its connect pieces and ticks are quadratic).
Prints one JSON line per workload with the card's name, power limit and SM clock.  `--size 97` makes a quick
run."""
import argparse
import json
import os
import pickle
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402

import oracle_skeleton  # noqa: E402
import skelmergeref  # noqa: E402
from igneous_b200 import _shim, kimimaro  # noqa: E402
from igneous_b200 import task_creation as tc  # noqa: E402
from igneous_b200._compat import Bbox, CloudFiles, CloudVolume, LocalTaskQueue  # noqa: E402
from igneous_b200.tasks import skeleton as task_module  # noqa: E402

ANISO = (16, 16, 40)
KW = dict(crop=0, dust_threshold=4000, tick_threshold=6000)


def card():
  q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                     stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()
  return q[0] if q else "unknown"


def voronoi(ctx, shape):
  raw = ctx.alloc(int(np.prod(shape)) * 4)
  _shim.check(ctx.lib.ign_synth_seg_dev(ctx.handle, _shim.ptr(raw), _shim.IGN_U32, *shape, 0, 0, 0, 16, 1 << 20, 0,
                                        0))
  out = np.empty(shape, np.uint32, order="F")
  ctx.d2h(out, raw)
  ctx.sync()
  raw.free()
  return out


def capsules(shape, seed=0):
  """a random tree of capsules: each new segment starts on an earlier one; label = 1 + segment // 6"""
  rng = np.random.default_rng(seed)
  img = np.zeros(shape, np.uint32)
  pts = [np.array(shape) / 2.0]
  for s in range(60):
    a = pts[int(rng.integers(0, len(pts)))]
    b = np.clip(a + rng.normal(0, 1, 3) / 1.0 * shape[0] / 4, 4, np.array(shape) - 5)
    lo = np.maximum(np.floor(np.minimum(a, b)) - 4, 0).astype(int)
    hi = np.minimum(np.ceil(np.maximum(a, b)) + 5, shape).astype(int)
    sub = np.stack(np.meshgrid(*[np.arange(l, h, dtype=np.float64) for l, h in zip(lo, hi)], indexing="ij"), -1)
    ab = b - a
    t = np.clip(((sub - a) @ ab) / max(ab @ ab, 1e-6), 0, 1)
    d = np.linalg.norm(sub - (a + t[..., None] * ab), axis=-1)
    view = img[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]]
    view[(d <= 3) & (view == 0)] = 1 + s // 6
    pts.append(b)
  return np.asfortranarray(img)


def fragments(path):
  vol = CloudVolume(path)
  cf = CloudFiles(vol.skeleton.path)
  out = {}
  for name in cf.list():
    m = task_module.SEGIDRE.search(name)
    if m:
      out.setdefault(int(m.group(1)), []).append((Bbox.from_filename(name), pickle.loads(cf.get(name))))
  return {k: out[k] for k in sorted(out)}


def run(ctx, root, name, img, ref_labels):
  path = "file://" + os.path.join(root, name)
  CloudVolume.from_numpy(img, path, resolution=ANISO, chunk_size=(128, 128, 64), layer_type="segmentation")
  half = (img.shape[0] + 1) // 2
  t0 = time.perf_counter()
  LocalTaskQueue().insert(tc.create_skeletonizing_tasks(path, mip=0, shape=(half, half, half),
                                                        teasar_params={"scale": 4, "const": 500}))
  t_skel = time.perf_counter() - t0
  frags = fragments(path)
  phases = {"list_get": 0.0, "unpickle": 0.0, "device": 0.0, "writes": 0.0}
  t0 = time.perf_counter()
  for t in tc.create_unsharded_skeleton_merge_tasks(path, magnitude=1, **KW):
    t.execute()
    p = task_module.last_phase_seconds
    phases["list_get"] += p["list"]
    phases["unpickle"] += p["unpickle"]
    phases["device"] += p["merge"]
    phases["writes"] += p["writes"]
  t_merge = time.perf_counter() - t0
  # the same batch in one call: device (after a warm-up) against the checkers
  segids, packed = kimimaro.pack_fragments(frags, crop=0, resolution=ANISO)
  kimimaro.merge_packed(packed, KW["dust_threshold"], KW["tick_threshold"], ctx=ctx)
  dev = []
  for _ in range(5):
    t0 = time.perf_counter()
    got, table = kimimaro.merge_packed(packed, KW["dust_threshold"], KW["tick_threshold"], ctx=ctx)
    dev.append(time.perf_counter() - t0)
  t0 = time.perf_counter()
  want, wtable = oracle_skeleton.merge(packed, KW["dust_threshold"], KW["tick_threshold"])
  t_c = time.perf_counter() - t0
  same = bool(np.array_equal(table, wtable) and bytes(got[:want.size]) == bytes(want))
  sub = segids[:ref_labels]
  t0 = time.perf_counter()
  for s in sub:
    sks = [(f.vertices, f.edges, f.radii, f.vertex_types) for _, f in frags[s]]
    skelmergeref.merge(sks, None, KW["dust_threshold"], KW["tick_threshold"])
  t_ref = time.perf_counter() - t0
  return {
    "workload": name, "shape": list(img.shape), "card": card(), "labels": len(frags),
    "fragments": int(sum(len(v) for v in frags.values())), "vertices": int(packed["radius"].size),
    "skeleton_tasks_s": round(t_skel, 3), "merge_tasks_s": round(t_merge, 3),
    "merge_phases_s": {k: round(v, 4) for k, v in phases.items()},
    "one_call_device_s": {"median": round(float(np.median(dev)), 4), "min": round(min(dev), 4)},
    "one_call_c_checker_s": round(t_c, 3), "numpy_restatement_s": round(t_ref, 3),
    "numpy_restatement_labels": len(sub), "device_equals_checker": same,
  }


def neuron(n, seed=0):
  """one label's fragments: a random tree of n vertices cut into 8 pieces (see the module docstring)"""
  rng = np.random.default_rng(seed)
  v = np.zeros((n, 3), np.float64)
  parent = np.zeros(n, np.int64)
  heading = np.array([1.0, 0.0, 0.0])
  tips = [0]
  for i in range(1, n):
    p = tips[-1] if rng.random() > 0.01 else int(rng.integers(0, i))
    if p != tips[-1]:
      tips.append(p)
    heading = heading + rng.normal(0, 0.3, 3)
    heading /= np.linalg.norm(heading)
    v[i] = v[p] + 40.0 * heading
    parent[i] = p
    tips[-1] = i
  cuts = np.linspace(0, n, 9).astype(int)
  frags = []
  for k in range(8):
    lo, hi = cuts[k], cuts[k + 1]
    keep = np.arange(max(lo - (k % 2 == 1), 0), hi)  # odd cuts share the end vertex of the previous piece
    local = {int(g): j for j, g in enumerate(keep)}
    e = [(local[int(g)], local[int(parent[g])]) for g in keep[1:] if int(parent[g]) in local]
    pts = v[keep].astype(np.float32)
    if k % 2 == 0 and k:
      pts = pts + np.float32(60.0)  # a gap to the previous piece, inside the radii
    frags.append((None, kimimaro.Skeleton(pts, np.array(e, np.uint32).reshape(-1, 2),
                                          np.full(len(keep), 200.0, np.float32), np.zeros(len(keep), np.uint8), 1)))
  return {1: frags}


def run_large(ctx, n, checker_max):
  frags = neuron(n)
  _, packed = kimimaro.pack_fragments(frags)
  got, table = kimimaro.merge_packed(packed, KW["dust_threshold"], KW["tick_threshold"], ctx=ctx)
  dev = []
  for _ in range(3):
    t0 = time.perf_counter()
    got, table = kimimaro.merge_packed(packed, KW["dust_threshold"], KW["tick_threshold"], ctx=ctx)
    dev.append(time.perf_counter() - t0)
  out = {"workload": "large", "card": card(), "vertices_in": int(packed["radius"].size),
         "vertices_out": int(table[0, 2]), "edges_out": int(table[0, 3]),
         "one_call_device_s": {"median": round(float(np.median(dev)), 4), "min": round(min(dev), 4)}}
  if n <= checker_max:
    t0 = time.perf_counter()
    want, wtable = oracle_skeleton.merge(packed, KW["dust_threshold"], KW["tick_threshold"])
    out["one_call_c_checker_s"] = round(time.perf_counter() - t0, 3)
    out["device_equals_checker"] = bool(np.array_equal(table, wtable) and bytes(got[:want.size]) == bytes(want))
  return out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--size", type=int, default=449)
  ap.add_argument("--ref-labels", type=int, default=50)
  ap.add_argument("--large", type=int, nargs="*", default=[20000, 100000])
  ap.add_argument("--checker-max", type=int, default=20000)
  ap.add_argument("--workloads", nargs="*", default=["voronoi", "capsules", "large"])
  args = ap.parse_args()
  ctx = _shim.default_context()
  shape = (args.size,) * 3
  root = tempfile.mkdtemp(prefix="skelmerge_")
  try:
    for name, img in (("voronoi", lambda: voronoi(ctx, shape)), ("capsules", lambda: capsules(shape))):
      if name in args.workloads:
        print(json.dumps(run(ctx, root, name, img(), args.ref_labels)), flush=True)
    if "large" in args.workloads:
      for n in args.large:
        print(json.dumps(run_large(ctx, n, args.checker_max)), flush=True)
  finally:
    shutil.rmtree(root, ignore_errors=True)


if __name__ == "__main__":
  main()
