"""Host-clock micro-benchmark of the compressed_segmentation codec entry points, each call followed by a
device synchronise.

Cases:
  one chunk   256 x 256 x 64 uint32 synth_seg, 8x8x8 and 8x4x2 blocks: ign_cseg_encode_dev, ign_cseg_decode_dev
  batch       64 chunks of 64^3 uint64 labels above 2^32 (the storage write path's shape), 8x8x8 blocks:
              ign_cseg_encode_batch_dev, ign_cseg_decode_batch_dev

Every call is checked: the decode gives back the labels.  --parent DIR runs the same calls with the tree in
DIR (another commit, already built) as well, alternated with this tree in every round, and checks that both
trees write identical streams.  Prints the card's name and power limit, one JSON line per round and tree,
and per case the median over rounds of each tree's per-round median in ms.

  python tools/microbench_cseg.py [--parent DIR] [--rounds N] [--reps N]
"""
import argparse
import ctypes as c
import hashlib
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
ONE = (256, 256, 64)
BATCH_CHUNK, BATCH_GRID = (64, 64, 64), (4, 4, 4)


def _inputs(tmp):
  """the labels of both cases, made once with this tree's oracle and shared with every worker"""
  sys.path.insert(0, ROOT)
  import numpy as np
  from oracle import oracle as O
  O.build()
  one = O.synth_seg(ONE, pitch=16, num_ids=1 << 20).astype(np.uint32)
  vol = O.synth_seg(tuple(c * g for c, g in zip(BATCH_CHUNK, BATCH_GRID)), pitch=16, num_ids=4096)
  vol = vol.astype(np.uint64) + np.uint64(2 ** 33)
  cx, cy, cz = BATCH_CHUNK
  chunks = [vol[i * cx:(i + 1) * cx, j * cy:(j + 1) * cy, k * cz:(k + 1) * cz]
            for k in range(BATCH_GRID[2]) for j in range(BATCH_GRID[1]) for i in range(BATCH_GRID[0])]
  packed = np.concatenate([ch.reshape(-1, order="F") for ch in chunks])
  np.save(os.path.join(tmp, "one.npy"), np.asfortranarray(one))
  np.save(os.path.join(tmp, "batch.npy"), packed)


def _timed(ctx, fn, reps):
  for _ in range(2):
    fn()
  ctx.sync()
  ts = []
  for _ in range(reps):
    t = time.perf_counter()
    fn()
    ctx.sync()
    ts.append((time.perf_counter() - t) * 1e3)
  ts.sort()
  return ts[len(ts) // 2]


def worker(tree, tmp, reps):
  """every case with the package of `tree`; prints one JSON line"""
  sys.path.insert(0, tree)
  import numpy as np
  from igneous_b200 import _shim
  ctx = _shim.default_context()
  lib = ctx.lib
  res = {}

  one = np.load(os.path.join(tmp, "one.npy"))
  d_one, d_dec = ctx.to_device(one), ctx.alloc(one.nbytes)
  for bs in ((8, 8, 8), (8, 4, 2)):
    g = 1
    for s, b in zip(ONE, bs):
      g *= -(-s // b)
    cap = 1 + 2 * g + 2 * g * bs[0] * bs[1] * bs[2]
    d_out, n = ctx.alloc(cap * 4), c.c_uint64(0)

    def enc():
      _shim.check(lib.ign_cseg_encode_dev(ctx.handle, _shim.ptr(d_one), _shim.IGN_U32, *ONE, 1, *bs, _shim.ptr(d_out),
                                          cap, c.byref(n)))

    def dec():
      _shim.check(lib.ign_cseg_decode_dev(ctx.handle, _shim.ptr(d_out), n.value, _shim.IGN_U32, *ONE, 1, *bs,
                                          _shim.ptr(d_dec)))
    name = "one %dx%dx%d u32 %dx%dx%d" % (ONE + bs)
    res[name + " encode"] = _timed(ctx, enc, reps)
    res[name + " decode"] = _timed(ctx, dec, reps)
    words = np.empty(n.value, np.uint32)
    ctx.d2h(words, d_out)
    back = ctx.to_host(d_dec, one.shape, one.dtype)
    if not np.array_equal(back, one):
      raise SystemExit("%s: the decode does not give back the labels" % name)
    res[name + " stream"] = hashlib.sha256(words.tobytes()).hexdigest()
    d_out.free()
  d_one.free(), d_dec.free()

  packed = np.load(os.path.join(tmp, "batch.npy"))
  nchunk = BATCH_GRID[0] * BATCH_GRID[1] * BATCH_GRID[2]
  shapes = np.ascontiguousarray(np.array([BATCH_CHUNK] * nchunk, dtype=np.uint32))
  g = (BATCH_CHUNK[0] // 8) * (BATCH_CHUNK[1] // 8) * (BATCH_CHUNK[2] // 8)
  cap = nchunk * (1 + 2 * g + 3 * g * 512)
  d_in, d_dec = ctx.to_device(packed), ctx.alloc(packed.nbytes)
  d_out, d_off, nw = ctx.alloc(cap * 4), ctx.alloc((nchunk + 1) * 8), c.c_uint64(0)
  woff = np.zeros(nchunk + 1, np.uint64)

  def benc():
    _shim.check(lib.ign_cseg_encode_batch_dev(ctx.handle, _shim.ptr(d_in), _shim.IGN_U64, nchunk, _shim.ptr(shapes),
                                              1, 8, 8, 8, _shim.ptr(d_out), cap, _shim.ptr(d_off), c.byref(nw)))

  def bdec():
    _shim.check(lib.ign_cseg_decode_batch_dev(ctx.handle, _shim.ptr(d_out), _shim.ptr(woff), nchunk, _shim.IGN_U64,
                                              _shim.ptr(shapes), 1, 8, 8, 8, _shim.ptr(d_dec)))
  name = "batch %d x %dx%dx%d u64 8x8x8" % ((nchunk,) + BATCH_CHUNK)
  res[name + " encode"] = _timed(ctx, benc, reps)
  ctx.d2h(woff, d_off)
  ctx.sync()
  res[name + " decode"] = _timed(ctx, bdec, reps)
  words = np.empty(nw.value, np.uint32)
  ctx.d2h(words, d_out)
  back = ctx.to_host(d_dec, packed.shape, packed.dtype)
  if not np.array_equal(back, packed):
    raise SystemExit("%s: the decode does not give back the labels" % name)
  res[name + " stream"] = hashlib.sha256(words.tobytes() + woff.tobytes()).hexdigest()
  print(json.dumps(res))


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--parent", help="tree of another commit (built) to alternate with and compare against")
  ap.add_argument("--rounds", type=int, default=5)
  ap.add_argument("--reps", type=int, default=30, help="timed calls per case, round and tree (the median is kept)")
  ap.add_argument("--worker", nargs=2, metavar=("TREE", "TMP"), help=argparse.SUPPRESS)
  args = ap.parse_args()
  if args.worker:
    return worker(args.worker[0], args.worker[1], args.reps)
  try:
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
  except OSError:
    gpu = "unknown"
  print(json.dumps({"gpu": gpu}))
  trees = {"this": ROOT}
  if args.parent:
    trees["parent"] = os.path.abspath(args.parent)
  tmp = tempfile.mkdtemp(prefix="ign_cseg_")
  times, streams = {}, {}
  try:
    _inputs(tmp)
    for r in range(args.rounds):
      names = list(trees) if r % 2 == 0 else list(trees)[::-1]
      for t in names:
        p = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", trees[t], tmp, "--reps",
                            str(args.reps)], capture_output=True, text=True)
        if p.returncode != 0:
          print(p.stdout + p.stderr[-3000:])
          raise SystemExit("worker failed on %s" % trees[t])
        res = json.loads(p.stdout.strip().splitlines()[-1])
        print(json.dumps(dict(res, tree=t, round=r)))
        for k, v in res.items():
          if k.endswith(" stream"):
            streams.setdefault(k, set()).add(v)
          else:
            times.setdefault(k, {}).setdefault(t, []).append(v)
  finally:
    shutil.rmtree(tmp, ignore_errors=True)
  for k, per in times.items():
    print(json.dumps({"case": k, **{t: {"median_ms": round(sorted(v)[len(v) // 2], 4), "min_ms": round(min(v), 4),
                                        "max_ms": round(max(v), 4)} for t, v in per.items()}}))
  same = all(len(v) == 1 for v in streams.values())
  print(json.dumps({"streams_identical": same}))
  return 0 if same else 1


if __name__ == "__main__":
  sys.exit(main())
