"""One TransferTask per workload on file:// layers in a temporary directory, with host-clock phase times.

Workloads (four mips each, 64^3 chunks, files stored without gzip):
  image-raw   2048 x 2048 x 128 uint8 image, raw -> raw
  image-jpeg  2048 x 2048 x 128 uint8 image, jpeg -> jpeg (quality 85)
  seg-cseg    1024 x 1024 x 256 uint64 segmentation (labels above 2^32), compressed_segmentation -> same

Phases (current tree): read files (CloudFiles.get), H2D (one copy of the files, or of a host image),
decode + place, pool (the device pyramid), cut + encode + D2H, writes (CloudFiles.put), and what is left
of the task (Python, info handling).  Each phase ends in a device synchronise, so its host-clock time
includes its kernels.

--parent DIR runs the same task with the tree in DIR (another commit, already built) as well, alternated
with this tree in every round, and checks that both write the same files (decompressed contents).

  python tools/microbench_transfer.py [--parent DIR] [--rounds N] [--workloads image-raw,image-jpeg,seg-cseg]
"""
import argparse
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
WORKLOADS = {
  "image-raw": ((2048, 2048, 128), "uint8", "raw"),
  "image-jpeg": ((2048, 2048, 128), "uint8", "jpeg"),
  "seg-cseg": ((1024, 1024, 256), "uint64", "compressed_segmentation"),
}
CHUNK = (64, 64, 64)
MIPS = 4


def _source(tmp, name):
  """the source layer of a workload, written once with this tree"""
  sys.path.insert(0, ROOT)
  import numpy as np
  from oracle import oracle as O
  from igneous_b200._compat import CloudVolume
  O.build()
  shape, dtype, enc = WORKLOADS[name]
  path = "file://" + os.path.join(tmp, "src-" + name)
  if dtype == "uint8":
    data = O.synth_image(shape)
  else:
    data = O.synth_seg(shape, pitch=16, num_ids=4096).astype(np.uint64) + np.uint64(2 ** 33)
  CloudVolume.from_numpy(data[..., np.newaxis], vol_path=path, resolution=(4, 4, 40), chunk_size=CHUNK,
                         encoding=enc, compress=None)
  return path


def _digest(path):
  """sha256 of every chunk file's decompressed content, by name"""
  from igneous_b200._compat import CloudFiles
  cf = CloudFiles(path)
  h = hashlib.sha256()
  names = [n for n in cf.list("") if n not in ("info", "provenance")]
  for n in names:
    h.update(n.encode())
    h.update(cf.get(n))
  return h.hexdigest(), len(names)


def worker(tree, src, dest):
  """one transfer task with the package of `tree`; prints a JSON line"""
  sys.path.insert(0, tree)
  import copy
  from igneous_b200 import _shim, downsample_scales
  from igneous_b200._compat import CloudVolume
  from igneous_b200.tasks import TransferTask
  ctx = _shim.default_context()
  info = copy.deepcopy(CloudVolume(src).info)
  CloudVolume(dest, info=info).commit_info()
  size = CloudVolume(dest).meta.volume_size(0)
  downsample_scales.create_downsample_scales(dest, 0, size, preserve_chunk_size=True, max_mips=MIPS)
  phases = _instrument(ctx)
  ctx.sync()
  t0 = time.perf_counter()
  TransferTask(src, dest, 0, tuple(int(v) for v in size), (0, 0, 0), compress=None, max_mips=MIPS)
  ctx.sync()
  total = time.perf_counter() - t0
  out = {"tree": tree, "seconds": total}
  if phases is not None:
    out["phases_s"] = dict(phases, **{"rest of the task": total - sum(phases.values())})
  out["digest"], out["files"] = _digest(dest)
  print(json.dumps(out))


def _instrument(ctx):
  """wrap the read / write path's steps in host-clock timers (exclusive of nested steps); None for a
  tree without the device paths"""
  from igneous_b200 import storage, tinybrain
  if not hasattr(storage.CloudVolume, "download_dev"):
    return None
  phases, stack = {}, []

  def timed(name, fn):
    def run(*a, **k):
      ctx.sync()
      stack.append(0.0)
      t = time.perf_counter()
      try:
        return fn(*a, **k)
      finally:
        ctx.sync()
        dt = time.perf_counter() - t
        inner = stack.pop()
        phases[name] = phases.get(name, 0.0) + dt - inner
        if stack:
          stack[-1] += dt
    return run

  storage.CloudFiles.get = timed("read files", storage.CloudFiles.get)
  storage.CloudFiles.put = timed("writes", storage.CloudFiles.put)
  storage._upload_bytes = timed("H2D", storage._upload_bytes)
  storage.DeviceCutout.from_host = classmethod(timed("H2D", storage.DeviceCutout.from_host.__func__))
  storage.CloudVolume._decode_into = timed("decode + place", storage.CloudVolume._decode_into)
  storage.CloudVolume._encode_boxes = timed("cut + encode + D2H", storage.CloudVolume._encode_boxes)
  tinybrain.downsample_dev = timed("pool", tinybrain.downsample_dev)
  return phases


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--parent", help="tree of another commit (built) to alternate with and compare against")
  ap.add_argument("--rounds", type=int, default=1)
  ap.add_argument("--workloads", default=",".join(WORKLOADS))
  ap.add_argument("--worker", nargs=3, metavar=("TREE", "SRC", "DEST"), help=argparse.SUPPRESS)
  args = ap.parse_args()
  if args.worker:
    return worker(*args.worker)
  try:
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
  except OSError:
    gpu = "unknown"
  print(json.dumps({"gpu": gpu}))
  trees = [ROOT] + ([os.path.abspath(args.parent)] if args.parent else [])
  tmp = tempfile.mkdtemp(prefix="ign_xfer_")
  ok = True
  try:
    for name in args.workloads.split(","):
      src = _source(tmp, name)
      digests = {}
      for r in range(args.rounds):
        order = trees if r % 2 == 0 else trees[::-1]
        for i, tree in enumerate(order):
          dest = "file://" + os.path.join(tmp, "dest-%s-%d-%d" % (name, r, i))
          p = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker", tree, src, dest],
                             capture_output=True, text=True)
          if p.returncode != 0:
            print(p.stdout + p.stderr[-3000:])
            raise SystemExit("worker failed: %s on %s" % (name, tree))
          res = json.loads(p.stdout.strip().splitlines()[-1])
          res.update(workload=name, round=r, tree="this" if tree == ROOT else "parent")
          digests.setdefault(res["tree"], set()).add(res["digest"])
          print(json.dumps(res))
          shutil.rmtree(dest[len("file://"):], ignore_errors=True)
      same = len(set().union(*digests.values())) == 1
      ok &= same
      print(json.dumps({"workload": name, "outputs_identical": same}))
  finally:
    shutil.rmtree(tmp, ignore_errors=True)
  return 0 if ok else 1


if __name__ == "__main__":
  sys.exit(main())
