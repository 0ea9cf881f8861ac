"""compute_rois and BlackoutTask on the device against a numpy / scipy run of the same rule on the host.

Layer: a 2048 x 2048 x 256 uint8 image (oracle.synth_image), raw, 256 x 256 x 64 chunks, one scale (so the
top mip is the whole layer), files gzipped (level 1) as the tasks write them, in a temporary directory.

  rois                compute_rois(suppress_faint_voxels=132, dust_threshold=10): one slab, pooled four times
                      to 128 x 128 x 256 (ceil(log2(2048^2 / 512^2)) mips); host: the layer read on the host, oracle averaging, np.greater,
                      scipy.ndimage.label (3x3x3), np.bincount, find_objects, boxes by first F-order voxel
  blackout-aligned    BlackoutTask of (0, 0, 64)-(2048, 2048, 128); host: np.full and the host raw write
  blackout-unaligned  BlackoutTask(non_aligned_writes=True) of (0, 0, 70)-(2048, 2048, 134), which reads and
                      rewrites the chunks of z 64-192; host: read the region, fill, write it back

Each timing is a host clock around a call that ends in a device synchronise (device runs) or returns host
data (host runs); the median of --rounds runs after one warm-up run, device and host alternated.  The device
and host results are compared: the same boxes, the same layer contents.

  python tools/microbench_rois.py [--rounds N] [--workloads rois,blackout-aligned,blackout-unaligned]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

SHAPE, CHUNK = (2048, 2048, 256), (256, 256, 64)
ALIGNED, UNALIGNED = ((0, 0, 64), (2048, 2048, 128)), ((0, 0, 70), (2048, 2048, 134))


def host_rois(path, suppress, dust, max_axial):
  """compute_rois's rule on the host (one slab)"""
  import numpy as np
  from scipy import ndimage
  from oracle import oracle as O
  from igneous_b200._compat import CloudVolume
  cv = CloudVolume(path, fill_missing=True)
  img = cv[cv.bounds][..., 0]
  sxy = img.shape[0] * img.shape[1]
  more = int(np.ceil(np.log2(sxy / max_axial ** 2))) if sxy > max_axial ** 2 else 0
  if more:
    img = O.downsample_with_averaging(np.asfortranarray(img), (2, 2, 1), num_mips=more)[-1]
  lab, n = ndimage.label(img > suppress, structure=np.ones((3, 3, 3), dtype=bool))
  sizes = np.bincount(lab.ravel())
  objs = ndimage.find_objects(lab)
  ids, first = np.unique(lab.ravel(order="F"), return_index=True)
  out = []
  z0 = int(cv.bounds.minpt[2])
  for _, l in sorted(zip(first, ids)):
    if l == 0 or sizes[l] < dust:
      continue
    s = objs[l - 1]
    lo = [s[0].start * 2 ** more, s[1].start * 2 ** more, s[2].start + z0]
    hi = [s[0].stop * 2 ** more - 1, s[1].stop * 2 ** more - 1, s[2].stop + z0 - 1]
    out.append(lo + hi)
  return out


def host_blackout(path, box, value):
  """the blackout on the host: a host array written through the raw host path"""
  import numpy as np
  from igneous_b200._compat import Bbox, CloudVolume
  vol = CloudVolume(path)
  box = Bbox(*box)
  region = Bbox.clamp(box.expand_to_chunk_size(vol.chunk_size, vol.voxel_offset), vol.bounds)
  img = vol[region] if not region == box else np.empty(tuple(box.size3()) + (1,), dtype=vol.dtype)
  img[tuple(slice(int(a - o), int(b - o)) for a, b, o in zip(box.minpt, box.maxpt, region.minpt))] = value
  vol[region] = img


def timed(fn, ctx=None):
  if ctx is not None:
    ctx.sync()
  t = time.perf_counter()
  out = fn()
  if ctx is not None:
    ctx.sync()
  return time.perf_counter() - t, out


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument("--rounds", type=int, default=3)
  ap.add_argument("--workloads", default="rois,blackout-aligned,blackout-unaligned")
  args = ap.parse_args()
  import numpy as np
  from oracle import oracle as O
  from igneous_b200 import _shim
  from igneous_b200._compat import CloudVolume
  from igneous_b200.task_creation import compute_rois
  from igneous_b200.tasks import BlackoutTask
  try:
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
  except OSError:
    gpu = "unknown"
  print(json.dumps({"gpu": gpu}), flush=True)
  ctx = _shim.default_context()
  O.build()
  data = O.synth_image(SHAPE)[..., np.newaxis]
  tmp = tempfile.mkdtemp(prefix="ign_rois_")
  ok = True
  try:
    paths = {}
    for name in ("dev", "host"):
      paths[name] = "file://" + os.path.join(tmp, name)
      CloudVolume.from_numpy(data, vol_path=paths[name], resolution=(4, 4, 40), chunk_size=CHUNK, compress="gzip")
      print("layer %s written" % name, file=sys.stderr, flush=True)
    work = {
      "rois": (lambda: [b.to_list() for b in compute_rois(paths["dev"], suppress_faint_voxels=132)],
               lambda: host_rois(paths["host"], 132, 10, 512)),
      "blackout-aligned": (lambda: BlackoutTask(paths["dev"], 0, (2048, 2048, 64), ALIGNED[0], value=17),
                           lambda: host_blackout(paths["host"], ALIGNED, 17)),
      "blackout-unaligned": (lambda: BlackoutTask(paths["dev"], 0, (2048, 2048, 64), UNALIGNED[0], value=23,
                                                  non_aligned_writes=True),
                             lambda: host_blackout(paths["host"], UNALIGNED, 23)),
    }
    for name in args.workloads.split(","):
      dev, host = work[name]
      times = {"device": [], "host": []}
      for r in range(args.rounds + 1):
        td, out_d = timed(dev, ctx)
        th, out_h = timed(host)
        print("%s round %d: device %.3f s, host %.3f s" % (name, r, td, th), file=sys.stderr, flush=True)
        if r:
          times["device"].append(td)
          times["host"].append(th)
      same = out_d == out_h if name == "rois" else \
          np.array_equal(CloudVolume(paths["dev"])[CloudVolume(paths["dev"]).bounds],
                         CloudVolume(paths["host"])[CloudVolume(paths["host"]).bounds])
      ok &= bool(same)
      res = {"workload": name, "device_s": float(np.median(times["device"])), "host_s": float(np.median(times["host"])),
             "device_runs_s": times["device"], "host_runs_s": times["host"], "results_identical": bool(same)}
      if name == "rois":
        res["boxes"] = len(out_d)
      print(json.dumps(res), flush=True)
  finally:
    shutil.rmtree(tmp, ignore_errors=True)
  return 0 if ok else 1


if __name__ == "__main__":
  sys.exit(main())
