"""In-tree build of libigneous_b200.so (sm_90a only).

nvcc cross-compiles without a GPU; the .so and objects are build products and
stay out of git.  `python -m igneous_b200.build [--force]`.
"""
import concurrent.futures
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
ASAN = bool(os.environ.get("IGN_ASAN"))
LIB = os.path.join(CSRC, "libigneous_b200_asan.so" if ASAN else "libigneous_b200.so")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
NVCC_FLAGS = [
  "-gencode", "arch=compute_90a,code=sm_90a",
  "-lineinfo", "-O3", "-std=c++17",
  "-Xcompiler", "-fPIC,-O3,-fvisibility=hidden",
  "--expt-relaxed-constexpr",
  "-Xptxas", "-v",
]


def _stale(target, deps):
  if not os.path.exists(target):
    return True
  t = os.path.getmtime(target)
  return any(os.path.getmtime(d) > t for d in deps)


# simplify.cu must match the CPU oracle bit for bit, and contrast.cu the float32 rules of
# DESIGN.md §5b (each product rounded on its own), geodesic.cu the penalty field of §5e, xsection.cu the
# membership test of §5i: no FMA contraction
PER_FILE_FLAGS = {"simplify.cu": ["-fmad=false"], "contrast.cu": ["-fmad=false"], "geodesic.cu": ["-fmad=false"],
                  "skelmerge.cu": ["-fmad=false"], "xsection.cu": ["-fmad=false"]}


def _compile(src, obj, log):
  extra = ["-Xcompiler", "-fsanitize=address,-fno-omit-frame-pointer", "-g"] if ASAN else []
  cmd = [NVCC] + NVCC_FLAGS + extra + PER_FILE_FLAGS.get(os.path.basename(src), []) + ["-c", src, "-o", obj]
  p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
  with open(log, "w") as f:
    f.write(" ".join(cmd) + "\n" + p.stdout)
  if p.returncode != 0:
    raise RuntimeError("nvcc failed for %s:\n%s" % (src, p.stdout[-4000:]))
  return obj


def build(force=False, verbose=False):
  srcs = sorted(glob.glob(os.path.join(CSRC, "*.cu")))
  hdrs = glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(CSRC, "*.h")) + \
      [os.path.join(os.path.dirname(HERE), "include", "igneous_b200.h")]
  os.makedirs(os.path.join(CSRC, "build"), exist_ok=True)
  jobs = []
  objs = []
  for s in srcs:
    base = os.path.splitext(os.path.basename(s))[0]
    o = os.path.join(CSRC, "build", base + (".asan.o" if ASAN else ".o"))
    objs.append(o)
    if force or _stale(o, [s] + hdrs):
      jobs.append((s, o, os.path.join(CSRC, "build", base + ".log")))
  if jobs:
    with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
      list(ex.map(lambda j: _compile(*j), jobs))
  if force or jobs or _stale(LIB, objs):
    cmd = [NVCC, "-shared", "-o", LIB] + objs + ["-lcudart_static", "-ldl", "-lrt", "-lpthread"] + \
        (["-Xcompiler", "-fsanitize=address"] if ASAN else [])
    p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if p.returncode != 0:
      raise RuntimeError("link failed:\n" + p.stdout[-4000:])
  if verbose:
    print("built", LIB, "(%d recompiled)" % len(jobs))
  return LIB


if __name__ == "__main__":
  build(force="--force" in sys.argv, verbose=True)
