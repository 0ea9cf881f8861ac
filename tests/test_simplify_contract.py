"""CPU: the simplifier's contract (tests/meshref.py) on every label the oracle simplifies.  The GPU is checked
bit for bit against the oracle elsewhere, so these tests are what pin the algorithm itself: on the benchmark
block, on a volume with labels in every size class, on the smallest closed labels, on labels of genus 1 to 3
and with a cavity, on labels cut by one to six faces of the task box, and on sparse noise with thousands of
tiny labels touching along edges and corners, over a sample of the factor / max_error / resolution /
voxel_centered grid.

Known gap: the per-face flip test does not keep a closed component whose size is below max_error from
flattening or turning inside out (test_small_closed_components_keep_their_volume, expected to fail).  The
volume of closed components is therefore checked on the labels that are large next to max_error only."""
import numpy as np
import pytest

from meshref import check_simplified

MAX_ROUNDS = 400


def bench_block(oracle):
  # a 129^3 block of the benchmark's mip-2 MeshTask volume: synth_seg pitch 64, seed 0, two 2x2x1 mode mips
  seg = oracle.synth_seg((516, 516, 129), pitch=64, num_ids=1 << 20, seed=0)
  return np.asfortranarray(oracle.downsample_segmentation(seg, (2, 2, 1), num_mips=2)[1].astype(np.uint32))


def class_volume(oracle):
  # 57 labels from 490 to 35,550 faces: every size class of k_simp_labels, and faces in global memory
  return np.asfortranarray(oracle.synth_seg((128, 128, 96), pitch=32, num_ids=64).astype(np.uint32))


def tiny_closed():
  """The smallest closed labels: one voxel, 1x1x2, rods of 3 and 6 along each axis, one-voxel sheets,
  2x2x1 and 2x2x2.  Simplified far enough they must end as tetrahedra, not as two coincident faces."""
  seg = np.zeros((40, 30, 14), dtype=np.uint32, order="F")
  seg[2, 2, 2] = 1
  seg[6, 2, 2:4] = 2
  seg[10, 2, 2:8] = 3
  seg[14:17, 2, 2] = 4
  seg[2, 6:12, 6] = 5
  seg[2:8, 14:20, 6] = 6
  seg[20, 2:7, 2:6] = 7
  seg[24:26, 2:4, 2:4] = 8
  seg[30:32, 2:4, 2] = 9
  seg[10:13, 10:13, 10] = 10
  seg[30:36, 10, 4:10] = 11
  return seg


def holes():
  """Slabs with one, two and three holes drilled through them (genus 1-3), and a cube with a cavity (an
  inner surface of negative volume)."""
  seg = np.zeros((26, 34, 24), dtype=np.uint32, order="F")
  for lab, y0 in ((1, 1), (2, 9), (3, 17)):
    seg[1:25, y0:y0 + 7, 1:7] = lab
    for h in range(lab):
      seg[3 + 7 * h:5 + 7 * h, y0 + 2:y0 + 5, 1:7] = 0
  seg[2:12, 25:33, 10:20] = 4
  seg[5:8, 28:30, 13:16] = 0
  return seg


def cut_by(k):
  """A label open on k = 1..6 faces of the task box (k = 6: three crossing bars)."""
  seg = np.zeros((18, 16, 14), dtype=np.uint32, order="F")
  if k == 6:
    seg[:, 6:10, 5:9] = 5
    seg[7:11, :, 5:9] = 5
    seg[7:11, 6:10, :] = 5
    return seg
  lo = [0, 0 if k >= 2 else 3, 0 if k >= 3 else 3]
  hi = [18 if k >= 4 else 11, 16 if k >= 5 else 10, 9]
  seg[lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]] = 5
  seg[lo[0] + 1:lo[0] + 3, lo[1] + 2:lo[1] + 4, 4:6] = 0 if k % 2 else 6   # a dent, or a second label in it
  return seg


def noise(seed=5):
  """Sparse noise: about 4,000 labels, each the voxels kept (p = 0.35) of one 3x3x3 cell, so voxels of one
  label and of neighbouring labels touch along edges and corners."""
  rng = np.random.default_rng(seed)
  n = 48
  x, y, z = np.meshgrid(np.arange(n), np.arange(n), np.arange(n), indexing="ij")
  cell = (x // 3) + 16 * ((y // 3) + 16 * (z // 3)) + 1
  keep = rng.random((n, n, n)) < 0.35
  return np.asfortranarray(np.where(keep, cell, 0).astype(np.uint32))


# (reduction factor, max_error, resolution, voxel_centered): every value of each parameter, in pairs that
# differ from volume to volume
GRID = [
  (2, 0.0, (1, 1, 1), False),
  (10, 1.0, (16, 16, 40), True),
  (100, 40.0, (4, 4, 40), True),
  (1000, 1e9, (1, 1, 1), True),
  (100, 1.0, (1, 1, 1), False),
  (1000, 40.0, (16, 16, 40), False),
  (10, 1e9, (4, 4, 40), False),
  (2, 40.0, (16, 16, 40), True),
  (1000, 0.0, (4, 4, 40), True),
  (100, 1e9, (16, 16, 40), False),
]
BENCH = (100, 40.0, (16, 16, 40), True)


def simplify_and_check(oracle, seg, factor, max_error, res, centered, volume=True):
  """Simplify every label of `seg` with the oracle and check the contract (volume: also the volume of
  closed components).  Returns the welded meshes, the oracle's output and rep, and the total output face
  count."""
  tl, tv = oracle.marching_cubes(seg)
  W = oracle.WeldedMeshes(tl, tv)
  out, rounds, rep = oracle.simplify_welded(W, res, factor, max_error, centered, MAX_ROUNDS, with_rep=True)
  before = {l: W.get(l, res, centered) for l in W.ids()}
  targets = {l: len(before[l][1]) // factor for l in W.ids()}
  total = check_simplified(before, out, rep, targets, max_error, rounds < MAX_ROUNDS, volume)
  return W, out, rep, total


def test_bench_block(oracle):
  # the benchmark's own parameters; before the tetrahedron rule 9 of its 299 labels held coincident faces
  W, out, _, total = simplify_and_check(oracle, bench_block(oracle), *BENCH)
  assert len(W.ids()) == 299
  assert total == 203814


def test_class_volume(oracle):
  seg = class_volume(oracle)
  simplify_and_check(oracle, seg, *GRID[5])


def test_tiny_closed_labels(oracle):
  seg = tiny_closed()
  for params in GRID:
    _, out, _, _ = simplify_and_check(oracle, seg, *params, volume=params[1] <= 1.0)
    if params[0] == 1000 and params[1] == 1e9:
      # nothing holds them back: every label ends as the smallest closed surface, a tetrahedron
      assert {l: len(f) for l, (v, f) in out.items()} == {l: 4 for l in out}, params


@pytest.mark.parametrize("params", GRID[::2] + GRID[1::2][:2])
def test_holes_and_cavity(oracle, params):
  simplify_and_check(oracle, holes(), *params, volume=params[1] <= 40.0)


@pytest.mark.parametrize("k", range(1, 7))
def test_cut_by_task_box(oracle, k):
  seg = cut_by(k)
  for params in GRID[k % 2::2]:
    simplify_and_check(oracle, seg, *params)


@pytest.mark.parametrize("params", [GRID[0], GRID[3], GRID[5], GRID[6]])
def test_noise(oracle, params):
  simplify_and_check(oracle, noise(), *params, volume=params[1] <= 1.0)


@pytest.mark.xfail(strict=True, reason="a collapse only checks that no face of its rings flips, so closed "
                   "components smaller than max_error can flatten or turn inside out")
@pytest.mark.parametrize("volume,params", [("tiny_closed", GRID[3]), ("noise", BENCH[:2] + ((4, 4, 40), True))])
def test_small_closed_components_keep_their_volume(oracle, volume, params):
  simplify_and_check(oracle, globals()[volume](), *params)
