"""The quadric simplifier on the GPU (k_simp_labels / k_simp_resume) against the CPU oracle: every mesh is
bit-identical to the oracle's on every memory path, size class, winner cap and lane-group width, and the
counters of ign_mesh_simplify_counters (c below; include/igneous_b200.h documents each word) show which
of those paths ran."""
import ctypes
import os
import re

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _simplify(seg, res, factor, max_error, centered, **env):
  """Mesh and simplify `seg` with IGN_SIMP_<NAME> set to each value of `env` (gmem=1, wcap=8, group=16,
  trace=1; None leaves it unset) and every other IGN_SIMP_* variable cleared.  Returns the meshes by label
  and the 17 counters of ign_mesh_simplify_counters."""
  from igneous_b200 import _shim, zmesh
  saved = {k: os.environ.pop(k) for k in list(os.environ) if k.startswith("IGN_SIMP_")}
  os.environ.update({"IGN_SIMP_" + k.upper(): str(v) for k, v in env.items() if v is not None})
  try:
    m = zmesh.Mesher(res)
    m.mesh(seg)
    meshes = {int(i): m.get(i, reduction_factor=factor, max_error=max_error, voxel_centered=centered)
              for i in m.ids()}
  finally:
    for k in [k for k in os.environ if k.startswith("IGN_SIMP_")]:
      del os.environ[k]
    os.environ.update(saved)
  counters = (ctypes.c_uint32 * 17)()
  _shim.check(m._ctx.lib.ign_mesh_simplify_counters(m._handle, counters))
  return meshes, list(counters)


_ORACLE = {}


def _oracle(oracle, name, seg, res, factor, max_error, centered):
  """The oracle's welded input and simplified meshes of the volume `name`, computed once per module."""
  key = (name, res, factor, max_error, centered)
  if key not in _ORACLE:
    tl, tv = oracle.marching_cubes(seg)
    W = oracle.WeldedMeshes(tl, tv)
    _ORACLE[key] = (W, oracle.simplify_welded(W, res, factor, max_error, centered)[0])
  return _ORACLE[key]


def _assert_same(got, want, *where):
  assert got.keys() == want.keys(), where
  for k in want:
    wv, wf = want[k]
    assert np.array_equal(got[k].vertices, wv) and np.array_equal(got[k].faces, wf), where + (k,)


@pytest.fixture(scope="module")
def bench_block(oracle):
  # a 129^3 block of the benchmark's mip-2 MeshTask volume: synth_seg pitch 64, seed 0, two 2x2x1 mode mips
  seg = oracle.synth_seg((516, 516, 129), pitch=64, num_ids=1 << 20, seed=0)
  return np.asfortranarray(oracle.downsample_segmentation(seg, (2, 2, 1), num_mips=2)[1].astype(np.uint32))


@pytest.fixture(scope="module")
def class_volume(oracle):
  # 57 labels from 490 to 35,550 faces: 6 fit a 256-thread CTA, 12 a 512-thread one, 39 need the whole SM,
  # and those over 16,384 faces keep their faces in global memory
  return np.asfortranarray(oracle.synth_seg((128, 128, 96), pitch=32, num_ids=64).astype(np.uint32))


def _box(n):
  # a closed box of (n - 2)^3 voxels: its faces in shared memory (n = 30, about 9,400 faces), in global
  # memory with keys, flags and states in shared memory (hybrid, n = 40, about 17,300), or everything in
  # global memory (n = 64, 46,124)
  data = np.zeros((n, n, n), dtype=np.uint32, order="F")
  data[1:-1, 1:-1, 1:-1] = 1
  return data


# ---- Size classes
# k_simp_labels runs each label in the smallest CTA whose shared-memory budget holds it (1024 threads
# alone on an SM, 512 threads two per SM, 256 threads four per SM).  A volume with labels in every size
# class: each class runs, and every mesh is bit-identical to the oracle, with the topology in shared
# memory and on the global-memory path (IGN_SIMP_GMEM=1).

@pytest.mark.parametrize("factor,max_error", [(100, 40.0), (10, 8.0)])
def test_simplify_size_classes_bit_exact(ctx, oracle, class_volume, factor, max_error):
  _, want = _oracle(oracle, "class_volume", class_volume, (16, 16, 40), factor, max_error, True)
  smem, c = _simplify(class_volume, (16, 16, 40), factor, max_error, True)
  rounds, n_smem, n_gmem, n_full, n_half, n_quarter = c[0:6]
  assert n_full > 0 and n_half > 0 and n_quarter > 0, c
  assert n_full + n_half + n_quarter == n_smem + n_gmem == len(want)
  assert n_gmem > 0  # labels over 16,384 faces keep their faces in global memory
  gmem, c_g = _simplify(class_volume, (16, 16, 40), factor, max_error, True, gmem=1)
  assert c_g[1] == 0 and c_g[2] == len(want) and c_g[3:6] == c[3:6], c_g
  _assert_same(smem, want)
  _assert_same(gmem, want)


# ---- Cost format
# The simplifier caches each edge's cost in the format of the label's key.  A label whose 3T half-edge ids fit
# 16 bits (3T <= 65536: 32-bit keys) keeps only the key's 16 cost bits, three per face in one 8-byte word; a
# larger label (64-bit keys) keeps the float costs.  Labels on both sides of the boundary (3T = 65,535 and
# 65,538) run next to a shared-memory label that migrates to smaller size classes, with their topology in
# shared memory / hybrid and with IGN_SIMP_GMEM=1 in global memory; the meshes stay bit-identical to the
# oracle and the key pass never meets an edge without a cost.

def _costfmt_volume(dents):
  # label 1: a 40 x 40 x 119 box in the volume's corner (an open surface: its face count can be odd), with
  # voxels taken out of its corner edges to set the count; label 2: a closed 28^3 box (9,404 faces)
  seg = np.zeros((72, 44, 124), dtype=np.uint32, order="F")
  seg[0:40, 0:40, 0:119] = 1
  for p in dents:
    seg[p] = 0
  seg[42:70, 8:36, 20:48] = 2
  return seg


@pytest.mark.parametrize("factor,max_error", [(100, 40.0), (10, 8.0)])
@pytest.mark.parametrize("dents,three_t", [([(0, 0, 20)], 65535), ([(0, 0, 0), (39, 0, 0)], 65538)])
def test_cost_format_boundary_bit_exact(ctx, oracle, dents, three_t, factor, max_error):
  seg = _costfmt_volume(dents)
  W, want = _oracle(oracle, "costfmt%d" % three_t, seg, (16, 16, 40), factor, max_error, True)
  assert W.ids() == [1, 2]
  assert [int(3 * (b - a)) for a, b in zip(W.f0, W.f1)] == [three_t, 28212]
  for gmem in (None, 1):
    got, c = _simplify(seg, (16, 16, 40), factor, max_error, True, gmem=gmem)
    _assert_same(got, want, gmem)
    assert c[13] == 0, c  # the key pass never meets an edge without a cost
    if gmem:
      assert c[1:3] == [0, 2] and c[6:9] == [0, 0, 0], c
    else:
      # label 1 keeps its faces in global memory (hybrid), label 2 runs in shared memory and migrates
      assert c[1:3] == [1, 1] and c[7] + c[8] > 0, c


# ---- Cached costs
# The simplifier caches the float cost of every edge.  k_simp_ecost costs every edge before the first round,
# and each collapse re-costs the edges of the vertex it moved right after it moved (E2d), so the key pass of a
# round only posts cached keys and never evaluates a cost.  Meshes stay bit-identical to the oracle on the
# benchmark block, on a volume with labels in every size class, and on closed boxes whose flat faces park
# many edges (topology in shared memory, in hybrid and in global memory), also with rounds split into several
# selection passes (IGN_SIMP_WCAP=8).

def _check_costs(oracle, name, seg, res, factor, max_error, centered, wcap):
  W, want = _oracle(oracle, name, seg, res, factor, max_error, centered)
  got, c = _simplify(seg, res, factor, max_error, centered, wcap=wcap)
  _assert_same(got, want)
  # every canonical half-edge (u < v) of the input is costed once before the first round
  f = np.asarray(W.faces, dtype=np.int64).reshape(-1, 3)
  canonical = int((f[:, 0] < f[:, 1]).sum() + (f[:, 1] < f[:, 2]).sum() + (f[:, 2] < f[:, 0]).sum())
  assert c[11] == canonical, (c, canonical)
  assert c[12] > 0, c  # collapses re-cost the edges of the vertices they move
  assert c[13] == 0, c  # the key pass never meets an edge without a cost
  return c


@pytest.mark.parametrize("wcap", [None, 8])
def test_costs_bench_block(ctx, oracle, bench_block, wcap):
  _check_costs(oracle, "bench_block", bench_block, (16, 16, 40), 100, 40.0, True, wcap)


@pytest.mark.parametrize("wcap", [None, 8])
def test_costs_size_classes(ctx, oracle, class_volume, wcap):
  c = _check_costs(oracle, "class_volume", class_volume, (16, 16, 40), 100, 40.0, True, wcap)
  assert min(c[3:6]) > 0 and c[2] > 0, c


@pytest.mark.parametrize("wcap", [None, 8])
@pytest.mark.parametrize("n,smem", [(30, True), (40, False), (64, False)])
def test_costs_box(ctx, oracle, n, smem, wcap):
  c = _check_costs(oracle, "box%d" % n, _box(n), (1, 1, 1), 100, 40.0, False, wcap)
  assert c[1:3] == ([1, 0] if smem else [0, 1]), c


# ---- Flip sides
# E2 of k_simp_labels flip-tests the faces of both rings of a winner that survive the collapse; a flip on
# either side rejects the winner.  The re-costs after a collapse take the kept vertex's new quadric and position
# from the lane group's registers (sl_recost_k) instead of reloading them.  The IGN_SIMP_TRACE summary counts
# the winners rejected by flips on the u side only, the v side only and both.  Meshes stay bit-identical to the
# oracle at every group width (IGN_SIMP_GROUP=8|16|32), and neither the simplifier counters nor the
# rejections depend on the width.

_FLIPS = re.compile(r"winners rejected by E2 flip tests: (\d+) on the u side only, (\d+) on the v side only, (\d+) on both")
_FLIP_RUNS = {}


def _flip_run(oracle, capfd, seg, group):
  """Simplify `seg` at the narrowest group width `group` with the trace on; check every mesh against the
  oracle and return the counters and the flip-test trace (rejected u side only, v side only, both)."""
  if group not in _FLIP_RUNS:
    _, want = _oracle(oracle, "bench_block", seg, (16, 16, 40), 100, 40.0, True)
    capfd.readouterr()
    got, c = _simplify(seg, (16, 16, 40), 100, 40.0, True, group=group, trace=1)
    err = capfd.readouterr().err
    _assert_same(got, want, group)
    lines = _FLIPS.findall(err)
    assert lines, err[-2000:]
    _FLIP_RUNS[group] = (c, [sum(int(x[i]) for x in lines) for i in range(3)])
  return _FLIP_RUNS[group]


@pytest.mark.parametrize("group", [8, 16, 32])
def test_flipsides_bench_block(ctx, oracle, capfd, bench_block, group):
  c, flips = _flip_run(oracle, capfd, bench_block, group)
  ref, ref_flips = _flip_run(oracle, capfd, bench_block, 8)
  assert c[:14] == ref[:14], (group, c, ref)
  assert sum(c[14:]) == sum(ref[14:]), (group, c, ref)
  assert flips == ref_flips, (group, flips, ref_flips)  # the same winners flip, whatever the width
  assert c[12] > 0 and c[13] == 0, c


def test_flipsides_one_sided_rejections(ctx, oracle, capfd, bench_block):
  # winners rejected only by a flip of a u-side face, and only by one of a v-side face
  _, flips = _flip_run(oracle, capfd, bench_block, 8)
  assert flips[0] > 0 and flips[1] > 0, flips


# ---- Lane groups
# E2 of k_simp_labels gives each winner one group of 8 lanes (16 or 32 when a ring holds more than 8 or 16
# faces), which runs its flip tests, link condition, collapse and re-costs with no barrier in between.
# IGN_SIMP_GROUP=16|32 sets the narrowest group, so that the wider sweeps take every winner.  Meshes stay
# bit-identical to the oracle for every group width and selection-pass cap, on shared-memory, hybrid and
# global-memory labels and on labels that migrate between size classes; the counters do not depend on the
# width, and the group counters c[14:17] show which sweeps ran.

GROUPS = (None, 16, 32)


def _groups_run(oracle, name, seg, res, factor, max_error, centered, wcap):
  _, want = _oracle(oracle, name, seg, res, factor, max_error, centered)
  runs = {}
  for g in GROUPS:
    got, c = _simplify(seg, res, factor, max_error, centered, wcap=wcap, group=g)
    _assert_same(got, want, g)
    runs[g] = c
  c = runs[None]
  for g in GROUPS:
    assert runs[g][:14] == c[:14], (g, runs[g], c)
    assert sum(runs[g][14:]) == sum(c[14:]), (g, runs[g], c)  # the same winners, whatever the width
  assert c[14] > 0, c
  assert runs[16][14] == 0 and runs[16][15] > 0, runs[16]
  assert runs[32][14:16] == [0, 0] and runs[32][16] == sum(c[14:]), runs[32]
  return c


@pytest.mark.parametrize("wcap", [None, 8])
def test_groups_bench_block(ctx, oracle, bench_block, wcap):
  c = _groups_run(oracle, "bench_block", bench_block, (16, 16, 40), 100, 40.0, True, wcap)
  assert c[15] + c[16] > 0, c  # rings over 8 faces took the wider sweeps


@pytest.mark.parametrize("wcap", [None, 8])
def test_groups_migrating_labels(ctx, oracle, bench_block, wcap):
  # factor 10: labels shrink into the 512- and 256-thread classes and resume there
  c = _groups_run(oracle, "bench_block", bench_block, (16, 16, 40), 10, 8.0, True, wcap)
  assert c[7] > 0 and c[8] > 0, c


@pytest.mark.parametrize("wcap", [None, 8])
def test_groups_size_classes(ctx, oracle, class_volume, wcap):
  c = _groups_run(oracle, "class_volume", class_volume, (16, 16, 40), 100, 40.0, True, wcap)
  assert min(c[3:6]) > 0 and c[2] > 0, c


@pytest.mark.parametrize("wcap", [None, 8])
@pytest.mark.parametrize("n,memory", [(30, [1, 0]), (40, [0, 1]), (64, [0, 1])])
def test_groups_box(ctx, oracle, n, memory, wcap):
  c = _groups_run(oracle, "box%d" % n, _box(n), (1, 1, 1), 100, 40.0, False, wcap)
  assert c[1:3] == memory, c


# ---- Migration
# A shared-memory label of k_simp_labels whose alive faces and vertices come to fit the next smaller
# size class continues there (1024 -> 512 -> 256 threads): its state is compacted, its faces and vertices
# renumbered, and the keys, cached costs, positions and quadrics are still addressed by the original ids.
# The meshes stay bit-identical to the oracle, and each label still counts once, in the class it started in.

@pytest.mark.parametrize("factor,max_error", [(100, 40.0), (10, 8.0)])
def test_migration_bench_block_bit_exact(ctx, oracle, bench_block, factor, max_error):
  _, want = _oracle(oracle, "bench_block", bench_block, (16, 16, 40), factor, max_error, True)
  got, c = _simplify(bench_block, (16, 16, 40), factor, max_error, True)
  _assert_same(got, want)
  n_full, n_half = c[3], c[4]
  resumed = c[6:9]
  assert c[3] + c[4] + c[5] == c[1] + c[2] == len(want), c
  assert resumed[0] == 0 and resumed[1] > 0 and resumed[2] > 0, c
  assert resumed[1] <= n_full and resumed[2] <= n_full + n_half, c
  if factor == 100:
    # more labels resumed in the 256-thread class than started in the 512-thread one: some of them
    # started in the 1024-thread class and migrated twice
    assert resumed[2] > n_half, c


@pytest.mark.parametrize("factor,max_error", [(100, 40.0), (10, 8.0)])
def test_migration_size_class_volume_bit_exact(ctx, oracle, class_volume, factor, max_error):
  # labels in every class, and over 16,384 faces (global-memory path, which never migrates)
  _, want = _oracle(oracle, "class_volume", class_volume, (16, 16, 40), factor, max_error, True)
  got, c = _simplify(class_volume, (16, 16, 40), factor, max_error, True)
  _assert_same(got, want)
  assert c[6] == 0 and c[7] + c[8] > 0, c
  assert c[7] <= c[3] - c[2], c  # only shared-memory labels of the full class
  got_g, c_g = _simplify(class_volume, (16, 16, 40), factor, max_error, True, gmem=1)
  _assert_same(got_g, want)
  assert c_g[6:9] == [0, 0, 0] and c_g[3:6] == c[3:6], (c_g, c)


# ---- Winner capacity
# k_simp_labels validates the winners of a round in as few passes as the label's shared memory allows: a
# shared-memory label takes as many winners per pass as its size class's budget leaves room for, and a round
# with more winners than that runs further passes.  IGN_SIMP_WCAP=n caps the winners per pass so that the
# extra passes run on any volume.  The meshes are bit-identical to the oracle whatever the cap, in shared
# and in global memory, and the cap never changes the class a label runs in.

@pytest.mark.parametrize("volume", ["bench_block", "class_volume"])
@pytest.mark.parametrize("gmem", [False, True])
def test_winner_capacity_bit_exact(ctx, oracle, request, volume, gmem):
  seg = request.getfixturevalue(volume)
  _, want = _oracle(oracle, volume, seg, (16, 16, 40), 100, 40.0, True)
  gmem = 1 if gmem else None
  got, c = _simplify(seg, (16, 16, 40), 100, 40.0, True, gmem=gmem)
  _assert_same(got, want)
  multi = {}
  for cap in (8, 32):
    got_c, c_c = _simplify(seg, (16, 16, 40), 100, 40.0, True, gmem=gmem, wcap=cap)
    _assert_same(got_c, want, cap)
    assert c_c[:6] == c[:6], (cap, c_c, c)  # the cap changes no label's class or memory path
    # winners rejected for a ring over 32 faces are the same ones whatever the cap
    assert c_c[10] == c[10], (cap, c_c, c)
    multi[cap] = c_c[9]
  # a smaller cap splits more rounds, and the default capacity splits fewer than either
  assert multi[8] >= multi[32] > c[9], (multi, c)
