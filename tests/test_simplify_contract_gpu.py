"""The simplifier's contract (tests/meshref.py) on the GPU: the volumes of test_simplify_contract.py go through
zmesh.Mesher on the default path and on the paths IGN_SIMP_GMEM=1 (topology in global memory),
IGN_SIMP_WCAP=8 (rounds split into selection passes of 8 winners) and IGN_SIMP_GROUP=32 (every winner in a
32-lane group) force.  Every mesh is bit-identical to the oracle's and meets the contract, with the oracle's
rep (the surviving vertex of each input vertex) standing for the GPU's; the counters show that each path ran."""
import numpy as np
import pytest

import test_simplify_contract as C
from meshref import check_simplified
from test_simplify_gpu import _simplify

pytestmark = pytest.mark.gpu

# (volume, parameters, check the volume of closed components): see test_simplify_contract.py
CASES = [("bench_block", C.BENCH, True), ("class_volume", C.GRID[5], True), ("tiny_closed", C.GRID[3], False),
         ("tiny_closed", C.GRID[4], True), ("holes", C.GRID[2], True), ("noise", C.GRID[6], False),
         ("noise", C.GRID[1], True)] + [("cut_by_%d" % k, C.GRID[k % 2 + 6], True) for k in range(1, 7)]
PATHS = [{}, {"gmem": 1}, {"wcap": 8}, {"group": 32}]

_VOLUMES, _ORACLE = {}, {}


def _volume(oracle, name):
  if name not in _VOLUMES:
    if name.startswith("cut_by_"):
      _VOLUMES[name] = C.cut_by(int(name[7:]))
    elif name in ("bench_block", "class_volume"):
      _VOLUMES[name] = getattr(C, name)(oracle)
    else:
      _VOLUMES[name] = getattr(C, name)()
  return _VOLUMES[name]


def _oracle(oracle, name, params):
  key = (name, params)
  if key not in _ORACLE:
    factor, max_error, res, centered = params
    tl, tv = oracle.marching_cubes(_volume(oracle, name))
    W = oracle.WeldedMeshes(tl, tv)
    want, _, rep = oracle.simplify_welded(W, res, factor, max_error, centered, C.MAX_ROUNDS, with_rep=True)
    before = {l: W.get(l, res, centered) for l in W.ids()}
    targets = {l: len(before[l][1]) // factor for l in W.ids()}
    _ORACLE[key] = (want, rep, before, targets)
  return _ORACLE[key]


@pytest.mark.parametrize("path", PATHS, ids=["default", "gmem", "wcap8", "group32"])
@pytest.mark.parametrize("name,params,volume", CASES)
def test_contract_gpu(ctx, oracle, name, params, volume, path):
  factor, max_error, res, centered = params
  want, rep, before, targets = _oracle(oracle, name, params)
  got, c = _simplify(_volume(oracle, name), res, factor, max_error, centered, **path)
  assert got.keys() == want.keys()
  for k in want:
    assert np.array_equal(got[k].vertices, want[k][0]) and np.array_equal(got[k].faces, want[k][1]), (path, k)
  after = {k: (m.vertices, m.faces) for k, m in got.items()}
  check_simplified(before, after, rep, targets, max_error, c[0] < C.MAX_ROUNDS, volume)
  n = len(want)
  assert c[1] + c[2] == c[3] + c[4] + c[5] == n, c
  assert c[13] == 0, c  # the key pass never meets an edge without a cached cost
  if path.get("gmem"):
    assert c[1:3] == [0, n] and c[6:9] == [0, 0, 0], c
  if path.get("group") == 32:
    assert c[14:16] == [0, 0] and c[16] > 0, c
  if path.get("wcap") and name in ("bench_block", "class_volume"):
    assert c[9] > 0, c  # rounds with more than 8 winners took several passes
  if name == "class_volume":
    assert min(c[3:6]) > 0, c  # every size class ran
  if name == "noise":
    assert n > 3000 and c[5] == n, c  # thousands of labels, all in the 256-thread class
