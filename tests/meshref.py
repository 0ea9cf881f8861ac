"""A plain numpy/scipy checker of the mesh simplifier's contract (DESIGN.md §5), sharing no code with
oracle/.  It takes the welded marching-cubes meshes of a task, the simplified meshes, the surviving vertex
each input vertex was collapsed into, and the parameters, and checks every label at once:

- the output is a valid indexed mesh: indices in range, every vertex used, no face repeats a vertex and
  no two faces have the same vertex set;
- every edge is used at most twice, an interior edge once in each direction (consistent winding), and
  every vertex's link is one cycle or one path wherever the input's links all are;
- per label, the multiset of connected components by (Euler characteristic, boundary loops) is kept;
- the boundary edges, as pairs of float32 positions, are kept bit for bit (chunks still stitch);
- every closed component encloses a non-zero volume of the sign of the input component it came from;
- no label grows, and each reaches its target face count unless its simplification stopped;
- max_error: the plane quadrics (float64, unit normals, degenerate faces skipped) of the input
  vertices merged into a surviving vertex, evaluated at its position, stay within max_error^2.  Every
  collapse checks that bound on the summed quadric at the new position, and later collapses only add
  to it, so the final sums are bounded too.
"""
import numpy as np
from scipy import sparse
from scipy.sparse import csgraph


class Concat:
  """Meshes of several labels in one vertex and face list."""

  def __init__(self, meshes, labels):
    vs, fs, vl, fl = [], [], [], []
    self.voff = {}
    n = 0
    for lab in labels:
      v, f = meshes[lab]
      f = np.asarray(f, dtype=np.int64).reshape(-1, 3)
      assert f.size == 0 or (f.min() >= 0 and f.max() < len(v)), ("face index out of range", lab)
      self.voff[lab] = n
      vs.append(np.asarray(v, dtype=np.float32).reshape(-1, 3))
      fs.append(f + n)
      vl.append(np.full(len(v), lab, dtype=np.uint64))
      fl.append(np.full(len(f), lab, dtype=np.uint64))
      n += len(v)
    self.v32 = np.concatenate(vs) if vs else np.zeros((0, 3), np.float32)
    self.v = self.v32.astype(np.float64)
    self.f = np.concatenate(fs) if fs else np.zeros((0, 3), np.int64)
    self.vlab = np.concatenate(vl) if vl else np.zeros(0, np.uint64)
    self.flab = np.concatenate(fl) if fl else np.zeros(0, np.uint64)
    self.V = n
    f = self.f
    self.he = np.stack([f, np.roll(f, -1, axis=1)], axis=2).reshape(-1, 2)   # directed half-edges
    und = np.sort(self.he, axis=1)
    key = und[:, 0] * max(n, 1) + und[:, 1]
    self.ekey, self.einv, self.euse = np.unique(key, return_inverse=True, return_counts=True)
    self.e = np.stack([self.ekey // max(n, 1), self.ekey % max(n, 1)], axis=1)  # undirected edges
    self.bedge = self.e[self.euse == 1]                                        # boundary edges

  def components(self):
    """Vertex components (scipy connected components over the edges): (count, component of each vertex)."""
    g = sparse.coo_matrix((np.ones(len(self.e)), (self.e[:, 0], self.e[:, 1])), shape=(self.V, self.V))
    return csgraph.connected_components(g, directed=False)

  def link_ok(self):
    """Per vertex: its link (the opposite edges of its faces) is connected.  Nodes are (vertex, link
    vertex) pairs, joined by each face's opposite edge."""
    f, n = self.f, max(self.V, 1)
    w = f.reshape(-1)
    x = np.roll(f, -1, axis=1).reshape(-1)
    y = np.roll(f, -2, axis=1).reshape(-1)
    keys, inv = np.unique(np.concatenate([w * n + x, w * n + y]), return_inverse=True)
    a, b = inv[:len(w)], inv[len(w):]
    g = sparse.coo_matrix((np.ones(len(a)), (a, b)), shape=(len(keys), len(keys)))
    nc, comp = csgraph.connected_components(g, directed=False)
    pairs = np.unique(keys // n * nc + comp)  # (vertex, link component)
    nlink = np.bincount(pairs // nc, minlength=self.V)
    return nlink <= 1

  def signed_volume(self, comp, ncomp):
    a, b, c = (self.v[self.f[:, k]] for k in range(3))
    vol = np.einsum("ij,ij->i", a, np.cross(b, c)) / 6.0
    return np.bincount(comp[self.f[:, 0]], weights=vol, minlength=ncomp) if len(self.f) else np.zeros(ncomp)


def _labels_where(mask, labs):
  return sorted({int(l) for l in np.asarray(labs)[mask]})


def _component_table(m, comp, ncomp):
  """(label, Euler characteristic, boundary loops) of each component."""
  nv = np.bincount(comp, minlength=ncomp)
  ne = np.bincount(comp[m.e[:, 0]], minlength=ncomp)
  nf = np.bincount(comp[m.f[:, 0]], minlength=ncomp) if len(m.f) else np.zeros(ncomp, np.int64)
  chi = nv - ne + nf
  loops = np.zeros(ncomp, np.int64)
  if len(m.bedge):
    bv, binv = np.unique(m.bedge, return_inverse=True)
    binv = binv.reshape(-1, 2)
    g = sparse.coo_matrix((np.ones(len(binv)), (binv[:, 0], binv[:, 1])), shape=(len(bv), len(bv)))
    nb, bcomp = csgraph.connected_components(g, directed=False)
    first = np.zeros(nb, np.int64)
    first[bcomp] = bv   # any vertex of each boundary loop
    loops = np.bincount(comp[first], minlength=ncomp)
  lab = np.zeros(ncomp, np.uint64)
  lab[comp] = m.vlab
  return lab, chi, loops


def _boundary_rows(m):
  """Boundary edges as rows (label, float32 bits of both endpoints, the smaller endpoint first)."""
  bits = m.v32.view(np.uint32).astype(np.uint64)
  p, q = bits[m.bedge[:, 0]], bits[m.bedge[:, 1]]
  order = _lex_less(q, p)
  lo = np.where(order[:, None], q, p)
  hi = np.where(order[:, None], p, q)
  rows = np.concatenate([m.vlab[m.bedge[:, 0]][:, None], lo, hi], axis=1)
  return rows[np.lexsort(rows.T[::-1])] if len(rows) else rows


def _lex_less(a, b):
  """Row-wise a < b, lexicographically."""
  less = np.zeros(len(a), bool)
  eq = np.ones(len(a), bool)
  for k in range(a.shape[1]):
    less |= eq & (a[:, k] < b[:, k])
    eq &= a[:, k] == b[:, k]
  return less


def check_simplified(before, after, rep, targets, max_error, stopped, volume=True):
  """Assert the simplifier's contract on every label.  before / after: {label: (vertices f32 [N, 3],
  faces [M, 3])}, the welded input and the simplified output, in the same physical units and frame;
  rep: {label: index of the output vertex each input vertex ended in}; targets: {label: target face
  count}; stopped: labels may have stopped above their target (the run ended by its stop rule rather
  than a round cap); volume=False skips the volume of closed components.  Returns the total output face
  count."""
  labels = sorted(before)
  assert sorted(after) == labels, "label sets differ"
  A, B = Concat(before, labels), Concat(after, labels)
  R = np.concatenate([np.asarray(rep[l], dtype=np.int64) + B.voff[l] for l in labels]) if labels else np.zeros(0, np.int64)
  assert len(R) == A.V and (R >= 0).all() and (R < max(B.V, 1)).all(), "rep out of range"
  assert (B.vlab[R] == A.vlab).all(), "rep crosses labels"

  # a valid indexed mesh
  used = np.bincount(B.f.reshape(-1), minlength=B.V) > 0
  assert used.all(), ("unused output vertices", _labels_where(~used, B.vlab))
  f = B.f
  rep_v = (f[:, 0] == f[:, 1]) | (f[:, 1] == f[:, 2]) | (f[:, 2] == f[:, 0])
  assert not rep_v.any(), ("face repeats a vertex", _labels_where(rep_v, B.flab))
  n = max(B.V, 1)
  assert n < 1 << 21
  s = np.sort(f, axis=1)
  _, inv, cnt = np.unique((s[:, 0] * n + s[:, 1]) * n + s[:, 2], return_inverse=True, return_counts=True)
  dup = cnt[inv.reshape(-1)] > 1
  assert not dup.any(), ("coincident faces (same vertex set)", _labels_where(dup, B.flab))

  # edge use and winding; vertex links where the input's are manifold
  over_in = np.array(_labels_where(A.euse > 2, A.vlab[A.e[:, 0]]), dtype=np.uint64)
  over = (B.euse > 2) & ~np.isin(B.vlab[B.e[:, 0]], over_in)
  assert not over.any(), ("edge used more than twice", _labels_where(over, B.vlab[B.e[:, 0]]))
  _, hinv, hcnt = np.unique(B.he[:, 0] * max(B.V, 1) + B.he[:, 1], return_inverse=True, return_counts=True)
  twice = (hcnt[hinv.reshape(-1)] > 1) & ~np.isin(B.vlab[B.he[:, 0]], over_in)
  assert not twice.any(), ("inconsistent winding: a directed edge is used twice", _labels_where(twice, B.vlab[B.he[:, 0]]))
  bad_in = np.union1d(np.array(_labels_where(~A.link_ok(), A.vlab), dtype=np.uint64), over_in)
  bad = ~B.link_ok() & ~np.isin(B.vlab, bad_in)
  assert not bad.any(), ("vertex link is not one cycle or path", _labels_where(bad, B.vlab))

  # components by (Euler characteristic, boundary loops), matched through rep
  nca, ca = A.components()
  ncb, cb = B.components()
  ta, tb = _component_table(A, ca, nca), _component_table(B, cb, ncb)
  pairs = np.unique(np.stack([ca, cb[R]], axis=1), axis=0)
  assert len(pairs) == nca == ncb, ("components merged or split", nca, ncb, len(pairs))
  ia, ib = pairs[:, 0], pairs[:, 1]
  for t in range(3):
    diff = ta[t][ia] != tb[t][ib]
    assert not diff.any(), ("component (label, Euler characteristic, boundary loops) changed",
                            [(int(ta[0][i]), int(ta[1][i]), int(ta[2][i]), int(tb[1][j]), int(tb[2][j]))
                             for i, j in zip(ia[diff], ib[diff])][:10])

  # boundary edges, bit for bit
  ra, rb = _boundary_rows(A), _boundary_rows(B)
  assert ra.shape == rb.shape and np.array_equal(ra, rb), ("boundary edges moved", len(ra), len(rb))

  # closed components keep a non-zero volume of the input's sign
  va, vb = A.signed_volume(ca, nca), B.signed_volume(cb, ncb)
  closed = ta[2][ia] == 0
  wrong = closed & ~(np.sign(va[ia]) * vb[ib] > 0) & volume
  assert not wrong.any(), ("closed component lost its volume", [(int(ta[0][i]), float(va[i]), float(vb[j]))
                                                                for i, j in zip(ia[wrong], ib[wrong])][:10])

  # face counts
  for lab in labels:
    n0, n1 = len(before[lab][1]), len(after[lab][1])
    assert n1 <= n0, ("label grew", lab, n0, n1)
    assert n1 <= targets[lab] or stopped, ("label above its target", lab, n1, targets[lab])

  # max_error: sum over the input corners merged into each surviving vertex k of the squared distance of
  # k's position to the corner's face plane (= p^T (sum of plane quadrics) p)
  a, b, c = (A.v[A.f[:, k]] for k in range(3))
  nrm = np.cross(b - a, c - a)
  ln = np.sqrt((nrm * nrm).sum(axis=1))
  ok = ln > 0
  nrm = nrm[ok] / ln[ok, None]
  d = -(nrm * a[ok]).sum(axis=1)
  corners = A.f[ok]
  k = R[corners.reshape(-1)]
  n3 = np.repeat(nrm, 3, axis=0)
  d3 = np.repeat(d, 3)
  p = B.v[k]
  r = (n3 * p).sum(axis=1) + d3
  cost = np.bincount(k, weights=r * r, minlength=B.V)
  # slack: the output positions are float32 roundings (off by at most one float32 ulp per coordinate), and
  # the simplifier evaluates p^T Q p in float64 from terms of size about (|n.p| + |d|)^2
  ulp = np.linalg.norm(np.spacing(np.abs(B.v32)).astype(np.float64), axis=1)
  slack = np.bincount(k, weights=2.0 * np.abs(r) * ulp[k] + ulp[k] ** 2, minlength=B.V)
  mag = np.bincount(k, weights=(np.abs((n3 * p)).sum(axis=1) + np.abs(d3)) ** 2, minlength=B.V)
  tol = slack + 1e-12 * mag
  over_err = cost - tol > float(max_error) ** 2
  assert not over_err.any(), ("max_error exceeded", _labels_where(over_err, B.vlab),
                              float(np.max(cost[over_err])), float(max_error) ** 2)
  return len(B.f)
