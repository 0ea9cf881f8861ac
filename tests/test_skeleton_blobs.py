"""The host splitter of packed neuroglancer precomputed skeletons (kimimaro.split_blobs) on the serial C
checker's merge output (oracle_skeleton/merge_oracle.c): every blob re-encoded by the numpy restatement
(tests/skelmergeref.py), and every array a view into the buffer.  No GPU."""
import numpy as np
import pytest

import oracle_skeleton as C
import skelmergeref as R
from igneous_b200 import kimimaro
from test_skelmergeref import random_batch


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("vertex_types", [True, False])
@pytest.mark.parametrize("dust", [0, 200])
def test_split_matches_restatement(seed, vertex_types, dust):
  batch = random_batch(seed, labels=12)
  segids, packed = kimimaro.pack_fragments(batch)
  buf, table = C.merge(packed, dust, 0, None, vertex_types)
  attrs = kimimaro.ATTRIBUTES[:2 if vertex_types else 1]
  skeletons, blobs = kimimaro.split_blobs(buf, table[:, 1:], segids, attrs)
  assert [s.id for s in skeletons] == segids and len(blobs) == len(segids)
  if dust:
    assert any(s.empty() for s in skeletons)
  for s, blob, (_, off, nv, ne) in zip(skeletons, blobs, table.tolist()):
    assert s.vertices.shape == (nv, 3) and s.edges.shape == (ne, 2) and s.radii.shape == s.vertex_types.shape == (nv,)
    assert s.vertices.dtype == s.radii.dtype == np.float32 and s.edges.dtype == np.uint32
    assert s.vertex_types.dtype == np.uint8
    assert blob.tobytes() == R.encode((s.vertices, s.edges, s.radii, s.vertex_types), vertex_types)
    assert blob.tobytes() == buf[off:off + blob.size].tobytes()
    for a in (s.vertices, s.edges, s.radii, blob) + ((s.vertex_types,) if vertex_types else ()):
      assert np.shares_memory(a, buf) or a.size == 0
    if not vertex_types:
      assert not np.shares_memory(s.vertex_types, buf) and not s.vertex_types.any()
  if not vertex_types:  # the zeros of different skeletons are different memory
    z = [s.vertex_types for s in skeletons if s.vertex_types.size]
    assert not any(np.shares_memory(a, b) for a, b in zip(z, z[1:]))


def test_split_attributes_in_any_order():
  """a uint8 attribute before a float32 one, a 3-component attribute, and a blob past the buffer's end"""
  rng = np.random.default_rng(3)
  v = rng.normal(size=(5, 3)).astype(np.float32)
  e = np.array([[0, 1], [1, 2], [3, 4]], np.uint32)
  t, r, n = np.arange(5, dtype=np.uint8), rng.random(5).astype(np.float32), rng.random((5, 3)).astype(np.float32)
  data = np.frombuffer(bytearray(np.array([5, 3], "<u4").tobytes() + v.tobytes() + e.tobytes() + t.tobytes() +
                                 r.tobytes() + n.tobytes()), np.uint8)
  attrs = kimimaro.ATTRIBUTES[::-1] + [{"id": "normal", "data_type": "float32", "num_components": 3}]
  (s,), (blob,) = kimimaro.split_blobs(data, [(0, 5, 3)], [9], attrs)
  assert s.id == 9 and blob.size == data.size
  assert np.array_equal(s.vertices, v) and np.array_equal(s.edges, e)
  assert np.array_equal(s.vertex_types, t) and np.array_equal(s.radii, r)
  assert np.shares_memory(s.radii, data) and s.radii.flags.writeable
  with pytest.raises(ValueError, match="past the"):
    kimimaro.split_blobs(data[:-1], [(0, 5, 3)], [9], attrs)
