"""Hashed label shards on the GPU: ign_shard_hash_dev bit for bit against the pure-Python restatement,
ign_skeleton_restrip_dev against a numpy re-encoding, and SkeletonTask -> UnshardedSkeletonMergeTask ->
create_sharded_skeletons_from_unsharded_tasks -> LocalTaskQueue end to end, read back with this file's own
numpy shard reader and with vol.skeleton.get."""
import gzip
import struct

import numpy as np
import pytest

from igneous_b200 import labelshard
from igneous_b200 import task_creation as tc
from igneous_b200._compat import CloudFiles, CloudVolume, LocalTaskQueue
from igneous_b200.sharding import murmurhash3_x86_128_u64
from test_label_shards import EDGES, locate, random_labels

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("preshift,mb,sb", [(0, 0, 0), (0, 9, 0), (0, 0, 11), (3, 6, 5), (0, 32, 32), (5, 2, 9)])
def test_hash_kernel_matches_the_restatement(ctx, preshift, mb, sb):
  labels = np.concatenate([np.array(EDGES, dtype=np.uint64), random_labels(3000, seed=sb)])
  got, loc, starts, shards = labelshard.shard_hash(labels, preshift, mb, sb, ctx)
  want = sorted(((*locate(l, preshift, mb, sb), l) for l in labels.tolist()))
  assert got.tolist() == [w[2] for w in want]
  assert loc.tolist() == [(s << mb) | m for s, m, _ in want]
  wshards = sorted({w[0] for w in want})
  assert shards.tolist() == wshards
  assert starts.tolist() == [next(i for i, w in enumerate(want) if w[0] == s) for s in wshards] + [len(want)]


def test_hash_kernel_on_a_million_labels(ctx):
  labels = random_labels(10 ** 6, seed=9)
  got, loc, starts, shards = labelshard.shard_hash(labels, 0, 9, 1, ctx)
  # every location bit for bit: the kernel's hash of each sorted label against the restatement on a sample,
  # and against the host hash (itself checked against the restatement) on all of them
  h = murmurhash3_x86_128_u64(got) & np.uint64((1 << 10) - 1)
  assert np.array_equal(loc, h)
  for i in np.random.default_rng(0).integers(0, 10 ** 6, 20000).tolist():
    s, m = locate(int(got[i]), 0, 9, 1)
    assert int(loc[i]) == (s << 9) | m
  assert np.array_equal(np.sort(got), np.sort(labels))
  key = loc.astype(object) * (1 << 64) + got.astype(object)
  assert all(a <= b for a, b in zip(key[:-1], key[1:]))
  assert shards.tolist() == [0, 1] and starts[0] == 0 and starts[-1] == 10 ** 6
  assert int(starts[1]) == int(np.count_nonzero(loc < np.uint64(512)))


def test_hash_kernel_no_labels(ctx):
  got, loc, starts, shards = labelshard.shard_hash(np.zeros(0, np.uint64), 0, 3, 3, ctx)
  assert got.size == loc.size == shards.size == 0 and starts.tolist() == [0]


# ------------------------------------------------------------------------ restrip
def blob(rng, nv, ne, attrs):
  parts = [struct.pack("<II", nv, ne), rng.normal(size=(nv, 3)).astype(np.float32).tobytes(),
           rng.integers(0, max(nv, 1), (ne, 2)).astype(np.uint32).tobytes()]
  sections = []
  for a in attrs:
    dt = np.dtype(a["data_type"])
    vals = rng.integers(0, 250, nv * a["num_components"]).astype(dt) if dt.kind in "ui" else \
        rng.normal(size=nv * a["num_components"]).astype(dt)
    sections.append(vals.tobytes())
  return b"".join(parts + sections), parts, sections


def numpy_restrip(parts, sections, attrs):
  return b"".join(parts + [s for s, a in zip(sections, attrs) if a["data_type"] in ("float32", "float64")])


ORDERS = [
  [{"id": "radius", "data_type": "float32", "num_components": 1},
   {"id": "vertex_types", "data_type": "uint8", "num_components": 1}],
  [{"id": "vertex_types", "data_type": "uint8", "num_components": 1},
   {"id": "radius", "data_type": "float32", "num_components": 1}],
  [{"id": "a", "data_type": "uint16", "num_components": 3},
   {"id": "thick", "data_type": "float64", "num_components": 2},
   {"id": "b", "data_type": "int32", "num_components": 1},
   {"id": "radius", "data_type": "float32", "num_components": 1}],
  [],
]


@pytest.mark.parametrize("attrs", ORDERS)
def test_restrip_matches_numpy(ctx, attrs):
  rng = np.random.default_rng(len(attrs))
  sizes = [(0, 0), (1, 0), (5, 4), (300, 299), (2, 7)] + [(int(n), int(rng.integers(0, n + 1))) for n in
                                                         rng.integers(0, 200, 200)]
  made = [blob(rng, nv, ne, attrs) for nv, ne in sizes]
  buf, offs = labelshard.restrip([m[0] for m in made], attrs, ctx=ctx)
  want = [numpy_restrip(m[1], m[2], attrs) for m in made]
  assert offs.tolist() == np.r_[0, np.cumsum([len(w) for w in want])].tolist()
  assert buf.tobytes() == b"".join(want)


def test_restrip_refuses_a_short_blob_naming_its_row(ctx):
  attrs = ORDERS[2]
  rng = np.random.default_rng(3)
  blobs = [blob(rng, 10, 9, attrs)[0] for _ in range(6)]
  blobs[4] = blobs[4][:-1]
  with pytest.raises(ValueError, match="row 4"):
    labelshard.restrip(blobs, attrs, ctx=ctx)
  with pytest.raises(ValueError, match="row 0"):
    labelshard.restrip([b"\x01\x00\x00"], attrs, ctx=ctx)


# ------------------------------------------------------------------------ end to end
def read_shard(data, index_encoding, data_encoding, minishard_bits):
  """{label: blob} of a whole shard file, from the published layout"""
  n = 16 << minishard_bits
  index = np.frombuffer(data[:n], "<u8").reshape(-1, 2)
  out = {}
  for start, end in index.tolist():
    if end == start:
      continue
    raw = data[n + start:n + end]
    raw = gzip.decompress(raw) if index_encoding == "gzip" else raw
    t = np.frombuffer(raw, "<u8").reshape(3, -1).astype(object)
    label, pos = 0, 0
    for d_id, d_start, size in zip(*t):
      label += d_id
      pos += d_start
      b = data[n + pos:n + pos + size]
      out[int(label)] = gzip.decompress(b) if data_encoding == "gzip" else b
      pos += size
  return out


def many_objects(seed, count):
  """count small bars, each its own label (some above 2^32), in a 96 x 96 x 48 volume"""
  rng = np.random.default_rng(seed)
  img = np.zeros((96, 96, 48), np.uint64)
  cells = [(x, y, z) for x in range(12) for y in range(12) for z in range(6)]
  labels = rng.choice(np.arange(1, 10 ** 6), count, replace=False).astype(np.uint64)
  labels[::7] += np.uint64(1 << 40)
  for (x, y, z), lab in zip([cells[i] for i in rng.permutation(len(cells))[:count]], labels):
    img[8 * x + 1:8 * x + 7, 8 * y + 3:8 * y + 6, 8 * z + 3:8 * z + 6] = lab
  return np.asfortranarray(img), sorted(int(l) for l in labels)


@pytest.mark.parametrize("data_encoding,index_encoding", [("gzip", "gzip"), ("raw", "raw"), ("raw", "gzip"),
                                                          ("gzip", "raw")])
def test_end_to_end(ctx, tmp_path, data_encoding, index_encoding):
  path = "file://" + str(tmp_path / "seg")
  img, labels = many_objects(0, 300)
  CloudVolume.from_numpy(img, path, resolution=(16, 16, 40), chunk_size=(48, 48, 48), layer_type="segmentation")
  LocalTaskQueue().insert(tc.create_skeletonizing_tasks(path, mip=0, shape=(48, 48, 48),
                                                        teasar_params={"scale": 4, "const": 50}, dust_threshold=0))
  vol = CloudVolume(path)
  vol.skeleton.meta.info["vertex_attributes"].append({"id": "vertex_types", "data_type": "uint8",
                                                      "num_components": 1})
  vol.skeleton.meta.commit_info()
  LocalTaskQueue().insert(tc.create_unsharded_skeleton_merge_tasks(path, magnitude=1, dust_threshold=0,
                                                                   tick_threshold=0))
  src = CloudVolume(path)
  assert [a["id"] for a in src.skeleton.meta.info["vertex_attributes"]] == ["radius", "vertex_types"]
  source = {l: src.skeleton.get(l) for l in labels}
  made = tc.create_sharded_skeletons_from_unsharded_tasks(path, path, shard_index_bytes=64, minishard_index_bytes=192,
                                                          data_encoding=data_encoding,
                                                          minishard_index_encoding=index_encoding,
                                                          skel_dir="skeletons_sharded")
  assert len(made) >= 8
  LocalTaskQueue().insert(made)
  dest = CloudVolume(path, skel_dir="skeletons_sharded")
  info = dest.skeleton.meta.info
  mb = info["sharding"]["minishard_bits"]
  assert mb == 2 and info["sharding"]["shard_bits"] == 4
  assert [a["id"] for a in info["vertex_attributes"]] == ["radius"]
  cf = CloudFiles(dest.skeleton.path)
  shards = [n for n in cf.list() if n.endswith(".shard")]
  assert len(shards) == len(made)
  got = {}
  minis = set()
  for name in shards:
    data = cf.get(name)
    part = read_shard(data, index_encoding, data_encoding, mb)
    assert not set(part) & set(got)
    got.update(part)
    index = np.frombuffer(data[:16 << mb], "<u8").reshape(-1, 2)
    minis |= {(name, m) for m, (a, b) in enumerate(index.tolist()) if b > a}
  assert len(minis) > len(shards)  # several minishards per shard
  assert sorted(got) == labels
  for l, s in source.items():
    b = np.frombuffer(got[l], np.uint8)
    nv, ne = (int(v) for v in b[:8].view(np.uint32))
    assert len(got[l]) == 8 + 16 * nv + 8 * ne
    assert b[8:8 + 12 * nv].tobytes() == s.vertices.tobytes()
    assert b[8 + 12 * nv:8 + 12 * nv + 8 * ne].tobytes() == s.edges.tobytes()
    assert b[8 + 12 * nv + 8 * ne:].tobytes() == s.radii.tobytes()
    r = dest.skeleton.get(l)
    assert r.vertices.tobytes() == s.vertices.tobytes() and r.edges.tobytes() == s.edges.tobytes()
    assert r.radii.tobytes() == s.radii.tobytes() and not r.vertex_types.any()
