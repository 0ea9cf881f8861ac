"""Hashed label shards on the host: murmurhash3_x86_128 against a byte-oriented pure-Python restatement, a
hashed shard synthesized and read back, and compute_shard_params_for_hashed (no GPU)."""
import gzip

import numpy as np
import pytest

from igneous_b200.sharding import LabelShardingSpecification, ShardingSpecification, murmurhash3_x86_128_u64
from igneous_b200.task_creation import compute_shard_params_for_hashed

M32 = 0xFFFFFFFF


def rotl(x, r):
  return ((x << r) | (x >> (32 - r))) & M32


def fmix(h):
  h ^= h >> 16
  h = (h * 0x85EBCA6B) & M32
  h ^= h >> 13
  h = (h * 0xC2B2AE35) & M32
  return h ^ (h >> 16)


def murmur3_x86_128(data, seed=0):
  """MurmurHash3_x86_128 of a byte string, as four 32-bit words, restated from the published algorithm"""
  c = (0x239B961B, 0xAB0E9789, 0x38B34AE5, 0xA1E38B93)
  rot_k, rot_h = (15, 16, 17, 18), (19, 17, 15, 13)
  add = (0x561CCD1B, 0x0BCAA747, 0x96CD1C35, 0x32AC3B17)
  h = [seed] * 4
  nblocks = len(data) // 16
  for b in range(nblocks):
    k = [int.from_bytes(data[16 * b + 4 * i:16 * b + 4 * i + 4], "little") for i in range(4)]
    for i in range(4):
      ki = (k[i] * c[i]) & M32
      ki = rotl(ki, rot_k[i])
      ki = (ki * c[(i + 1) % 4]) & M32
      h[i] ^= ki
      h[i] = rotl(h[i], rot_h[i])
      h[i] = (h[i] + h[(i + 1) % 4]) & M32
      h[i] = (h[i] * 5 + add[i]) & M32
  tail = data[16 * nblocks:]
  for i in range(4):
    chunk = tail[4 * i:4 * i + 4]
    if chunk:
      ki = int.from_bytes(chunk, "little")
      ki = (ki * c[i]) & M32
      ki = rotl(ki, rot_k[i])
      ki = (ki * c[(i + 1) % 4]) & M32
      h[i] ^= ki
  h = [x ^ len(data) for x in h]
  h[0] = (h[0] + h[1] + h[2] + h[3]) & M32
  for i in (1, 2, 3):
    h[i] = (h[i] + h[0]) & M32
  h = [fmix(x) for x in h]
  h[0] = (h[0] + h[1] + h[2] + h[3]) & M32
  for i in (1, 2, 3):
    h[i] = (h[i] + h[0]) & M32
  return h


def locate(label, preshift, mb, sb):
  h = murmur3_x86_128((label >> preshift).to_bytes(8, "little"))
  h64 = h[0] | (h[1] << 32)
  return (h64 >> mb) & ((1 << sb) - 1), h64 & ((1 << mb) - 1)


EDGES = [0, 1, 2 ** 32 - 1, 2 ** 32, 2 ** 63, 2 ** 64 - 1]


def random_labels(n, seed=0):
  rng = np.random.default_rng(seed)
  return rng.integers(0, 2 ** 64 - 1, size=n, dtype=np.uint64, endpoint=True)


def test_restatement_on_longer_keys_is_consistent():
  # the empty key with seed 0 hashes to zero; keys of every tail length and whole blocks run without error
  assert murmur3_x86_128(b"") == [0, 0, 0, 0]
  assert len({tuple(murmur3_x86_128(bytes(range(n)))) for n in range(40)}) == 40


def test_host_hash_matches_the_restatement():
  labels = np.concatenate([np.array(EDGES, dtype=np.uint64), random_labels(100000)])
  got = murmurhash3_x86_128_u64(labels)
  for lab, h in zip(labels.tolist(), got.tolist()):
    w = murmur3_x86_128(int(lab).to_bytes(8, "little"))
    assert h == w[0] | (w[1] << 32), lab


@pytest.mark.parametrize("preshift,mb,sb", [(0, 0, 0), (0, 9, 0), (0, 0, 11), (3, 6, 5), (17, 2, 1), (0, 32, 32)])
def test_locate_matches_the_restatement(preshift, mb, sb):
  spec = LabelShardingSpecification({"preshift_bits": preshift, "minishard_bits": mb, "shard_bits": sb,
                                     "hash": "murmurhash3_x86_128"})
  labels = np.concatenate([np.array(EDGES, dtype=np.uint64), random_labels(2000, seed=preshift + mb + sb)])
  shards, minis = spec.locate_many(labels)
  for lab, s, m in zip(labels.tolist(), shards.tolist(), minis.tolist()):
    assert (s, m) == locate(lab, preshift, mb, sb), lab
  assert spec.locate(EDGES[-1]) == locate(EDGES[-1], preshift, mb, sb)


def test_image_spec_still_refuses_the_hash_and_label_spec_refuses_identity():
  d = {"preshift_bits": 0, "minishard_bits": 1, "shard_bits": 1, "hash": "murmurhash3_x86_128"}
  with pytest.raises(NotImplementedError):
    ShardingSpecification(d)
  with pytest.raises(ValueError):
    LabelShardingSpecification(dict(d, hash="identity"))
  with pytest.raises(ValueError):
    LabelShardingSpecification(dict(d, data_encoding="zstd"))
  assert LabelShardingSpecification(d).to_dict()["hash"] == "murmurhash3_x86_128"


@pytest.mark.parametrize("data_encoding", ["raw", "gzip"])
@pytest.mark.parametrize("index_encoding", ["raw", "gzip"])
def test_synthesized_shard_reads_back_every_label(data_encoding, index_encoding):
  spec = LabelShardingSpecification({"preshift_bits": 0, "minishard_bits": 3, "shard_bits": 2,
                                     "hash": "murmurhash3_x86_128", "data_encoding": data_encoding,
                                     "minishard_index_encoding": index_encoding})
  rng = np.random.default_rng(5)
  labels = np.unique(np.concatenate([np.array(EDGES, dtype=np.uint64), random_labels(600, seed=5)]))
  shards, minis = spec.locate_many(labels)
  for s in range(4):
    mine = labels[shards == s]
    chunks = {int(l): rng.bytes(int(rng.integers(0, 50))) for l in mine}
    data = spec.synthesize_shard(chunks)
    assert len(data) >= 16 * 8
    for l, blob in chunks.items():
      assert spec.read_chunk(data, l) == blob
    assert spec.chunk_ids(data) == sorted(chunks)
    other = labels[shards != s][:5]
    assert all(spec.read_chunk(data, int(l)) is None for l in other)
    # the payloads are in (minishard, label) order, back to back after the shard index
    if data_encoding == "raw" and chunks:
      order = sorted(chunks, key=lambda l: (spec.locate(l)[1], l))
      assert data[16 * 8:16 * 8 + sum(len(chunks[l]) for l in order)] == b"".join(chunks[l] for l in order)
  with pytest.raises(ValueError, match="shards"):
    spec.synthesize_shard({int(l): b"x" for l in labels[:50]})


def test_minishard_index_is_gzip_level_6_without_mtime():
  spec = LabelShardingSpecification({"preshift_bits": 0, "minishard_bits": 0, "shard_bits": 0,
                                     "hash": "murmurhash3_x86_128", "data_encoding": "gzip",
                                     "minishard_index_encoding": "gzip"})
  data = spec.synthesize_shard({7: b"abc", 3: b"de"})
  start, end = np.frombuffer(data[:16], "<u8").tolist()
  idx = data[16 + start:16 + end]
  table = np.frombuffer(gzip.decompress(idx), "<u8").reshape(3, 2)
  assert table[0].tolist() == [3, 4] and table[1, 1] == 0
  assert idx == gzip.compress(table.tobytes(), compresslevel=6, mtime=0)


@pytest.mark.parametrize("n,want", [(10 ** 9, (11, 9, 0)), (10 ** 7, (4, 9, 0)), (10 ** 6, (1, 9, 0)), (0, (0, 0, 0)),
                                    (1000, (0, 0, 0)), (5000, (0, 2, 0)), (7 * 10 ** 5, (0, 9, 0))])
def test_shard_params_for_hashed(n, want):
  assert compute_shard_params_for_hashed(n) == want


def test_shard_params_min_shards_and_small_indices():
  assert compute_shard_params_for_hashed(10 ** 6, min_shards=8) == (3, 7, 0)
  assert compute_shard_params_for_hashed(300, shard_index_bytes=64, minishard_index_bytes=192) == (4, 2, 0)
  assert compute_shard_params_for_hashed(10, min_shards=4) == (2, 0, 0)
