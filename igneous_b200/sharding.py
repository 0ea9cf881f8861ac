"""neuroglancer_uint64_sharded_v1 for image chunks: the container either side of
ImageShardDownsampleTask (igneous/tasks/image/image.py:672-843).  LabelShardingSpecification is the same
container keyed by label with the murmurhash3_x86_128 hash, for skeleton layers (DESIGN.md §5l).

The reference gets all of this from cloudvolume (`ShardingSpecification`,
`create_sharded_image_info`, `image.make_shard[_chunks]`), which is not installed
here; this module restates the PUBLISHED container format (neuroglancer's
"sharded format" document) so that the `file://` stand-in can write and read
sharded scales.  Host-side byte shuffling only -- the voxels inside the chunks
come from the GPU (pooling, renumber / remap, compressed_segmentation).

  chunk id      compressed Morton code of the chunk's grid position
  shard file    [shard index: 2^minishard_bits x (start, end) u64le]
                [chunk payloads ...][minishard indices ...]
  minishard idx u64le array [3, n]: delta-coded chunk ids, delta-coded start
                offsets (relative to the end of the shard index; each start is
                coded against the END of the previous chunk), byte sizes

The choice of preshift / minishard / shard bits in `create_sharded_image_info`
follows cloudvolume's documented limits (8 KiB shard index, ~40 kB minishard
index, shard payload <= the memory target) but not its exact code: any choice
gives a valid dataset because readers follow the spec stored in the info file.
"""
import gzip
import math
import struct

import numpy as np

SHARDING_TYPE = "neuroglancer_uint64_sharded_v1"


def _bits(n):
  """bits needed to address n grid cells"""
  return int(math.ceil(math.log2(n))) if n > 1 else 0


def grid_bits(dataset_size, chunk_size):
  grid = [int(math.ceil(int(d) / int(c))) for d, c in zip(dataset_size, chunk_size)]
  return grid, [_bits(g) for g in grid]


def compressed_morton_code(gridpt, grid_size):
  """Interleave the bits of (x, y, z) from the LSB up, skipping a dimension once its
  own bits are exhausted.  Vectorised over an [n, 3] array of grid points."""
  pts = np.atleast_2d(np.asarray(gridpt, dtype=np.uint64))
  nb = [_bits(int(g)) for g in grid_size]
  if sum(nb) > 64:
    raise ValueError("grid %r needs more than 64 chunk-id bits" % (tuple(grid_size),))
  for d in range(3):
    if np.any(pts[:, d] >= max(int(grid_size[d]), 1)):
      raise ValueError("grid point outside grid %r" % (tuple(grid_size),))
  code = np.zeros(len(pts), dtype=np.uint64)
  j = 0
  for i in range(max(nb) if nb else 0):
    for d in range(3):
      if i < nb[d]:
        code |= ((pts[:, d] >> np.uint64(i)) & np.uint64(1)) << np.uint64(j)
        j += 1
  return code if np.ndim(gridpt) > 1 else int(code[0])


class ShardingSpecification:
  """The `sharding` member of a scale (same keys as the info file)."""

  def __init__(self, spec):
    if spec.get("@type", SHARDING_TYPE) != SHARDING_TYPE:
      raise ValueError("unknown sharding type %r" % spec.get("@type"))
    self.preshift_bits = int(spec["preshift_bits"])
    self.minishard_bits = int(spec["minishard_bits"])
    self.shard_bits = int(spec["shard_bits"])
    self.hash = spec.get("hash", "identity")
    self.minishard_index_encoding = spec.get("minishard_index_encoding", "raw")
    self.data_encoding = spec.get("data_encoding", "raw")
    if self.hash != "identity":
      # image scales use the identity hash (a shard = a box of the chunk grid); the murmur
      # variant belongs to mesh / skeleton shards, which are outside this path
      raise NotImplementedError("shard hash %r (only 'identity' image shards are supported)" % self.hash)
    for enc in (self.minishard_index_encoding, self.data_encoding):
      if enc not in ("raw", "gzip"):
        raise ValueError("unknown shard encoding %r" % enc)

  def to_dict(self):
    return {"@type": SHARDING_TYPE, "preshift_bits": self.preshift_bits, "hash": self.hash,
            "minishard_bits": self.minishard_bits, "shard_bits": self.shard_bits,
            "minishard_index_encoding": self.minishard_index_encoding, "data_encoding": self.data_encoding}

  def locate(self, chunk_id):
    """-> (shard number, minishard number)"""
    h = int(chunk_id) >> self.preshift_bits
    mini = h & ((1 << self.minishard_bits) - 1)
    shard = (h >> self.minishard_bits) & ((1 << self.shard_bits) - 1)
    return shard, mini

  def shard_filename(self, shard_number):
    return "%0*x.shard" % (max(int(math.ceil(self.shard_bits / 4.0)), 1), int(shard_number))

  @property
  def index_length(self):
    return 16 << self.minishard_bits

  # ---- writer
  def synthesize_shard(self, chunks):
    """{chunk id: encoded chunk bytes} (all of one shard) -> the bytes of the shard file."""
    keys = list(chunks)
    ids = np.fromiter((int(c) for c in keys), dtype=np.uint64, count=len(keys))
    shards, minis = self.locate_many(ids)
    if len(ids) and np.any(shards != shards[0]):
      other = shards[np.argmax(shards != shards[0])]
      raise ValueError("chunks of shards %x and %x in one synthesize_shard call" % (int(shards[0]), int(other)))
    order = np.lexsort((ids, minis))
    blobs = [chunks[keys[i]] for i in order]
    if self.data_encoding == "gzip":
      blobs = [gzip.compress(b, compresslevel=6, mtime=0) for b in blobs]
    return pack_shard(self.minishard_bits, self.minishard_index_encoding, minis[order], ids[order], blobs)

  def locate_many(self, chunk_ids):
    """-> (shard numbers, minishard numbers) of a uint64 array of chunk ids"""
    h = np.asarray(chunk_ids, dtype=np.uint64) >> np.uint64(self.preshift_bits)
    mini = h & np.uint64((1 << self.minishard_bits) - 1)
    shard = (h >> np.uint64(self.minishard_bits)) & np.uint64((1 << self.shard_bits) - 1)
    return shard, mini

  # ---- reader
  def minishard_table(self, shard_bytes, minishard):
    n = self.index_length
    start, end = struct.unpack_from("<QQ", shard_bytes, 16 * minishard)
    if end <= start:
      return np.zeros((3, 0), dtype=np.uint64)
    raw = shard_bytes[n + start:n + end]
    if self.minishard_index_encoding == "gzip":
      raw = gzip.decompress(raw)
    table = np.frombuffer(raw, dtype="<u8").reshape(3, -1).astype(np.uint64)
    ids = np.cumsum(table[0])
    sizes = table[2]
    starts = np.zeros_like(ids)
    pos = 0
    for i in range(table.shape[1]):
      pos += int(table[1, i])
      starts[i] = pos
      pos += int(sizes[i])
    return np.stack([ids, starts, sizes])

  def read_chunk(self, shard_bytes, chunk_id):
    """-> encoded chunk bytes or None"""
    _, mini = self.locate(chunk_id)
    t = self.minishard_table(shard_bytes, mini)
    hit = np.nonzero(t[0] == np.uint64(chunk_id))[0]
    if len(hit) == 0:
      return None
    n = self.index_length
    s, size = int(t[1, hit[0]]), int(t[2, hit[0]])
    blob = shard_bytes[n + s:n + s + size]
    return gzip.decompress(blob) if self.data_encoding == "gzip" else bytes(blob)

  def chunk_ids(self, shard_bytes):
    out = []
    for m in range(1 << self.minishard_bits):
      out.extend(int(v) for v in self.minishard_table(shard_bytes, m)[0])
    return sorted(out)


_U32 = np.uint64(0xFFFFFFFF)


def _rotl32(x, r):
  return ((x << np.uint64(r)) | (x >> np.uint64(32 - r))) & _U32


def _fmix32(h):
  h ^= h >> np.uint64(16)
  h = (h * np.uint64(0x85EBCA6B)) & _U32
  h ^= h >> np.uint64(13)
  h = (h * np.uint64(0xC2B2AE35)) & _U32
  return h ^ (h >> np.uint64(16))


def murmurhash3_x86_128_u64(keys):
  """MurmurHash3_x86_128 with seed 0 of the 8 little-endian bytes of each uint64 key, low 64 bits (h1 | h2 << 32).
  Vectorised; 32-bit words are held in uint64 and masked after every product (DESIGN.md §5l)."""
  keys = np.asarray(keys, dtype=np.uint64)
  c1, c2, c3 = np.uint64(0x239B961B), np.uint64(0xAB0E9789), np.uint64(0x38B34AE5)
  k1, k2 = keys & _U32, keys >> np.uint64(32)
  # an 8-byte key has no 16-byte block: bytes 4..7 are tail word k2, bytes 0..3 tail word k1
  h2 = (_rotl32((k2 * c2) & _U32, 16) * c3) & _U32
  h1 = (_rotl32((k1 * c1) & _U32, 15) * c2) & _U32
  h3 = np.zeros_like(keys)
  h4 = np.zeros_like(keys)
  h1, h2, h3, h4 = (h ^ np.uint64(8) for h in (h1, h2, h3, h4))  # the length
  h1 = (h1 + h2 + h3 + h4) & _U32
  h2, h3, h4 = ((h + h1) & _U32 for h in (h2, h3, h4))
  h1, h2, h3, h4 = (_fmix32(h) for h in (h1, h2, h3, h4))
  h1 = (h1 + h2 + h3 + h4) & _U32
  h2 = (h2 + h1) & _U32
  return h1 | (h2 << np.uint64(32))


class LabelShardingSpecification(ShardingSpecification):
  """The `sharding` member of a skeleton (or mesh) info: neuroglancer_uint64_sharded_v1 keyed by label with
  the murmurhash3_x86_128 hash (DESIGN.md §5l).  The container is the image shards' own; only the hash
  differs: h = murmur(label >> preshift_bits), minishard = h & (2^minishard_bits - 1),
  shard = (h >> minishard_bits) & (2^shard_bits - 1)."""

  HASH = "murmurhash3_x86_128"

  def __init__(self, spec):
    spec = dict(spec)
    if spec.get("hash", self.HASH) != self.HASH:
      raise ValueError("LabelShardingSpecification: hash %r (only %r)" % (spec.get("hash"), self.HASH))
    super().__init__(dict(spec, hash="identity"))
    self.hash = self.HASH
    if not (0 <= self.preshift_bits < 64 and 0 <= self.minishard_bits and 0 <= self.shard_bits
            and self.minishard_bits + self.shard_bits <= 64):
      raise ValueError("LabelShardingSpecification: preshift_bits %d, minishard_bits %d, shard_bits %d"
                       % (self.preshift_bits, self.minishard_bits, self.shard_bits))

  def locate_many(self, labels):
    h = murmurhash3_x86_128_u64(np.asarray(labels, dtype=np.uint64) >> np.uint64(self.preshift_bits))
    mini = h & np.uint64((1 << self.minishard_bits) - 1)
    shard = (h >> np.uint64(self.minishard_bits)) & np.uint64((1 << self.shard_bits) - 1) \
        if self.minishard_bits < 64 else np.zeros_like(h)
    return shard, mini

  def locate(self, label):
    """-> (shard number, minishard number)"""
    shard, mini = self.locate_many(np.array([int(label)], dtype=np.uint64))
    return int(shard[0]), int(mini[0])


def pack_shard(minishard_bits, minishard_index_encoding, minis, ids, blobs):
  """The bytes of a shard file whose entries are already in (minishard, id) order: minis and ids the
  minishard and id of each entry, blobs its payload as stored (already data-encoded).  The payloads go back to
  back after the shard index, then each non-empty minishard's index ([3, n] u64le: delta-coded ids,
  delta-coded starts, sizes), encoded with minishard_index_encoding, in minishard order."""
  minis = np.asarray(minis, dtype=np.uint64)
  ids = np.asarray(ids, dtype=np.uint64)
  sizes = np.fromiter((len(b) for b in blobs), dtype=np.uint64, count=len(blobs))
  starts = np.zeros(len(blobs), dtype=np.uint64)
  if len(blobs):
    np.cumsum(sizes[:-1], out=starts[1:])
  pos = int(sizes.sum())
  shard_index = np.zeros((1 << minishard_bits, 2), dtype="<u8")
  tail = []
  bounds = np.searchsorted(minis, np.arange((1 << minishard_bits) + 1, dtype=np.uint64))
  for m in range(1 << minishard_bits):
    a, b = int(bounds[m]), int(bounds[m + 1])
    if a == b:
      shard_index[m] = (pos, pos)  # empty minishard
      continue
    table = np.zeros((3, b - a), dtype="<u8")
    table[0, 0], table[0, 1:] = ids[a], np.diff(ids[a:b])
    table[1, 0] = starts[a]  # every later payload starts where the previous one ends
    table[2] = sizes[a:b]
    raw = table.tobytes(order="C")
    raw = gzip.compress(raw, compresslevel=6, mtime=0) if minishard_index_encoding == "gzip" else raw
    shard_index[m] = (pos, pos + len(raw))
    tail.append(raw)
    pos += len(raw)
  return shard_index.tobytes(order="C") + b"".join(bytes(b) for b in blobs) + b"".join(tail)


def create_sharded_image_info(dataset_size, chunk_size, encoding, dtype, uncompressed_shard_bytesize=int(3.5e9),
                              max_shard_index_bytes=8192, max_minishard_index_bytes=40000,
                              data_encoding="gzip", minishard_index_encoding="gzip"):
  """Sharding spec for an image scale: one shard holds a power-of-two block of chunks whose
  uncompressed size fits `uncompressed_shard_bytesize`; identity hash so that a shard is a
  contiguous box of the chunk grid (what ImageShardDownsampleTask relies on)."""
  _, nb = grid_bits(dataset_size, chunk_size)
  total_bits = sum(nb)
  chunk_bytes = int(np.prod([int(c) for c in chunk_size])) * np.dtype(dtype).itemsize
  per_shard = max(int(uncompressed_shard_bytesize) // max(chunk_bytes, 1), 1)
  shape_bits = min(int(math.floor(math.log2(per_shard))), total_bits)
  shard_bits = total_bits - shape_bits
  preshift = min(shape_bits, int(math.floor(math.log2(max(max_minishard_index_bytes // 24, 1)))))
  minishard = shape_bits - preshift
  max_mini = int(math.floor(math.log2(max(max_shard_index_bytes // 16, 1))))
  if minishard > max_mini:
    preshift += minishard - max_mini
    minishard = max_mini
  if encoding in ("jpeg", "png", "jxl", "compresso", "crackle", "fpzip", "kempressed", "zfpc"):
    data_encoding = "raw"  # already entropy coded: a second gzip pass buys nothing
  return {"@type": SHARDING_TYPE, "preshift_bits": int(preshift), "hash": "identity",
          "minishard_bits": int(minishard), "shard_bits": int(shard_bits),
          "minishard_index_encoding": minishard_index_encoding, "data_encoding": data_encoding}
