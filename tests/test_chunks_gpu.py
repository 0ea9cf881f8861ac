"""ign_chunks_place_dev / ign_chunks_cut_dev against numpy slicing, and the compressed_segmentation
batch entries against the CPU oracle's encoder and decoder, chunk by chunk."""
import ctypes as c

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

DTYPES = [np.uint8, np.uint16, np.uint32, np.uint64, np.float32]


def _place(ctx, chunks, rows, cutout_host):
  from igneous_b200 import _shim
  from igneous_b200.storage import DeviceCutout, _upload_bytes
  out = DeviceCutout.from_host(cutout_host, ctx)
  packed, offs = _upload_bytes(ctx, [np.asfortranarray(ch).tobytes(order="F") for ch in chunks])
  table = np.ascontiguousarray(np.array([list(ch.shape[:3]) + [o] + list(r) for ch, o, r in zip(chunks, offs, rows)],
                                        dtype=np.uint64))
  _shim.check(ctx.lib.ign_chunks_place_dev(ctx.handle, _shim.ptr(packed), _shim.dtype_code(out.dtype), out.shape[3],
                                           _shim.ptr(table), len(rows), out.ptr, *out.shape[:3]))
  return out


def _cut(ctx, cutout, boxes, background=0):
  from igneous_b200 import _shim
  from igneous_b200.storage import _packed_offsets
  nc, es = cutout.shape[3], cutout.dtype.itemsize
  offs = _packed_offsets([int(np.prod(b[3:])) * nc * es for b in boxes])
  table = np.ascontiguousarray(np.array([list(b) + [o] for b, o in zip(boxes, offs[:-1])], dtype=np.uint64))
  packed, flags = ctx.alloc(max(int(offs[-1]), 8)), ctx.alloc(4 * len(boxes))
  bg = np.array([background], dtype=cutout.dtype).view("u%d" % es)[0]
  _shim.check(ctx.lib.ign_chunks_cut_dev(ctx.handle, cutout.ptr, _shim.dtype_code(cutout.dtype), *cutout.shape[:3], nc,
                                         _shim.ptr(table), len(boxes), int(bg), _shim.ptr(packed), _shim.ptr(flags)))
  host, fl = np.empty(int(offs[-1]), np.uint8), np.empty(len(boxes), np.uint32)
  ctx.d2h(host, packed)
  ctx.d2h(fl, flags)
  ctx.sync()
  return [host[offs[i]:offs[i + 1]] for i in range(len(boxes))], fl != 0


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("nc", [1, 4])
def test_place_and_cut_random_boxes(ctx, dtype, nc):
  rng = np.random.default_rng(7 + nc)
  X, Y, Z = 70, 45, 33
  fill = (rng.random((X, Y, Z, nc)) * 200).astype(dtype)
  want = fill.copy(order="F")
  chunks, rows = [], []
  cells = [(x, y, z) for z in range(0, Z - 11, 12) for y in range(0, Y - 11, 12) for x in range(0, X - 11, 12)]
  for i in rng.permutation(len(cells))[:24]:  # rows write disjoint boxes, as a cutout's chunks do
    cs = rng.integers(1, 20, 3)
    ch = (rng.random(tuple(cs) + (nc,)) * 250).astype(dtype)
    size = [int(rng.integers(1, min(s, 12) + 1)) for s in cs]  # partial edge boxes included
    src = [int(rng.integers(0, s - z + 1)) for s, z in zip(cs, size)]
    dst = [int(c + rng.integers(0, 12 - z + 1)) for c, z in zip(cells[i], size)]
    chunks.append(ch)
    rows.append(src + size + dst)
    want[tuple(slice(d, d + z) for d, z in zip(dst, size))] = ch[tuple(slice(s, s + z) for s, z in zip(src, size))]
  got = _place(ctx, chunks, rows, fill).to_host()
  assert np.array_equal(got, want)  # voxels no row covers keep the fill
  boxes = []
  for _ in range(30):
    size = [int(rng.integers(1, d + 1)) for d in (X, Y, Z)]
    lo = [int(rng.integers(0, d - z + 1)) for d, z in zip((X, Y, Z), size)]
    boxes.append(lo + size)
  boxes.append([3, 4, 5, 2, 2, 2])
  dev = _place(ctx, [], [], want)
  dev_zero = _place(ctx, [], [], np.zeros_like(want))
  files, flags = _cut(ctx, dev, boxes)
  for b, f, fl in zip(boxes, files, flags):
    block = np.asfortranarray(want[b[0]:b[0] + b[3], b[1]:b[1] + b[4], b[2]:b[2] + b[5]])
    assert f.tobytes() == block.tobytes(order="F")
    assert bool(fl) == (not np.any(block != 0))
  _, zflags = _cut(ctx, dev_zero, boxes[:3])
  assert zflags.all()


def test_place_past_2_32_voxels(ctx):
  """a 2^32 + 2^20 voxel uint8 cutout: rows that land past voxel 2^32 are placed and cut back"""
  from igneous_b200.storage import DeviceCutout
  X, Y, Z = 4096, 4096, 257
  out = DeviceCutout.empty((X, Y, Z, 1), np.uint8, ctx)
  ctx.memset(out.buf, 0, out.nbytes)
  ch = np.arange(64 * 64 * 2, dtype=np.uint64).astype(np.uint8).reshape(64, 64, 2, 1, order="F")
  from igneous_b200 import _shim
  from igneous_b200.storage import _upload_bytes
  packed, _ = _upload_bytes(ctx, [ch.tobytes(order="F")])
  table = np.array([[64, 64, 2, 0, 0, 0, 0, 64, 64, 2, X - 64, Y - 64, Z - 2]], dtype=np.uint64)
  _shim.check(ctx.lib.ign_chunks_place_dev(ctx.handle, _shim.ptr(packed), _shim.IGN_U8, 1, _shim.ptr(table), 1,
                                           out.ptr, X, Y, Z))
  files, flags = _cut(ctx, out, [[X - 64, Y - 64, Z - 2, 64, 64, 2], [0, 0, 0, 64, 64, 2]])
  assert files[0].tobytes() == ch.tobytes(order="F")
  assert not flags[0] and flags[1]
  del out


def test_place_refuses_unsupported_dtype_and_bad_rows(ctx):
  from igneous_b200 import _shim
  buf = ctx.alloc(64)
  table = np.array([[4, 4, 4, 0, 0, 0, 0, 4, 4, 4, 0, 0, 0]], dtype=np.uint64)
  with pytest.raises(NotImplementedError):
    _shim.check(ctx.lib.ign_chunks_place_dev(ctx.handle, _shim.ptr(buf), 99, 1, _shim.ptr(table), 1, _shim.ptr(buf),
                                             4, 4, 4))
  table[0, 10] = 1  # the box would end past the cutout
  with pytest.raises(_shim.IgneousB200Error, match="row 0 writes outside"):
    _shim.check(ctx.lib.ign_chunks_place_dev(ctx.handle, _shim.ptr(buf), _shim.IGN_U8, 1, _shim.ptr(table), 1,
                                             _shim.ptr(buf), 4, 4, 4))


def _mixed_chunks(dtype, sc, rng):
  big = 2 ** 40 if dtype == np.uint64 else 2 ** 20
  out = []
  for shape in [(64, 64, 64), (17, 64, 9), (1, 64, 64), (64, 1, 3), (5, 7, 1), (1, 1, 1), (30, 31, 29)]:
    out.append((rng.integers(0, 6, shape + (sc,)) + big).astype(dtype))
  out.append(np.full((16, 16, 16, sc), big + 3, dtype=dtype))  # a single label
  many = (np.arange(64 * 64 * 20 * sc, dtype=np.uint64).reshape((64, 64, 20, sc)) * 7 + big).astype(dtype)
  out.append(many)  # > 2^16 labels
  out.append(np.repeat(out[0][:8, :8, :8], 2, axis=0))  # repeated tables inside and across chunks
  return out


@pytest.mark.parametrize("dtype", [np.uint32, np.uint64])
@pytest.mark.parametrize("block", [(8, 8, 8), (4, 4, 2)])
@pytest.mark.parametrize("sc", [1, 2])
def test_cseg_batch_equals_oracle(ctx, oracle, dtype, block, sc):
  from igneous_b200 import codecs
  from igneous_b200.storage import DeviceCutout, _upload_bytes
  chunks = _mixed_chunks(dtype, sc, np.random.default_rng(3))
  packed, _ = _upload_bytes(ctx, [np.asfortranarray(ch).tobytes(order="F") for ch in chunks])
  shapes = [ch.shape[:3] for ch in chunks]
  files = codecs.cseg_encode_batch_dev(packed, dtype, shapes, sc, block, ctx)
  for ch, f in zip(chunks, files):
    assert f == oracle.cseg_encode(ch, block).tobytes()
  streams, offs = _upload_bytes(ctx, files)
  out = DeviceCutout.empty((sum(int(np.prod(ch.shape)) for ch in chunks),), dtype, ctx)
  codecs.cseg_decode_batch_dev(streams, offs, dtype, shapes, sc, block, out.buf, ctx)
  flat, at = out.to_host(), 0
  for ch, f in zip(chunks, files):
    n = int(np.prod(ch.shape))
    got = flat[at:at + n].reshape(ch.shape, order="F")
    assert np.array_equal(got, ch)
    assert np.array_equal(got, oracle.cseg_decode(np.frombuffer(f, np.uint32), ch.shape, dtype, block))
    at += n


def test_cseg_batch_hash_collisions(ctx, oracle, monkeypatch):
  """IGN_CSEG_HASH_BITS=2 makes most tables share a hash, across chunks too: owners are still found by
  content inside each chunk's channel"""
  from igneous_b200 import codecs
  from igneous_b200.storage import _upload_bytes
  monkeypatch.setenv("IGN_CSEG_HASH_BITS", "2")
  chunks = _mixed_chunks(np.uint64, 2, np.random.default_rng(5))[:4]
  packed, _ = _upload_bytes(ctx, [ch.tobytes(order="F") for ch in chunks])
  files = codecs.cseg_encode_batch_dev(packed, np.uint64, [ch.shape[:3] for ch in chunks], 2, (8, 8, 8), ctx)
  monkeypatch.delenv("IGN_CSEG_HASH_BITS")
  for ch, f in zip(chunks, files):
    assert f == oracle.cseg_encode(ch, (8, 8, 8)).tobytes()


def test_cseg_batch_refusals(ctx, oracle):
  from igneous_b200 import _shim, codecs
  from igneous_b200.storage import _upload_bytes
  chunks = _mixed_chunks(np.uint32, 1, np.random.default_rng(1))[:3]
  shapes = np.ascontiguousarray(np.array([ch.shape[:3] for ch in chunks], dtype=np.uint32))
  packed, _ = _upload_bytes(ctx, [ch.tobytes(order="F") for ch in chunks])
  need = sum(len(oracle.cseg_encode(ch)) for ch in chunks)
  out, offs, nw = ctx.alloc(need * 4), ctx.alloc(32), c.c_uint64(0)
  with pytest.raises(_shim.IgneousB200Error, match="words needed"):
    _shim.check(ctx.lib.ign_cseg_encode_batch_dev(ctx.handle, _shim.ptr(packed), _shim.IGN_U32, 3, _shim.ptr(shapes),
                                                  1, 8, 8, 8, _shim.ptr(out), need - 1, _shim.ptr(offs), c.byref(nw)))
  assert nw.value == need
  _shim.check(ctx.lib.ign_cseg_encode_batch_dev(ctx.handle, _shim.ptr(packed), _shim.IGN_U32, 3, _shim.ptr(shapes),
                                                1, 8, 8, 8, _shim.ptr(out), need, _shim.ptr(offs), c.byref(nw)))
  with pytest.raises(NotImplementedError):
    _shim.check(ctx.lib.ign_cseg_encode_batch_dev(ctx.handle, _shim.ptr(packed), _shim.IGN_U16, 3, _shim.ptr(shapes),
                                                  1, 8, 8, 8, _shim.ptr(out), need, _shim.ptr(offs), c.byref(nw)))
  files = [oracle.cseg_encode(ch).tobytes() for ch in chunks]
  files[1] = files[1][:len(files[1]) // 8 * 4]  # truncated to half its words
  streams, boffs = _upload_bytes(ctx, files)
  dec = ctx.alloc(sum(ch.nbytes for ch in chunks))
  with pytest.raises(_shim.IgneousB200Error, match="stream 1 is malformed"):
    codecs.cseg_decode_batch_dev(streams, boffs, np.uint32, shapes, 1, (8, 8, 8), dec, ctx)
