"""Argument checks at the entry points: a CCL call refuses an output dtype other than u16 / u32 /
u64, and a label entry point refuses a dtype code other than u8 / u16 / u32 / u64, before it
launches anything and whatever the data.  ign_ccl6_dev and ign_ccl6_volume_dev are one
implementation: the same labels from the same launches."""
import ctypes as c

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

SHAPE = (24, 20, 8)
N = SHAPE[0] * SHAPE[1] * SHAPE[2]
UNKNOWN = (0, 6, 99)
PROF_CLASSES = (0, 1, 2)  # ccl_local, ccl_merge, ccl_label


def _labels(dtype, empty=False):
  if empty:
    return np.zeros(SHAPE, dtype=dtype, order="F")
  rng = np.random.default_rng(3)
  return np.asfortranarray(rng.integers(0, 4, size=SHAPE).astype(dtype))


@pytest.fixture
def dev(ctx):
  """device buffers, each room for N u64 elements, freed after the test"""
  bufs = []

  def alloc(src=None):
    b = ctx.alloc(N * 8)
    if src is not None:
      ctx.h2d(b, src)
      ctx.sync()
    bufs.append(b)
    return b
  yield alloc
  for b in bufs:
    b.free()


@pytest.fixture
def prof(ctx):
  """per-class CCL launch counts recorded since the last reset"""
  lib = ctx.lib

  def counts():
    out = []
    for cls in PROF_CLASSES:
      ms, n = c.c_float(0), c.c_uint64(0)
      assert lib.ign_prof_read(ctx.handle, cls, c.byref(ms), c.byref(n)) == 0
      out.append(n.value)
    return out

  def reset():
    assert lib.ign_prof_enable(ctx.handle, 1) == 0
  reset()
  yield counts, reset
  lib.ign_prof_enable(ctx.handle, 0)


def _refused(ctx, call, error):
  before = ctx.launch_count()
  with pytest.raises(error):
    call()
  assert ctx.launch_count() == before


# ------------------------------------------------------------------ CCL output dtype
BAD_OUT = (1, 5, 99)  # IGN_U8, IGN_F32, an unknown code


@pytest.mark.parametrize("out_dtype", BAD_OUT)
@pytest.mark.parametrize("empty", [True, False], ids=["zeros", "labels"])
@pytest.mark.parametrize("entry", ["ign_ccl6", "ign_ccl6_dev", "ign_ccl6_volume_dev", "ign_ccl6_volume_finish_dev"])
def test_ccl_refuses_out_dtype(ctx, dev, entry, empty, out_dtype):
  from igneous_b200 import _shim
  lib = ctx.lib
  labels = _labels(np.uint32, empty)
  n = c.c_uint64(0)
  if entry == "ign_ccl6":
    out = np.zeros(N * 8, np.uint8)
    _refused(ctx, lambda: _shim.check(lib.ign_ccl6(ctx.handle, _shim.ptr(labels), _shim.IGN_U32, *SHAPE,
                                                   _shim.ptr(out), out_dtype, c.byref(n))), NotImplementedError)
    return
  d_in, d_out = dev(labels), dev()
  if entry == "ign_ccl6_volume_finish_dev":
    v = c.c_void_p()
    _shim.check(lib.ign_ccl6_volume_begin_dev(ctx.handle, _shim.ptr(d_in), _shim.IGN_U32, *SHAPE, None, None, None,
                                              None, c.byref(v), c.byref(n)))
    # the refused finish still consumes the volume
    _refused(ctx, lambda: _shim.check(lib.ign_ccl6_volume_finish_dev(v, None, n.value, _shim.ptr(d_out), out_dtype)),
             NotImplementedError)
    return
  fn = getattr(lib, entry)
  _refused(ctx, lambda: _shim.check(fn(ctx.handle, _shim.ptr(d_in), _shim.IGN_U32, *SHAPE, _shim.ptr(d_out), out_dtype,
                                       c.byref(n))), NotImplementedError)


# ------------------------------------------------------------------ unknown label dtypes
def _calls(ctx, dev, code):
  """name -> (call, raises) for every entry point that dispatches on a label dtype.  Device forms and
  host-only entries raise NotImplementedError through _shim.check; a host form with a device twin
  stages no bytes for a dtype of no size, so it may fail on those first."""
  from igneous_b200 import _shim
  lib, h = ctx.lib, ctx.handle
  labels = _labels(np.uint32)
  d_in, d_out, d_aux = dev(labels), dev(), dev()
  out_host = np.zeros(N * 8, np.uint8)
  aux_host = np.zeros(N * 8, np.uint8)
  n = c.c_uint64(0)
  keys = np.array([1, 2, 3], np.uint64)
  vals = np.array([3, 2, 1], np.uint64)
  aniso = (c.c_float * 3)(1.0, 1.0, 1.0)
  mip = (SHAPE[0] // 2) * (SHAPE[1] // 2) * SHAPE[2] * 8
  d_mip = dev()
  mip_host = np.zeros(mip, np.uint8)
  p, dp, o, do, a, da = (_shim.ptr(labels), _shim.ptr(d_in), _shim.ptr(out_host), _shim.ptr(d_out),
                         _shim.ptr(aux_host), _shim.ptr(d_aux))
  host_outs, dev_outs = _shim.void_pp([mip_host.ctypes.data]), _shim.void_pp([d_mip.ptr])
  rails = (1 << 40,) * 3
  table = [
    ("ign_ccl6", lambda: lib.ign_ccl6(h, p, code, *SHAPE, o, _shim.IGN_U32, c.byref(n)), False),
    ("ign_ccl6_dev", lambda: lib.ign_ccl6_dev(h, dp, code, *SHAPE, do, _shim.IGN_U32, c.byref(n)), True),
    ("ign_ccl6_volume_dev", lambda: lib.ign_ccl6_volume_dev(h, dp, code, *SHAPE, do, _shim.IGN_U32, c.byref(n)), True),
    ("ign_ccl6_volume_begin_dev",
     lambda: lib.ign_ccl6_volume_begin_dev(h, dp, code, *SHAPE, None, None, None, None, c.byref(c.c_void_p()),
                                           c.byref(n)), True),
    ("ign_dust", lambda: lib.ign_dust(h, p, code, *SHAPE, 2), False),
    ("ign_dust_dev", lambda: lib.ign_dust_dev(h, dp, code, *SHAPE, 2), True),
    ("ign_ccl_task", lambda: lib.ign_ccl_task(h, p, code, *SHAPE, 0, 0.0, 0, 0.0, *rails, 0, 0, o, c.byref(n)), False),
    ("ign_ccl_task_dev",
     lambda: lib.ign_ccl_task_dev(h, dp, code, *SHAPE, 0, 0.0, 0, 0.0, *rails, 0, 0, do, c.byref(n)), True),
    ("ign_renumber", lambda: lib.ign_renumber(h, p, code, N, o, a, N, c.byref(n)), False),
    ("ign_renumber_dev", lambda: lib.ign_renumber_dev(h, dp, code, N, do, da, N, c.byref(n)), True),
    ("ign_remap", lambda: lib.ign_remap(h, p, code, N, _shim.ptr(keys), _shim.ptr(vals), len(keys), 1), False),
    ("ign_remap_dev", lambda: lib.ign_remap_dev(h, dp, code, N, _shim.ptr(keys), _shim.ptr(vals), len(keys), 1), True),
    ("ign_mask", lambda: lib.ign_mask(h, p, code, N, _shim.ptr(keys), len(keys), 0, 0), True),
    ("ign_unique", lambda: lib.ign_unique(h, p, code, N, o, a, N, c.byref(n)), True),
    ("ign_inverse_component_map",
     lambda: lib.ign_inverse_component_map(h, p, p, code, N, o, c.byref(c.c_uint64(N // 2))), True),
    ("ign_cast_dev in", lambda: lib.ign_cast_dev(h, dp, code, do, _shim.IGN_U32, N), True),
    ("ign_cast_dev out", lambda: lib.ign_cast_dev(h, dp, _shim.IGN_U32, do, code, N), True),
    ("ign_find_objects", lambda: lib.ign_find_objects(h, p, code, *SHAPE, c.byref(c.c_uint64(0)), o), False),
    ("ign_find_objects_dev", lambda: lib.ign_find_objects_dev(h, dp, code, *SHAPE, c.byref(c.c_uint64(0)), do), True),
    ("ign_edt", lambda: lib.ign_edt(h, p, code, *SHAPE, aniso, 0, 0, o), False),
    ("ign_edt_dev", lambda: lib.ign_edt_dev(h, dp, code, *SHAPE, aniso, 0, 0, do), True),
    ("ign_dilate_multilabel", lambda: lib.ign_dilate_multilabel(h, p, code, *SHAPE, o), False),
    ("ign_dilate_multilabel_dev", lambda: lib.ign_dilate_multilabel_dev(h, dp, code, *SHAPE, do), True),
    ("ign_fill_holes", lambda: lib.ign_fill_holes(h, p, code, *SHAPE, 0, 100, o, a), False),
    ("ign_fill_holes_dev", lambda: lib.ign_fill_holes_dev(h, dp, code, *SHAPE, 0, 100, do, da), True),
    ("ign_pool_mode_2x2x1", lambda: lib.ign_pool_mode_2x2x1(h, p, code, *SHAPE, 1, 0, host_outs), False),
    ("ign_pool_mode_2x2x1_dev", lambda: lib.ign_pool_mode_2x2x1_dev(h, dp, code, *SHAPE, 1, 0, dev_outs), True),
    ("ign_pool_select", lambda: lib.ign_pool_select(h, p, code, *SHAPE, 2, 2, 1, 1, 0, host_outs), False),
    ("ign_pool_select_dev", lambda: lib.ign_pool_select_dev(h, dp, code, *SHAPE, 2, 2, 1, 1, 0, dev_outs), True),
    ("ign_synth_seg_dev", lambda: lib.ign_synth_seg_dev(h, do, code, *SHAPE, 0, 0, 0, 4, 8, 0, 1), True),
  ]
  return {name: (call, NotImplementedError if strict else Exception) for name, call, strict in table}


ENTRIES = ["ign_ccl6", "ign_ccl6_dev", "ign_ccl6_volume_dev", "ign_ccl6_volume_begin_dev", "ign_dust", "ign_dust_dev",
           "ign_ccl_task", "ign_ccl_task_dev", "ign_renumber", "ign_renumber_dev", "ign_remap", "ign_remap_dev",
           "ign_mask", "ign_unique", "ign_inverse_component_map", "ign_cast_dev in", "ign_cast_dev out",
           "ign_find_objects", "ign_find_objects_dev", "ign_edt", "ign_edt_dev", "ign_dilate_multilabel",
           "ign_dilate_multilabel_dev", "ign_fill_holes", "ign_fill_holes_dev", "ign_pool_mode_2x2x1",
           "ign_pool_mode_2x2x1_dev", "ign_pool_select", "ign_pool_select_dev", "ign_synth_seg_dev"]


@pytest.mark.parametrize("code", UNKNOWN)
@pytest.mark.parametrize("entry", ENTRIES)
def test_label_entry_refuses_unknown_dtype(ctx, dev, entry, code):
  from igneous_b200 import _shim
  calls = _calls(ctx, dev, code)
  assert sorted(calls) == sorted(ENTRIES)
  call, error = calls[entry]
  _refused(ctx, lambda: _shim.check(call()), error)


# ------------------------------------------------------------------ one CCL path
@pytest.mark.parametrize("empty", [False, True], ids=["labels", "zeros"])
@pytest.mark.parametrize("dtype", [np.uint8, np.uint16, np.uint32, np.uint64])
def test_ccl6_dev_is_volume_dev(ctx, dev, prof, dtype, empty):
  from igneous_b200 import _shim
  counts, reset = prof
  labels = _labels(dtype, empty)
  d_in = dev(labels)
  got = []
  for entry in ("ign_ccl6_dev", "ign_ccl6_volume_dev"):
    d_out = dev()
    n = c.c_uint64(0)
    reset()
    before = ctx.launch_count()
    _shim.check(getattr(ctx.lib, entry)(ctx.handle, _shim.ptr(d_in), _shim.dtype_code(dtype), *SHAPE,
                                        _shim.ptr(d_out), _shim.IGN_U32, c.byref(n)))
    launches = ctx.launch_count() - before
    got.append((ctx.to_host(d_out, SHAPE, np.uint32), n.value, launches, counts()))
  (a, na, la, pa), (b, nb, lb, pb) = got
  assert a.tobytes() == b.tobytes() and na == nb and la == lb and pa == pb
  assert (na == 0) == empty and la > 0
