"""The C-ABI library loads and exports every symbol include/igneous_b200.h
declares, with the header's argument types (no compute calls: runs without a GPU)."""
import ast
import ctypes
import glob
import os

import pytest

from igneous_b200 import _shim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
  lib = _shim.load()
  names = sorted(_shim.prototypes())
  assert len(names) >= 45
  missing = [n for n in names if not hasattr(lib, n)]
  assert not missing, missing


def test_every_declared_function_has_the_header_types():
  lib = _shim.load()
  for name, (restype, argtypes) in _shim.prototypes().items():
    fn = getattr(lib, name)
    assert fn.restype is restype and fn.argtypes == argtypes, name
  assert lib.ign_last_error.restype is ctypes.c_char_p and lib.ign_version.argtypes == []
  assert lib.ign_mesh_simplify.argtypes == [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_float]
  assert lib.ign_ccl_task.argtypes[7] is ctypes.c_double and lib.ign_synth_seg_dev.argtypes[6] is ctypes.c_int64
  assert lib.ign_pool_select.argtypes[6] is ctypes.c_uint32 and lib.ign_dust.argtypes[6] is ctypes.c_uint64


def test_bad_arguments_fail_before_native_code():
  lib = _shim.load()
  with pytest.raises(ctypes.ArgumentError):
    lib.ign_timer_start(None, 1.5)  # a float for `int slot`
  with pytest.raises(ctypes.ArgumentError):
    lib.ign_dev_alloc(None, ctypes.c_int(8), None)  # a c_int for `uint64_t bytes`
  timer_start = lib.ign_timer_start
  with pytest.raises(TypeError):
    timer_start(None)


def test_unmapped_header_type_or_missing_export_raises_at_load(monkeypatch, tmp_path):
  header = tmp_path / "igneous_b200.h"
  monkeypatch.setattr(_shim, "HEADER", str(header))
  monkeypatch.setattr(_shim, "_lib", None)
  header.write_text("IGN_API int ign_version(void);\nIGN_API int ign_sync(ign_ctx* ctx, size_t n);\n")
  with pytest.raises(ValueError, match="size_t n"):
    _shim.load()
  header.write_text("IGN_API int ign_version(void);\nIGN_API int ign_not_exported(int x);\n")
  with pytest.raises(AttributeError, match="ign_not_exported"):
    _shim.load()
  assert _shim._lib is None


def test_call_sites_pass_as_many_arguments_as_the_header_declares():
  """ctypes rejects too few arguments but passes extra ones on: every `<lib>.ign_*(...)` call without
  *args in the package, the tools, the tests and bench.py matches its prototype's arity."""
  protos = _shim.prototypes()
  paths = [os.path.join(ROOT, "bench.py")]
  for d in ("igneous_b200", "tools", "tests"):
    paths += glob.glob(os.path.join(ROOT, d, "**", "*.py"), recursive=True)
  checked, wrong = 0, []
  for path in paths:
    with open(path) as f:
      tree = ast.parse(f.read(), path)
    for node in ast.walk(tree):
      if not (isinstance(node, ast.Call) and isinstance(node.func, ast.Attribute) and node.func.attr in protos):
        continue
      if any(isinstance(a, ast.Starred) for a in node.args) or node.keywords:
        continue
      checked += 1
      want = len(protos[node.func.attr][1])
      if len(node.args) != want:
        wrong.append("%s:%d %s: %d arguments, the header declares %d"
                     % (os.path.relpath(path, ROOT), node.lineno, node.func.attr, len(node.args), want))
  assert checked >= 100
  assert not wrong, "\n".join(wrong)


def test_version_and_error_string():
  lib = _shim.load()
  assert lib.ign_version() >= 100
  assert isinstance(lib.ign_last_error(), bytes)


def test_no_oracle_import_in_product():
  # the product must never route through the CPU oracle
  pkg = os.path.join(ROOT, "igneous_b200")
  for dirpath, _, files in os.walk(pkg):
    for f in files:
      if f.endswith((".py", ".cu", ".cuh", ".h")):
        src = open(os.path.join(dirpath, f), errors="replace").read()
        assert "import oracle" not in src and "from oracle" not in src, f
        assert "liboracle" not in src, f


def test_fails_loudly_without_a_gpu():
  """No CPU fallback: on a box without a CUDA device every compute entry point
  must raise instead of silently computing on the host."""
  import numpy as np
  import pytest
  if _shim.device_count() > 0:
    pytest.skip("a CUDA device is visible")
  with pytest.raises(_shim.IgneousB200Error):
    _shim.Context(0)
  from igneous_b200 import tinybrain, cc3d, zmesh, fastremap
  img = np.zeros((8, 8, 8), dtype=np.uint32)
  for call in (lambda: tinybrain.downsample_segmentation(img, (2, 2, 1)),
               lambda: cc3d.connected_components(img, connectivity=6),
               lambda: fastremap.renumber(img + 1),
               lambda: zmesh.Mesher((1, 1, 1)).mesh(img)):
    with pytest.raises(_shim.IgneousB200Error):
      call()


def test_missing_library_is_an_error(monkeypatch, tmp_path):
  import importlib
  import pytest
  monkeypatch.setenv("IGNEOUS_B200_LIB", str(tmp_path / "nope.so"))
  monkeypatch.setattr(_shim, "_lib", None)
  with pytest.raises(_shim.NativeLibraryMissing):
    _shim.load()
  monkeypatch.delenv("IGNEOUS_B200_LIB")
  monkeypatch.setattr(_shim, "_lib", None)
  assert _shim.load() is not None
