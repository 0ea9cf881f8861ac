"""Drop-in for the `zmesh` calls on the igneous hot path, running on H100.

Reference call sites (seung-lab/igneous):
  igneous/tasks/mesh/mesh.py:151      zmesh.Mesher(self._volume.resolution)
  igneous/tasks/mesh/mesh.py:245      self._mesher.mesh(data, preserve_order=False)
  igneous/tasks/mesh/mesh.py:374-381  for obj_id in mesher.ids(): mesher.get(obj_id,
                                        reduction_factor=, max_error=, voxel_centered=True)
  igneous/tasks/mesh/mesh.py:443-448  mesh.to_precomputed()
  igneous/tasks/mesh/mesh.py:239      zmesh.Mesh.concatenate(a, b, id=segid)

Vertices are float32 physical coordinates
  (half_voxel/2 + (0.5 if voxel_centered else 0)) * resolution,
faces uint32.  Vertex order is (z,y,x)-sorted, face order is cube raster order
(zmesh's own orders are hash-map dependent; parity is defined on the
canonicalised mesh, see DESIGN.md).
"""
import ctypes
import struct

import numpy as np

from . import _shim

__all__ = ["Mesher", "Mesh"]


class Mesh:
  def __init__(self, vertices, faces, normals=None, id=None):
    self.vertices = np.asarray(vertices, dtype=np.float32).reshape(-1, 3)
    self.faces = np.asarray(faces, dtype=np.uint32).reshape(-1, 3)
    self.normals = normals
    self.id = id

  def __len__(self):
    return self.vertices.shape[0]

  def __eq__(self, other):
    return (isinstance(other, Mesh) and np.array_equal(self.vertices, other.vertices)
            and np.array_equal(self.faces, other.faces))

  def clone(self):
    return Mesh(self.vertices.copy(), self.faces.copy(), self.normals, self.id)

  def to_precomputed(self):
    """Neuroglancer legacy fragment: u32 Nv | f32[3*Nv] | u32[3*Nf], little endian."""
    v = np.ascontiguousarray(self.vertices, dtype="<f4")
    f = np.ascontiguousarray(self.faces, dtype="<u4")
    return struct.pack("<I", v.shape[0]) + v.tobytes("C") + f.tobytes("C")

  @classmethod
  def from_precomputed(cls, binary, id=None):
    n = struct.unpack("<I", binary[:4])[0]
    v = np.frombuffer(binary, dtype="<f4", count=3 * n, offset=4).reshape(n, 3)
    f = np.frombuffer(binary, dtype="<u4", offset=4 + 12 * n).reshape(-1, 3)
    return cls(v.copy(), f.copy(), id=id)

  @classmethod
  def concatenate(cls, *meshes, id=None):
    verts, faces, off = [], [], 0
    for m in meshes:
      verts.append(m.vertices)
      faces.append(m.faces + np.uint32(off))
      off += m.vertices.shape[0]
    if not verts:
      return cls(np.zeros((0, 3), np.float32), np.zeros((0, 3), np.uint32), id=id)
    return cls(np.concatenate(verts), np.concatenate(faces), id=id)


class Mesher:
  def __init__(self, voxel_res, ctx=None):
    self.voxel_res = np.asarray(voxel_res, dtype=np.float32).reshape(3)
    self._ctx = ctx
    self._handle = None
    self._export = {}
    self._simp = None  # (reduction_factor, max_error) the resident meshes were simplified with

  # -- lifecycle
  def _free(self):
    if self._handle is not None:
      _shim.load().ign_mesh_free(self._handle)
      self._handle = None
    self._export = {}
    self._simp = None

  def clear(self):
    self._free()

  def __del__(self):
    try:
      self._free()
    except Exception:
      pass

  # -- zmesh API
  def mesh(self, data, close=False, preserve_order=False):
    """Marching cubes over every label of a 3-D unsigned integer volume."""
    if close:
      raise NotImplementedError("igneous_b200.zmesh: close=True is not implemented "
                                "(igneous pads the volume itself, mesh.py:267-303)")
    arr = np.asarray(data)
    while arr.ndim > 3 and arr.shape[-1] == 1:
      arr = arr[..., 0]
    if arr.ndim != 3:
      raise ValueError("Mesher.mesh expects a 3-D array, got shape %r" % (arr.shape,))
    if arr.dtype == np.bool_:
      arr = arr.view(np.uint8)
    arr = np.asfortranarray(arr)
    self._free()
    ctx = self._ctx or _shim.default_context()
    self._ctx = ctx
    h = ctypes.c_void_p()
    sx, sy, sz = arr.shape
    _shim.check(ctx.lib.ign_mesh_begin(ctx.handle, _shim.ptr(arr), _shim.dtype_code(arr.dtype), sx, sy, sz,
                                       ctypes.byref(h)))
    self._handle = h

  def ids(self):
    if self._handle is None:
      return []
    lib = self._ctx.lib
    n = ctypes.c_uint64(0)
    _shim.check(lib.ign_mesh_num_ids(self._handle, ctypes.byref(n)))
    ids = np.zeros(int(n.value), dtype=np.uint64)
    if n.value:
      _shim.check(lib.ign_mesh_ids(self._handle, _shim.ptr(ids), n.value))
    return [int(i) for i in ids]

  def _simplify(self, reduction_factor, max_error):
    want = (int(reduction_factor), float(max_error)) if reduction_factor and reduction_factor > 0 else None
    if want == self._simp:
      return
    if self._simp is not None or (want is None and self._simp is not None):
      raise ValueError("igneous_b200.zmesh: the resident meshes were simplified with %r; call mesh() "
                       "again to extract with %r" % (self._simp, want))
    res = (ctypes.c_float * 3)(*[float(r) for r in self.voxel_res])
    _shim.check(self._ctx.lib.ign_mesh_simplify(self._handle, res, *want))
    self._simp = want
    self._export = {}

  def _exported(self, voxel_centered):
    key = bool(voxel_centered)
    if key not in self._export:
      lib = self._ctx.lib
      nv, nf = ctypes.c_uint64(0), ctypes.c_uint64(0)
      _shim.check(lib.ign_mesh_totals(self._handle, ctypes.byref(nv), ctypes.byref(nf)))
      ids = self.ids()
      verts = np.zeros((int(nv.value), 3), dtype=np.float32)
      faces = np.zeros((int(nf.value), 3), dtype=np.uint32)
      voff = np.zeros(len(ids) + 1, dtype=np.uint64)
      foff = np.zeros(len(ids) + 1, dtype=np.uint64)
      res = (ctypes.c_float * 3)(*[float(r) for r in self.voxel_res])
      _shim.check(lib.ign_mesh_export(self._handle, res, int(key), _shim.ptr(verts),
                                      _shim.ptr(faces), _shim.ptr(voff), _shim.ptr(foff)))
      index = {i: j for j, i in enumerate(ids)}
      self._export[key] = (verts, faces, voff, foff, index)
    return self._export[key]

  def get(self, label, normals=False, reduction_factor=0, max_error=40, voxel_centered=False):
    """Mesh of one label.  reduction_factor > 0 requests quadric edge-collapse
    simplification towards nf/reduction_factor faces within max_error."""
    if self._handle is None:
      raise ValueError("Mesher.get called before Mesher.mesh")
    if normals:
      raise NotImplementedError("igneous_b200.zmesh: normals=True is not implemented")
    self._simplify(reduction_factor, max_error)
    verts, faces, voff, foff, index = self._exported(voxel_centered)
    label = int(label)
    if label not in index:
      raise KeyError(label)
    j = index[label]
    v = verts[int(voff[j]):int(voff[j + 1])].copy()
    f = faces[int(foff[j]):int(foff[j + 1])].copy()
    return Mesh(v, f, id=label)

  def get_mesh(self, *args, **kwargs):  # legacy alias
    return self.get(*args, **kwargs)

  def erase(self, label):
    pass  # results live in one pooled buffer; freed by clear()/mesh()
