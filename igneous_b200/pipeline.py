"""Device-resident downsample -> CCL -> mesh pipeline over one volume (one GPU
holds one z-slab of the dataset; BASELINE.json config C5 / the headline metric).

The three stages are exactly the per-task bodies of the reference, chained in
HBM instead of through CloudVolume files:
  * DownsampleTask          igneous/tasks/image/image.py:518-549 (2 mode mips)
  * CCL passes 1-4          igneous/tasks/image/ccl.py:126-420
  * MeshTask (mip 2, 256^3) igneous/tasks/mesh/mesh.py:140-265
Host code only sequences kernels; all arithmetic runs in libigneous_b200.
"""
import ctypes as c

import numpy as np

from . import _shim

PROF_CLASSES = {"ccl_local": 0, "ccl_merge": 1, "ccl_label": 2, "pool": 3, "mc": 4, "simp_labels": 5}


class VolumePipeline:
  def __init__(self, ctx, shape, dtype=np.uint32, num_mips=2, mesh_shape=(256, 256, 256),
               resolution=(16, 16, 40), pitch=64, num_ids=1 << 20, seed=0, offset=(0, 0, 0),
               ccl_out_dtype=np.uint32, simplification_factor=100, max_simplification_error=40,
               group=None, mesh_streams=8, id_base=0):
    self.ctx = ctx
    self.lib = ctx.lib
    self.shape = tuple(int(s) for s in shape)
    self.dtype = np.dtype(dtype)
    self.code = _shim.dtype_code(self.dtype)
    self.num_mips = int(num_mips)
    self.mesh_shape = tuple(mesh_shape)
    self.resolution = tuple(resolution)
    self.pitch, self.num_ids, self.seed, self.offset = pitch, num_ids, seed, tuple(offset)
    self.id_base = int(id_base)
    self.ccl_out_dtype = np.dtype(ccl_out_dtype)
    self.simplification_factor = simplification_factor
    self.max_simplification_error = max_simplification_error
    self.group = group
    sx, sy, sz = self.shape
    self.n = sx * sy * sz
    es = self.dtype.itemsize
    self.d_in = ctx.alloc(self.n * es)
    self.mip_shapes = []
    x, y = sx, sy
    for _ in range(self.num_mips):
      x, y = (x + 1) // 2, (y + 1) // 2
      self.mip_shapes.append((x, y, sz))
    self.d_mips = [ctx.alloc(int(np.prod(s)) * es) for s in self.mip_shapes]
    self.d_cc = ctx.alloc(self.n * self.ccl_out_dtype.itemsize)
    mx, my, mz = self.mesh_shape
    self.d_task = ctx.alloc((mx + 1) * (my + 1) * (mz + 1) * es)
    # MeshTask bodies are independent and latency bound (sorts, simplification
    # rounds): run several of them concurrently, each on its own ign_ctx (own
    # stream, scratch arena and mesher pool) of the same device.
    # The main context's stream is left free during the mesh stage so that the D2H
    # of the CCL labels / mips (e2e) overlaps with meshing.
    self.mesh_streams = max(1, int(mesh_streams))
    # Whole-volume passes (pooling, CCL) run on a high-priority stream: their thread blocks are
    # dispatched first whenever a MeshTask CTA retires (k_simp_labels runs one label per CTA), so the
    # CCL is not stretched over the mesh stage it shares the SMs with.  A second context
    # drains finished products to the host while the main stream keeps uploading / computing.
    ctx.set_priority(True)
    self._dl = _shim.Context(ctx.device)
    self._workers = []
    for _ in range(self.mesh_streams):
      wctx = _shim.Context(ctx.device)
      self._workers.append((wctx, wctx.alloc((mx + 1) * (my + 1) * (mz + 1) * es)))
    self.n_components = 0
    self.mesh_stats = {}
    self.mesh_task_counts = np.zeros((0, 5), dtype=np.int64)

  def free(self):
    for b in [self.d_in, self.d_cc, self.d_task] + self.d_mips:
      b.free()
    for wctx, buf in self._workers:
      buf.free()
      wctx.close()
    self._dl.close()

  # ------------------------------------------------------------------ inputs
  def synth(self):
    sx, sy, sz = self.shape
    ox, oy, oz = self.offset
    _shim.check(self.lib.ign_synth_seg_dev(self.ctx.handle, _shim.ptr(self.d_in), self.code, sx, sy, sz, ox, oy, oz,
                                           self.pitch, self.num_ids, self.seed, self.id_base))

  def load_host(self, arr):
    self.ctx.h2d(self.d_in, arr)

  # ------------------------------------------------------------------ stages
  def pool(self):
    sx, sy, sz = self.shape
    if self.num_mips:
      _shim.check(self.lib.ign_pool_mode_2x2x1_dev(self.ctx.handle, _shim.ptr(self.d_in), self.code, sx, sy, sz,
                                                   self.num_mips, 0, _shim.void_pp([m.ptr for m in self.d_mips])))
    self.ctx.timer_start(15)  # "mips ready" mark for the mesh streams

  def ccl(self):
    sx, sy, sz = self.shape
    n = c.c_uint64(0)
    if self.group is not None:
      n_glob = self.group.ccl_sharded(self, n)
      self.n_components = n_glob
      return
    _shim.check(self.lib.ign_ccl6_volume_dev(self.ctx.handle, _shim.ptr(self.d_in), self.code, sx, sy, sz,
                                             _shim.ptr(self.d_cc), _shim.dtype_code(self.ccl_out_dtype), c.byref(n)))
    self.n_components = int(n.value)

  def mesh_tasks(self):
    """(x0,y0,z0,bx,by,bz) cutouts of the mesh mip: task shape + 1 voxel high padding
    (igneous/tasks/mesh/mesh.py:158-160), clamped to the volume."""
    msx, msy, msz = self.mip_shapes[-1] if self.num_mips else self.shape
    mx, my, mz = self.mesh_shape
    for z0 in range(0, msz, mz):
      for y0 in range(0, msy, my):
        for x0 in range(0, msx, mx):
          yield (x0, y0, z0, min(mx + 1, msx - x0), min(my + 1, msy - y0), min(mz + 1, msz - z0))

  def _mesh_one(self, wctx, d_task, task, export):
    lib = wctx.lib
    src = self.d_mips[-1] if self.num_mips else self.d_in
    msx, msy, msz = self.mip_shapes[-1] if self.num_mips else self.shape
    x0, y0, z0, bx, by, bz = task
    _shim.check(lib.ign_copy_box_dev(wctx.handle, _shim.ptr(src), self.code, msx, msy, msz, x0, y0, z0, bx, by, bz,
                                     _shim.ptr(d_task)))
    h = c.c_void_p()
    _shim.check(lib.ign_mesh_begin_dev(wctx.handle, _shim.ptr(d_task), self.code, bx, by, bz, c.byref(h)))
    try:
      nv0, nf0 = c.c_uint64(0), c.c_uint64(0)
      _shim.check(lib.ign_mesh_totals(h, c.byref(nv0), c.byref(nf0)))  # marching-cubes output (host counters)
      if self.simplification_factor and self.simplification_factor > 0:
        _shim.check(lib.ign_mesh_simplify(h, (c.c_float * 3)(*[float(r) for r in self.resolution]),
                                          int(self.simplification_factor), float(self.max_simplification_error)))
      nv, nf, nl = c.c_uint64(0), c.c_uint64(0), c.c_uint64(0)
      _shim.check(lib.ign_mesh_totals(h, c.byref(nv), c.byref(nf)))
      _shim.check(lib.ign_mesh_num_ids(h, c.byref(nl)))
      if export is not None:
        export(task, h, int(nv.value), int(nf.value), int(nl.value), wctx)
      return int(nf.value), int(nv.value), int(nl.value), int(nf0.value), int(nv0.value)
    finally:
      lib.ign_mesh_free(h)

  def mesh(self, export=None, wait_for=None):
    """MeshTask bodies over the mesh mip.  `export(task, mesher, nv, nf, nl, ctx)` may
    pull results to the host (e2e); without it only the totals are read back.
    `wait_for(task)` (streamed step) blocks the calling mesh thread until the host
    has enqueued the mip planes the task reads and returns the event slot recorded after
    them; the mesh stream then waits on the device for exactly that event (not for whatever
    the main stream has enqueued since)."""
    tasks = list(self.mesh_tasks())
    if wait_for is None:
      for wctx, _ in self._workers:  # mesh streams start when the mip pyramid is complete
        _shim.check(self.lib.ign_stream_wait_mark(wctx.handle, self.ctx.handle, 15))
    results = []
    from concurrent.futures import ThreadPoolExecutor

    def run(widx):
      wctx, buf = self._workers[widx]
      out = []
      for i in range(widx, len(tasks), self.mesh_streams):
        t = tasks[i]
        if wait_for is not None:
          mark = wait_for(t)  # the mark the main stream recorded after the last layer this task reads
          _shim.check(self.lib.ign_stream_wait_mark(wctx.handle, self.ctx.handle, mark))
        out.append((i, self._mesh_one(wctx, buf, t, export)))
      wctx.sync()
      return out
    if self.mesh_streams == 1:
      results = run(0)
    else:
      with ThreadPoolExecutor(max_workers=self.mesh_streams) as ex:
        for part in ex.map(run, range(self.mesh_streams)):
          results.extend(part)
    # per task, in mesh_tasks() order: (triangles, vertices, label fragments, triangles in, vertices in)
    self.mesh_task_counts = np.array([r for _, r in sorted(results)], dtype=np.int64).reshape(-1, 5)
    results = [r for _, r in results]
    self.mesh_stats = {"tasks": len(tasks), "triangles": int(sum(r[0] for r in results)),
                       "vertices": int(sum(r[1] for r in results)),
                       "label_fragments": int(sum(r[2] for r in results)),
                       "triangles_in": int(sum(r[3] for r in results)), "vertices_in": int(sum(r[4] for r in results)),
                       "streams": self.mesh_streams}

  def launch_count(self):
    return self.ctx.launch_count() + sum(w[0].launch_count() for w in self._workers)

  def step(self, timers=True):
    """One pass of the hot path over the resident volume."""
    ctx = self.ctx
    if timers:
      ctx.timer_start(1)
    self.pool()
    if timers:
      ctx.timer_stop(1)
      ctx.timer_start(2)
    self.ccl()
    if timers:
      ctx.timer_stop(2)
      ctx.timer_start(3)
    self.mesh()
    if timers:
      ctx.timer_stop(3)

  def step_streamed(self, host_in, host_out=None, export=None):
    """One pass of the hot path from a HOST volume: the volume is uploaded in z-layers
    of the mesh task height; each layer is pooled as soon as it has landed (2x2x1
    pooling never mixes z planes) and the MeshTasks of a layer start when the layer
    above it is pooled (they read one plane of it: mesh.py:158-160 high padding), so
    meshing overlaps the rest of the upload, the CCL passes and the D2H of the
    products.  Results are identical to load_host() + step()."""
    import threading
    sx, sy, sz = self.shape
    es = self.dtype.itemsize
    mz = self.mesh_shape[2]
    # upload granularity: a quarter of the mesh task height -- a task needs its own planes and ONE plane
    # of the layer above, so it can start after 5 quarter-layers instead of 2 whole layers
    lz = max(1, mz // 4)
    n_layers = -(-sz // lz)
    cond = threading.Condition()
    state = {"ready": 0, "error": None}

    def layer_mark(k):  # one event per layer (slots 16..63; a reused slot only makes a late waiter wait longer)
      return 16 + k % 48

    def wait_for(task):
      top = min(sz, task[2] + task[5])          # first plane the task does not read (2x2x1 pooling keeps z)
      need = min(n_layers, -(-top // lz))
      with cond:
        cond.wait_for(lambda: state["ready"] >= need or state["error"] is not None)
        if state["error"] is not None:
          raise RuntimeError("upload failed") from state["error"]
      return layer_mark(need - 1)

    mesh_err = []

    def mesh_thread():
      try:
        self.mesh(export=export, wait_for=wait_for)
      except BaseException as e:  # re-raised on the caller's thread
        mesh_err.append(e)

    import os, time
    trace = os.environ.get("IGN_PIPE_TRACE") is not None
    # finished products are downloaded on a second context's stream while the main stream keeps
    # uploading / computing (ign_d2h only enqueues)
    def download(mark, dst, srcp, nbytes):
      _shim.check(self.lib.ign_stream_wait_mark(self._dl.handle, self.ctx.handle, mark))
      _shim.check(self.lib.ign_d2h(self._dl.handle, dst, srcp, nbytes))

    t_host0 = time.perf_counter()
    th = threading.Thread(target=mesh_thread)
    th.start()
    try:
      src = host_in.ctypes.data
      if trace:
        self.ctx.timer_start(10)
      for k in range(n_layers):
        z0, z1 = k * lz, min(sz, (k + 1) * lz)
        off = z0 * sx * sy * es
        _shim.check(self.lib.ign_h2d(self.ctx.handle, self.d_in.ptr + off, src + off, (z1 - z0) * sx * sy * es))
        if self.num_mips:
          outs = [m.ptr + z0 * s[0] * s[1] * es for m, s in zip(self.d_mips, self.mip_shapes)]
          _shim.check(self.lib.ign_pool_mode_2x2x1_dev(self.ctx.handle, self.d_in.ptr + off, self.code, sx, sy, z1 - z0,
                                                       self.num_mips, 0, _shim.void_pp(outs)))
        self.ctx.timer_start(layer_mark(k))
        if host_out is not None and self.num_mips:
          # the mip planes of this layer are final: download them now (the D2H engine is idle
          # while the volume is still being uploaded), on the second context's stream
          for dst, m, s3 in zip(host_out["mips"], self.d_mips, self.mip_shapes):
            o = z0 * s3[0] * s3[1] * es
            download(layer_mark(k), dst.ctypes.data + o, m.ptr + o, (z1 - z0) * s3[0] * s3[1] * es)
        with cond:
          state["ready"] = k + 1
          cond.notify_all()
      if trace:
        self.ctx.timer_stop(10)
        self.ctx.timer_start(11)
      self.ccl()
      if trace:
        self.ctx.timer_stop(11)
        self.ctx.timer_start(12)
      if host_out is not None:
        self.ctx.timer_start(14)
        download(14, host_out["cc"].ctypes.data, self.d_cc.ptr, host_out["cc"].nbytes)
      if trace:
        self.ctx.timer_stop(12)
    except BaseException as e:
      with cond:
        state["error"] = e
        cond.notify_all()
      th.join()
      raise
    th.join()
    t_mesh = time.perf_counter()
    if mesh_err:
      raise mesh_err[0]
    self._dl.sync()
    self.ctx.sync()
    if trace:
      import sys
      print("step_streamed: upload+pool %.0f ms, ccl %.0f ms, (label d2h queued %.0f ms) (stream time); mesh threads done at %.0f ms, "
            "all done at %.0f ms (host clock)" % (self.ctx.timer_ms(10), self.ctx.timer_ms(11), self.ctx.timer_ms(12),
                                                  1e3 * (t_mesh - t_host0), 1e3 * (time.perf_counter() - t_host0)), file=sys.stderr)

  def stage_ms(self):
    return {"pool_ms": self.ctx.timer_ms(1), "ccl_ms": self.ctx.timer_ms(2),
            "mesh_ms": self.ctx.timer_ms(3)}

  # --------------------------------------------------------------- profiling
  def prof_enable(self, on=True):
    for ctx in [self.ctx] + [w[0] for w in self._workers]:
      _shim.check(self.lib.ign_prof_enable(ctx.handle, int(on)))

  def prof_read(self):
    """(total ms, launches) per kernel class, summed over the main context and the mesh
    streams (kernels of different mesh streams overlap: their sum can exceed the wall time)."""
    out = {}
    for name, cls in PROF_CLASSES.items():
      tot, n = 0.0, 0
      for ctx in [self.ctx] + [w[0] for w in self._workers]:
        ms, cnt = c.c_float(0), c.c_uint64(0)
        _shim.check(self.lib.ign_prof_read(ctx.handle, cls, c.byref(ms), c.byref(cnt)))
        tot += float(ms.value)
        n += int(cnt.value)
      out[name] = (tot, n)
    return out

  # ------------------------------------------------------------- host results
  def results_to_host(self, host):
    """D2H of every product of one step into preallocated (pinned) arrays."""
    for dst, src in zip(host["mips"], self.d_mips):
      self.ctx.d2h(dst, src)
    self.ctx.d2h(host["cc"], self.d_cc)
