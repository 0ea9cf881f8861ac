// common.cuh -- shared host/device helpers for libigneous_b200 (sm_90a only)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include <vector>

#include "../../include/igneous_b200.h"

#if defined(__CUDA_ARCH__) && (__CUDA_ARCH__ != 900)
#error "libigneous_b200 targets sm_90a (Hopper H100) only"
#endif

namespace ign {

void set_error(const char* fmt, ...);

#define IGN_CUDA(call)                                                          \
  do {                                                                          \
    cudaError_t _e = (call);                                                    \
    if (_e != cudaSuccess) {                                                    \
      ign::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call,              \
                     cudaGetErrorString(_e));                                   \
      return IGN_ERR_CUDA;                                                      \
    }                                                                           \
  } while (0)

#define IGN_TRY(call)                 \
  do {                                \
    int _s = (call);                  \
    if (_s != IGN_OK) return _s;      \
  } while (0)

#define IGN_REQUIRE(cond, status, ...)   \
  do {                                   \
    if (!(cond)) {                       \
      ign::set_error(__VA_ARGS__);       \
      return (status);                   \
    }                                    \
  } while (0)

static inline int dtype_size(int dt) {
  switch (dt) {
    case IGN_U8: return 1;
    case IGN_U16: return 2;
    case IGN_U32: return 4;
    case IGN_U64: return 8;
    case IGN_F32: return 4;
    default: return 0;
  }
}

// Calls f(T{}) with T the unsigned type of label dtype IGN_U8 / U16 / U32 / U64 and returns what f
// returns; any other code is IGN_ERR_UNSUPPORTED, reported as `who`'s.
template <typename F>
int dispatch_label(int dtype, const char* who, F&& f) {
  switch (dtype) {
    case IGN_U8: return f(uint8_t{});
    case IGN_U16: return f(uint16_t{});
    case IGN_U32: return f(uint32_t{});
    case IGN_U64: return f(uint64_t{});
  }
  set_error("%s: unsupported label dtype %d", who, dtype);
  return IGN_ERR_UNSUPPORTED;
}

// f(T{}) with T the element type of dtype: the label types, and float for IGN_F32 (whose comparisons
// then follow float rules, as numpy's do)
template <typename F>
int dispatch_chunk(int dtype, const char* who, F&& f) {
  if (dtype == IGN_F32) return f(float{});
  return dispatch_label(dtype, who, f);
}

}  // namespace ign

constexpr int IGN_TIMER_SLOTS = 64;  // CUDA event pairs per context: timers and cross-stream marks

struct ign_ctx {
  int device;
  int sm_count;
  cudaStream_t stream;
  cudaStream_t copy_stream;
  // device scratch arena, bump allocated through ign::ScratchFrame
  struct ScratchBlock { char* base; size_t bytes, used; };
  std::vector<ScratchBlock> scratch;  // normally one block
  size_t scratch_lin;                 // bytes taken, as if the blocks were one
  size_t scratch_high;                // largest scratch_lin reached: the size a coalesced block needs
  int scratch_frames;                 // open frames
  char* pinned;  // staging for scalars / small results
  size_t pinned_bytes;
  cudaEvent_t timers[IGN_TIMER_SLOTS][2];
  uint64_t launches;
  // optional per-kernel-class profiling (ign_prof_enable): CUDA events recorded
  // on the ctx stream around selected launches
  int prof_on;
  struct ProfRec { int cls; cudaEvent_t a, b; };
  ProfRec* prof;
  int prof_n, prof_cap;
  // grow-only pool for the result buffers of the (normally single) live mesher:
  // cudaMalloc/cudaFree per task serialise on the driver lock
  char* mesh_pool;
  size_t mesh_pool_bytes;
  int mesh_pool_busy;
  // mapped pinned window for small control transfers (see ign::small_d2h)
  char* win;      // host address
  char* win_dev;  // the same bytes as seen by kernels
  size_t win_fetch_used, win_push_used;
  struct FetchRec { void* dst; size_t off, bytes; };
  FetchRec fetch[32];
  int fetch_n;
};

enum { IGN_PROF_CCL_LOCAL = 0, IGN_PROF_CCL_MERGE = 1, IGN_PROF_CCL_LABEL = 2, IGN_PROF_POOL = 3,
       IGN_PROF_MC = 4, IGN_PROF_SIMP = 5, IGN_PROF_CLASSES = 8 };

namespace ign {

// Make `ctx->device` current (one ctx per process is the contract, but be safe).
int activate(ign_ctx* ctx);
// A scope of device scratch.  Opening a frame records the arena's bump offsets and closing
// it restores them, on every return path, so what a frame takes lives exactly as long
// as the frame.  Frames nest and close in reverse order: a nested call opens its own frame on
// top of its caller's.  A take goes to the first device block with room at its end, else to a
// new block of its own size (rounded up to 1 MiB), so nothing an open frame has taken is ever
// moved or freed.  When the last frame closes on an arena of several blocks, the stream is synchronised
// and the blocks are replaced by one block of the high-water size: calls of the same shapes then
// bump-allocate from one block without cudaMalloc, cudaFree or a synchronisation.
class ScratchFrame {
 public:
  explicit ScratchFrame(ign_ctx* ctx);
  ~ScratchFrame();
  ScratchFrame(const ScratchFrame&) = delete;
  ScratchFrame& operator=(const ScratchFrame&) = delete;
  // *p = 256-byte aligned room for `bytes` bytes, or for `count` elements of T
  int take(void** p, size_t bytes);
  template <typename T>
  int take(T** p, size_t count) { return take((void**)p, count * sizeof(T)); }
  // release everything taken in this frame (a data-dependent retry starts over)
  void rewind();
  // no frame opened after this one is still open
  bool innermost() const;

 private:
  ign_ctx* ctx_;
  std::vector<size_t> mark_;  // `used` of every block when the frame opened
  size_t mark_lin_;
  int depth_;
};

static inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// One host buffer of a host-buffer entry point.  `from` is copied to the device before the call and
// the device buffer back to `to` after it; both set = one device buffer used in place, both null = the
// call gets a null pointer.  The call may lower `bytes` of an output whose size only its result gives.
struct HostBuf {
  const void* from;
  void* to;
  size_t bytes;
};

// Runs call(d) on device buffers d[i] for bufs[i], taken from one ScratchFrame, and returns its status.
// The copies are cudaMemcpyAsync on the ctx stream; after a successful call the outputs are copied
// back and the stream is synchronised, after a failed one nothing is copied back.
template <typename F>
int staged(ign_ctx* ctx, std::vector<HostBuf>& bufs, F&& call) {
  IGN_TRY(activate(ctx));
  ScratchFrame f(ctx);
  std::vector<void*> d(bufs.size(), nullptr);
  for (size_t i = 0; i < bufs.size(); i++) {
    if (!bufs[i].from && !bufs[i].to) continue;
    IGN_TRY(f.take(&d[i], bufs[i].bytes));
    if (bufs[i].from)
      IGN_CUDA(cudaMemcpyAsync(d[i], bufs[i].from, bufs[i].bytes, cudaMemcpyHostToDevice, ctx->stream));
  }
  IGN_TRY(call(d.data()));
  for (size_t i = 0; i < bufs.size(); i++)
    if (bufs[i].to) IGN_CUDA(cudaMemcpyAsync(bufs[i].to, d[i], bufs[i].bytes, cudaMemcpyDeviceToHost, ctx->stream));
  IGN_CUDA(cudaStreamSynchronize(ctx->stream));
  return IGN_OK;
}
template <typename F>
int staged(ign_ctx* ctx, std::vector<HostBuf>&& bufs, F&& call) {
  return staged(ctx, bufs, call);
}

// Small control transfers (counters, per-label offset tables) that sit between kernels
// of one call.  cudaMemcpyAsync would put them on a copy engine, where they queue behind
// multi-GB transfers issued by other contexts of the same device (the volume upload /
// label download that overlap the mesh stage).  Instead a copy kernel on the ctx stream
// moves them through a mapped pinned window, so only the SMs and the stream order are
// involved.  Transfers that do not fit the window fall back to cudaMemcpyAsync.
//   small_d2h: host_dst is valid after small_sync().
//   small_h2d: host_src is consumed before the call returns.
//   small_sync: cudaStreamSynchronize(ctx->stream) + delivery of pending small_d2h results.
int small_d2h(ign_ctx* ctx, void* host_dst, const void* dev_src, size_t bytes);
// bulk device -> pinned host copy issued as a kernel on the ctx stream (falls back to the copy engine for pageable memory)
int d2h_by_kernel(ign_ctx* ctx, void* host_dst, const void* dev_src, size_t bytes);
int small_h2d(ign_ctx* ctx, void* dev_dst, const void* host_src, size_t bytes);
int small_sync(ign_ctx* ctx);

// launch bookkeeping: every kernel launch in this library goes through
// IGN_LAUNCH so ign_launch_count() is exact.
#define IGN_LAUNCH(ctx, kernel, grid, block, smem, ...)                          \
  do {                                                                           \
    kernel<<<(grid), (block), (smem), (ctx)->stream>>>(__VA_ARGS__);             \
    (ctx)->launches++;                                                           \
    IGN_CUDA(cudaGetLastError());                                                \
  } while (0)

// profiled launch: like IGN_LAUNCH, plus an event pair when profiling is on
int prof_begin(ign_ctx* ctx, int cls);
void prof_end(ign_ctx* ctx, int slot);
// event pair around the work a scope enqueues on ctx->stream (end() closes it early)
struct ProfSpan {
  ign_ctx* ctx;
  int slot;
  ProfSpan(ign_ctx* c, int cls) : ctx(c), slot(prof_begin(c, cls)) {}
  void end() {
    prof_end(ctx, slot);
    slot = -1;
  }
  ~ProfSpan() { end(); }
};
#define IGN_LAUNCH_PROF(ctx, cls, kernel, grid, block, smem, ...)                 \
  do {                                                                           \
    const int _slot = ign::prof_begin((ctx), (cls));                             \
    kernel<<<(grid), (block), (smem), (ctx)->stream>>>(__VA_ARGS__);             \
    (ctx)->launches++;                                                           \
    ign::prof_end((ctx), _slot);                                                 \
    IGN_CUDA(cudaGetLastError());                                                \
  } while (0)

static inline unsigned blocks_for(uint64_t n, unsigned threads) {
  return (unsigned)((n + threads - 1) / threads);
}

}  // namespace ign

// ------------------------------------------------------------------ device
#ifdef __CUDACC__
namespace ign {

__device__ __forceinline__ uint4 ld_stream(const void* p) {
  // streaming 128-bit load: read-only path, do not allocate in L1
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ void st_stream(void* p, uint4 v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x),
               "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}
__device__ __forceinline__ void st_stream(void* p, uint2 v) {
  asm volatile("st.global.L1::no_allocate.v2.u32 [%0], {%1,%2};" ::"l"(p), "r"(v.x), "r"(v.y)
               : "memory");
}

__device__ __forceinline__ uint64_t mix64(uint64_t z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

}  // namespace ign
#endif
