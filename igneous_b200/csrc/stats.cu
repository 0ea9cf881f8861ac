// stats.cu -- per-label bounding boxes of a label volume (scipy.ndimage.find_objects,
// igneous/tasks/spatial_index.py:10-20), sm_90a.
//
//   k_fo_max     largest label, only when the caller does not pass it
//   k_fo_boxes   min / max of x, y and z of every label 1..N, in one read of the volume
//   k_fo_pack    the structure-of-arrays boxes -> [N][6] rows
//
// k_fo_boxes gives each warp tiles of 32 x-adjacent voxels by FO_ROWS consecutive rows (a row
// is one (y, z)).  Per row the warp splits its 32 voxels into runs of equal labels with one
// shuffle and two ballots.  Each lane keeps one open box (label + six bounds) in registers.
// A run goes to the first lane inside it whose open box has the run's label, which widens that
// box; if no lane inside it has one, the run's first lane flushes its own box to global memory
// and opens a new one.  Labels are spatially coherent, so a box usually absorbs the label's
// runs over many rows (one label filling the volume is flushed once per lane); the worst case,
// every voxel its own label, flushes once per voxel, to consecutive addresses.  A flush is six
// atomicMin / atomicMax on a structure of arrays in global memory (one array per bound).
#include <algorithm>

#include "common.cuh"

namespace ign {

namespace {

constexpr int FO_THREADS = 256;
constexpr int FO_WARPS = FO_THREADS / 32;
constexpr uint64_t FO_ROWS = 64;  // rows per tile
constexpr int FO_BATCH = 8;       // rows whose loads are issued together
constexpr uint32_t FULL = 0xFFFFFFFFu;

template <typename T>
__device__ __forceinline__ T ld_label(const T* p) {
  if constexpr (sizeof(T) == 1) return (T)__ldcs((const unsigned char*)p);
  if constexpr (sizeof(T) == 2) return (T)__ldcs((const unsigned short*)p);
  if constexpr (sizeof(T) == 4) return (T)__ldcs((const unsigned int*)p);
  return (T)__ldcs((const unsigned long long*)p);
}

template <typename T>
__device__ __forceinline__ T shfl_up1(T v) {
  if constexpr (sizeof(T) == 8) return (T)__shfl_up_sync(FULL, (unsigned long long)v, 1);
  return (T)__shfl_up_sync(FULL, (unsigned)v, 1);
}

// soa = [min x | min y | min z | max x | max y | max z], N entries each; label l is entry l - 1
__device__ __forceinline__ void fo_flush(uint32_t* soa, uint64_t N, uint32_t label, uint32_t x0, uint32_t x1,
                                         uint32_t y0, uint32_t y1, uint32_t z0, uint32_t z1) {
  uint32_t* p = soa + (label - 1);
  atomicMin(p, x0);
  atomicMin(p + N, y0);
  atomicMin(p + 2 * N, z0);
  atomicMax(p + 3 * N, x1);
  atomicMax(p + 4 * N, y1);
  atomicMax(p + 5 * N, z1);
}

template <typename T>
__global__ void __launch_bounds__(FO_THREADS) k_fo_boxes(const T* __restrict__ in, uint32_t sx, uint32_t sy,
                                                         uint64_t nrows, uint64_t N, uint32_t nxw, uint64_t ntiles,
                                                         uint32_t* __restrict__ soa) {
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t upto = FULL >> (31 - lane);  // lanes 0..lane
  uint32_t open = 0, x0 = 0, x1 = 0, y0 = 0, y1 = 0, z0 = 0, z1 = 0;  // open == 0: no box
  const uint64_t stride = (uint64_t)gridDim.x * FO_WARPS;
  for (uint64_t t = blockIdx.x * (uint64_t)FO_WARPS + (threadIdx.x >> 5); t < ntiles; t += stride) {
    const uint32_t xw = (uint32_t)(t % nxw) * 32;
    const uint64_t r0 = (t / nxw) * FO_ROWS;
    const uint64_t r1 = r0 + FO_ROWS < nrows ? r0 + FO_ROWS : nrows;
    const bool valid = xw + lane < sx;
    const uint32_t last = (sx - xw < 32 ? sx - xw : 32) - 1;  // last valid lane
    uint32_t y = (uint32_t)(r0 % sy), z = (uint32_t)(r0 / sy);
    const T* p = in + r0 * sx + xw + lane;
    for (uint64_t r = r0; r < r1; r += FO_BATCH, p += (uint64_t)FO_BATCH * sx) {
      T v[FO_BATCH];
#pragma unroll
      for (int b = 0; b < FO_BATCH; ++b) v[b] = (valid && r + b < r1) ? ld_label(p + (uint64_t)b * sx) : T(0);
#pragma unroll
      for (int b = 0; b < FO_BATCH; ++b) {
        if (r + b < r1) {  // warp-uniform
          const T lab = v[b];
          const T prev = shfl_up1(lab);
          const uint32_t starts = __ballot_sync(FULL, valid && (lane == 0 || lab != prev));
          const bool hit = valid && open != 0 && lab == (T)open;
          const uint32_t hits = __ballot_sync(FULL, hit);
          const uint32_t head = 31 - __clz(starts & upto);  // lane 0 is valid, so starts & upto != 0
          const uint32_t later = starts & ~upto;
          const uint32_t end = later ? __ffs(later) - 2 : last;
          const uint32_t in_run = hits & (FULL >> (31 - end)) & (FULL << head);
          const uint32_t owner = in_run ? __ffs(in_run) - 1 : head;
          if (valid && owner == lane && lab != 0 && (uint64_t)lab <= N) {
            const uint32_t xa = xw + head, xb = xw + end;
            if (hit) {
              x0 = min(x0, xa);
              x1 = max(x1, xb);
              y0 = min(y0, y);
              y1 = max(y1, y);
              z0 = min(z0, z);
              z1 = max(z1, z);
            } else {
              if (open) fo_flush(soa, N, open, x0, x1, y0, y1, z0, z1);
              open = (uint32_t)lab;
              x0 = xa;
              x1 = xb;
              y0 = y1 = y;
              z0 = z1 = z;
            }
          }
          if (++y == sy) {
            y = 0;
            ++z;
          }
        }
      }
    }
  }
  if (open) fo_flush(soa, N, open, x0, x1, y0, y1, z0, z1);
}

template <typename T>
__global__ void __launch_bounds__(256) k_fo_max(const T* __restrict__ in, uint64_t n,
                                                unsigned long long* __restrict__ out) {
  unsigned long long m = 0;
  for (uint64_t i = blockIdx.x * 256ull + threadIdx.x; i < n; i += (uint64_t)gridDim.x * 256)
    m = max(m, (unsigned long long)ld_label(in + i));
#pragma unroll
  for (int o = 16; o; o >>= 1) m = max(m, __shfl_xor_sync(FULL, m, o));
  if ((threadIdx.x & 31) == 0 && m) atomicMax(out, m);
}

__global__ void __launch_bounds__(256) k_fo_pack(const uint32_t* __restrict__ soa, uint64_t N,
                                                 uint32_t* __restrict__ out) {
  const uint64_t i = blockIdx.x * 256ull + threadIdx.x;
  if (i >= N) return;
#pragma unroll
  for (int k = 0; k < 6; ++k) out[6 * i + k] = soa[k * N + i];
}

template <typename T>
int find_max(ign_ctx* ctx, const void* in, uint64_t n, uint64_t* max_label) {
  ScratchFrame f(ctx);
  unsigned long long* d;
  IGN_TRY(f.take(&d, 1));
  IGN_CUDA(cudaMemsetAsync(d, 0, 8, ctx->stream));
  const unsigned grid = (unsigned)std::min<uint64_t>(blocks_for(n, 256), (uint64_t)ctx->sm_count * 8);
  IGN_LAUNCH(ctx, k_fo_max<T>, grid, 256, 0, (const T*)in, n, d);
  IGN_TRY(small_d2h(ctx, max_label, d, 8));
  return small_sync(ctx);
}

template <typename T>
int find_boxes(ign_ctx* ctx, const void* in, uint64_t sx, uint64_t sy, uint64_t sz, uint64_t N, uint32_t* boxes) {
  ScratchFrame f(ctx);
  uint32_t* soa;
  IGN_TRY(f.take(&soa, 6 * N));
  IGN_CUDA(cudaMemsetAsync(soa, 0xFF, 3 * N * sizeof(uint32_t), ctx->stream));
  IGN_CUDA(cudaMemsetAsync(soa + 3 * N, 0, 3 * N * sizeof(uint32_t), ctx->stream));
  const uint64_t nrows = sy * sz;
  if (sx && nrows) {
    const uint32_t nxw = (uint32_t)((sx + 31) / 32);
    const uint64_t ntiles = nxw * ((nrows + FO_ROWS - 1) / FO_ROWS);
    const unsigned grid = (unsigned)std::min<uint64_t>((ntiles + FO_WARPS - 1) / FO_WARPS, (uint64_t)ctx->sm_count * 8);
    IGN_LAUNCH(ctx, k_fo_boxes<T>, grid, FO_THREADS, 0, (const T*)in, (uint32_t)sx, (uint32_t)sy, nrows, N, nxw,
               ntiles, soa);
  }
  IGN_LAUNCH(ctx, k_fo_pack, blocks_for(N, 256), 256, 0, soa, N, boxes);
  return IGN_OK;
}

int fo_check(int dtype, uint64_t sx, uint64_t sy, uint64_t sz, const uint64_t* max_label) {
  IGN_REQUIRE(dtype == IGN_U8 || dtype == IGN_U16 || dtype == IGN_U32 || dtype == IGN_U64, IGN_ERR_UNSUPPORTED,
              "find_objects: label dtype %d is not u8 / u16 / u32 / u64", dtype);
  IGN_REQUIRE(max_label, IGN_ERR_INVALID, "find_objects: null max_label");
  IGN_REQUIRE(sx < (1ull << 31) && sy < (1ull << 31) && sz < (1ull << 31), IGN_ERR_OVERFLOW,
              "find_objects: volume %llu x %llu x %llu (each side below 2^31)", (unsigned long long)sx,
              (unsigned long long)sy, (unsigned long long)sz);
  IGN_REQUIRE(*max_label < (1ull << 32), IGN_ERR_UNSUPPORTED,
              "find_objects: largest label %llu is 2^32 or more; renumber the labels first (fastremap.renumber)",
              (unsigned long long)*max_label);
  return IGN_OK;
}

}  // namespace

}  // namespace ign

using namespace ign;

extern "C" {

int ign_find_objects_dev(ign_ctx* ctx, const void* labels, int dtype, uint64_t sx, uint64_t sy, uint64_t sz,
                         uint64_t* max_label, uint32_t* boxes) {
  IGN_TRY(activate(ctx));
  IGN_TRY(fo_check(dtype, sx, sy, sz, max_label));
  const uint64_t n = sx * sy * sz;
  IGN_REQUIRE(labels || !n, IGN_ERR_INVALID, "null buffer");
  IGN_REQUIRE((uintptr_t)labels % dtype_size(dtype) == 0, IGN_ERR_INVALID,
              "find_objects: labels not aligned to their element size");
  if (*max_label == 0) {
    if (!n) return IGN_OK;
    IGN_TRY(dispatch_label(dtype, "find_objects",
                           [&](auto v) { return find_max<decltype(v)>(ctx, labels, n, max_label); }));
    return fo_check(dtype, sx, sy, sz, max_label);
  }
  IGN_REQUIRE(boxes, IGN_ERR_INVALID, "null buffer");
  IGN_REQUIRE((uintptr_t)boxes % 4 == 0, IGN_ERR_INVALID, "find_objects: boxes not aligned to 4 bytes");
  const uint64_t N = *max_label;
  return dispatch_label(dtype, "find_objects",
                        [&](auto v) { return find_boxes<decltype(v)>(ctx, labels, sx, sy, sz, N, boxes); });
}

int ign_find_objects(ign_ctx* ctx, const void* labels, int dtype, uint64_t sx, uint64_t sy, uint64_t sz,
                     uint64_t* max_label, uint32_t* boxes) {
  IGN_TRY(fo_check(dtype, sx, sy, sz, max_label));
  const uint64_t n = sx * sy * sz;
  const uint64_t N = *max_label;
  return staged(ctx, {{labels, nullptr, n * dtype_size(dtype)}, {nullptr, N ? boxes : nullptr, N * 24}},
                [&](void* const* d) {
                  return ign_find_objects_dev(ctx, d[0], dtype, sx, sy, sz, max_label, (uint32_t*)d[1]);
                });
}

}  // extern "C"
