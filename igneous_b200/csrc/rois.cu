// rois.cu -- the device half of compute_rois: threshold a slab, then the boxes of its 26-connected parts
//
// compute_rois (igneous/task_creation/image.py:1995-2058) thresholds each z slab of the top mip, labels it
// with cc3d (26-connected), drops dust and keeps cc3d.statistics' bounding boxes.  Only the boxes are
// wanted, so nothing per voxel leaves the device:
//   init    L[i] = i on a non-zero voxel, BG elsewhere
//   merge   union-find over the 13 neighbours that come earlier in F order; a union links the larger
//           root under the smaller (atomicMin), so every root is its component's smallest F-order index
//   flatten L[i] = root
//   roots   the roots in ascending order (per-segment counts, cub scan): a component's rank among them
//           is cc3d's label
//   stats   per component {count, min x, min y, min z, max x, max y, max z} from runs along x: a thread
//           walks 32 voxels of one row and issues its atomics once per run of one component
//   dust    the rows of components of at least dust_threshold voxels, in rank order (flags, cub scan)
// L holds 32-bit voxel indices: a slab of 2^32 - 1 voxels or more is refused.
#include <string.h>

#include <cub/cub.cuh>

#include <algorithm>
#include <type_traits>

#include "common.cuh"

namespace ign {

namespace {

constexpr uint32_t kBg = 0xFFFFFFFFu;
constexpr int kSeg = 32;  // voxels of a row one stats thread walks

struct BoxRow {
  uint32_t w[IGN_BOX_ROW];  // count, min x, min y, min z, max x, max y, max z
};

template <typename T>
__global__ void __launch_bounds__(256) k_threshold(const T* __restrict__ in, uint64_t n, T t, uint8_t* __restrict__ out) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    out[i] = in[i] > t;
}

__global__ void __launch_bounds__(256) k_uf_init(const uint8_t* __restrict__ mask, uint64_t n, uint32_t* __restrict__ L) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    L[i] = mask[i] ? (uint32_t)i : kBg;
}

// links only ever point to smaller indices, so the walk ends; L2 reads (__ldcg) see other SMs' links sooner
__device__ __forceinline__ uint32_t uf_find(const uint32_t* L, uint32_t i) {
  uint32_t p = __ldcg(L + i);
  while (p != i) {
    i = p;
    p = __ldcg(L + i);
  }
  return i;
}

// Playne & Hawick's lock-free union: link the larger root under the smaller; when the atomic finds the
// larger one already linked elsewhere, carry on with what it was linked to
__device__ __forceinline__ void uf_union(uint32_t* L, uint32_t a, uint32_t b) {
  bool done;
  do {
    a = uf_find(L, a);
    b = uf_find(L, b);
    if (a < b) {
      const uint32_t old = atomicMin(L + b, a);
      done = old == b;
      b = old;
    } else if (b < a) {
      const uint32_t old = atomicMin(L + a, b);
      done = old == a;
      a = old;
    } else {
      done = true;
    }
  } while (!done);
}

// One thread per voxel.  The neighbours before (x, y, z) in F order are (x-1, y, z), (x-1..x+1, y-1, z) and
// (x-1..x+1, y-1..y+1, z-1).  When (x-1, y, z) is set and joined, the neighbours it shares with (x, y, z)
// are joined through it, which leaves (x+1, y-1, z) and (x+1, y-1..y+1, z-1).
__global__ void __launch_bounds__(256) k_uf_merge(const uint8_t* __restrict__ mask, uint64_t sx, uint64_t sy,
                                                 uint64_t sz, uint32_t* L) {
  const uint64_t n = sx * sy * sz, sxy = sx * sy;
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    if (!mask[i]) continue;
    const uint64_t x = i % sx, y = (i / sx) % sy, z = i / sxy;
    const bool left = x > 0 && mask[i - 1];
    if (left) uf_union(L, (uint32_t)i, (uint32_t)(i - 1));
    const int64_t dx0 = left ? 1 : -1;
    for (int64_t dz = -1; dz <= 0; dz++) {
      if (dz < 0 && z == 0) continue;
      for (int64_t dy = -1; dy <= (dz < 0 ? 1 : -1); dy++) {
        if ((dy < 0 && y == 0) || (dy > 0 && y + 1 == sy)) continue;
        for (int64_t dx = dx0; dx <= 1; dx++) {
          if ((dx < 0 && x == 0) || (dx > 0 && x + 1 == sx)) continue;
          const uint64_t j = (uint64_t)((int64_t)i + dx + dy * (int64_t)sx + dz * (int64_t)sxy);
          if (mask[j]) uf_union(L, (uint32_t)i, (uint32_t)j);
        }
      }
    }
  }
}

__global__ void __launch_bounds__(256) k_uf_flatten(uint64_t n, uint32_t* L) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    if (__ldcg(L + i) != kBg) L[i] = uf_find(L, (uint32_t)i);
}

// per segment of kSeg voxels of a row (segments in F order): WRITE = false counts its roots into cnt
// (cnt[segments] = 0 closes the table), WRITE = true writes them in order from roots[at[segment]]
template <bool WRITE>
__global__ void __launch_bounds__(256) k_seg_roots(const uint32_t* __restrict__ L, uint64_t sx, uint64_t rows,
                                                  uint32_t* __restrict__ cnt, const uint32_t* __restrict__ at,
                                                  uint32_t* __restrict__ roots) {
  const uint64_t segs = (sx + kSeg - 1) / kSeg, total = segs * rows;
  for (uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; t <= total; t += (uint64_t)gridDim.x * blockDim.x) {
    if (t == total) {
      if (!WRITE) cnt[t] = 0;
      continue;
    }
    const uint64_t row = t / segs, x0 = (t % segs) * kSeg, x1 = std::min<uint64_t>(x0 + kSeg, sx);
    uint32_t c = 0;
    for (uint64_t i = row * sx + x0; i < row * sx + x1; i++) {
      if (L[i] != (uint32_t)i) continue;
      if (WRITE) roots[at[t] + c] = (uint32_t)i;
      c++;
    }
    if (!WRITE) cnt[t] = c;
  }
}

__global__ void __launch_bounds__(256) k_keep_flags(const BoxRow* __restrict__ rows, uint64_t k, uint64_t threshold,
                                                   uint32_t* __restrict__ keep) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i <= k; i += (uint64_t)gridDim.x * blockDim.x)
    keep[i] = i < k && rows[i].w[0] >= threshold;
}

__global__ void __launch_bounds__(256) k_keep_rows(const BoxRow* __restrict__ rows, uint64_t k,
                                                  const uint32_t* __restrict__ keep, const uint32_t* __restrict__ at,
                                                  BoxRow* __restrict__ out) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < k; i += (uint64_t)gridDim.x * blockDim.x)
    if (keep[i]) out[at[i]] = rows[i];
}

__global__ void __launch_bounds__(256) k_rows_init(BoxRow* rows, uint64_t k) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < k; i += (uint64_t)gridDim.x * blockDim.x) {
    BoxRow r;
    r.w[0] = 0;
    r.w[1] = r.w[2] = r.w[3] = kBg;
    r.w[4] = r.w[5] = r.w[6] = 0;
    rows[i] = r;
  }
}

// the rank of root r among the k roots (ascending, r is one of them)
__device__ __forceinline__ uint32_t root_rank(const uint32_t* roots, uint32_t k, uint32_t r) {
  uint32_t lo = 0, hi = k;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (roots[mid] < r) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

__device__ __forceinline__ void flush_run(BoxRow* rows, const uint32_t* roots, uint32_t k, uint32_t root, uint32_t cnt,
                                          uint32_t xa, uint32_t xb, uint32_t y, uint32_t z) {
  uint32_t* w = rows[root_rank(roots, k, root)].w;
  atomicAdd(w + 0, cnt);
  atomicMin(w + 1, xa);
  atomicMin(w + 2, y);
  atomicMin(w + 3, z);
  atomicMax(w + 4, xb);
  atomicMax(w + 5, y);
  atomicMax(w + 6, z);
}

__global__ void __launch_bounds__(256) k_box_stats(const uint32_t* __restrict__ L, uint64_t sx, uint64_t sy, uint64_t sz,
                                                  const uint32_t* __restrict__ roots, uint32_t k, BoxRow* rows) {
  const uint64_t segs = (sx + kSeg - 1) / kSeg, total = segs * sy * sz;
  for (uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; t < total; t += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t s = t % segs, row = t / segs;
    const uint32_t y = (uint32_t)(row % sy), z = (uint32_t)(row / sy);
    const uint64_t x0 = s * kSeg, x1 = std::min<uint64_t>(x0 + kSeg, sx);
    const uint32_t* line = L + row * sx;
    uint32_t cur = kBg, cnt = 0, xa = 0, xb = 0;
    for (uint64_t x = x0; x < x1; x++) {
      const uint32_t r = line[x];
      if (r != cur) {
        if (cur != kBg) flush_run(rows, roots, k, cur, cnt, xa, xb, y, z);
        cur = r;
        cnt = 0;
        xa = (uint32_t)x;
      }
      if (r != kBg) {
        cnt++;
        xb = (uint32_t)x;
      }
    }
    if (cur != kBg) flush_run(rows, roots, k, cur, cnt, xa, xb, y, z);
  }
}

static unsigned grid_for(ign_ctx* ctx, uint64_t n) {
  return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(blocks_for(n, 256), (uint64_t)ctx->sm_count * 32));
}

}  // namespace

}  // namespace ign

using namespace ign;

extern "C" {

int ign_threshold_dev(ign_ctx* ctx, const void* in, int dtype, uint64_t n, uint64_t t, uint8_t* out) {
  IGN_TRY(activate(ctx));
  IGN_REQUIRE(n == 0 || (in && out), IGN_ERR_INVALID, "threshold: null buffer");
  return dispatch_chunk(dtype, "threshold", [&](auto v) -> int {
    using T = decltype(v);
    if (n == 0) return IGN_OK;
    T tt;
    if constexpr (std::is_same<T, float>::value) {
      const uint32_t bits = (uint32_t)t;
      memcpy(&tt, &bits, 4);
    } else if (t > (uint64_t)(T)~(T)0) {  // above every value of T: nothing is greater
      IGN_CUDA(cudaMemsetAsync(out, 0, n, ctx->stream));
      return IGN_OK;
    } else {
      tt = (T)t;
    }
    IGN_LAUNCH(ctx, k_threshold<T>, grid_for(ctx, n), 256, 0, (const T*)in, n, tt, out);
    return IGN_OK;
  });
}

int ign_mask_boxes_dev(ign_ctx* ctx, const uint8_t* mask, uint64_t sx, uint64_t sy, uint64_t sz,
                       uint64_t dust_threshold, uint32_t* rows, uint64_t capacity, uint64_t* n) {
  IGN_TRY(activate(ctx));
  IGN_REQUIRE(n, IGN_ERR_INVALID, "mask_boxes: null count");
  *n = 0;
  IGN_REQUIRE(sx < (1ull << 32) && sy < (1ull << 32) && sz < (1ull << 32), IGN_ERR_UNSUPPORTED,
              "mask_boxes: a side of %llu x %llu x %llu is 2^32 or more", (unsigned long long)sx,
              (unsigned long long)sy, (unsigned long long)sz);
  const uint64_t nv = sx * sy * sz;
  IGN_REQUIRE(nv < (uint64_t)kBg, IGN_ERR_UNSUPPORTED,
              "mask_boxes: %llu voxels (the labels are 32-bit voxel indices: fewer than 2^32 - 1)",
              (unsigned long long)nv);
  if (nv == 0) return IGN_OK;
  IGN_REQUIRE(mask && (rows || capacity == 0), IGN_ERR_INVALID, "mask_boxes: null buffer");
  ScratchFrame f(ctx);
  uint32_t *L, *roots;
  BoxRow *all, *kept;
  IGN_TRY(f.take(&L, nv));
  const unsigned g = grid_for(ctx, nv);
  IGN_LAUNCH(ctx, k_uf_init, g, 256, 0, mask, nv, L);
  IGN_LAUNCH(ctx, k_uf_merge, g, 256, 0, mask, sx, sy, sz, L);
  IGN_LAUNCH(ctx, k_uf_flatten, g, 256, 0, nv, L);
  // the roots in ascending order: counted per segment, then written at the exclusive sum of the counts
  const uint64_t segs = (sx + kSeg - 1) / kSeg * sy * sz;
  uint32_t *cnt, *at;
  IGN_TRY(f.take(&cnt, segs + 1));
  IGN_TRY(f.take(&at, segs + 1));
  IGN_LAUNCH(ctx, k_seg_roots<false>, grid_for(ctx, segs + 1), 256, 0, L, sx, sy * sz, cnt, nullptr, nullptr);
  size_t tb = 0;
  IGN_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, cnt, at, (int64_t)segs + 1, ctx->stream));
  void* tmp;
  IGN_TRY(f.take(&tmp, tb));
  IGN_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tb, cnt, at, (int64_t)segs + 1, ctx->stream));
  ctx->launches += 2;
  uint32_t hk = 0;
  IGN_TRY(small_d2h(ctx, &hk, at + segs, 4));
  IGN_TRY(small_sync(ctx));
  if (hk == 0) return IGN_OK;
  const uint32_t k = hk;
  IGN_TRY(f.take(&roots, k));
  IGN_LAUNCH(ctx, k_seg_roots<true>, grid_for(ctx, segs), 256, 0, L, sx, sy * sz, nullptr, at, roots);
  IGN_TRY(f.take(&all, k));
  IGN_TRY(f.take(&kept, k));
  IGN_LAUNCH(ctx, k_rows_init, grid_for(ctx, k), 256, 0, all, k);
  IGN_LAUNCH(ctx, k_box_stats, grid_for(ctx, segs), 256, 0, L, sx, sy, sz, roots, k, all);
  // dust: the kept rows, in rank order, at the exclusive sum of their flags (keep[k] = 0: pos[k] = the number kept)
  uint32_t *keep, *pos;
  IGN_TRY(f.take(&keep, (uint64_t)k + 1));
  IGN_TRY(f.take(&pos, (uint64_t)k + 1));
  IGN_LAUNCH(ctx, k_keep_flags, grid_for(ctx, (uint64_t)k + 1), 256, 0, all, k, dust_threshold, keep);
  size_t tb2 = 0;
  IGN_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb2, keep, pos, (int64_t)k + 1, ctx->stream));
  void* tmp2;
  IGN_TRY(f.take(&tmp2, tb2));
  IGN_CUDA(cub::DeviceScan::ExclusiveSum(tmp2, tb2, keep, pos, (int64_t)k + 1, ctx->stream));
  ctx->launches += 2;
  IGN_LAUNCH(ctx, k_keep_rows, grid_for(ctx, k), 256, 0, all, k, keep, pos, kept);
  uint32_t hn = 0;
  IGN_TRY(small_d2h(ctx, &hn, pos + k, 4));
  IGN_TRY(small_sync(ctx));
  *n = (uint64_t)hn;
  if (*n && *n <= capacity) {
    IGN_CUDA(cudaMemcpyAsync(rows, kept, *n * sizeof(BoxRow), cudaMemcpyDeviceToHost, ctx->stream));
    IGN_CUDA(cudaStreamSynchronize(ctx->stream));
  }
  return IGN_OK;
}

}  // extern "C"
