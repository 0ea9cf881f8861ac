// parts.cu -- the connected parts of a label volume under 6-, 18- or 26-connectivity (DESIGN.md §5k)
//
// Two neighbours join when they hold the same non-zero label.  Parts are numbered by first voxel in F order
// (cc3d's numbering), parts of fewer than dust_threshold voxels are dropped and the rest keep their order:
//   init    L[i] = i on a non-zero voxel, BG elsewhere
//   merge   union-find over the neighbours that come earlier in F order; a union links the larger root
//           under the smaller (atomicMin), so every root is its part's smallest F-order index
//   flatten L[i] = root
//   roots   the roots in ascending order (per-segment counts, cub scan): a part's rank among them is its
//           number
//   stats   per part {count, min x, min y, min z, max x, max y, max z} from runs along x: a thread walks
//           32 voxels of one row and issues its atomics once per run of one part (only when rows or dust
//           need them)
//   dust    a keep flag per part and their exclusive sum: the kept parts' new ranks, the kept rows in order
//   parts   optional: each voxel's new rank + 1, 0 on label 0 and on dust
// L holds 32-bit voxel indices: a volume of 2^32 - 1 voxels or more is refused.
#include <cub/cub.cuh>

#include <algorithm>

#include "common.cuh"

namespace ign {

namespace {

constexpr uint32_t kBg = 0xFFFFFFFFu;
constexpr int kSeg = 32;  // voxels of a row one stats thread walks

struct BoxRow {
  uint32_t w[IGN_BOX_ROW];  // count, min x, min y, min z, max x, max y, max z
};

template <typename T>
__global__ void __launch_bounds__(256) k_uf_init(const T* __restrict__ lab, uint64_t n, uint32_t* __restrict__ L) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    L[i] = lab[i] ? (uint32_t)i : kBg;
}

// links only ever point to smaller indices, so the walk ends; path halving (each visited entry skips to its
// grandparent, also an ancestor) keeps the chains of a part that fills the volume short; L2 reads (__ldcg)
// see other SMs' links sooner
__device__ __forceinline__ uint32_t uf_find(uint32_t* L, uint32_t i) {
  uint32_t p = __ldcg(L + i);
  while (p != i) {
    const uint32_t g = __ldcg(L + p);
    if (g != p) L[i] = g;  // i is not a root
    i = p;
    p = g;
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

// One thread per voxel.  (dx, dy, dz) is a neighbour when |dx| + |dy| + |dz| <= reach (1, 2, 3 for 6, 18,
// 26); the ones before (x, y, z) in F order are (x-1, y, z), (x-1..x+1, y-1, z) and (x-1..x+1, y-1..y+1, z-1).
// (x-1, y, z) unites with each of its own earlier neighbours of its label.  When it holds this voxel's label,
// those that are neighbours of both, dx <= 0 and |dx + 1| + |dy| + |dz| <= reach, are joined through it:
// that leaves the 4 with dx = 1 at 26, (1, -1, 0), (1, 0, -1), (0, -1, -1), (0, 1, -1) at 18, all 3 at 6.
template <typename T>
__global__ void __launch_bounds__(256) k_uf_merge(const T* __restrict__ lab, uint64_t sx, uint64_t sy, uint64_t sz,
                                                 int reach, uint32_t* L) {
  const uint64_t n = sx * sy * sz, sxy = sx * sy;
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const T l = lab[i];
    if (!l) continue;
    const uint64_t x = i % sx, y = (i / sx) % sy, z = i / sxy;
    const bool left = x > 0 && lab[i - 1] == l;
    if (left) uf_union(L, (uint32_t)i, (uint32_t)(i - 1));
    for (int dz = -1; dz <= 0; dz++) {
      if (dz < 0 && z == 0) continue;
      for (int dy = -1; dy <= (dz < 0 ? 1 : -1); dy++) {
        if ((dy < 0 && y == 0) || (dy > 0 && y + 1 == sy)) continue;
        for (int dx = -1; dx <= 1; dx++) {
          if ((dx < 0 && x == 0) || (dx > 0 && x + 1 == sx)) continue;
          if (abs(dx) + abs(dy) + abs(dz) > reach) continue;
          if (left && dx <= 0 && abs(dx + 1) + abs(dy) + abs(dz) <= reach) continue;
          const uint64_t j = (uint64_t)((int64_t)i + dx + dy * (int64_t)sx + dz * (int64_t)sxy);
          if (lab[j] == l) uf_union(L, (uint32_t)i, (uint32_t)j);
        }
      }
    }
  }
}

// a read-only walk: a halving store here could replace an entry that another thread has already set to its
// root by a mere ancestor
__global__ void __launch_bounds__(256) k_uf_flatten(uint64_t n, uint32_t* L) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t r = __ldcg(L + i);
    if (r == kBg) continue;
    for (uint32_t p = __ldcg(L + r); p != r; p = __ldcg(L + r)) r = p;
    L[i] = r;
  }
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

// rows is NULL when the stats did not run, which is only when dust_threshold <= 1 keeps every part
__global__ void __launch_bounds__(256) k_keep_flags(const BoxRow* __restrict__ rows, uint64_t k, uint64_t threshold,
                                                   uint32_t* __restrict__ keep) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i <= k; i += (uint64_t)gridDim.x * blockDim.x)
    keep[i] = i < k && (!rows || rows[i].w[0] >= threshold);
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

// the kept parts' ranks: pos[rank] + 1 where keep[rank], 0 on label 0 and on dust
__global__ void __launch_bounds__(256) k_parts(const uint32_t* __restrict__ L, uint64_t n,
                                              const uint32_t* __restrict__ roots, uint32_t k,
                                              const uint32_t* __restrict__ keep, const uint32_t* __restrict__ pos,
                                              uint32_t* __restrict__ out) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t r = L[i];
    uint32_t v = 0;
    if (r != kBg) {
      const uint32_t j = root_rank(roots, k, r);
      if (keep[j]) v = pos[j] + 1;
    }
    out[i] = v;
  }
}

static unsigned grid_for(ign_ctx* ctx, uint64_t n) {
  return (unsigned)std::max<uint64_t>(1, std::min<uint64_t>(blocks_for(n, 256), (uint64_t)ctx->sm_count * 32));
}

template <typename T>
int label_parts(ign_ctx* ctx, const T* lab, uint64_t sx, uint64_t sy, uint64_t sz, int reach, uint64_t dust_threshold,
                uint32_t* parts_out, uint32_t* rows, uint64_t capacity, uint64_t* n) {
  const uint64_t nv = sx * sy * sz;
  ScratchFrame f(ctx);
  uint32_t *L, *roots;
  IGN_TRY(f.take(&L, nv));
  const unsigned g = grid_for(ctx, nv);
  IGN_LAUNCH(ctx, k_uf_init<T>, g, 256, 0, lab, nv, L);
  IGN_LAUNCH(ctx, k_uf_merge<T>, g, 256, 0, lab, sx, sy, sz, reach, L);
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
  if (hk == 0) {
    if (parts_out) IGN_CUDA(cudaMemsetAsync(parts_out, 0, nv * 4, ctx->stream));
    return IGN_OK;
  }
  const uint32_t k = hk;
  IGN_TRY(f.take(&roots, k));
  IGN_LAUNCH(ctx, k_seg_roots<true>, grid_for(ctx, segs), 256, 0, L, sx, sy * sz, nullptr, at, roots);
  BoxRow* all = nullptr;
  if (rows || dust_threshold > 1) {
    IGN_TRY(f.take(&all, k));
    IGN_LAUNCH(ctx, k_rows_init, grid_for(ctx, k), 256, 0, all, k);
    IGN_LAUNCH(ctx, k_box_stats, grid_for(ctx, segs), 256, 0, L, sx, sy, sz, roots, k, all);
  }
  // dust: the kept parts in rank order, at the exclusive sum of their flags (keep[k] = 0: pos[k] = the number kept)
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
  if (parts_out) IGN_LAUNCH(ctx, k_parts, g, 256, 0, L, nv, roots, k, keep, pos, parts_out);
  uint32_t hn = 0;
  IGN_TRY(small_d2h(ctx, &hn, pos + k, 4));
  IGN_TRY(small_sync(ctx));
  *n = (uint64_t)hn;
  if (rows && *n && *n <= capacity) {
    BoxRow* kept;
    IGN_TRY(f.take(&kept, *n));
    IGN_LAUNCH(ctx, k_keep_rows, grid_for(ctx, k), 256, 0, all, k, keep, pos, kept);
    IGN_CUDA(cudaMemcpyAsync(rows, kept, *n * sizeof(BoxRow), cudaMemcpyDeviceToHost, ctx->stream));
    IGN_CUDA(cudaStreamSynchronize(ctx->stream));
  }
  return IGN_OK;
}

}  // namespace

}  // namespace ign

using namespace ign;

extern "C" {

int ign_label_parts_dev(ign_ctx* ctx, const void* labels, int dtype, uint64_t sx, uint64_t sy, uint64_t sz,
                        int connectivity, uint64_t dust_threshold, uint32_t* parts_out, uint32_t* rows,
                        uint64_t capacity, uint64_t* n) {
  IGN_TRY(activate(ctx));
  IGN_REQUIRE(n, IGN_ERR_INVALID, "label_parts: null count");
  *n = 0;
  IGN_REQUIRE(connectivity == 6 || connectivity == 18 || connectivity == 26, IGN_ERR_INVALID,
              "label_parts: connectivity %d (6, 18 or 26)", connectivity);
  const int reach = connectivity == 6 ? 1 : connectivity == 18 ? 2 : 3;
  IGN_REQUIRE(sx < (1ull << 32) && sy < (1ull << 32) && sz < (1ull << 32), IGN_ERR_UNSUPPORTED,
              "label_parts: a side of %llu x %llu x %llu is 2^32 or more", (unsigned long long)sx,
              (unsigned long long)sy, (unsigned long long)sz);
  const uint64_t sxy = sx * sy, nv = sxy * sz;  // sides below 2^32: sxy does not wrap, and nv only when refused
  IGN_REQUIRE(sz == 0 || sxy <= (kBg - 1) / sz, IGN_ERR_UNSUPPORTED,
              "label_parts: %llu x %llu x %llu voxels (the union-find links are 32-bit voxel indices: fewer than "
              "2^32 - 1)", (unsigned long long)sx, (unsigned long long)sy, (unsigned long long)sz);
  return dispatch_label(dtype, "label_parts", [&](auto v) -> int {
    using T = decltype(v);
    if (nv == 0) return IGN_OK;
    IGN_REQUIRE(labels && (rows || capacity == 0), IGN_ERR_INVALID, "label_parts: null buffer");
    return label_parts<T>(ctx, (const T*)labels, sx, sy, sz, reach, dust_threshold, parts_out, rows, capacity, n);
  });
}

}  // extern "C"
