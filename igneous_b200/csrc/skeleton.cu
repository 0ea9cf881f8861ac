// skeleton.cu -- the per-label export of a chunk's TEASAR skeleton (ign_teasar_paths_dev's compacted
// output) into neuroglancer precomputed skeletons, one blob per label, sm_90a.  The rule is
// DESIGN.md §5g: a label's vertices are its skeleton voxels in ascending linear index, each vertex
// fl32((double)fl32(fl32(c) * a) + offset) per axis, one edge (min, max) of local vertex indices per
// voxel whose next voxel is another, the edges of a label sorted by (lo, hi).
//
//   k_sx_keys     the label of every skeleton voxel; checks the voxels are ascending, inside the volume and
//                 on labels 1..K (the host reads the flags back and refuses bad input before any other pass)
//   (sort)        stable radix sort of (label, position): a label's voxels keep their ascending order
//   k_sx_heads    1 where a label's run of sorted positions starts; an inclusive sum gives the run number
//   k_sx_rank     rank[position] = sorted position; per run its first sorted position and its label
//   k_sx_edges    per voxel with next != itself: the next voxel's rank by binary search in the ascending
//                 index list, the key (lo rank << 32) | hi rank; a next voxel off the skeleton or on
//                 another label fails the call before any output is written
//   (sort)        the edge keys: runs are contiguous in rank, so this is the order (label, lo, hi)
//   (encode)      skelblob_encode (skelblob.cuh): a row per run, the sorted positions as final vertices
//   k_sx_boxes    one warp per run: min / max of its vertices
//
// Every voxel's vertex is computed by sx_vertex, so the boxes are the min / max of the written values.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>

#include "common.cuh"
#include "skelblob.cuh"

namespace ign {

namespace {

struct SxCtl {
  uint32_t err;  // bit b: a voxel failed check b of sx_fail_host
  uint32_t pad;
  unsigned long long bad[5];  // per check, the lowest linear index that failed it
  unsigned long long ne;      // edges
  unsigned long long bytes;   // end of the last blob
};

__device__ __forceinline__ void sx_fail(SxCtl* ctl, int bit, uint64_t voxel) {
  atomicOr(&ctl->err, 1u << bit);
  atomicMin(&ctl->bad[bit], (unsigned long long)voxel);
}

__device__ __forceinline__ float sx_coord(uint64_t c, float a, double off) {
  return __double2float_rn(__dadd_rn((double)__fmul_rn(__ull2float_rn(c), a), off));
}

__device__ __forceinline__ void sx_vertex(uint64_t v, uint64_t sx, uint64_t sy, float a0, float a1, float a2,
                                          double o0, double o1, double o2, float out[3]) {
  const uint64_t x = v % sx, yz = v / sx;
  out[0] = sx_coord(x, a0, o0);
  out[1] = sx_coord(yz % sy, a1, o1);
  out[2] = sx_coord(yz / sy, a2, o2);
}

__global__ void __launch_bounds__(256) k_sx_keys(const uint32_t* __restrict__ lab, uint64_t n,
                                                 const uint32_t* __restrict__ skel, uint64_t count, uint64_t K,
                                                 uint32_t* __restrict__ key, uint32_t* __restrict__ val, SxCtl* ctl) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= count) return;
  const uint32_t v = skel[i];
  uint32_t l = 0;
  if (v >= n) {
    sx_fail(ctl, 0, (uint64_t)v);
  } else {
    if (i && skel[i - 1] >= v) sx_fail(ctl, 1, (uint64_t)v);
    l = lab[v];
    if (l == 0 || l > K) sx_fail(ctl, 2, (uint64_t)v);
  }
  key[i] = l;
  val[i] = (uint32_t)i;
}

__global__ void __launch_bounds__(256) k_sx_heads(const uint32_t* __restrict__ key_s, uint64_t count,
                                                  uint32_t* __restrict__ head) {
  const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p < count) head[p] = (p == 0 || key_s[p] != key_s[p - 1]) ? 1u : 0u;
}

// run[p] = 1-based run of sorted position p
__global__ void __launch_bounds__(256) k_sx_rank(const uint32_t* __restrict__ key_s, const uint32_t* __restrict__ val_s,
                                                 const uint32_t* __restrict__ head, const uint32_t* __restrict__ run,
                                                 uint64_t count, uint32_t* __restrict__ rank,
                                                 uint32_t* __restrict__ start, uint32_t* __restrict__ label) {
  const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= count) return;
  rank[val_s[p]] = (uint32_t)p;
  if (head[p]) {
    start[run[p] - 1] = (uint32_t)p;
    label[run[p] - 1] = key_s[p];
  }
}

__global__ void __launch_bounds__(256) k_sx_edges(const uint32_t* __restrict__ lab, uint64_t n,
                                                  const uint32_t* __restrict__ skel, const uint32_t* __restrict__ next,
                                                  uint64_t count, const uint32_t* __restrict__ rank,
                                                  uint64_t* __restrict__ ekey, SxCtl* ctl) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  bool edge = false;
  if (i < count) {
    const uint32_t v = skel[i], u = next[i];
    uint64_t k = count << 32;  // sorts after every edge
    if (u != v && v < n) {
      uint64_t lo = 0, hi = count;  // first position with skel >= u
      while (lo < hi) {
        const uint64_t mid = (lo + hi) >> 1;
        if (skel[mid] < u) lo = mid + 1; else hi = mid;
      }
      if (u >= n || lo == count || skel[lo] != u) {
        sx_fail(ctl, 3, (uint64_t)v);
      } else if (lab[u] != lab[v]) {
        sx_fail(ctl, 4, (uint64_t)v);
      } else {
        const uint32_t r0 = rank[i], r1 = rank[lo];
        k = ((uint64_t)min(r0, r1) << 32) | max(r0, r1);
        edge = true;
      }
    }
    ekey[i] = k;
  }
  // one atomic per warp for the edge count
  const unsigned m = __ballot_sync(0xFFFFFFFFu, edge);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(&ctl->ne, (unsigned long long)__popc(m));
}

// the rows of skelblob_encode: one per run; final vertex j is sorted position j
struct SxSource {
  const uint32_t *start, *labels, *run, *val_s, *skel;
  const float* radius;
  uint64_t runs, count, sx, sy;
  float a0, a1, a2;
  double o0, o1, o2;
  __device__ uint64_t vstart(uint64_t g) const { return g < runs ? start[g] : count; }
  __device__ uint64_t label(uint64_t g) const { return labels[g]; }
  __device__ uint32_t row(uint64_t j) const { return run[j] - 1; }
  __device__ void vertex(uint64_t j, float c[3], float& r, uint8_t& t) const {
    const uint32_t i = val_s[j];
    sx_vertex(skel[i], sx, sy, a0, a1, a2, o0, o1, o2, c);
    r = radius[i];
    t = 0;
  }
};

__global__ void __launch_bounds__(256) k_sx_boxes(const uint32_t* __restrict__ skel, const uint32_t* __restrict__ val_s,
                                                  const uint32_t* __restrict__ start, uint64_t runs, uint64_t count,
                                                  uint64_t sx, uint64_t sy, float a0, float a1, float a2, double o0,
                                                  double o1, double o2, float* __restrict__ boxes) {
  const uint64_t g = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (g >= runs) return;  // whole warps leave together
  const uint64_t a = start[g], b = g + 1 < runs ? start[g + 1] : count;
  float lo[3] = {INFINITY, INFINITY, INFINITY}, hi[3] = {-INFINITY, -INFINITY, -INFINITY};
  for (uint64_t p = a + lane; p < b; p += 32) {
    float c[3];
    sx_vertex(skel[val_s[p]], sx, sy, a0, a1, a2, o0, o1, o2, c);
    for (int d = 0; d < 3; ++d) {
      lo[d] = fminf(lo[d], c[d]);
      hi[d] = fmaxf(hi[d], c[d]);
    }
  }
  for (int s = 16; s; s >>= 1)
    for (int d = 0; d < 3; ++d) {
      lo[d] = fminf(lo[d], __shfl_xor_sync(0xFFFFFFFFu, lo[d], s));
      hi[d] = fmaxf(hi[d], __shfl_xor_sync(0xFFFFFFFFu, hi[d], s));
    }
  if (lane < 3) {
    boxes[6 * g + lane] = lo[lane];
    boxes[6 * g + 3 + lane] = hi[lane];
  }
}

int bit_width(uint64_t v) {
  int b = 0;
  while (v) {
    ++b;
    v >>= 1;
  }
  return b;
}

uint64_t export_bound(uint64_t count, uint64_t max_label) {
  return count * 25 + std::min(max_label, count) * 16;
}

int sx_fail_host(const SxCtl& h) {
  static const char* what[5] = {
    "lies outside the volume", "is not above the one before it (the voxels must be ascending)",
    "lies on label 0 or above max_label", "has a next voxel that is not a skeleton voxel",
    "has its next voxel on another label (a corrupt next field; no edge crosses labels)"};
  for (int b = 0; b < 5; ++b)
    IGN_REQUIRE(!(h.err & (1u << b)), IGN_ERR_INVALID, "skeleton_export: the skeleton voxel at linear index %llu %s",
                h.bad[b], what[b]);
  return IGN_OK;
}

}  // namespace
}  // namespace ign

using namespace ign;

extern "C" {

int ign_skeleton_export_capacity(uint64_t count, uint64_t max_label, uint64_t* bytes) {
  IGN_REQUIRE(bytes, IGN_ERR_INVALID, "skeleton_export: null bytes");
  IGN_REQUIRE(count < (1ull << 31), IGN_ERR_OVERFLOW, "skeleton_export: %llu skeleton voxels (fewer than 2^31)",
              (unsigned long long)count);
  *bytes = export_bound(count, max_label);
  return IGN_OK;
}

int ign_skeleton_export_dev(ign_ctx* ctx, const uint32_t* labels, uint64_t sx, uint64_t sy, uint64_t sz,
                            uint64_t max_label, const uint32_t* skel, const uint32_t* next, const float* radius,
                            uint64_t count, const float anisotropy[3], const double offset[3], int vertex_types,
                            uint8_t* blobs_out, uint64_t capacity, uint64_t* table_out, float* boxes_out,
                            uint64_t* n_skeletons, uint64_t* nbytes) {
  IGN_TRY(activate(ctx));
  IGN_REQUIRE(n_skeletons && nbytes && anisotropy && offset, IGN_ERR_INVALID, "skeleton_export: null argument");
  *n_skeletons = 0;
  *nbytes = 0;
  const uint64_t n = sx * sy * sz;
  IGN_REQUIRE(sx < (1ull << 30) && sy < (1ull << 30) && sz < (1ull << 30) && n < 0xFFFFFFFFull, IGN_ERR_INVALID,
              "skeleton_export: volume (%llu, %llu, %llu): each side below 2^30, fewer than 2^32 - 1 voxels",
              (unsigned long long)sx, (unsigned long long)sy, (unsigned long long)sz);
  IGN_REQUIRE(max_label < (1ull << 32), IGN_ERR_UNSUPPORTED, "skeleton_export: max_label %llu (below 2^32)",
              (unsigned long long)max_label);
  IGN_REQUIRE(count < (1ull << 31) && count <= n, IGN_ERR_OVERFLOW,
              "skeleton_export: %llu skeleton voxels (fewer than 2^31 and at most the volume's)",
              (unsigned long long)count);
  for (int i = 0; i < 3; ++i) {
    IGN_REQUIRE(anisotropy[i] > 0.f && isfinite(anisotropy[i]), IGN_ERR_INVALID,
                "skeleton_export: anisotropy[%d] = %g (positive and finite)", i, (double)anisotropy[i]);
    IGN_REQUIRE(isfinite(offset[i]), IGN_ERR_INVALID, "skeleton_export: offset[%d] = %g (finite)", i, offset[i]);
  }
  const uint64_t bound = export_bound(count, max_label);
  IGN_REQUIRE(capacity >= bound, IGN_ERR_INVALID,
              "skeleton_export: capacity %llu bytes is below the bound count * 25 + min(max_label, count) * 16 = %llu",
              (unsigned long long)capacity, (unsigned long long)bound);
  if (count == 0) return IGN_OK;
  IGN_REQUIRE(labels && skel && next && radius && blobs_out && table_out && boxes_out, IGN_ERR_INVALID,
              "skeleton_export: null buffer");
  IGN_REQUIRE(((uintptr_t)blobs_out & 7) == 0 && ((uintptr_t)table_out & 7) == 0 && ((uintptr_t)boxes_out & 3) == 0,
              IGN_ERR_INVALID, "skeleton_export: an output buffer is not aligned (blobs and table to 8 bytes)");
  const uint64_t rows = std::max<uint64_t>(std::min(max_label, count), 1);
  ScratchFrame f(ctx);
  SxCtl* ctl;
  uint32_t *key, *val, *key_s, *val_s, *head, *run, *rank, *start, *label;
  uint64_t *ekey, *ekey_s;
  IGN_TRY(f.take(&ctl, 1));
  IGN_TRY(f.take(&key, count));
  IGN_TRY(f.take(&val, count));
  IGN_TRY(f.take(&key_s, count));
  IGN_TRY(f.take(&val_s, count));
  IGN_TRY(f.take(&head, count));
  IGN_TRY(f.take(&run, count));
  IGN_TRY(f.take(&rank, count));
  IGN_TRY(f.take(&ekey, count));
  IGN_TRY(f.take(&ekey_s, count));
  IGN_TRY(f.take(&start, rows));
  IGN_TRY(f.take(&label, rows));
  const int items = (int)count;
  const int label_bits = std::max(1, bit_width(max_label));
  const int edge_bits = 32 + bit_width(count);
  size_t tb = 0, t;
  IGN_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, t, key, key_s, val, val_s, items, 0, label_bits, ctx->stream));
  tb = std::max(tb, t);
  IGN_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, t, ekey, ekey_s, items, 0, edge_bits, ctx->stream));
  tb = std::max(tb, t);
  IGN_CUDA(cub::DeviceScan::InclusiveSum(nullptr, t, head, run, items, ctx->stream));
  tb = std::max(tb, t);
  void* tmp;
  IGN_TRY(f.take(&tmp, tb));

  SxCtl init{};
  for (int b = 0; b < 5; ++b) init.bad[b] = ~0ull;
  IGN_TRY(small_h2d(ctx, ctl, &init, sizeof(SxCtl)));
  const unsigned grid = blocks_for(count, 256);
  IGN_LAUNCH(ctx, k_sx_keys, grid, 256, 0, labels, n, skel, count, max_label, key, val, ctl);
  // every later pass relies on the voxels being ascending, inside the volume and on labels 1..K (the run
  // count then stays within rows and the sort's bits cover every key): refuse bad input first
  SxCtl h{};
  IGN_TRY(small_d2h(ctx, &h, ctl, sizeof(SxCtl)));
  IGN_TRY(small_sync(ctx));
  IGN_TRY(sx_fail_host(h));
  IGN_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tb, key, key_s, val, val_s, items, 0, label_bits, ctx->stream));
  IGN_LAUNCH(ctx, k_sx_heads, grid, 256, 0, key_s, count, head);
  IGN_CUDA(cub::DeviceScan::InclusiveSum(tmp, tb, head, run, items, ctx->stream));
  IGN_LAUNCH(ctx, k_sx_rank, grid, 256, 0, key_s, val_s, head, run, count, rank, start, label);
  IGN_LAUNCH(ctx, k_sx_edges, grid, 256, 0, labels, n, skel, next, count, rank, ekey, ctl);
  uint32_t runs32 = 0;
  IGN_TRY(small_d2h(ctx, &h, ctl, sizeof(SxCtl)));
  IGN_TRY(small_d2h(ctx, &runs32, run + (count - 1), 4));
  IGN_TRY(small_sync(ctx));
  IGN_TRY(sx_fail_host(h));
  const uint64_t runs = runs32;
  IGN_CUDA(cub::DeviceRadixSort::SortKeys(tmp, tb, ekey, ekey_s, items, 0, edge_bits, ctx->stream));
  const float a0 = anisotropy[0], a1 = anisotropy[1], a2 = anisotropy[2];
  const double o0 = offset[0], o1 = offset[1], o2 = offset[2];
  const SxSource src{start, label, run, val_s, skel, radius, runs, count, sx, sy, a0, a1, a2, o0, o1, o2};
  IGN_TRY(skelblob_encode(ctx, f, src, runs, count, ekey_s, h.ne, &ctl->ne, vertex_types, table_out, blobs_out,
                          &ctl->bytes));
  IGN_LAUNCH(ctx, k_sx_boxes, blocks_for(runs * 32, 256), 256, 0, skel, val_s, start, runs, count, sx, sy, a0, a1, a2,
             o0, o1, o2, boxes_out);
  IGN_TRY(small_d2h(ctx, &h, ctl, sizeof(SxCtl)));
  IGN_TRY(small_sync(ctx));
  *n_skeletons = runs;
  *nbytes = h.bytes;
  return IGN_OK;
}

}  // extern "C"
