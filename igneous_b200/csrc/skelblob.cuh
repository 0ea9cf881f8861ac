// skelblob.cuh -- the neuroglancer precomputed skeleton encoder of ign_skeleton_export_dev (skeleton.cu) and
// ign_skeleton_merge_dev (skelmerge.cu), and the blob layout ign_skeleton_restrip_dev (labelshard.cu) reads,
// sm_90a: the only code under csrc/ that knows the blob layout (DESIGN.md §5g).  The caller numbers its final vertices label-major, sorts its edges as keys (lo << 32) | hi
// of those numbers, and describes its G rows with a source, a device functor with
//   vstart(g), g <= G      the first final vertex of row g (vstart(G) is the vertex count)
//   label(g)               column 0 of the table
//   row(j)                 the row of final vertex j
//   vertex(j, xyz, r, t)   its coordinates, radius and type
// The kernels only move integers and copy values: any float arithmetic stays in the sources.
#pragma once

#include <cub/device/device_scan.cuh>

#include "common.cuh"

namespace ign {

namespace {

__device__ __forceinline__ uint64_t sb_lower(const uint64_t* __restrict__ a, uint64_t n, uint64_t x) {
  uint64_t lo = 0, hi = n;
  while (lo < hi) {
    const uint64_t mid = (lo + hi) >> 1;
    if (a[mid] < x) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// a blob: uint32 nv, ne, float32 vertices[nv][3], uint32 edges[ne][2], then one section per vertex attribute,
// each nv values; sb_head_bytes is where the first attribute section starts
__device__ __forceinline__ uint64_t sb_head_bytes(uint64_t nv, uint64_t ne) { return 8 + 12 * nv + 8 * ne; }

// the blob of the encoder below: radius float32, then vertex_types uint8 when vt
__device__ __forceinline__ uint64_t sb_blob_bytes(uint64_t nv, uint64_t ne, int vt) {
  return sb_head_bytes(nv, ne) + (vt ? 5 : 4) * nv;
}

template <class Src>
__global__ void __launch_bounds__(256) k_sb_sizes(Src src, uint64_t G, const uint64_t* __restrict__ key,
                                                  const unsigned long long* __restrict__ ne_all, int vt,
                                                  uint32_t* __restrict__ vstart, uint32_t* __restrict__ estart,
                                                  uint64_t* __restrict__ size) {
  const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g > G) return;
  const uint64_t ne = *ne_all, v0 = src.vstart(g), e0 = sb_lower(key, ne, v0 << 32);
  vstart[g] = (uint32_t)v0;
  estart[g] = (uint32_t)e0;
  if (g < G) {
    const uint64_t v1 = src.vstart(g + 1), e1 = sb_lower(key, ne, v1 << 32);
    size[g] = (sb_blob_bytes(v1 - v0, e1 - e0, vt) + 7) & ~7ull;
  }
}

template <class Src>
__global__ void __launch_bounds__(256) k_sb_table(Src src, uint64_t G, const uint32_t* __restrict__ vstart,
                                                  const uint32_t* __restrict__ estart,
                                                  const uint64_t* __restrict__ off, int vt,
                                                  uint64_t* __restrict__ table, uint8_t* __restrict__ blobs,
                                                  unsigned long long* __restrict__ bytes) {
  const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= G) return;
  const uint64_t nv = vstart[g + 1] - vstart[g], ne = estart[g + 1] - estart[g];
  table[4 * g + 0] = src.label(g);
  table[4 * g + 1] = off[g];
  table[4 * g + 2] = nv;
  table[4 * g + 3] = ne;
  uint32_t* h = (uint32_t*)(blobs + off[g]);
  h[0] = (uint32_t)nv;
  h[1] = (uint32_t)ne;
  const uint64_t end = off[g] + sb_blob_bytes(nv, ne, vt);
  for (uint64_t b = end; b & 7; ++b) blobs[b] = 0;  // the padding up to the next blob
  if (g + 1 == G) *bytes = end;
}

template <class Src>
__global__ void __launch_bounds__(256) k_sb_verts(Src src, uint64_t G, uint64_t vmax,
                                                  const uint32_t* __restrict__ vstart,
                                                  const uint32_t* __restrict__ estart,
                                                  const uint64_t* __restrict__ off, int vt,
                                                  uint8_t* __restrict__ blobs) {
  const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= vmax || j >= vstart[G]) return;
  const uint32_t g = src.row(j);
  const uint64_t i = j - vstart[g], o = off[g], nv = vstart[g + 1] - vstart[g], ne = estart[g + 1] - estart[g];
  float c[3], r;
  uint8_t t;
  src.vertex(j, c, r, t);
  float* vert = (float*)(blobs + o + 8) + 3 * i;
  vert[0] = c[0];
  vert[1] = c[1];
  vert[2] = c[2];
  ((float*)(blobs + o + sb_head_bytes(nv, ne)))[i] = r;
  if (vt) blobs[o + sb_head_bytes(nv, ne) + 4 * nv + i] = t;
}

template <class Src>
__global__ void __launch_bounds__(256) k_sb_edges(Src src, const uint64_t* __restrict__ key,
                                                  const unsigned long long* __restrict__ ne_all,
                                                  const uint32_t* __restrict__ vstart,
                                                  const uint32_t* __restrict__ estart,
                                                  const uint64_t* __restrict__ off, uint8_t* __restrict__ blobs) {
  const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= *ne_all) return;
  const uint32_t lo = (uint32_t)(key[e] >> 32), hi = (uint32_t)key[e], g = src.row(lo);
  const uint64_t nv = vstart[g + 1] - vstart[g];
  uint32_t* edge = (uint32_t*)(blobs + off[g] + 8 + 12 * nv) + 2 * (e - estart[g]);
  edge[0] = lo - vstart[g];
  edge[1] = hi - vstart[g];
}

// Writes the G >= 1 blobs and table rows of src.  key: the sorted edge keys, *ne_all of them live (anything
// after them sorts above every live key); vmax and emax: host bounds on the final vertices and the live
// edges; *bytes receives the end of the last blob.  Takes its scratch from f; four launches at most, no
// synchronisation.
template <class Src>
int skelblob_encode(ign_ctx* ctx, ScratchFrame& f, const Src& src, uint64_t G, uint64_t vmax,
                    const uint64_t* key, uint64_t emax, const unsigned long long* ne_all, int vt,
                    uint64_t* table, uint8_t* blobs, unsigned long long* bytes) {
  uint32_t *vstart, *estart;
  uint64_t *size, *off;
  IGN_TRY(f.take(&vstart, G + 1));
  IGN_TRY(f.take(&estart, G + 1));
  IGN_TRY(f.take(&size, G));
  IGN_TRY(f.take(&off, G));
  size_t tb = 0;
  IGN_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, size, off, (int)G, ctx->stream));
  void* tmp;
  IGN_TRY(f.take(&tmp, tb));
  IGN_LAUNCH(ctx, k_sb_sizes<Src>, blocks_for(G + 1, 256), 256, 0, src, G, key, ne_all, vt, vstart, estart, size);
  IGN_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tb, size, off, (int)G, ctx->stream));
  IGN_LAUNCH(ctx, k_sb_table<Src>, blocks_for(G, 256), 256, 0, src, G, vstart, estart, off, vt, table, blobs, bytes);
  if (vmax)
    IGN_LAUNCH(ctx, k_sb_verts<Src>, blocks_for(vmax, 256), 256, 0, src, G, vmax, vstart, estart, off, vt, blobs);
  if (emax)
    IGN_LAUNCH(ctx, k_sb_edges<Src>, blocks_for(emax, 256), 256, 0, src, key, ne_all, vstart, estart, off, blobs);
  return IGN_OK;
}

}  // namespace
}  // namespace ign
