// mesh.cu -- multi-label marching cubes (K8) + per-label vertex welding (K9)
//
// Replaces zmesh.Mesher.mesh / ids / get as called from
// igneous/tasks/mesh/mesh.py:151,245,371-383.
//
//   renumber   labels -> dense 1..K (shares remap.cu's hash table kernels)
//   count      one thread per 2x2x2 cube (x fastest, corners through L1): for
//              every distinct non-zero corner label the 256-case table gives a
//              triangle count; one total per CTA.  A pass over the lattice
//              edges counts vertex records (below) per warp.
//   emit       an exclusive scan of the totals gives each CTA (warp) its base;
//              its records go to base + in-CTA (in-warp) prefix, so they land in
//              raster order with no atomics: (label, cube<<11 | case<<3 | t).
//   sort       stable radix sort on the label bits alone -> (label, cube, t).
//   weld       a vertex of label L sits on every lattice edge with one endpoint
//              L != 0 and the other != L (every case of mc_table.h uses exactly
//              the edges whose endpoint bits differ).  Edges are enumerated in
//              raster order of the half-voxel lattice, one record per non-zero
//              side, and stably sorted on the label: that is the unique vertex
//              order (label, z2, y2, x2).  Per-warp record masks give each
//              face corner the emission index of its vertex record, and the
//              sort's inverse permutation its vertex id.
// Roofline: HBM-bound streaming over the label volume for count/emit
// (algorithmic bytes = sizeof(label) per voxel); the sorts are bound by the
// surface size, not the volume.
#include <cub/block/block_scan.cuh>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <atomic>
#include <climits>
#include <vector>

#include "common.cuh"
#include "mc_table.h"

namespace ign {

constexpr unsigned MFULL = 0xFFFFFFFFu;
constexpr int V_COORD_BITS = 11;
constexpr int V_LABEL_SHIFT = 3 * V_COORD_BITS;  // 33
constexpr int TRI_CASE_SHIFT = 3, TRI_CUBE_SHIFT = 11;  // triangle record: cube << 11 | case << 3 | t
using BlockScan256 = cub::BlockScan<uint32_t, 256>;

__constant__ int8_t c_edge_mid[12][3] = {{1, 0, 0}, {2, 1, 0}, {1, 2, 0}, {0, 1, 0},
                                         {1, 0, 2}, {2, 1, 2}, {1, 2, 2}, {0, 1, 2},
                                         {0, 0, 1}, {2, 0, 1}, {2, 2, 1}, {0, 2, 1}};

struct McTables {
  int8_t tri[256][16];
  uint8_t ntri[256];
};
__constant__ McTables c_mc;

// Lattice edges in raster order of the half-voxel lattice (z2, y2, x2): per plane z, the x-edges
// then the y-edges of each row y, then the plane's z-edges in (y, x) order.  An edge's slot in that
// order is its id (< 3 * 1023^3 < 2^32); slots of edges that leave the volume hold no vertex.
struct Lattice {
  uint32_t sx, sy, sz;
  __device__ __forceinline__ uint32_t plane() const { return 3 * sx * sy; }
  // slot -> lower endpoint voxel and direction (0 x, 1 y, 2 z)
  __device__ __forceinline__ void edge(uint32_t g, uint32_t& x, uint32_t& y, uint32_t& z, uint32_t& dir) const {
    z = g / plane();
    uint32_t r = g - z * plane();
    if (r < 2 * sx * sy) {
      y = r / (2 * sx);
      r -= y * 2 * sx;
      dir = r >= sx;
      x = r - dir * sx;
    } else {
      r -= 2 * sx * sy;
      dir = 2;
      y = r / sx;
      x = r - y * sx;
    }
  }
  // half-voxel coordinates of an edge midpoint -> slot
  __device__ __forceinline__ uint32_t slot(uint32_t X2, uint32_t Y2, uint32_t Z2) const {
    const uint32_t base = (Z2 >> 1) * plane();
    if (Z2 & 1) return base + 2 * sx * sy + (Y2 >> 1) * sx + (X2 >> 1);
    return base + (Y2 >> 1) * 2 * sx + ((Y2 & 1) ? sx : 0) + (X2 >> 1);
  }
};

// corner k of Bourke's numbering -> offset (dx,dy,dz)
__device__ __forceinline__ void cube_corners(const uint32_t* __restrict__ lab, uint32_t sx,
                                             uint32_t sxy, uint32_t base, uint32_t (&c)[8]) {
  c[0] = lab[base];
  c[1] = lab[base + 1];
  c[2] = lab[base + 1 + sx];
  c[3] = lab[base + sx];
  c[4] = lab[base + sxy];
  c[5] = lab[base + 1 + sxy];
  c[6] = lab[base + 1 + sx + sxy];
  c[7] = lab[base + sx + sxy];
}

// EMIT=false: triangles per CTA into cta[blockIdx.x]; EMIT=true: records at the CTA's scanned base
template <bool EMIT>
__global__ void __launch_bounds__(256)
    k_mc(const uint32_t* __restrict__ lab, uint32_t sx, uint32_t sy, uint32_t sz,
         unsigned long long* __restrict__ cta, uint32_t* __restrict__ tlabel, uint64_t* __restrict__ trec) {
  __shared__ uint8_t s_ntri[256];
  __shared__ typename BlockScan256::TempStorage s_scan;
  for (int i = threadIdx.x; i < 256; i += blockDim.x) s_ntri[i] = c_mc.ntri[i];
  __syncthreads();
  const uint32_t cx = sx - 1, cy = sy - 1, cz = sz - 1;
  const uint64_t ncubes = (uint64_t)cx * cy * cz;
  const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  uint32_t mine = 0;
  uint32_t c[8];
  uint32_t x = 0, y = 0, z = 0;
  bool active = false;
  if (t < ncubes) {
    x = (uint32_t)(t % cx);
    y = (uint32_t)((t / cx) % cy);
    z = (uint32_t)(t / ((uint64_t)cx * cy));
    cube_corners(lab, sx, sx * sy, (z * sy + y) * sx + x, c);
    const uint32_t o = c[0] | c[1] | c[2] | c[3] | c[4] | c[5] | c[6] | c[7];
    const bool same = (c[0] == c[1]) & (c[0] == c[2]) & (c[0] == c[3]) & (c[0] == c[4]) &
                      (c[0] == c[5]) & (c[0] == c[6]) & (c[0] == c[7]);
    active = (o != 0) && !same;
  }
  uint8_t idxs[8];
  if (active) {
#pragma unroll
    for (int k = 0; k < 8; k++) {
      const uint32_t L = c[k];
      bool first = (L != 0);
#pragma unroll
      for (int j = 0; j < 8; j++)
        if (j < k) first = first && (c[j] != L);
      uint32_t idx = 0;
#pragma unroll
      for (int j = 0; j < 8; j++) idx |= (uint32_t)(c[j] == L) << j;
      idxs[k] = first ? (uint8_t)idx : 0;  // case 0 emits nothing
      mine += s_ntri[idxs[k]];
    }
  }
  uint32_t pre, total;
  BlockScan256(s_scan).ExclusiveSum(mine, pre, total);
  if (!EMIT) {
    if (threadIdx.x == 0) cta[blockIdx.x] = total;
    return;
  }
  if (!active) return;
  uint64_t pos = cta[blockIdx.x] + pre;
  const uint64_t cube = (uint64_t)t;
#pragma unroll
  for (int k = 0; k < 8; k++) {
    const uint32_t n = s_ntri[idxs[k]];
    for (uint32_t tt = 0; tt < n; tt++) {
      tlabel[pos] = c[k];
      trec[pos] = (cube << TRI_CUBE_SHIFT) | ((uint64_t)idxs[k] << TRI_CASE_SHIFT) | tt;
      pos++;
    }
  }
}

// Vertex records are counted per warp of 32 edge slots: bit j of the warp's mask is set when slot j
// holds at least one record, bit 32 + j when it holds two.  With the scanned warp bases that gives the
// emission index of any record without storing one per edge.
__device__ __forceinline__ uint64_t record_index(const uint64_t* __restrict__ wmask,
                                                 const unsigned long long* __restrict__ wbase, uint32_t g) {
  const uint64_t mk = wmask[g >> 5];
  const uint32_t below = (1u << (g & 31)) - 1;
  return wbase[g >> 5] + __popc((uint32_t)mk & below) + __popc((uint32_t)(mk >> 32) & below);
}

// EMIT=false: masks and record counts per warp; EMIT=true: (label, edge slot) records at the warp's
// scanned base, the side of the lower endpoint first
template <bool EMIT>
__global__ void __launch_bounds__(256)
    k_edges(const uint32_t* __restrict__ lab, Lattice lt, uint64_t* __restrict__ wmask,
            unsigned long long* __restrict__ wcount, uint32_t* __restrict__ vlabel, uint32_t* __restrict__ vedge) {
  const uint64_t nslots = 3ull * lt.sx * lt.sy * lt.sz;
  const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  uint32_t a = 0, b = 0, mine = 0;
  if (t < nslots) {
    uint32_t x, y, z, dir;
    lt.edge((uint32_t)t, x, y, z, dir);
    const bool inside = dir == 0 ? x + 1 < lt.sx : dir == 1 ? y + 1 < lt.sy : z + 1 < lt.sz;
    if (inside) {
      const uint64_t i = ((uint64_t)z * lt.sy + y) * lt.sx + x;
      a = lab[i];
      b = lab[i + (dir == 0 ? 1ull : dir == 1 ? (uint64_t)lt.sx : (uint64_t)lt.sx * lt.sy)];
      if (a != b) mine = (a != 0) + (b != 0);
    }
  }
  const uint32_t m1 = __ballot_sync(MFULL, mine >= 1), m2 = __ballot_sync(MFULL, mine == 2);
  if (!EMIT) {
    if ((threadIdx.x & 31) == 0) {
      wmask[t >> 5] = m1 | ((uint64_t)m2 << 32);
      wcount[t >> 5] = __popc(m1) + __popc(m2);
    }
    return;
  }
  if (!mine) return;
  uint64_t pos = record_index(wmask, wcount, (uint32_t)t);
  if (a) {
    vlabel[pos] = a;
    vedge[pos] = (uint32_t)t;
    pos++;
  }
  if (b) {
    vlabel[pos] = b;
    vedge[pos] = (uint32_t)t;
  }
}

// emission index of the record of label L on edge slot g, whose lower endpoint is labelled a
__device__ __forceinline__ uint64_t side_index(const uint64_t* __restrict__ wmask,
                                               const unsigned long long* __restrict__ wbase, uint32_t g,
                                               uint32_t a, uint32_t L) {
  return record_index(wmask, wbase, g) + (L != a && a != 0);
}

// sorted vertex records -> packed vertex keys [label | z2 | y2 | x2], and the sorted position of
// every record by its emission index
__global__ void __launch_bounds__(256)
    k_vertex_keys(const uint32_t* __restrict__ lab, Lattice lt, const uint64_t* __restrict__ wmask,
                  const unsigned long long* __restrict__ wbase, const uint32_t* __restrict__ vlabel,
                  const uint32_t* __restrict__ vedge, uint64_t U, uint64_t* __restrict__ uniq_vkeys,
                  uint32_t* __restrict__ sorted_pos) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= U) return;
  const uint32_t L = vlabel[i], g = vedge[i];
  uint32_t x, y, z, dir;
  lt.edge(g, x, y, z, dir);
  const uint64_t vx = 2 * x + (dir == 0), vy = 2 * y + (dir == 1), vz = 2 * z + (dir == 2);
  uniq_vkeys[i] = ((uint64_t)L << V_LABEL_SHIFT) | (vz << (2 * V_COORD_BITS)) | (vy << V_COORD_BITS) | vx;
  const uint32_t a = lab[((uint64_t)z * lt.sy + y) * lt.sx + x];
  sorted_pos[side_index(wmask, wbase, g, a, L)] = (uint32_t)i;
}

// sorted triangle records -> faces as vertex ids local to the label
__global__ void __launch_bounds__(256)
    k_faces(const uint32_t* __restrict__ lab, Lattice lt, const uint32_t* __restrict__ tlabel,
            const uint64_t* __restrict__ trec, uint64_t T, const uint64_t* __restrict__ wmask,
            const unsigned long long* __restrict__ wbase, const uint32_t* __restrict__ sorted_pos,
            const uint32_t* __restrict__ vert_off, uint32_t* __restrict__ faces) {
  const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (t >= T) return;
  const uint32_t L = tlabel[t];
  const uint64_t rec = trec[t];
  const uint32_t cube = (uint32_t)(rec >> TRI_CUBE_SHIFT);
  const uint32_t cs = (uint32_t)(rec >> TRI_CASE_SHIFT) & 255u, tt = (uint32_t)rec & 7u;
  const uint32_t cx = lt.sx - 1, cy = lt.sy - 1;
  const uint32_t x = cube % cx, y = (cube / cx) % cy, z = cube / (cx * cy);
  const int8_t* row = c_mc.tri[cs];
  const uint32_t off = vert_off[L];
#pragma unroll
  for (int v = 0; v < 3; v++) {
    // table winds clockwise seen from outside for "bit = inside"; reverse it so
    // that normals point out of the label (oracle.marching_cubes flip=True)
    const int e = row[3 * tt + (2 - v)];
    const uint32_t X2 = 2 * x + c_edge_mid[e][0], Y2 = 2 * y + c_edge_mid[e][1], Z2 = 2 * z + c_edge_mid[e][2];
    const uint32_t a = lab[((uint64_t)(Z2 >> 1) * lt.sy + (Y2 >> 1)) * lt.sx + (X2 >> 1)];
    faces[3 * t + v] = sorted_pos[side_index(wmask, wbase, lt.slot(X2, Y2, Z2), a, L)] - off;
  }
}

// boundaries in a sorted array of labels -> per-label [start) markers
__global__ void __launch_bounds__(256)
    k_label_starts(const uint32_t* __restrict__ labels, uint64_t n, uint32_t* __restrict__ start /* [K+2], prefilled with n */) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t label = labels[i];
  if (i == 0 || labels[i - 1] != label) start[label] = (uint32_t)i;
}

__global__ void __launch_bounds__(256) k_fill_u32(uint32_t* a, uint32_t value, uint32_t n) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] = value;
}

__global__ void __launch_bounds__(256)
    k_vertex_positions(const uint64_t* __restrict__ uniq_vkeys, uint64_t first, uint64_t count,
                       float rx, float ry, float rz, float shift, float* __restrict__ out) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= count) return;
  const uint64_t k = uniq_vkeys[first + i];
  const float x = (float)(k & ((1u << V_COORD_BITS) - 1));
  const float y = (float)((k >> V_COORD_BITS) & ((1u << V_COORD_BITS) - 1));
  const float z = (float)((k >> (2 * V_COORD_BITS)) & ((1u << V_COORD_BITS) - 1));
  out[3 * i + 0] = __fmul_rn(__fadd_rn(__fmul_rn(x, 0.5f), shift), rx);
  out[3 * i + 1] = __fmul_rn(__fadd_rn(__fmul_rn(y, 0.5f), shift), ry);
  out[3 * i + 2] = __fmul_rn(__fadd_rn(__fmul_rn(z, 0.5f), shift), rz);
}

}  // namespace ign

#include "mesher.h"

namespace ign {
int simp_export_positions(ign_ctx* ctx, const float* pos_f, uint64_t first, uint64_t count,
                          const float shift[3], float* d_out);
}
using namespace ign;

// positions of vertices [first, first+count) into d_out (device), whichever form the mesher holds
static int mesher_positions(ign_mesher* m, uint64_t first, uint64_t count, const float resolution[3],
                            int voxel_centered, float* d_out) {
  ign_ctx* ctx = m->ctx;
  if (m->simplified) {
    IGN_REQUIRE(resolution[0] == m->res[0] && resolution[1] == m->res[1] && resolution[2] == m->res[2],
                IGN_ERR_INVALID, "resolution differs from the one the mesher was simplified with");
    const float shift[3] = {voxel_centered ? 0.5f * m->res[0] : 0.0f, voxel_centered ? 0.5f * m->res[1] : 0.0f,
                            voxel_centered ? 0.5f * m->res[2] : 0.0f};
    return simp_export_positions(ctx, m->d_pos_f, first, count, shift, d_out);
  }
  IGN_LAUNCH(ctx, k_vertex_positions, blocks_for(count, 256), 256, 0, m->d_uniq_vkeys, first, count,
             resolution[0], resolution[1], resolution[2], voxel_centered ? 0.5f : 0.0f, d_out);
  return IGN_OK;
}

// one flag per device; set after the upload has completed (mesh streams of one device share it)
static std::atomic<bool> g_tables_loaded[64];

static int load_tables(ign_ctx* ctx) {
  if (ctx->device < 64 && g_tables_loaded[ctx->device]) return IGN_OK;
  McTables h;
  memcpy(h.tri, mc_tri_table, sizeof(h.tri));
  memcpy(h.ntri, mc_tri_count, sizeof(h.ntri));
  IGN_CUDA(cudaMemcpyToSymbolAsync(c_mc, &h, sizeof(h), 0, cudaMemcpyHostToDevice, ctx->stream));
  IGN_CUDA(cudaStreamSynchronize(ctx->stream));
  if (ctx->device < 64) g_tables_loaded[ctx->device] = true;
  return IGN_OK;
}

static int bits_for(uint64_t v) {
  int b = 1;
  while (b < 64 && (1ull << b) <= v) b++;
  return b;
}

extern "C" {

int ign_mesh_free(ign_mesher* m) {
  if (!m) return IGN_OK;
  cudaSetDevice(m->ctx->device);
  if (m->pooled) {
    m->ctx->mesh_pool_busy = 0;
  } else {
    if (m->d_uniq_vkeys) cudaFree(m->d_uniq_vkeys);
    if (m->d_faces) cudaFree(m->d_faces);
  }
  delete m;
  return IGN_OK;
}

int ign_mesh_begin_dev(ign_ctx* ctx, const void* labels, int dtype, uint64_t sx, uint64_t sy,
                       uint64_t sz, ign_mesher** out) {
  IGN_TRY(activate(ctx));
  IGN_REQUIRE(labels && out, IGN_ERR_INVALID, "null argument");
  *out = nullptr;
  ProfSpan prof(ctx, IGN_PROF_MC);
  IGN_REQUIRE(sx >= 1 && sy >= 1 && sz >= 1, IGN_ERR_INVALID, "empty volume");
  IGN_REQUIRE(sx <= 1023 && sy <= 1023 && sz <= 1023, IGN_ERR_UNSUPPORTED,
              "mesher: task of %llux%llux%llu exceeds the 1023^3 limit of the packed vertex format",
              (unsigned long long)sx, (unsigned long long)sy, (unsigned long long)sz);
  IGN_TRY(load_tables(ctx));
  const uint64_t n = sx * sy * sz;

  ign_mesher* m = new ign_mesher();
  m->ctx = ctx;
  m->K = m->T = m->U = 0;
  m->d_uniq_vkeys = nullptr;
  m->d_faces = nullptr;
  m->pooled = false;
  m->simplified = false;
  m->d_pos_f = nullptr;
  m->simp_factor = 0;
  m->simp_max_error = 0;
  // a failed build frees the half-built mesher
  struct Guard {
    ign_mesher* m;
    ~Guard() { ign_mesh_free(m); }
  } guard{m};
  ScratchFrame f(ctx);

  // ---- dense labels
  uint32_t* d_lab;
  IGN_TRY(f.take(&d_lab, n));
  uint64_t K = 0;
  {
    ScratchFrame fu(ctx);  // only d_lab outlives the renumber
    uint64_t* d_uniq;
    IGN_TRY(fu.take(&d_uniq, n));
    IGN_TRY(ign_renumber_dev(ctx, labels, dtype, n, d_lab, d_uniq, n, &K));
    m->K = K;
    m->ids.resize(K);
    if (K) {
      IGN_TRY(small_d2h(ctx, m->ids.data(), d_uniq, K * 8));
      IGN_TRY(small_sync(ctx));
    }
  }
  m->tri_off.assign(K + 2, 0);
  m->vert_off.assign(K + 2, 0);
  if (K == 0 || sx < 2 || sy < 2 || sz < 2) {
    guard.m = nullptr;
    *out = m;
    return IGN_OK;
  }
  IGN_REQUIRE(K < (1ull << 31), IGN_ERR_OVERFLOW, "mesher: too many labels");

  // ---- count: triangles per CTA of cubes, vertex records per warp of edge slots.  An exclusive scan
  // of each (one slot past the end, zeroed) gives every CTA's or warp's base and, last, the total.
  const Lattice lt{(uint32_t)sx, (uint32_t)sy, (uint32_t)sz};
  const uint64_t ncubes = (sx - 1) * (sy - 1) * (sz - 1), nwarps = (3 * n + 31) / 32;
  const unsigned grid = blocks_for(ncubes, 256), egrid = blocks_for(3 * n, 256);
  unsigned long long *tcnt, *tbase, *wcnt, *wbase;
  uint64_t* wmask;
  IGN_TRY(f.take(&tcnt, grid + 1));
  IGN_TRY(f.take(&tbase, grid + 1));
  IGN_TRY(f.take(&wcnt, nwarps + 1));
  IGN_TRY(f.take(&wbase, nwarps + 1));
  IGN_TRY(f.take(&wmask, nwarps));
  size_t scanb = 0, sortt = 0, sortv = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, scanb, tcnt, tbase, (int64_t)nwarps + 1);
  void* scan_tmp;
  IGN_TRY(f.take(&scan_tmp, scanb));
  IGN_CUDA(cudaMemsetAsync(tcnt + grid, 0, 8, ctx->stream));
  IGN_CUDA(cudaMemsetAsync(wcnt + nwarps, 0, 8, ctx->stream));
  IGN_LAUNCH(ctx, (k_mc<false>), grid, 256, 0, d_lab, (uint32_t)sx, (uint32_t)sy, (uint32_t)sz, tcnt,
             (uint32_t*)nullptr, (uint64_t*)nullptr);
  IGN_LAUNCH(ctx, (k_edges<false>), egrid, 256, 0, d_lab, lt, wmask, wcnt, (uint32_t*)nullptr, (uint32_t*)nullptr);
  size_t tb = scanb;
  IGN_CUDA(cub::DeviceScan::ExclusiveSum(scan_tmp, tb, tcnt, tbase, (int64_t)grid + 1, ctx->stream));
  tb = scanb;
  IGN_CUDA(cub::DeviceScan::ExclusiveSum(scan_tmp, tb, wcnt, wbase, (int64_t)nwarps + 1, ctx->stream));
  ctx->launches += 4;
  unsigned long long tot[2];
  IGN_TRY(small_d2h(ctx, &tot[0], tbase + grid, 8));
  IGN_TRY(small_d2h(ctx, &tot[1], wbase + nwarps, 8));
  IGN_TRY(small_sync(ctx));
  const unsigned long long T = tot[0], U = tot[1];
  m->T = T;
  if (T == 0) {
    guard.m = nullptr;
    *out = m;
    return IGN_OK;
  }
  // the sorts take int item counts: 3T corners must fit an int (and U <= 3T: every vertex is a corner)
  IGN_REQUIRE(3 * T <= (unsigned long long)INT_MAX, IGN_ERR_OVERFLOW,
              "mesher: %llu triangles exceed 2^31 - 1 corners; split the volume into tasks", T);
  m->U = U;

  // ---- emit + sort buffers
  cub::DeviceRadixSort::SortPairs(nullptr, sortt, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                  (const uint64_t*)nullptr, (uint64_t*)nullptr, (int)T);
  cub::DeviceRadixSort::SortPairs(nullptr, sortv, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                  (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)U);
  const size_t tmp_bytes = sortt > sortv ? sortt : sortv;
  uint32_t *tlabel, *tlabel_s, *vlabel, *vlabel_s, *vedge, *vedge_s, *sorted_pos, *d_tri_off, *d_vert_off;
  uint64_t *trec, *trec_s;
  void* tmp;
  IGN_TRY(f.take(&tlabel, T));
  IGN_TRY(f.take(&tlabel_s, T));
  IGN_TRY(f.take(&trec, T));
  IGN_TRY(f.take(&trec_s, T));
  IGN_TRY(f.take(&vlabel, U));
  IGN_TRY(f.take(&vlabel_s, U));
  IGN_TRY(f.take(&vedge, U));
  IGN_TRY(f.take(&vedge_s, U));
  IGN_TRY(f.take(&sorted_pos, U));
  IGN_TRY(f.take(&d_tri_off, K + 2));
  IGN_TRY(f.take(&d_vert_off, K + 2));
  IGN_TRY(f.take(&tmp, tmp_bytes));

  // ---- emit in raster order; a stable sort on the label bits then gives (label, cube, t) and
  // (label, z2, y2, x2)
  const int label_bits = bits_for(K);
  IGN_LAUNCH(ctx, (k_mc<true>), grid, 256, 0, d_lab, (uint32_t)sx, (uint32_t)sy, (uint32_t)sz, tbase, tlabel,
             trec);
  tb = tmp_bytes;
  IGN_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tb, tlabel, tlabel_s, trec, trec_s, (int)T, 0, label_bits,
                                           ctx->stream));
  ctx->launches += 2;
  IGN_LAUNCH(ctx, (k_edges<true>), egrid, 256, 0, d_lab, lt, wmask, wbase, vlabel, vedge);
  tb = tmp_bytes;
  IGN_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tb, vlabel, vlabel_s, vedge, vedge_s, (int)U, 0, label_bits,
                                           ctx->stream));
  ctx->launches += 2;
  {
    const size_t fbytes = align_up(3 * T * 4, 256), vbytes = align_up(U * 12, 256);  // 12: float3 after simplify
    if (!ctx->mesh_pool_busy) {
      if (ctx->mesh_pool_bytes < fbytes + vbytes) {
        IGN_CUDA(cudaStreamSynchronize(ctx->stream));
        if (ctx->mesh_pool) cudaFree(ctx->mesh_pool);
        ctx->mesh_pool = nullptr;
        ctx->mesh_pool_bytes = 0;
        const size_t want = (fbytes + vbytes) * 5 / 4;
        IGN_CUDA(cudaMalloc((void**)&ctx->mesh_pool, want));
        ctx->mesh_pool_bytes = want;
      }
      m->d_faces = (uint32_t*)ctx->mesh_pool;
      m->d_uniq_vkeys = (uint64_t*)(ctx->mesh_pool + fbytes);
      m->pooled = true;
      ctx->mesh_pool_busy = 1;
    } else {
      IGN_CUDA(cudaMalloc((void**)&m->d_faces, 3 * T * 4));
      IGN_CUDA(cudaMalloc((void**)&m->d_uniq_vkeys, U * 12));  // 12: float3 positions after simplification
    }
  }
  IGN_LAUNCH(ctx, k_vertex_keys, blocks_for(U, 256), 256, 0, d_lab, lt, wmask, wbase, vlabel_s, vedge_s,
             (uint64_t)U, m->d_uniq_vkeys, sorted_pos);

  // ---- per-label offsets (labels are 1..K; slot K+1 is the end sentinel)
  IGN_LAUNCH(ctx, k_fill_u32, blocks_for(K + 2, 256), 256, 0, d_tri_off, (uint32_t)T, (uint32_t)(K + 2));
  IGN_LAUNCH(ctx, k_fill_u32, blocks_for(K + 2, 256), 256, 0, d_vert_off, (uint32_t)U, (uint32_t)(K + 2));
  IGN_LAUNCH(ctx, k_label_starts, blocks_for(T, 256), 256, 0, tlabel_s, (uint64_t)T, d_tri_off);
  IGN_LAUNCH(ctx, k_label_starts, blocks_for(U, 256), 256, 0, vlabel_s, (uint64_t)U, d_vert_off);
  IGN_TRY(small_d2h(ctx, m->tri_off.data(), d_tri_off, (K + 2) * 4));
  IGN_TRY(small_d2h(ctx, m->vert_off.data(), d_vert_off, (K + 2) * 4));
  IGN_TRY(small_sync(ctx));
  // absent labels hold the end marker: a suffix minimum turns starts into offsets
  for (int64_t l = (int64_t)K; l >= 0; l--) {
    if (m->tri_off[l] > m->tri_off[l + 1]) m->tri_off[l] = m->tri_off[l + 1];
    if (m->vert_off[l] > m->vert_off[l + 1]) m->vert_off[l] = m->vert_off[l + 1];
  }
  IGN_TRY(small_h2d(ctx, d_vert_off, m->vert_off.data(), (K + 2) * 4));
  IGN_LAUNCH(ctx, k_faces, blocks_for(T, 256), 256, 0, d_lab, lt, tlabel_s, trec_s, (uint64_t)T, wmask, wbase,
             sorted_pos, d_vert_off, m->d_faces);
  IGN_CUDA(cudaStreamSynchronize(ctx->stream));
  for (uint64_t l = 1; l <= K; l++)
    if (m->tri_off[l + 1] > m->tri_off[l]) m->present.push_back(m->ids[l - 1]);
  guard.m = nullptr;
  *out = m;
  return IGN_OK;
}

int ign_mesh_begin(ign_ctx* ctx, const void* labels, int dtype, uint64_t sx, uint64_t sy, uint64_t sz,
                   ign_mesher** out) {
  // the mesher keeps no reference to its labels: they can go when the staging frame closes
  return staged(ctx, {{labels, nullptr, sx * sy * sz * dtype_size(dtype)}},
                [&](void* const* d) { return ign_mesh_begin_dev(ctx, d[0], dtype, sx, sy, sz, out); });
}

int ign_mesh_num_ids(ign_mesher* m, uint64_t* n) {
  IGN_REQUIRE(m && n, IGN_ERR_INVALID, "null argument");
  *n = m->present.size();
  return IGN_OK;
}

int ign_mesh_ids(ign_mesher* m, uint64_t* ids, uint64_t capacity) {
  IGN_REQUIRE(m && ids, IGN_ERR_INVALID, "null argument");
  const uint64_t k = m->present.size() < capacity ? m->present.size() : capacity;
  for (uint64_t i = 0; i < k; i++) ids[i] = m->present[i];
  return IGN_OK;
}

int ign_mesh_totals(ign_mesher* m, uint64_t* nv, uint64_t* nf) {
  IGN_REQUIRE(m && nv && nf, IGN_ERR_INVALID, "null argument");
  *nv = m->U;
  *nf = m->T;
  return IGN_OK;
}

static int64_t dense_of(ign_mesher* m, uint64_t id) {
  // ids[] is in first-appearance order, not sorted: linear scan is fine for the
  // per-id API (bulk export does not need it)
  for (uint64_t i = 0; i < m->ids.size(); i++)
    if (m->ids[i] == id) return (int64_t)i + 1;
  return -1;
}

int ign_mesh_counts(ign_mesher* m, uint64_t id, uint64_t* nv, uint64_t* nf) {
  IGN_REQUIRE(m && nv && nf, IGN_ERR_INVALID, "null argument");
  const int64_t l = dense_of(m, id);
  IGN_REQUIRE(l > 0, IGN_ERR_KEY, "%llu", (unsigned long long)id);
  *nv = m->vert_off[l + 1] - m->vert_off[l];
  *nf = m->tri_off[l + 1] - m->tri_off[l];
  return IGN_OK;
}

int ign_mesh_get(ign_mesher* m, uint64_t id, const float resolution[3], int reduction_factor,
                 float max_error, int voxel_centered, float* vertices, uint32_t* faces, uint64_t* nv,
                 uint64_t* nf) {
  IGN_REQUIRE(m && resolution && nv && nf, IGN_ERR_INVALID, "null argument");
  ign_ctx* ctx = m->ctx;
  IGN_TRY(activate(ctx));
  if (reduction_factor > 0 && !m->simplified) IGN_TRY(ign_mesh_simplify(m, resolution, reduction_factor, max_error));
  if (m->simplified) {
    IGN_REQUIRE(reduction_factor == m->simp_factor && max_error == m->simp_max_error, IGN_ERR_INVALID,
                "mesher was simplified with reduction_factor=%d max_error=%g; call mesh() again to change",
                m->simp_factor, (double)m->simp_max_error);
  }
  const int64_t l = dense_of(m, id);
  IGN_REQUIRE(l > 0, IGN_ERR_KEY, "%llu", (unsigned long long)id);
  const uint64_t v0 = m->vert_off[l], v1 = m->vert_off[l + 1];
  const uint64_t t0 = m->tri_off[l], t1 = m->tri_off[l + 1];
  *nv = v1 - v0;
  *nf = t1 - t0;
  if (*nv == 0 || vertices == nullptr || faces == nullptr) return IGN_OK;
  ScratchFrame f(ctx);
  float* d_pos;
  IGN_TRY(f.take(&d_pos, (v1 - v0) * 3));
  IGN_TRY(mesher_positions(m, v0, v1 - v0, resolution, voxel_centered, d_pos));
  IGN_CUDA(cudaMemcpyAsync(vertices, d_pos, (v1 - v0) * 12, cudaMemcpyDeviceToHost, ctx->stream));
  IGN_CUDA(cudaMemcpyAsync(faces, m->d_faces + 3 * t0, (t1 - t0) * 12, cudaMemcpyDeviceToHost, ctx->stream));
  IGN_CUDA(cudaStreamSynchronize(ctx->stream));
  return IGN_OK;
}

int ign_mesh_export(ign_mesher* m, const float resolution[3], int voxel_centered, float* vertices,
                    uint32_t* faces, uint64_t* vert_offsets, uint64_t* face_offsets) {
  IGN_REQUIRE(m && resolution && vert_offsets && face_offsets, IGN_ERR_INVALID, "null argument");
  ign_ctx* ctx = m->ctx;
  IGN_TRY(activate(ctx));
  uint64_t j = 0;
  for (uint64_t l = 1; l <= m->K; l++) {
    if (m->tri_off[l + 1] > m->tri_off[l]) {
      vert_offsets[j] = m->vert_off[l];
      face_offsets[j] = m->tri_off[l];
      j++;
    }
  }
  vert_offsets[j] = m->U;
  face_offsets[j] = m->T;
  if (m->U == 0 || vertices == nullptr || faces == nullptr) return IGN_OK;
  ScratchFrame f(ctx);
  float* d_pos;
  IGN_TRY(f.take(&d_pos, m->U * 3));
  IGN_TRY(mesher_positions(m, 0, m->U, resolution, voxel_centered, d_pos));
  IGN_TRY(d2h_by_kernel(ctx, vertices, d_pos, m->U * 12));
  IGN_TRY(d2h_by_kernel(ctx, faces, m->d_faces, m->T * 12));
  IGN_CUDA(cudaStreamSynchronize(ctx->stream));
  return IGN_OK;
}

}  // extern "C"
