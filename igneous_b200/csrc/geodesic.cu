// geodesic.cu -- single-source shortest paths on the voxel lattice for every label of a volume in
// the same launches (the `dijkstra3d` wheel that kimimaro's TEASAR reads its distance-from-root and
// parent fields from), the per-label argmax around it and the TEASAR penalty field, sm_90a.  The
// rule is DESIGN.md §5e: voxels p, q are joined when they are neighbours under the connectivity and
// carry the same non-zero label; d[source] = 0 and d[q] = fl32(d[p] + w(p -> q)), one float32
// addition per edge, least over all paths from a source of q's label; +inf elsewhere.  float32
// addition is monotone in its first argument, so the least fixed point of the relaxation is unique
// whatever order it runs in, and equals what a heap Dijkstra computes with the same additions.
//
//   k_geo_init     d = +inf, parents = 0; the field weights are checked here (finite and >= 0).
//   k_geo_sources  d[source] = 0; the source's brick goes on the first dirty list, and so does every
//                  neighbouring brick whose halo holds the source: a source never falls, so no
//                  sweep would wake them, and it may be the only voxel joining two bricks.
//   k_geo_relax    one round of the label-correcting solver.  A CTA takes a dirty brick of
//                  32 x 8 x 8 voxels, stages its labels and distances with a one-voxel halo in
//                  shared memory, and pulls d[q] = min(d[q], fl32(d[p] + w)) over the brick (every
//                  thread owns a z-column; all read, barrier, all write, barrier) until a sweep
//                  changes nothing.  Only the brick's own voxels are written, so no two CTAs write
//                  one word.  Every neighbouring brick whose halo holds a lowered voxel is put on
//                  the next round's list (a flag per brick keeps it there once).  A CTA may stage a
//                  halo word (__ldcg) while the CTA that owns it stores to it in the same launch:
//                  by design.  The word is aligned and only ever falls, so the reader gets the old
//                  or the new value, both upper bounds; and the owner puts the reader on the next
//                  list after every store, whichever the reader saw, so it is staged again in a
//                  later launch, which sees the store.  A racecheck report on dist[] between
//                  those two accesses is this and nothing else.
//   k_geo_parents  after convergence: the first neighbour p, in the neighbour order below, with
//                  fl32(d[p] + w) == d[q] and (d[p], p) < (d[q], q).
//
// Rounds are chained without the host: the grid is fixed, the list and its length live on the
// device, and a round whose list is empty returns at once.  The host reads the length back every
// GEO_ROUNDS_PER_SYNC rounds and stops when it is zero.  A shortest path that crosses k brick faces
// is final after round k + 1, and a simple path crosses fewer faces than the volume has voxels, so
// geo_round_cap() bounds the loop; reaching it is reported as an error.  The sweep loop inside a brick
// is bounded the same way by the brick's voxel count (a brick that reaches it puts itself back on
// the list), so every launch ends whatever the data.
//
// Neighbour order: (dz, dy, dx) in raster order, dx fastest, each from -1 to 1, the centre left
// out, keeping |dx| + |dy| + |dz| <= 1 / 2 / 3 for connectivity 6 / 18 / 26: ascending linear index.
//
// Compiled with -fmad=false: k_teasar_pdrf's float32 expression is rounded operation by operation.
#include <math.h>

#include <algorithm>

#include "common.cuh"

namespace ign {

namespace {

constexpr int BX = 32, BY = 8, BZ = 8;
constexpr int HX = BX + 2, HY = BY + 2, HZ = BZ + 2, HN = HX * HY * HZ;
constexpr int GEO_THREADS = BX * BY;               // one thread per z-column of the brick
constexpr int GEO_MAX_SWEEPS = BX * BY * BZ;       // a path inside a brick has at most this many voxels
constexpr int GEO_ROUNDS_PER_SYNC = 8;
constexpr uint32_t INF_BITS = 0x7F800000u;
constexpr uint32_t SOURCE_MARK = 0xFFFFFFFFu;      // parents[] of a source until k_geo_parents clears it
constexpr uint32_t FULL = 0xFFFFFFFFu;
enum { ERR_WEIGHT = 1, ERR_SOURCE_RANGE = 2, ERR_SOURCE_ZERO = 4, ERR_NO_PARENT = 8 };

struct Nbrs {
  int n, maxdiag;
  int8_t dx[26], dy[26], dz[26];
  float w[26];  // euclidean edge lengths
};

// device-resident control block of one solve
struct GeoCtl {
  uint32_t count[3];  // length of the list of round r at count[r % 3]
  uint32_t err;
  unsigned long long visits, rounds;
  unsigned long long orphan;  // 1 + the highest linear index of a reached voxel without a parent
};

thread_local uint64_t g_stats[3];  // rounds, brick visits, host synchronisations of the last solve

uint64_t geo_round_cap(uint64_t n) { return n + 1; }

Nbrs make_nbrs(int connectivity, const float* a) {
  Nbrs nb{};
  nb.maxdiag = connectivity == 6 ? 1 : connectivity == 18 ? 2 : 3;
  for (int dz = -1; dz <= 1; ++dz)
    for (int dy = -1; dy <= 1; ++dy)
      for (int dx = -1; dx <= 1; ++dx) {
        const int m = abs(dx) + abs(dy) + abs(dz);
        if (m == 0 || m > nb.maxdiag) continue;
        nb.dx[nb.n] = (int8_t)dx;
        nb.dy[nb.n] = (int8_t)dy;
        nb.dz[nb.n] = (int8_t)dz;
        if (a) {
          const double x = (double)a[0] * dx, y = (double)a[1] * dy, z = (double)a[2] * dz;
          nb.w[nb.n] = (float)sqrt(x * x + y * y + z * z);
        }
        ++nb.n;
      }
  return nb;
}

__device__ __forceinline__ bool weight_ok(float w) { return w >= 0.f && w < __uint_as_float(INF_BITS); }

__global__ void __launch_bounds__(256) k_geo_init(uint32_t* __restrict__ dist, uint32_t* __restrict__ parents,
                                                  const float* __restrict__ W, uint64_t n, GeoCtl* ctl) {
  bool bad = false;
  for (uint64_t i = blockIdx.x * 256ull + threadIdx.x; i < n; i += (uint64_t)gridDim.x * 256) {
    dist[i] = INF_BITS;
    if (parents) parents[i] = 0;
    if (W && !weight_ok(W[i])) bad = true;
  }
  if (__any_sync(FULL, bad) && (threadIdx.x & 31) == 0) atomicOr(&ctl->err, ERR_WEIGHT);
}

__device__ __forceinline__ void mark_brick(uint32_t b, uint32_t* flags, uint32_t* list, uint32_t* count) {
  if (atomicExch(flags + b, 1u) == 0u) list[atomicAdd(count, 1u)] = b;
}

template <typename T>
__global__ void __launch_bounds__(256) k_geo_sources(const T* __restrict__ lab, const uint64_t* __restrict__ src,
                                                     uint64_t ns, uint64_t n, uint64_t sx, uint64_t sy,
                                                     uint32_t nbx, uint32_t nby, uint32_t nbz, int maxdiag,
                                                     uint32_t* dist, uint32_t* parents, GeoCtl* ctl, uint32_t* list,
                                                     uint32_t* flags) {
  const uint64_t i = blockIdx.x * 256ull + threadIdx.x;
  if (i >= ns) return;
  const uint64_t s = src[i];
  if (s >= n) {
    atomicOr(&ctl->err, ERR_SOURCE_RANGE);
    return;
  }
  if (lab[s] == T(0)) {
    atomicOr(&ctl->err, ERR_SOURCE_ZERO);
    return;
  }
  dist[s] = 0;
  if (parents) parents[s] = SOURCE_MARK;
  const uint64_t x = s % sx, y = (s / sx) % sy, z = s / (sx * sy);
  const int64_t bx = x / BX, by = y / BY, bz = z / BZ;
  const int ex = x % BX == 0 ? -1 : x % BX == BX - 1 ? 1 : 0, ey = y % BY == 0 ? -1 : y % BY == BY - 1 ? 1 : 0,
            ez = z % BZ == 0 ? -1 : z % BZ == BZ - 1 ? 1 : 0;
  for (int m = 0; m < 8; ++m) {  // the brick itself (m == 0) and those across the faces the source lies on
    if (((m & 1) && !ex) || ((m & 2) && !ey) || ((m & 4) && !ez) || __popc(m) > maxdiag) continue;
    const int64_t qx = bx + ((m & 1) ? ex : 0), qy = by + ((m & 2) ? ey : 0), qz = bz + ((m & 4) ? ez : 0);
    if (qx < 0 || qy < 0 || qz < 0 || qx >= nbx || qy >= nby || qz >= nbz) continue;
    mark_brick((uint32_t)(qx + nbx * (qy + (int64_t)nby * qz)), flags, list, &ctl->count[0]);
  }
}

template <typename T, bool FIELD>
__global__ void __launch_bounds__(GEO_THREADS) k_geo_relax(const T* __restrict__ lab, const float* __restrict__ W,
                                                           uint32_t* dist, uint64_t sx, uint64_t sy, uint64_t sz,
                                                           uint32_t nbx, uint32_t nby, uint32_t nbz, Nbrs nb,
                                                           GeoCtl* ctl, uint32_t* lists, uint32_t* flags,
                                                           uint32_t nbricks, uint32_t round /* mod 6 */) {
  __shared__ T sl[HN];
  __shared__ uint32_t sd[HN];
  __shared__ int soff[26];
  __shared__ float sw[26];
  __shared__ uint32_t smarks;
  const uint32_t* cur_list = lists + (round & 1) * (uint64_t)nbricks;
  uint32_t* cur_flags = flags + (round & 1) * (uint64_t)nbricks;
  uint32_t* next_list = lists + ((round + 1) & 1) * (uint64_t)nbricks;
  uint32_t* next_flags = flags + ((round + 1) & 1) * (uint64_t)nbricks;
  uint32_t* next_count = &ctl->count[(round + 1) % 3];
  const uint32_t ncur = ctl->count[round % 3];
  const int tid = threadIdx.x, tx = tid & (BX - 1), ty = tid / BX;
  if (blockIdx.x == 0 && tid == 0) {
    ctl->count[(round + 2) % 3] = 0;  // the list after next; no CTA of this launch reads or appends to it
    ctl->visits += ncur;
    ctl->rounds += ncur ? 1 : 0;
  }
  if (tid < nb.n) {
    soff[tid] = nb.dx[tid] + HX * (nb.dy[tid] + HY * nb.dz[tid]);
    sw[tid] = nb.w[tid];
  }
  for (uint32_t li = blockIdx.x; li < ncur; li += gridDim.x) {
    const uint32_t b = cur_list[li];
    const uint32_t bx = b % nbx, by = (b / nbx) % nby, bz = b / (nbx * nby);
    if (tid == 0) {
      cur_flags[b] = 0;
      smarks = 0;
    }
    for (int i = tid; i < HN; i += GEO_THREADS) {
      const int64_t gx = (int64_t)bx * BX + i % HX - 1, gy = (int64_t)by * BY + (i / HX) % HY - 1,
                    gz = (int64_t)bz * BZ + i / (HX * HY) - 1;
      const bool in = gx >= 0 && gy >= 0 && gz >= 0 && gx < (int64_t)sx && gy < (int64_t)sy && gz < (int64_t)sz;
      const uint64_t g = (uint64_t)gx + sx * ((uint64_t)gy + sy * (uint64_t)gz);
      sl[i] = in ? lab[g] : T(0);
      sd[i] = in ? __ldcg(dist + g) : INF_BITS;
    }
    __syncthreads();
    // this thread's column: which neighbours share the voxel's label, its distance and entry cost
    const int c0 = (tx + 1) + HX * ((ty + 1) + HY);
    const uint64_t gx = (uint64_t)bx * BX + tx, gy = (uint64_t)by * BY + ty;
    uint32_t m[BZ], cur[BZ], fell = 0;  // fell: bit z set once cur[z] dropped
    float w[BZ];
#pragma unroll
    for (int z = 0; z < BZ; ++z) {
      const int c = c0 + z * HX * HY;
      const T l = sl[c];
      uint32_t mk = 0;
      if (l != T(0))
        for (int k = 0; k < nb.n; ++k) mk |= (uint32_t)(sl[c + soff[k]] == l) << k;
      m[z] = mk;
      cur[z] = sd[c];
      w[z] = 0.f;
      if (FIELD && mk) {
        const float v = W[gx + sx * (gy + sy * ((uint64_t)bz * BZ + z))];
        w[z] = weight_ok(v) ? v : __uint_as_float(INF_BITS);  // a refused weight lowers nothing
      }
    }
    int sweeps = 0;
    for (;;) {
      bool changed = false;
#pragma unroll
      for (int z = 0; z < BZ; ++z) {
        const int c = c0 + z * HX * HY;
        uint32_t best = cur[z];
        for (int k = 0; k < nb.n; ++k)
          if (m[z] >> k & 1)
            best = min(best, __float_as_uint(__uint_as_float(sd[c + soff[k]]) + (FIELD ? w[z] : sw[k])));
        if (best < cur[z]) fell |= 1u << z;
        changed |= best < cur[z];
        cur[z] = best;
      }
      __syncthreads();
      if (changed) {
#pragma unroll
        for (int z = 0; z < BZ; ++z) sd[c0 + z * HX * HY] = cur[z];
      }
      ++sweeps;
      if (!__syncthreads_or(changed) || sweeps >= GEO_MAX_SWEEPS) break;
    }
    // write back what fell, and collect the neighbouring bricks whose halo holds such a voxel
    uint32_t marks = (sweeps >= GEO_MAX_SWEEPS && tid == 0) ? 1u << 13 : 0u;
#pragma unroll
    for (int z = 0; z < BZ; ++z) {
      if (fell >> z & 1) {
        dist[gx + sx * (gy + sy * ((uint64_t)bz * BZ + z))] = cur[z];
        const int ex = tx == 0 ? -1 : tx == BX - 1 ? 1 : 0, ey = ty == 0 ? -1 : ty == BY - 1 ? 1 : 0,
                  ez = z == 0 ? -1 : z == BZ - 1 ? 1 : 0;
        for (int s = 1; s < 8; ++s) {
          const int ox = (s & 1) ? ex : 0, oy = (s & 2) ? ey : 0, oz = (s & 4) ? ez : 0;
          if (((s & 1) && !ex) || ((s & 2) && !ey) || ((s & 4) && !ez) || __popc(s) > nb.maxdiag) continue;
          marks |= 1u << ((ox + 1) + 3 * (oy + 1) + 9 * (oz + 1));
        }
      }
    }
    marks = __reduce_or_sync(FULL, marks);
    if ((tid & 31) == 0 && marks) atomicOr(&smarks, marks);
    __syncthreads();
    if (tid < 27 && (smarks >> tid & 1)) {
      const int64_t qx = (int64_t)bx + tid % 3 - 1, qy = (int64_t)by + (tid / 3) % 3 - 1, qz = (int64_t)bz + tid / 9 - 1;
      if (qx >= 0 && qy >= 0 && qz >= 0 && qx < nbx && qy < nby && qz < nbz)
        mark_brick((uint32_t)(qx + nbx * (qy + (int64_t)nby * qz)), next_flags, next_list, next_count);
    }
    __syncthreads();
  }
}

template <typename T, bool FIELD>
__global__ void __launch_bounds__(256) k_geo_parents(const T* __restrict__ lab, const float* __restrict__ W,
                                                     const uint32_t* __restrict__ dist, uint32_t* __restrict__ parents,
                                                     uint64_t sx, uint64_t sy, uint64_t sz, Nbrs nb, GeoCtl* ctl) {
  const uint64_t n = sx * sy * sz;
  for (uint64_t q = blockIdx.x * 256ull + threadIdx.x; q < n; q += (uint64_t)gridDim.x * 256) {
    if (parents[q] == SOURCE_MARK) {
      parents[q] = 0;
      continue;
    }
    const T l = lab[q];
    const uint32_t dq = dist[q];
    if (l == T(0) || dq == INF_BITS) continue;
    const int64_t x = q % sx, y = (q / sx) % sy, z = q / (sx * sy);
    const float wq = FIELD ? W[q] : 0.f;
    uint32_t found = 0;
    for (int k = 0; k < nb.n && !found; ++k) {
      const int64_t px = x + nb.dx[k], py = y + nb.dy[k], pz = z + nb.dz[k];
      if (px < 0 || py < 0 || pz < 0 || px >= (int64_t)sx || py >= (int64_t)sy || pz >= (int64_t)sz) continue;
      const uint64_t p = (uint64_t)px + sx * ((uint64_t)py + sy * (uint64_t)pz);
      if (lab[p] != l) continue;
      const uint32_t dp = dist[p];
      if (__float_as_uint(__uint_as_float(dp) + (FIELD ? wq : nb.w[k])) == dq && (dp < dq || (dp == dq && p < q)))
        found = (uint32_t)p + 1;
    }
    if (found) parents[q] = found;
    else {
      atomicOr(&ctl->err, ERR_NO_PARENT);
      atomicMax(&ctl->orphan, (unsigned long long)q + 1);
    }
  }
}

int geo_fail(uint32_t err, unsigned long long orphan = 0) {
  IGN_REQUIRE(!(err & ERR_WEIGHT), IGN_ERR_INVALID, "geodesic: a field weight is negative, infinite or NaN");
  IGN_REQUIRE(!(err & ERR_SOURCE_RANGE), IGN_ERR_INVALID, "geodesic: a source lies outside the volume");
  IGN_REQUIRE(!(err & ERR_SOURCE_ZERO), IGN_ERR_INVALID, "geodesic: a source lies on label 0");
  IGN_REQUIRE(!(err & ERR_NO_PARENT), IGN_ERR_INVALID,
              "geodesic: the reached voxel q at linear index %llu (and maybe others below it) has no predecessor p "
              "with fl32(d[p] + w) == d[q] and (d[p], p) < (d[q], q): a float32 plateau entered from a higher "
              "index; no parent field was completed",
              orphan - 1);
  return IGN_OK;
}

template <typename T, bool FIELD>
int geo_run(ign_ctx* ctx, const void* labels, uint64_t sx, uint64_t sy, uint64_t sz, const Nbrs& nb,
            const float* W, const uint64_t* sources, uint64_t ns, float* dist_out, uint32_t* parents) {
  const T* lab = (const T*)labels;
  uint32_t* dist = (uint32_t*)dist_out;
  const uint64_t n = sx * sy * sz;
  const uint32_t nbx = (uint32_t)((sx + BX - 1) / BX), nby = (uint32_t)((sy + BY - 1) / BY),
                 nbz = (uint32_t)((sz + BZ - 1) / BZ);
  const uint64_t nbricks64 = (uint64_t)nbx * nby * nbz;
  IGN_REQUIRE(nbricks64 < (1ull << 31), IGN_ERR_OVERFLOW, "geodesic: %llu bricks of %d x %d x %d (below 2^31)",
              (unsigned long long)nbricks64, BX, BY, BZ);
  const uint32_t nbricks = (uint32_t)nbricks64;
  ScratchFrame f(ctx);
  GeoCtl* ctl;
  uint32_t *lists, *flags;
  IGN_TRY(f.take(&ctl, 1));
  IGN_TRY(f.take(&lists, 2 * (uint64_t)nbricks));
  IGN_TRY(f.take(&flags, 2 * (uint64_t)nbricks));
  IGN_CUDA(cudaMemsetAsync(ctl, 0, sizeof(GeoCtl), ctx->stream));
  IGN_CUDA(cudaMemsetAsync(flags, 0, 2 * (uint64_t)nbricks * 4, ctx->stream));
  const unsigned vgrid = (unsigned)std::min<uint64_t>(blocks_for(n, 256), (uint64_t)ctx->sm_count * 16);
  IGN_LAUNCH(ctx, k_geo_init, vgrid, 256, 0, dist, parents, W, n, ctl);
  if (ns)
    IGN_LAUNCH(ctx, k_geo_sources<T>, blocks_for(ns, 256), 256, 0, lab, sources, ns, n, sx, sy, nbx, nby, nbz,
               nb.maxdiag, dist, parents, ctl, lists, flags);
  const unsigned grid = std::min<uint32_t>(nbricks, (uint32_t)ctx->sm_count * 8);
  const uint64_t cap = geo_round_cap(n);
  GeoCtl h{};
  uint64_t syncs = 0;
  for (uint64_t r = 0;;) {
    for (int i = 0; i < GEO_ROUNDS_PER_SYNC; ++i, ++r)
      IGN_LAUNCH(ctx, (k_geo_relax<T, FIELD>), grid, GEO_THREADS, 0, lab, W, dist, sx, sy, sz, nbx, nby, nbz, nb, ctl,
                 lists, flags, nbricks, (uint32_t)(r % 6));
    IGN_TRY(small_d2h(ctx, &h, ctl, sizeof(GeoCtl)));
    IGN_TRY(small_sync(ctx));
    ++syncs;
    g_stats[0] = h.rounds;
    g_stats[1] = h.visits;
    g_stats[2] = syncs;
    IGN_TRY(geo_fail(h.err));
    if (h.count[r % 3] == 0) break;
    IGN_REQUIRE(r < cap, IGN_ERR_INVALID, "geodesic: not converged after %llu rounds (the bound for %llu voxels)",
                (unsigned long long)r, (unsigned long long)n);
  }
  if (parents) {
    IGN_LAUNCH(ctx, (k_geo_parents<T, FIELD>), vgrid, 256, 0, lab, W, dist, parents, sx, sy, sz, nb, ctl);
    IGN_TRY(small_d2h(ctx, &h, ctl, sizeof(GeoCtl)));
    IGN_TRY(small_sync(ctx));
    g_stats[2] = syncs + 1;
    IGN_TRY(geo_fail(h.err, h.orphan));
  }
  return IGN_OK;
}

int geo_check(int dtype, uint64_t sx, uint64_t sy, uint64_t sz, int connectivity, const float* a, bool field,
              bool parents) {
  IGN_REQUIRE(dtype == IGN_U8 || dtype == IGN_U16 || dtype == IGN_U32 || dtype == IGN_U64, IGN_ERR_UNSUPPORTED,
              "geodesic: label dtype %d is not u8 / u16 / u32 / u64", dtype);
  IGN_REQUIRE(connectivity == 6 || connectivity == 18 || connectivity == 26, IGN_ERR_INVALID,
              "geodesic: connectivity %d is not 6, 18 or 26", connectivity);
  IGN_REQUIRE(sx < (1ull << 30) && sy < (1ull << 30) && sz < (1ull << 30), IGN_ERR_OVERFLOW,
              "geodesic: volume %llu x %llu x %llu (each side below 2^30)", (unsigned long long)sx,
              (unsigned long long)sy, (unsigned long long)sz);
  // each side is below 2^30, so sx * sy cannot wrap; the third factor is bounded by a division
  IGN_REQUIRE(sz == 0 || sx * sy <= (1ull << 62) / sz, IGN_ERR_OVERFLOW,
              "geodesic: volume %llu x %llu x %llu holds more than 2^62 voxels", (unsigned long long)sx,
              (unsigned long long)sy, (unsigned long long)sz);
  IGN_REQUIRE(!parents || sx * sy * sz < 0xFFFFFFFFull, IGN_ERR_OVERFLOW,
              "geodesic: %llu voxels; the uint32 parent field holds fewer than 2^32 - 1",
              (unsigned long long)(sx * sy * sz));
  if (!field) {
    IGN_REQUIRE(a, IGN_ERR_INVALID, "geodesic: null anisotropy");
    for (int i = 0; i < 3; ++i)
      IGN_REQUIRE(a[i] > 0.f && isfinite(a[i]), IGN_ERR_INVALID, "geodesic: anisotropy[%d] = %g (positive and finite)",
                  i, (double)a[i]);
  }
  return IGN_OK;
}

// order-preserving map of a float onto uint32; 0 is below every float
__device__ __forceinline__ uint32_t ord_of(float v) {
  const uint32_t b = __float_as_uint(v + 0.f);  // -0 counts as +0
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float ord_to(uint32_t k) {
  return __uint_as_float((k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k);
}

template <typename T, bool SECOND>
__global__ void __launch_bounds__(256) k_argmax(const T* __restrict__ lab, const float* __restrict__ field, uint64_t n,
                                                uint64_t max_label, uint32_t* __restrict__ keys,
                                                unsigned long long* __restrict__ index) {
  for (uint64_t i = blockIdx.x * 256ull + threadIdx.x; i < n; i += (uint64_t)gridDim.x * 256) {
    const uint64_t l = lab[i];
    if (l == 0 || l > max_label) continue;
    const float v = field[i];
    if (!isfinite(v)) continue;
    if (!SECOND) atomicMax(keys + l, ord_of(v));
    else if (keys[l] == ord_of(v)) atomicMin(index + l, (unsigned long long)i);
  }
}

__global__ void __launch_bounds__(256) k_argmax_values(const uint32_t* __restrict__ keys, uint64_t count,
                                                       float* __restrict__ value) {
  const uint64_t l = blockIdx.x * 256ull + threadIdx.x;
  if (l < count) value[l] = keys[l] ? ord_to(keys[l]) : -__uint_as_float(INF_BITS);
}

template <typename T>
__global__ void __launch_bounds__(256) k_teasar_pdrf(const T* __restrict__ lab, const float* __restrict__ dbf,
                                                     const float* __restrict__ daf, const float* __restrict__ dbf_max,
                                                     const float* __restrict__ daf_max, uint64_t n, uint64_t max_label,
                                                     float scale, int exponent, float* __restrict__ out) {
  for (uint64_t i = blockIdx.x * 256ull + threadIdx.x; i < n; i += (uint64_t)gridDim.x * 256) {
    const uint64_t l = lab[i];
    const float a = daf[i];
    float r = 0.f;
    if (l != 0 && l <= max_label && a < __uint_as_float(INF_BITS)) {
      const float t = 1.f - dbf[i] / (1.01f * dbf_max[l]);
      float p = t;
      for (int e = 1; e < exponent; ++e) p = p * t;
      const float am = daf_max[l];
      r = scale * p + (am > 0.f ? a / am : 0.f);
    }
    out[i] = r;
  }
}

}  // namespace

}  // namespace ign

using namespace ign;

extern "C" {

int ign_geodesic_dev(ign_ctx* ctx, const void* labels, int dtype, uint64_t sx, uint64_t sy, uint64_t sz,
                     int connectivity, const float anisotropy[3], const float* weights, const uint64_t* sources,
                     uint64_t n_sources, float* dist_out, uint32_t* parents_out) {
  IGN_TRY(activate(ctx));
  IGN_TRY(geo_check(dtype, sx, sy, sz, connectivity, anisotropy, weights != nullptr, parents_out != nullptr));
  g_stats[0] = g_stats[1] = g_stats[2] = 0;
  if (sx * sy * sz == 0) return IGN_OK;
  IGN_REQUIRE(labels && dist_out && (sources || !n_sources), IGN_ERR_INVALID, "geodesic: null buffer");
  IGN_REQUIRE((uintptr_t)labels % dtype_size(dtype) == 0 && (uintptr_t)dist_out % 4 == 0 &&
                  (uintptr_t)weights % 4 == 0 && (uintptr_t)parents_out % 4 == 0 && (uintptr_t)sources % 8 == 0,
              IGN_ERR_INVALID, "geodesic: a buffer is not aligned to its element size");
  const Nbrs nb = make_nbrs(connectivity, weights ? nullptr : anisotropy);
  return dispatch_label(dtype, "geodesic", [&](auto v) -> int {
    using T = decltype(v);
    if (weights)
      return geo_run<T, true>(ctx, labels, sx, sy, sz, nb, weights, sources, n_sources, dist_out, parents_out);
    return geo_run<T, false>(ctx, labels, sx, sy, sz, nb, nullptr, sources, n_sources, dist_out, parents_out);
  });
}

int ign_geodesic(ign_ctx* ctx, const void* labels, int dtype, uint64_t sx, uint64_t sy, uint64_t sz, int connectivity,
                 const float anisotropy[3], const float* weights, const uint64_t* sources, uint64_t n_sources,
                 float* dist_out, uint32_t* parents_out) {
  IGN_TRY(geo_check(dtype, sx, sy, sz, connectivity, anisotropy, weights != nullptr, parents_out != nullptr));
  const uint64_t n = sx * sy * sz;
  return staged(ctx,
                {{labels, nullptr, n * dtype_size(dtype)},
                 {weights, nullptr, n * 4},
                 {n_sources ? sources : nullptr, nullptr, n_sources * 8},
                 {nullptr, dist_out, n * 4},
                 {nullptr, parents_out, n * 4}},
                [&](void* const* d) {
                  return ign_geodesic_dev(ctx, d[0], dtype, sx, sy, sz, connectivity, anisotropy, (const float*)d[1],
                                          (const uint64_t*)d[2], n_sources, (float*)d[3], (uint32_t*)d[4]);
                });
}

int ign_geodesic_round_cap(uint64_t sx, uint64_t sy, uint64_t sz, uint64_t* cap) {
  IGN_REQUIRE(cap, IGN_ERR_INVALID, "geodesic: null cap");
  IGN_TRY(geo_check(IGN_U8, sx, sy, sz, 6, nullptr, true, false));
  *cap = geo_round_cap(sx * sy * sz);
  return IGN_OK;
}

int ign_geodesic_last_stats(uint64_t stats[3]) {
  IGN_REQUIRE(stats, IGN_ERR_INVALID, "geodesic: null stats");
  for (int i = 0; i < 3; ++i) stats[i] = g_stats[i];
  return IGN_OK;
}

int ign_label_argmax_dev(ign_ctx* ctx, const void* labels, int dtype, uint64_t n, const float* field,
                         uint64_t max_label, uint64_t* index_out, float* value_out) {
  IGN_TRY(activate(ctx));
  IGN_REQUIRE(max_label < (1ull << 32), IGN_ERR_UNSUPPORTED,
              "label_argmax: largest label %llu does not fit 32 bits (renumber the labels first)",
              (unsigned long long)max_label);
  IGN_REQUIRE(index_out && value_out && (n == 0 || (labels && field)), IGN_ERR_INVALID, "label_argmax: null buffer");
  return dispatch_label(dtype, "label_argmax", [&](auto v) -> int {
    using T = decltype(v);
    ScratchFrame f(ctx);
    uint32_t* keys;
    IGN_TRY(f.take(&keys, max_label + 1));
    IGN_CUDA(cudaMemsetAsync(keys, 0, (max_label + 1) * 4, ctx->stream));
    IGN_CUDA(cudaMemsetAsync(index_out, 0xFF, (max_label + 1) * 8, ctx->stream));
    if (n) {
      const unsigned grid = (unsigned)std::min<uint64_t>(blocks_for(n, 256), (uint64_t)ctx->sm_count * 16);
      IGN_LAUNCH(ctx, (k_argmax<T, false>), grid, 256, 0, (const T*)labels, field, n, max_label, keys,
                 (unsigned long long*)index_out);
      IGN_LAUNCH(ctx, (k_argmax<T, true>), grid, 256, 0, (const T*)labels, field, n, max_label, keys,
                 (unsigned long long*)index_out);
    }
    IGN_LAUNCH(ctx, k_argmax_values, blocks_for(max_label + 1, 256), 256, 0, keys, max_label + 1, value_out);
    return IGN_OK;
  });
}

int ign_teasar_pdrf_dev(ign_ctx* ctx, const void* labels, int dtype, uint64_t n, const float* dbf, const float* daf,
                        const float* dbf_max, const float* daf_max, uint64_t max_label, float scale, int exponent,
                        float* out) {
  IGN_TRY(activate(ctx));
  IGN_REQUIRE(exponent >= 1 && exponent <= 64, IGN_ERR_INVALID, "teasar_pdrf: exponent %d (a whole number from 1 to 64)",
              exponent);
  IGN_REQUIRE(isfinite(scale) && scale >= 0.f, IGN_ERR_INVALID, "teasar_pdrf: scale %g (finite and >= 0)", (double)scale);
  if (n == 0) return IGN_OK;
  IGN_REQUIRE(labels && dbf && daf && dbf_max && daf_max && out, IGN_ERR_INVALID, "teasar_pdrf: null buffer");
  return dispatch_label(dtype, "teasar_pdrf", [&](auto v) -> int {
    using T = decltype(v);
    const unsigned grid = (unsigned)std::min<uint64_t>(blocks_for(n, 256), (uint64_t)ctx->sm_count * 16);
    IGN_LAUNCH(ctx, k_teasar_pdrf<T>, grid, 256, 0, (const T*)labels, dbf, daf, dbf_max, daf_max, n, max_label, scale,
               exponent, out);
    return IGN_OK;
  });
}

}  // extern "C"
