// xsection.cu -- cross-sectional areas at skeleton vertices (kimimaro.cross_sectional_area), sm_90a.  The rule
// is DESIGN.md §5i: each point has a voxel c, a label and a normal n (float64, physical units); voxel q of the
// label is cut when |s| < h with s = n0 d0 + n1 d1 + n2 d2, d_i = (q_i - c_i) a_i and
// h = ((|n0| a0 + |n1| a1) + |n2| a2) / 2, all float64 without FMA (the file is built with -fmad=false); the
// section is the set of cut voxels 26-connected to c through cut voxels; its area is the float64 sum over the
// section of the exact area of the plane inside each voxel's box, rounded to float32.
//
//   k_xs_small  one warp per point (taken from a counter): breadth-first walk with a shared-memory hash set
//               (1024 slots) and queue (512 voxels) of offsets from c.  A section that outgrows either, or
//               reaches 512 voxels from c, stops and appends its point to the large list.
//   k_xs_large  one 512-thread CTA per large point (taken from a counter), over a pool of slots in global
//               memory: a level-synchronous walk whose visited set is a bitmap over the plane's projection
//               along its dominant axis (the axis of the largest |n_k| a_k): at most three voxels of a column
//               are cut, so one byte per column holds them, bit q_k - floor(t) + 3 where t is the real q_k on
//               the plane.  The queue holds 3 voxels per column.  The CTA clears the bytes it set before it takes
//               the next point.
//
// ign_cross_section_normals is the host pass that gives every vertex of a skeleton its normal: an O(V w)
// walk over the tree of each component, too little work and too many dependent steps for the device.
#include <algorithm>
#include <cmath>
#include <vector>

#include "common.cuh"

namespace ign {

namespace {

constexpr int XS_WARPS = 8;       // warps per k_xs_small CTA
constexpr int XS_HCAP = 1024;     // hash slots per warp
constexpr int XS_QCAP = 512;      // queued voxels per warp: a larger section goes to k_xs_large
constexpr int XS_REACH = 511;     // offsets from c the packed key holds
constexpr int XS_LARGE = 512;     // threads per k_xs_large CTA
constexpr uint32_t XS_EMPTY = 0xFFFFFFFFu;
constexpr uint64_t XS_SLOT_BUDGET = 512ull << 20;  // bytes of bitmaps and queues for the large points at once

struct XsCtl {
  unsigned long long next;        // next point of k_xs_small
  unsigned long long next_large;  // next entry of the large list
  unsigned long long n_large;     // points appended to the large list
  unsigned long long voxels;      // voxels of every finished section
  unsigned long long abandoned;   // voxels k_xs_small visited in sections it handed on
  unsigned long long bad;         // lowest point with a voxel outside the volume or a non-finite normal
  uint32_t err;                   // bit 0: bad point; bit 1: a large section broke its column or queue bound
  uint32_t pad;
};

// Everything a point's walk needs, set up by xs_point.
struct XsPoint {
  double n[3], h, nn;  // normal, half band, |n|
  double e[3];         // |n_i| a_i / 2, descending: the first m are the nonzero components
  double inv;          // |n| / (prod of the nonzero |n_i|) (times 1/2 with three nonzero)
  double zprod;        // product of a_i over the zero components
  int m;               // nonzero components
  uint32_t cx, cy, cz;
};

__device__ __forceinline__ void xs_order(double& x, double& y) {
  const double lo = fmin(x, y);
  x = fmax(x, y);
  y = lo;
}

// false: the point gets area 0 and contacts 0 (zero normal, or its voxel holds another label)
template <typename T>
__device__ bool xs_point(const T* __restrict__ lab, uint32_t sx, uint32_t sy, uint32_t sz,
                         const uint64_t* __restrict__ voxel, const uint64_t* __restrict__ plabel,
                         const double* __restrict__ normal, uint64_t p, double a0, double a1, double a2, XsCtl* ctl,
                         XsPoint& P) {
  const uint64_t n = (uint64_t)sx * sy * sz;
  const uint64_t c = voxel[p];
  const double n0 = normal[3 * p], n1 = normal[3 * p + 1], n2 = normal[3 * p + 2];
  if (c >= n || !isfinite(n0) || !isfinite(n1) || !isfinite(n2)) {
    atomicOr(&ctl->err, 1u);
    atomicMin(&ctl->bad, (unsigned long long)p);
    return false;
  }
  if ((n0 == 0.0 && n1 == 0.0 && n2 == 0.0) || (uint64_t)lab[c] != plabel[p]) return false;
  P.n[0] = n0;
  P.n[1] = n1;
  P.n[2] = n2;
  P.h = 0.5 * ((fabs(n0) * a0 + fabs(n1) * a1) + fabs(n2) * a2);
  P.nn = sqrt((n0 * n0 + n1 * n1) + n2 * n2);
  P.m = (n0 != 0.0) + (n1 != 0.0) + (n2 != 0.0);
  P.zprod = (n0 == 0.0 ? a0 : 1.0) * (n1 == 0.0 ? a1 : 1.0) * (n2 == 0.0 ? a2 : 1.0);
  const double prod = (n0 != 0.0 ? fabs(n0) : 1.0) * (n1 != 0.0 ? fabs(n1) : 1.0) * (n2 != 0.0 ? fabs(n2) : 1.0);
  P.inv = P.nn / (P.m == 3 ? 2.0 * prod : prod);
  P.e[0] = fabs(n0) * a0 * 0.5;
  P.e[1] = fabs(n1) * a1 * 0.5;
  P.e[2] = fabs(n2) * a2 * 0.5;
  xs_order(P.e[0], P.e[1]);
  xs_order(P.e[1], P.e[2]);
  xs_order(P.e[0], P.e[1]);
  P.cx = (uint32_t)(c % sx);
  P.cy = (uint32_t)((c / sx) % sy);
  P.cz = (uint32_t)(c / sx / sy);
  return true;
}

__device__ __forceinline__ double xs_s(const XsPoint& P, int dx, int dy, int dz, double a0, double a1, double a2) {
  return (P.n[0] * ((double)dx * a0) + P.n[1] * ((double)dy * a1)) + P.n[2] * ((double)dz * a2);
}

// The area of the plane n.y = -s inside the box [-a/2, a/2] around a cut voxel: |n| times the derivative of
// the box's volume below the plane, by inclusion-exclusion over the corners of its nonzero axes.
__device__ double xs_area(const XsPoint& P, double s) {
  if (P.m == 1) return P.zprod;
  const double t = -s;
  const double e0 = P.e[0], e1 = P.e[1];
  double f = 0.0;
  if (P.m == 2) {
    for (int k = 0; k < 4; ++k) {
      const double u0 = (k & 1) ? e0 : -e0, u1 = (k & 2) ? e1 : -e1;
      const double w = t - (u0 + u1);
      if (w > 0.0) f += (__popc(k) & 1) ? -w : w;
    }
    return P.zprod * (f * P.inv);
  }
  const double e2 = P.e[2];
  for (int k = 0; k < 8; ++k) {
    const double u0 = (k & 1) ? e0 : -e0, u1 = (k & 2) ? e1 : -e1, u2 = (k & 4) ? e2 : -e2;
    const double w = t - ((u0 + u1) + u2);
    if (w > 0.0) f += (__popc(k) & 1) ? -(w * w) : w * w;
  }
  return f * P.inv;
}

__device__ __forceinline__ uint32_t xs_faces(uint32_t x, uint32_t y, uint32_t z, uint32_t sx, uint32_t sy,
                                             uint32_t sz) {
  return (x == 0 ? 1u : 0u) | (x == sx - 1 ? 2u : 0u) | (y == 0 ? 4u : 0u) | (y == sy - 1 ? 8u : 0u) |
         (z == 0 ? 16u : 0u) | (z == sz - 1 ? 32u : 0u);
}

__device__ __forceinline__ uint32_t xs_key(int dx, int dy, int dz) {
  return (uint32_t)(dx + 512) | ((uint32_t)(dy + 512) << 10) | ((uint32_t)(dz + 512) << 20);
}

__device__ __forceinline__ double warp_sum(double v) {
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xFFFFFFFFu, v, o);
  return v;
}

template <typename T>
__global__ void __launch_bounds__(XS_WARPS * 32) k_xs_small(
    const T* __restrict__ lab, uint32_t sx, uint32_t sy, uint32_t sz, const uint64_t* __restrict__ voxel,
    const uint64_t* __restrict__ plabel, const double* __restrict__ normal, uint64_t np, double a0, double a1,
    double a2, float* __restrict__ area, uint8_t* __restrict__ contacts, uint32_t* __restrict__ large, XsCtl* ctl) {
  __shared__ uint32_t s_tab[XS_WARPS][XS_HCAP];
  __shared__ uint32_t s_q[XS_WARPS][XS_QCAP];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  uint32_t* tab = s_tab[w];
  uint32_t* q = s_q[w];
  const uint32_t lt = (1u << lane) - 1;
  for (;;) {
    unsigned long long p = 0;
    if (lane == 0) p = atomicAdd(&ctl->next, 1ull);
    p = __shfl_sync(0xFFFFFFFFu, p, 0);
    if (p >= np) return;
    XsPoint P;
    if (!xs_point(lab, sx, sy, sz, voxel, plabel, normal, p, a0, a1, a2, ctl, P)) {
      if (lane == 0) {
        area[p] = 0.f;
        contacts[p] = 0;
      }
      continue;
    }
    const T L = lab[voxel[p]];
    for (int i = lane; i < XS_HCAP; i += 32) tab[i] = XS_EMPTY;
    __syncwarp();
    const uint32_t k0 = xs_key(0, 0, 0);
    if (lane == 0) {
      tab[(k0 * 2654435761u) >> 22] = k0;
      q[0] = k0;
    }
    __syncwarp();
    uint32_t head = 0, tail = 1;
    bool over = false;
    double acc = 0.0;
    uint32_t con = 0;
    while (head < tail && !over) {
      const uint32_t i = head + lane, end = min(head + 32, tail);  // this round's items: [head, end)
      const bool act = i < end;
      int dx = 0, dy = 0, dz = 0;
      if (act) {
        const uint32_t k = q[i];
        dx = (int)(k & 1023) - 512;
        dy = (int)((k >> 10) & 1023) - 512;
        dz = (int)(k >> 20) - 512;
        acc += xs_area(P, xs_s(P, dx, dy, dz, a0, a1, a2));
        con |= xs_faces(P.cx + dx, P.cy + dy, P.cz + dz, sx, sy, sz);
      }
      for (int nb = 0; nb < 27; ++nb) {
        if (nb == 13) continue;
        const int ex = dx + nb % 3 - 1, ey = dy + (nb / 3) % 3 - 1, ez = dz + nb / 9 - 1;
        bool fresh = false;
        uint32_t key = 0;
        if (act) {
          const long long x = (long long)P.cx + ex, y = (long long)P.cy + ey, z = (long long)P.cz + ez;
          if (x >= 0 && y >= 0 && z >= 0 && x < sx && y < sy && z < sz &&
              fabs(xs_s(P, ex, ey, ez, a0, a1, a2)) < P.h && lab[(uint64_t)x + sx * ((uint64_t)y + (uint64_t)sy * z)] == L) {
            if (max(abs(ex), max(abs(ey), abs(ez))) > XS_REACH) {
              over = true;
            } else {
              key = xs_key(ex, ey, ez);
              uint32_t slot = (key * 2654435761u) >> 22;
              int probe = 0;
              for (; probe < XS_HCAP; ++probe, slot = (slot + 1) & (XS_HCAP - 1)) {
                const uint32_t old = atomicCAS(&tab[slot], XS_EMPTY, key);
                if (old == XS_EMPTY) { fresh = true; break; }
                if (old == key) break;
              }
              if (probe == XS_HCAP) over = true;
            }
          }
        }
        const uint32_t b = __ballot_sync(0xFFFFFFFFu, fresh);
        if (fresh) {
          const uint32_t pos = tail + __popc(b & lt);
          if (pos < XS_QCAP) q[pos] = key;
        }
        tail += __popc(b);
      }
      over = __any_sync(0xFFFFFFFFu, over) || tail > XS_QCAP;
      head = end;
      __syncwarp();
    }
    if (over) {
      if (lane == 0) {
        large[atomicAdd(&ctl->n_large, 1ull)] = (uint32_t)p;
        atomicAdd(&ctl->abandoned, (unsigned long long)min(tail, (uint32_t)XS_QCAP));
      }
    } else {
      acc = warp_sum(acc);
      con = __reduce_or_sync(0xFFFFFFFFu, con);
      if (lane == 0) {
        area[p] = (float)acc;
        contacts[p] = (uint8_t)con;
        atomicAdd(&ctl->voxels, (unsigned long long)tail);
      }
    }
    __syncwarp();
  }
}

// The byte of voxel (q_i, q_j, *) of a large point's bitmap, and the bit of q_k in it (8: outside the byte).
struct XsCols {
  int k, i, j;                 // dominant axis, then the other two ascending
  uint32_t si;                 // extent along i
  long long ci, cj;            // c_i, c_j
  double ai, aj, ni, nj, nk_ak, base;  // n_k a_k; the real c_k before the terms of i and j
};

__device__ __forceinline__ uint32_t xs_sel(uint32_t x, uint32_t y, uint32_t z, int axis) {
  return axis == 0 ? x : (axis == 1 ? y : z);
}
__device__ __forceinline__ double xs_sel(double x, double y, double z, int axis) {
  return axis == 0 ? x : (axis == 1 ? y : z);
}

__device__ __forceinline__ uint64_t xs_col(const XsCols& C, uint32_t x, uint32_t y, uint32_t z) {
  return (uint64_t)xs_sel(x, y, z, C.i) + (uint64_t)C.si * xs_sel(x, y, z, C.j);
}

__device__ __forceinline__ uint32_t xs_bit(const XsCols& C, uint32_t x, uint32_t y, uint32_t z) {
  const double di = (double)((long long)xs_sel(x, y, z, C.i) - C.ci) * C.ai;
  const double dj = (double)((long long)xs_sel(x, y, z, C.j) - C.cj) * C.aj;
  const double t = C.base - (C.ni * di + C.nj * dj) / C.nk_ak;
  const long long b = (long long)xs_sel(x, y, z, C.k) - ((long long)floor(t) - 3);
  return (b >= 0 && b < 8) ? (uint32_t)b : 8u;
}

template <typename T>
__global__ void __launch_bounds__(XS_LARGE) k_xs_large(
    const T* __restrict__ lab, uint32_t sx, uint32_t sy, uint32_t sz, const uint64_t* __restrict__ voxel,
    const uint64_t* __restrict__ plabel, const double* __restrict__ normal, double a0, double a1, double a2,
    const uint32_t* __restrict__ large, uint32_t* __restrict__ maps, uint64_t map_words,
    uint32_t* __restrict__ queues, uint64_t qcap, float* __restrict__ area, uint8_t* __restrict__ contacts,
    XsCtl* ctl) {
  __shared__ unsigned long long s_p;
  __shared__ uint32_t s_tail, s_con, s_bad;
  __shared__ double s_acc[XS_LARGE / 32];
  uint32_t* map = maps + blockIdx.x * map_words;
  uint32_t* q = queues + blockIdx.x * qcap;
  const uint32_t lane = threadIdx.x & 31, lt = (1u << lane) - 1;
  for (;;) {
    if (threadIdx.x == 0) {
      s_p = atomicAdd(&ctl->next_large, 1ull);
      s_tail = 1;
      s_con = 0;
      s_bad = 0;
    }
    __syncthreads();
    if (s_p >= ctl->n_large) return;
    const uint64_t p = large[s_p];
    XsPoint P;
    xs_point(lab, sx, sy, sz, voxel, plabel, normal, p, a0, a1, a2, ctl, P);  // true: it was in k_xs_small
    const T L = lab[voxel[p]];
    XsCols C;
    const double e0 = fabs(P.n[0]) * a0, e1 = fabs(P.n[1]) * a1, e2 = fabs(P.n[2]) * a2;
    C.k = e1 > e0 ? (e2 > e1 ? 2 : 1) : (e2 > e0 ? 2 : 0);
    C.i = C.k == 0 ? 1 : 0;
    C.j = C.k == 2 ? 1 : 2;
    C.si = xs_sel(sx, sy, sz, C.i);
    C.ci = xs_sel(P.cx, P.cy, P.cz, C.i);
    C.cj = xs_sel(P.cx, P.cy, P.cz, C.j);
    C.ai = xs_sel(a0, a1, a2, C.i);
    C.aj = xs_sel(a0, a1, a2, C.j);
    C.ni = xs_sel(P.n[0], P.n[1], P.n[2], C.i);
    C.nj = xs_sel(P.n[0], P.n[1], P.n[2], C.j);
    C.nk_ak = xs_sel(P.n[0], P.n[1], P.n[2], C.k) * xs_sel(a0, a1, a2, C.k);
    C.base = (double)xs_sel(P.cx, P.cy, P.cz, C.k);
    if (threadIdx.x == 0) {
      const uint64_t col = xs_col(C, P.cx, P.cy, P.cz);
      atomicOr(&map[col >> 2], 1u << ((col & 3) * 8 + xs_bit(C, P.cx, P.cy, P.cz)));  // bit 3: t is c_k
      q[0] = (uint32_t)voxel[p];
    }
    __syncthreads();
    uint32_t lo = 0, hi = 1;
    double acc = 0.0;
    uint32_t con = 0;
    while (lo < hi) {
      for (uint32_t base = lo; base < hi; base += XS_LARGE) {
        const uint32_t idx = base + threadIdx.x;
        const bool act = idx < hi;
        uint32_t x = 0, y = 0, z = 0;
        if (act) {
          const uint32_t v = q[idx];
          x = v % sx;
          y = (v / sx) % sy;
          z = v / sx / sy;
          acc += xs_area(P, xs_s(P, (int)x - (int)P.cx, (int)y - (int)P.cy, (int)z - (int)P.cz, a0, a1, a2));
          con |= xs_faces(x, y, z, sx, sy, sz);
        }
        for (int nb = 0; nb < 27; ++nb) {
          if (nb == 13) continue;
          const long long nx = (long long)x + nb % 3 - 1, ny = (long long)y + (nb / 3) % 3 - 1,
                          nz = (long long)z + nb / 9 - 1;
          bool fresh = false;
          uint32_t v = 0;
          if (act && nx >= 0 && ny >= 0 && nz >= 0 && nx < sx && ny < sy && nz < sz) {
            v = (uint32_t)((uint64_t)nx + sx * ((uint64_t)ny + (uint64_t)sy * nz));
            if (fabs(xs_s(P, (int)(nx - P.cx), (int)(ny - P.cy), (int)(nz - P.cz), a0, a1, a2)) < P.h && lab[v] == L) {
              const uint32_t b = xs_bit(C, (uint32_t)nx, (uint32_t)ny, (uint32_t)nz);
              const uint64_t col = xs_col(C, (uint32_t)nx, (uint32_t)ny, (uint32_t)nz);
              if (b == 8) {
                s_bad = 1;
              } else {
                const uint32_t m = 1u << ((col & 3) * 8 + b);
                fresh = !(atomicOr(&map[col >> 2], m) & m);
              }
            }
          }
          const uint32_t bal = __ballot_sync(0xFFFFFFFFu, fresh);
          uint32_t start = 0;
          if (lane == 0 && bal) start = atomicAdd(&s_tail, (uint32_t)__popc(bal));
          start = __shfl_sync(0xFFFFFFFFu, start, 0);
          if (fresh) {
            const uint32_t pos = start + __popc(bal & lt);
            if (pos < qcap) q[pos] = v; else s_bad = 1;
          }
        }
      }
      __syncthreads();
      lo = hi;
      hi = (uint32_t)min((uint64_t)s_tail, qcap);
      __syncthreads();
    }
    acc = warp_sum(acc);
    con = __reduce_or_sync(0xFFFFFFFFu, con);
    if (lane == 0) {
      s_acc[threadIdx.x >> 5] = acc;
      atomicOr(&s_con, con);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      double sum = 0.0;
      for (int i = 0; i < XS_LARGE / 32; ++i) sum += s_acc[i];
      area[p] = (float)sum;
      contacts[p] = (uint8_t)s_con;
      atomicAdd(&ctl->voxels, (unsigned long long)hi);
      if (s_bad) atomicOr(&ctl->err, 2u);
    }
    // clear what this point set: every word holding a visited column is this point's alone
    for (uint32_t idx = threadIdx.x; idx < hi; idx += XS_LARGE) {
      const uint32_t v = q[idx];
      map[xs_col(C, v % sx, (v / sx) % sy, v / sx / sy) >> 2] = 0;
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------- normals (host)

struct Graph {
  std::vector<uint64_t> off;
  std::vector<uint32_t> adj;
};

// breadth-first hop distances from src over the component; the visit order is returned in `order`
void bfs(const Graph& g, uint32_t src, std::vector<int64_t>& dist, std::vector<uint32_t>& order) {
  order.clear();
  order.push_back(src);
  dist[src] = 0;
  for (size_t h = 0; h < order.size(); ++h) {
    const uint32_t u = order[h];
    for (uint64_t e = g.off[u]; e < g.off[u + 1]; ++e) {
      const uint32_t w = g.adj[e];
      if (dist[w] < 0) {
        dist[w] = dist[u] + 1;
        order.push_back(w);
      }
    }
  }
}

// numpy's 'symmetric' padding of positions 0..len-1
int64_t reflect(int64_t j, int64_t len) {
  int64_t m = j % (2 * len);
  if (m < 0) m += 2 * len;
  return m < len ? m : 2 * len - 1 - m;
}

}  // namespace
}  // namespace ign

using namespace ign;

extern "C" {

int ign_cross_section_normals(uint64_t n_vertices, const int64_t* voxels, uint64_t n_edges, const uint32_t* edges,
                              const double anisotropy[3], uint64_t window, double* normals_out) {
  IGN_REQUIRE(anisotropy, IGN_ERR_INVALID, "cross_section_normals: null anisotropy");
  for (int i = 0; i < 3; ++i)
    IGN_REQUIRE(anisotropy[i] > 0.0 && std::isfinite(anisotropy[i]), IGN_ERR_INVALID,
                "cross_section_normals: anisotropy[%d] = %g (positive and finite)", i, anisotropy[i]);
  IGN_REQUIRE(window >= 1, IGN_ERR_INVALID, "cross_section_normals: window 0 (at least 1)");
  IGN_REQUIRE(n_vertices < (1ull << 32), IGN_ERR_UNSUPPORTED, "cross_section_normals: %llu vertices (below 2^32)",
              (unsigned long long)n_vertices);
  if (n_vertices == 0) return IGN_OK;
  IGN_REQUIRE(voxels && normals_out && (edges || !n_edges), IGN_ERR_INVALID, "cross_section_normals: null buffer");
  const uint32_t V = (uint32_t)n_vertices;
  Graph g;
  g.off.assign(V + 1, 0);
  for (uint64_t e = 0; e < n_edges; ++e) {
    const uint32_t u = edges[2 * e], w = edges[2 * e + 1];
    IGN_REQUIRE(u < V && w < V, IGN_ERR_INVALID, "cross_section_normals: edge %llu (%u, %u) with %u vertices",
                (unsigned long long)e, u, w, V);
    if (u == w) continue;
    g.off[u + 1]++;
    g.off[w + 1]++;
  }
  for (uint32_t v = 0; v < V; ++v) g.off[v + 1] += g.off[v];
  g.adj.resize(g.off[V]);
  {
    std::vector<uint64_t> fill(g.off.begin(), g.off.end() - 1);
    for (uint64_t e = 0; e < n_edges; ++e) {
      const uint32_t u = edges[2 * e], w = edges[2 * e + 1];
      if (u == w) continue;
      g.adj[fill[u]++] = w;
      g.adj[fill[w]++] = u;
    }
  }
  std::vector<int64_t> ds(V, -1), depth(V, -1);
  std::vector<uint32_t> order, comp, parent(V), best(V), down(V);
  std::vector<uint8_t> has_child(V);
  const double* a = anisotropy;
  const int64_t half = (int64_t)(window / 2), w = (int64_t)window;
  std::vector<uint32_t> seg;  // a path's vertices around v, by position
  for (uint32_t s = 0; s < V; ++s) {
    if (ds[s] >= 0) continue;
    bfs(g, s, ds, comp);  // s is the lowest vertex of its component: every lower one was seen before
    uint32_t r = s;
    for (uint32_t u : comp)
      if (ds[u] > ds[r] || (ds[u] == ds[r] && u < r)) r = u;
    if (comp.size() == 1) {
      normals_out[3 * s] = normals_out[3 * s + 1] = normals_out[3 * s + 2] = 0.0;
      continue;
    }
    bfs(g, r, depth, order);
    for (uint32_t u : order) {
      has_child[u] = 0;
      parent[u] = u;
      if (u == r) continue;
      for (uint64_t e = g.off[u]; e < g.off[u + 1]; ++e) {
        const uint32_t x = g.adj[e];
        if (depth[x] == depth[u] - 1 && (parent[u] == u || x < parent[u])) parent[u] = x;
      }
    }
    for (uint32_t u : order)
      if (u != r) has_child[parent[u]] = 1;
    for (uint32_t u : order) best[u] = has_child[u] ? UINT32_MAX : u;
    // deepest first: every child settles its best leaf before its parent compares it
    for (size_t h = order.size(); h-- > 1;) {
      const uint32_t u = order[h], p = parent[u], b = best[u];
      const uint32_t c = best[p];
      if (c == UINT32_MAX || depth[b] < depth[c] || (depth[b] == depth[c] && b < c)) {
        best[p] = b;
        down[p] = u;
      }
    }
    for (uint32_t v : order) {
      const int64_t L = depth[best[v]], i = L - depth[v];  // positions 0 (the leaf) .. L (the root)
      const int64_t lo = std::max<int64_t>(0, i - w), hi = std::min<int64_t>(L, i + w);
      seg.assign((size_t)(hi - lo + 1), 0);
      uint32_t u = v;
      for (int64_t pos = i; pos >= lo; --pos) {
        seg[pos - lo] = u;
        if (pos > lo) u = down[u];
      }
      u = v;
      for (int64_t pos = i; pos <= hi; ++pos) {
        seg[pos - lo] = u;
        if (pos < hi) u = parent[u];
      }
      // d at path position pos: c_u - c_parent(u), the root taking the step of position L - 1
      auto step = [&](int64_t pos, int64_t out[3]) {
        const uint32_t x = seg[(pos == L ? L - 1 : pos) - lo];
        for (int k = 0; k < 3; ++k) out[k] = voxels[3 * (uint64_t)x + k] - voxels[3 * (uint64_t)parent[x] + k];
      };
      int64_t sum[3] = {0, 0, 0}, d[3];
      for (int64_t j = i - half; j < i - half + w; ++j) {
        step(reflect(j, L + 1), d);
        for (int k = 0; k < 3; ++k) sum[k] += d[k];
      }
      if (sum[0] == 0 && sum[1] == 0 && sum[2] == 0) {
        step(i, d);
        for (int k = 0; k < 3; ++k) sum[k] = d[k];
      }
      for (int k = 0; k < 3; ++k) normals_out[3 * (uint64_t)v + k] = (double)sum[k] * a[k];
    }
  }
  return IGN_OK;
}

int ign_cross_section_dev(ign_ctx* ctx, const void* labels, int dtype, uint64_t sx, uint64_t sy, uint64_t sz,
                          const uint64_t* voxel, const uint64_t* label, const double* normal, uint64_t n_points,
                          const double anisotropy[3], float* area_out, uint8_t* contacts_out, uint64_t stats[4]) {
  IGN_TRY(activate(ctx));
  IGN_REQUIRE(anisotropy && stats, IGN_ERR_INVALID, "cross_section: null argument");
  stats[0] = stats[1] = stats[2] = stats[3] = 0;
  for (int i = 0; i < 3; ++i)
    IGN_REQUIRE(anisotropy[i] > 0.0 && std::isfinite(anisotropy[i]), IGN_ERR_INVALID,
                "cross_section: anisotropy[%d] = %g (positive and finite)", i, anisotropy[i]);
  IGN_REQUIRE(sx && sy && sz, IGN_ERR_INVALID, "cross_section: an empty volume");
  IGN_REQUIRE(sx < (1ull << 32) && sy < (1ull << 32) && sz < (1ull << 32) && sx * sy < (1ull << 32) &&
                  sx * sy * sz < (1ull << 32),
              IGN_ERR_UNSUPPORTED, "cross_section: volume (%llu, %llu, %llu) (fewer than 2^32 voxels)",
              (unsigned long long)sx, (unsigned long long)sy, (unsigned long long)sz);
  IGN_REQUIRE(n_points < (1ull << 32), IGN_ERR_UNSUPPORTED, "cross_section: %llu points (below 2^32)",
              (unsigned long long)n_points);
  if (n_points == 0) return IGN_OK;
  IGN_REQUIRE(labels && voxel && label && normal && area_out && contacts_out, IGN_ERR_INVALID,
              "cross_section: null buffer");
  const uint64_t n = sx * sy * sz;
  const double a0 = anisotropy[0], a1 = anisotropy[1], a2 = anisotropy[2];
  ScratchFrame f(ctx);
  XsCtl* ctl;
  uint32_t* large;
  IGN_TRY(f.take(&ctl, 1));
  IGN_TRY(f.take(&large, n_points));
  XsCtl init{};
  init.bad = ~0ull;
  IGN_TRY(small_h2d(ctx, ctl, &init, sizeof(XsCtl)));
  const unsigned small_grid = (unsigned)std::min<uint64_t>(blocks_for(n_points, XS_WARPS), 4ull * ctx->sm_count);
  IGN_TRY(dispatch_label(dtype, "cross_section", [&](auto t) -> int {
    using T = decltype(t);
    IGN_LAUNCH(ctx, k_xs_small<T>, small_grid, XS_WARPS * 32, 0, (const T*)labels, (uint32_t)sx, (uint32_t)sy,
               (uint32_t)sz, voxel, label, normal, n_points, a0, a1, a2, area_out, contacts_out, large, ctl);
    return IGN_OK;
  }));
  XsCtl h{};
  IGN_TRY(small_d2h(ctx, &h, ctl, sizeof(XsCtl)));
  IGN_TRY(small_sync(ctx));
  IGN_REQUIRE(!(h.err & 1u), IGN_ERR_INVALID,
              "cross_section: point %llu has a voxel outside the volume or a non-finite normal", h.bad);
  if (h.n_large) {
    // one slot per concurrent CTA: a byte per column of the largest projection, and a queue of 3 voxels per
    // column (|q_k - t| < 1.5 cuts at most 3 voxels of a column; a section past the queue fails the call)
    const uint64_t proj = std::max({sx * sy, sx * sz, sy * sz});
    const uint64_t words = (proj + 3) / 4, qcap = std::min(3 * proj, n);
    const uint64_t per_slot = words * 4 + qcap * 4;
    const uint64_t slots = std::max<uint64_t>(
        1, std::min<uint64_t>({h.n_large, (uint64_t)ctx->sm_count, XS_SLOT_BUDGET / per_slot}));
    uint32_t *maps, *queues;
    IGN_TRY(f.take(&maps, words * slots));
    IGN_TRY(f.take(&queues, qcap * slots));
    IGN_CUDA(cudaMemsetAsync(maps, 0, words * slots * 4, ctx->stream));
    IGN_TRY(dispatch_label(dtype, "cross_section", [&](auto t) -> int {
      using T = decltype(t);
      IGN_LAUNCH(ctx, k_xs_large<T>, (unsigned)slots, XS_LARGE, 0, (const T*)labels, (uint32_t)sx, (uint32_t)sy,
                 (uint32_t)sz, voxel, label, normal, a0, a1, a2, large, maps, words, queues, qcap, area_out,
                 contacts_out, ctl);
      return IGN_OK;
    }));
    IGN_TRY(small_d2h(ctx, &h, ctl, sizeof(XsCtl)));
    IGN_TRY(small_sync(ctx));
    stats[3] = slots;
    IGN_REQUIRE(!(h.err & 2u), IGN_ERR_OVERFLOW,
                "cross_section: a large section outgrew its queue of 3 voxels per column of its projection, or "
                "a cut voxel fell outside its column's byte");
  }
  stats[0] = h.voxels;
  stats[1] = h.n_large;
  stats[2] = h.abandoned;
  return IGN_OK;
}

}  // extern "C"
