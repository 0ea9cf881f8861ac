// skelmerge.cu -- the merge stage of skeletonization, sm_90a: every label's skeleton fragments are cropped,
// fused, consolidated and postprocessed (dust, loops, connect pieces, ticks), then encoded as neuroglancer
// precomputed skeletons, for a whole batch of labels in one call.  The rule is DESIGN.md §5h.
//
// Bulk passes over the batch:
//   k_mg_ranges / k_mg_verts / k_mg_edges  input checks: CSR ranges, finite vertices, edge indices inside their
//                 fragment (read back and refused before any other pass)
//   k_mg_keys     per vertex: crop test against its fragment's box; the keys (label, x, y, z) as orderable
//                 32-bit words, -0.0 folded into 0.0; a cropped vertex gets label ~0 and sorts last
//   (sort x4)     LSD radix sort of the positions by z, y, x, label: stable, so a run starts at the first occurrence
//   k_mg_heads    1 where a run of equal keys starts; an inclusive sum numbers the unique vertices
//   k_mg_uid      the unique vertex of every input vertex, and of every unique vertex its first occurrence
//   k_mg_ekeys    per input edge: (min, max) of the unique ends, ~0 for a self-loop or a cropped end
//   (sort)        64-bit edge keys: the order (label, lo, hi), since unique vertices are label-major
//   k_mg_eheads / k_mg_used / k_mg_compact  unique edges, vertices with an edge, compacted arrays
//   k_mg_label_ranges  per label its vertex and edge ranges
// Per label, one CTA (k_mg_post): cable length against max_cable_length, dust, loops (thread 0: cycles are
// rare), connect pieces (Borůvka rounds, every thread searching candidates), ticks (block-wide argmin per
// removal).  Edges live in a per-label slice of 2 * ne + nv + 1 entries of global vertex indices.
// Final consolidate and encode: the vertices left with an edge numbered by a scan (fnew) and listed in that
// order (k_mg_src), the live edges sorted as 64-bit keys of the new numbers, then skelblob_encode
// (skelblob.cuh) with a row per label.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>

#include "common.cuh"
#include "skelblob.cuh"

namespace ign {

namespace {

constexpr uint32_t MG_NONE = 0xFFFFFFFFu;
constexpr int MG_THREADS = 256;

struct MgCtl {
  uint32_t err;  // bit b: check b of mg_fail_host failed
  uint32_t pad;
  unsigned long long bad[3];  // per check, the lowest index that failed it
  unsigned long long ne;      // live edges after postprocessing
  unsigned long long bytes;   // end of the last blob
};

struct MgEdge {
  uint32_t a, b;  // global vertex indices, a < b
};

__device__ __forceinline__ void mg_fail(MgCtl* ctl, int bit, uint64_t i) {
  atomicOr(&ctl->err, 1u << bit);
  atomicMin(&ctl->bad[bit], (unsigned long long)i);
}

// the largest i < n with a[i] <= x (a ascending, a[0] <= x)
__device__ __forceinline__ uint64_t mg_owner(const uint64_t* __restrict__ a, uint64_t n, uint64_t x) {
  uint64_t lo = 0, hi = n;
  while (hi - lo > 1) {
    const uint64_t mid = (lo + hi) >> 1;
    if (a[mid] <= x) lo = mid; else hi = mid;
  }
  return lo;
}

__device__ __forceinline__ uint32_t mg_order(float f) {
  uint32_t u = __float_as_uint(__fadd_rn(f, 0.0f));  // -0.0 -> 0.0
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// float32 edge length: every operation rounded on its own
__device__ __forceinline__ float mg_len(const float* __restrict__ v, uint32_t a, uint32_t b) {
  const float dx = __fsub_rn(v[3 * b], v[3 * a]), dy = __fsub_rn(v[3 * b + 1], v[3 * a + 1]);
  const float dz = __fsub_rn(v[3 * b + 2], v[3 * a + 2]);
  return __fsqrt_rn(__fadd_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)), __fmul_rn(dz, dz)));
}

__device__ __forceinline__ double mg_dist(const float* __restrict__ v, uint32_t a, uint32_t b) {
  const double dx = __dsub_rn((double)v[3 * a], (double)v[3 * b]);
  const double dy = __dsub_rn((double)v[3 * a + 1], (double)v[3 * b + 1]);
  const double dz = __dsub_rn((double)v[3 * a + 2], (double)v[3 * b + 2]);
  return __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
}

// ------------------------------------------------------------------ checks
__global__ void __launch_bounds__(256) k_mg_ranges(const uint64_t* __restrict__ label_frag, uint64_t L,
                                                   const uint64_t* __restrict__ frag_vert,
                                                   const uint64_t* __restrict__ frag_edge, uint64_t F, uint64_t V,
                                                   uint64_t E, MgCtl* ctl) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i <= L) {
    const bool bad = i == 0 ? label_frag[0] != 0 : (label_frag[i] < label_frag[i - 1] || (i == L && label_frag[L] != F));
    if (bad) mg_fail(ctl, 0, i);
  }
  if (i <= F) {
    bool bad = i == 0 ? (frag_vert[0] != 0 || frag_edge[0] != 0)
                      : (frag_vert[i] < frag_vert[i - 1] || frag_edge[i] < frag_edge[i - 1]);
    if (i == F) bad |= frag_vert[F] != V || frag_edge[F] != E;
    if (bad) mg_fail(ctl, 0, i);
  }
}

__global__ void __launch_bounds__(256) k_mg_verts(const float* __restrict__ vert, uint64_t V, MgCtl* ctl) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < V && !(isfinite(vert[3 * i]) && isfinite(vert[3 * i + 1]) && isfinite(vert[3 * i + 2]))) mg_fail(ctl, 1, i);
}

__global__ void __launch_bounds__(256) k_mg_edges(const uint64_t* __restrict__ frag_vert,
                                                  const uint64_t* __restrict__ frag_edge, uint64_t F,
                                                  const uint32_t* __restrict__ edges, uint64_t E, MgCtl* ctl) {
  const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const uint64_t f = mg_owner(frag_edge, F + 1, e);
  const uint64_t nv = frag_vert[f + 1] - frag_vert[f];
  if (edges[2 * e] >= nv || edges[2 * e + 1] >= nv) mg_fail(ctl, 2, e);
}

// ------------------------------------------------------------------ fuse and consolidate
__global__ void __launch_bounds__(256) k_mg_keys(const uint64_t* __restrict__ label_frag, uint64_t L,
                                                 const uint64_t* __restrict__ frag_vert, uint64_t F,
                                                 const double* __restrict__ box, const float* __restrict__ vert,
                                                 uint64_t V, uint32_t* __restrict__ kl, uint32_t* __restrict__ kx,
                                                 uint32_t* __restrict__ ky, uint32_t* __restrict__ kz,
                                                 uint32_t* __restrict__ perm) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= V) return;
  const uint64_t f = mg_owner(frag_vert, F + 1, i);
  const uint64_t l = mg_owner(label_frag, L + 1, f);
  bool in = true;
  for (int d = 0; d < 3; ++d) {
    const double c = (double)vert[3 * i + d];
    in &= box[6 * f + d] <= c && c <= box[6 * f + 3 + d];
  }
  kl[i] = in ? (uint32_t)l : MG_NONE;
  kx[i] = mg_order(vert[3 * i]);
  ky[i] = mg_order(vert[3 * i + 1]);
  kz[i] = mg_order(vert[3 * i + 2]);
  perm[i] = (uint32_t)i;
}

__global__ void __launch_bounds__(256) k_mg_gather(const uint32_t* __restrict__ key, const uint32_t* __restrict__ perm,
                                                   uint64_t n, uint32_t* __restrict__ out) {
  const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p < n) out[p] = key[perm[p]];
}

__global__ void __launch_bounds__(256) k_mg_heads(const uint32_t* __restrict__ perm, uint64_t V,
                                                  const uint32_t* __restrict__ kl, const uint32_t* __restrict__ kx,
                                                  const uint32_t* __restrict__ ky, const uint32_t* __restrict__ kz,
                                                  uint32_t* __restrict__ head) {
  const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= V) return;
  const uint32_t i = perm[p];
  uint32_t h = kl[i] != MG_NONE;
  if (h && p) {
    const uint32_t j = perm[p - 1];
    h = kl[i] != kl[j] || kx[i] != kx[j] || ky[i] != ky[j] || kz[i] != kz[j];
  }
  head[p] = h;
}

__global__ void __launch_bounds__(256) k_mg_uid(const uint32_t* __restrict__ perm, uint64_t V,
                                                const uint32_t* __restrict__ kl, const uint32_t* __restrict__ head,
                                                const uint32_t* __restrict__ run, uint32_t* __restrict__ uid,
                                                uint32_t* __restrict__ first) {
  const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= V) return;
  const uint32_t i = perm[p];
  uid[i] = kl[i] == MG_NONE ? MG_NONE : run[p] - 1;
  if (head[p]) first[run[p] - 1] = i;
}

__global__ void __launch_bounds__(256) k_mg_ekeys(const uint64_t* __restrict__ frag_vert,
                                                  const uint64_t* __restrict__ frag_edge, uint64_t F,
                                                  const uint32_t* __restrict__ edges, uint64_t E,
                                                  const uint32_t* __restrict__ uid, uint64_t* __restrict__ ekey) {
  const uint64_t e = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= E) return;
  const uint64_t f = mg_owner(frag_edge, F + 1, e);
  const uint32_t a = uid[frag_vert[f] + edges[2 * e]], b = uid[frag_vert[f] + edges[2 * e + 1]];
  ekey[e] = (a == MG_NONE || b == MG_NONE || a == b) ? ~0ull : ((uint64_t)min(a, b) << 32) | max(a, b);
}

__global__ void __launch_bounds__(256) k_mg_eheads(const uint64_t* __restrict__ k, uint64_t n,
                                                   uint32_t* __restrict__ head) {
  const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p < n) head[p] = k[p] != ~0ull && (p == 0 || k[p] != k[p - 1]);
}

__global__ void __launch_bounds__(256) k_mg_used(const uint64_t* __restrict__ k, const uint32_t* __restrict__ head,
                                                 uint64_t n, uint32_t* __restrict__ used) {
  const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p < n && head[p]) {
    used[k[p] >> 32] = 1;
    used[(uint32_t)k[p]] = 1;
  }
}

// unique vertex u with an edge -> compacted vertex vnew[u]; unique edge -> compacted edge
__global__ void __launch_bounds__(256) k_mg_compact_v(const uint32_t* __restrict__ used, const uint32_t* __restrict__ vnew,
                                                      const uint32_t* __restrict__ first, uint64_t U,
                                                      const uint32_t* __restrict__ kl, const float* __restrict__ vert,
                                                      const float* __restrict__ rad, const uint8_t* __restrict__ vt,
                                                      float* __restrict__ cv, float* __restrict__ cr,
                                                      uint8_t* __restrict__ ct, uint32_t* __restrict__ clab) {
  const uint64_t u = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (u >= U || !used[u]) return;
  const uint32_t i = first[u], j = vnew[u];
  cv[3 * j] = vert[3 * i];
  cv[3 * j + 1] = vert[3 * i + 1];
  cv[3 * j + 2] = vert[3 * i + 2];
  cr[j] = rad[i];
  ct[j] = vt[i];
  clab[j] = kl[i];
}

__global__ void __launch_bounds__(256) k_mg_compact_e(const uint64_t* __restrict__ k, const uint32_t* __restrict__ head,
                                                      const uint32_t* __restrict__ enew, uint64_t n,
                                                      const uint32_t* __restrict__ vnew, MgEdge* __restrict__ ce) {
  const uint64_t p = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p < n && head[p]) ce[enew[p]] = MgEdge{vnew[k[p] >> 32], vnew[(uint32_t)k[p]]};
}

__device__ __forceinline__ uint32_t mg_lower_lab(const uint32_t* __restrict__ lab, uint32_t n, uint32_t x) {
  uint32_t lo = 0, hi = n;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (lab[mid] < x) lo = mid + 1; else hi = mid;
  }
  return lo;
}

__device__ __forceinline__ uint32_t mg_lower_edge(const MgEdge* __restrict__ e, uint32_t n, uint32_t v) {
  uint32_t lo = 0, hi = n;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (e[mid].a < v) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// per label l: vertices [vs[l], vs[l + 1]), edges [es[l], es[l + 1]) (entry L closes the ranges)
__global__ void __launch_bounds__(256) k_mg_label_ranges(const uint32_t* __restrict__ clab, uint32_t nv,
                                                         const MgEdge* __restrict__ ce, uint32_t ne, uint64_t L,
                                                         uint32_t* __restrict__ vs, uint32_t* __restrict__ es) {
  const uint64_t l = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (l > L) return;
  const uint32_t v = l == L ? nv : mg_lower_lab(clab, nv, (uint32_t)l);
  vs[l] = v;
  es[l] = mg_lower_edge(ce, ne, v);
}

// ------------------------------------------------------------------ postprocess, one CTA per label
struct MgPost {
  const float* v;     // compacted vertices (global)
  const float* r;
  const MgEdge* ce;
  const uint32_t* vs;
  const uint32_t* es;
  MgEdge* pe;         // per label: 2 * ne + nv + 1 entries from 2 * es[l] + vs[l] + l
  uint8_t* alive;     // per entry
  uint32_t* deg;      // per vertex
  uint32_t* uf;       // per vertex
  uint32_t* aux;      // per vertex: DFS predecessor / tick end
  uint32_t* aux2;     // per vertex: path / stack / leaf list / Borůvka partner
  uint32_t* off;      // per vertex + 1 per label: adjacency offsets
  uint32_t* adj;      // per entry * 2
  uint32_t* eid;      // per entry * 2
  double* dv;         // per vertex: cable per root / best candidate distance / tick length
  uint32_t* tend;     // per vertex: the end of the j-th leaf's tick
  double dust, tick, max_cable;
};

__device__ uint32_t mg_find(uint32_t* p, uint32_t x) {
  while (p[x] != x) {
    p[x] = p[p[x]];
    x = p[x];
  }
  return x;
}

__device__ bool mg_union(uint32_t* p, uint32_t a, uint32_t b) {
  a = mg_find(p, a);
  b = mg_find(p, b);
  if (a == b) return false;
  if (a < b) p[b] = a; else p[a] = b;
  return true;
}

// union-find over the live entries, local vertex indices (base subtracted)
__device__ void mg_forest(const MgPost& P, uint32_t* uf, const MgEdge* pe, const uint8_t* alive, uint32_t m,
                          uint32_t n, uint32_t base) {
  for (uint32_t i = 0; i < n; ++i) uf[i] = i;
  for (uint32_t q = 0; q < m; ++q)
    if (alive[q]) mg_union(uf, pe[q].a - base, pe[q].b - base);
}

// drop the dead entries, keeping the order
__device__ uint32_t mg_squeeze(MgEdge* pe, uint8_t* alive, uint32_t m) {
  uint32_t w = 0;
  for (uint32_t q = 0; q < m; ++q)
    if (alive[q]) {
      pe[w] = pe[q];
      alive[w++] = 1;
    }
  for (uint32_t q = w; q < m; ++q) alive[q] = 0;
  return w;
}

__device__ void mg_kill(MgEdge* pe, uint8_t* alive, uint32_t m, uint32_t a, uint32_t b, uint32_t* deg, uint32_t base) {
  if (a > b) { const uint32_t s = a; a = b; b = s; }
  uint32_t lo = 0, hi = m;  // entries are sorted by (a, b) during the loop step
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (pe[mid].a < a || (pe[mid].a == a && pe[mid].b < b)) lo = mid + 1; else hi = mid;
  }
  if (lo < m && pe[lo].a == a && pe[lo].b == b && alive[lo]) {
    alive[lo] = 0;
    deg[a - base]--;
    deg[b - base]--;
  }
}

// one cycle (DESIGN.md §5h, loops); false when the live edges form a forest.  Thread 0 only.
__device__ bool mg_one_loop(const MgPost& P, MgEdge* pe, uint8_t* alive, uint32_t& m, uint32_t n, uint32_t base,
                            uint32_t* deg, uint32_t* uf, uint32_t* prev, uint32_t* path, uint32_t* off,
                            uint32_t* adj) {
  m = mg_squeeze(pe, alive, m);
  for (uint32_t i = 0; i < n; ++i) uf[i] = i;
  uint32_t c = m;
  for (uint32_t q = 0; q < m; ++q)
    if (!mg_union(uf, pe[q].a - base, pe[q].b - base)) {
      c = q;
      break;
    }
  if (c == m) return false;
  for (uint32_t i = 0; i <= n; ++i) off[i] = 0;
  for (uint32_t q = 0; q < c; ++q) {
    off[pe[q].a - base + 1]++;
    off[pe[q].b - base + 1]++;
  }
  for (uint32_t i = 0; i < n; ++i) off[i + 1] += off[i];
  for (uint32_t i = 0; i < n; ++i) prev[i] = off[i];
  for (uint32_t q = 0; q < c; ++q) {
    const uint32_t a = pe[q].a - base, b = pe[q].b - base;
    adj[prev[a]++] = b;
    adj[prev[b]++] = a;
  }
  const uint32_t a = pe[c].a - base, b = pe[c].b - base;
  for (uint32_t i = 0; i < n; ++i) prev[i] = MG_NONE;
  prev[a] = a;
  uint32_t* stack = uf;
  uint32_t top = 0;
  stack[top++] = a;
  while (top) {
    const uint32_t x = stack[--top];
    for (uint32_t j = off[x]; j < off[x + 1]; ++j)
      if (prev[adj[j]] == MG_NONE) {
        prev[adj[j]] = x;
        stack[top++] = adj[j];
      }
  }
  uint32_t k = 0;
  for (uint32_t x = b;; x = prev[x]) {
    path[k++] = x;
    if (x == a) break;
  }
  for (uint32_t i = 0; i < k / 2; ++i) {
    const uint32_t s = path[i];
    path[i] = path[k - 1 - i];
    path[k - 1 - i] = s;
  }
  uint32_t br[2], nb = 0;
  for (uint32_t i = 0; i < k; ++i)
    if (deg[path[i]] >= 3) {
      if (nb < 2) br[nb] = i;
      nb++;
    }
  const float* v = P.v;
  auto ring = [&](uint32_t i) { mg_kill(pe, alive, m, path[i] + base, path[(i + 1) % k] + base, deg, base); };
  if (nb == 0) {
    for (uint32_t i = 0; i < k; ++i) ring(i);
  } else if (nb == 1) {
    const uint32_t bv = path[br[0]];
    uint32_t f = bv;
    double best = -1.0;
    for (uint32_t i = 0; i < k; ++i) {
      const double d = mg_dist(v, bv + base, path[i] + base);
      if (d > best || (d == best && path[i] < f)) {
        best = d;
        f = path[i];
      }
    }
    for (uint32_t i = 0; i < k; ++i) ring(i);
    // insert (bv, f) in order, or revive it
    const uint32_t x = min(bv, f) + base, y = max(bv, f) + base;
    uint32_t lo = 0, hi = m;
    while (lo < hi) {
      const uint32_t mid = (lo + hi) >> 1;
      if (pe[mid].a < x || (pe[mid].a == x && pe[mid].b < y)) lo = mid + 1; else hi = mid;
    }
    if (!(lo < m && pe[lo].a == x && pe[lo].b == y)) {
      for (uint32_t q = m; q > lo; --q) {
        pe[q] = pe[q - 1];
        alive[q] = alive[q - 1];
      }
      pe[lo] = MgEdge{x, y};
      alive[lo] = 0;
      m++;
    }
    if (!alive[lo]) {
      alive[lo] = 1;
      deg[x - base]++;
      deg[y - base]++;
    }
  } else if (nb == 2) {
    const uint32_t i = br[0], j = br[1], len1 = j - i, len2 = k - len1;
    uint32_t m1 = MG_NONE, m2 = MG_NONE;
    for (uint32_t q = i + 1; q < j; ++q) m1 = min(m1, path[q]);
    for (uint32_t q = j + 1; q < k + i; ++q) m2 = min(m2, path[q % k]);
    const bool keep1 = len1 != len2 ? len1 < len2 : m1 < m2;
    if (keep1) {
      for (uint32_t q = j; q < k + i; ++q) ring(q % k);
    } else {
      for (uint32_t q = i; q < j; ++q) ring(q);
    }
  } else {
    uint32_t bi = 0, ba = MG_NONE, bb = MG_NONE;
    float bl = -1.0f;
    for (uint32_t i = 0; i < k; ++i) {
      const uint32_t x = min(path[i], path[(i + 1) % k]), y = max(path[i], path[(i + 1) % k]);
      const float l = mg_len(v, x + base, y + base);
      if (l > bl || (l == bl && (x < ba || (x == ba && y < bb)))) {
        bl = l;
        ba = x;
        bb = y;
        bi = i;
      }
    }
    ring(bi);
  }
  return true;
}

// walk from a leaf to the first vertex of degree >= 3; the tick's length and end.  With kill, the tick's edges
// are removed on the way.
__device__ double mg_walk(const MgPost& P, uint32_t leaf, uint32_t base, const uint32_t* off, const uint32_t* adj,
                          const uint32_t* eid, uint8_t* alive, uint32_t* deg, bool kill, uint32_t& end) {
  uint32_t prv = MG_NONE, x = leaf;
  double len = 0.0;
  for (;;) {
    uint32_t y = MG_NONE, q = 0;
    for (uint32_t j = off[x]; j < off[x + 1]; ++j)
      if (alive[eid[j]] && adj[j] != prv) {
        y = adj[j];
        q = eid[j];
        break;
      }
    len = __dadd_rn(len, (double)mg_len(P.v, min(x, y) + base, max(x, y) + base));
    const uint32_t dy = deg[y];
    if (kill) {
      alive[q] = 0;
      deg[x]--;
      deg[y]--;
    }
    prv = x;
    x = y;
    if (dy >= 3) break;
  }
  end = x;
  return len;
}

__global__ void __launch_bounds__(MG_THREADS) k_mg_post(MgPost P) {
  const uint32_t l = blockIdx.x, t = threadIdx.x;
  const uint32_t base = P.vs[l], n = P.vs[l + 1] - base;
  const uint32_t e0 = P.es[l], ne = P.es[l + 1] - e0;
  const uint64_t pbase = 2ull * e0 + base + l;
  MgEdge* pe = P.pe + pbase;
  uint8_t* alive = P.alive + pbase;
  const uint32_t cap = 2 * ne + n + 1;
  uint32_t* deg = P.deg + base;
  uint32_t* uf = P.uf + base;
  uint32_t* aux = P.aux + base;
  uint32_t* aux2 = P.aux2 + base;
  uint32_t* off = P.off + base + l;
  uint32_t* adj = P.adj + 2 * pbase;
  uint32_t* eid = P.eid + 2 * pbase;
  double* dv = P.dv + base;
  uint32_t* tend = P.tend + base;
  __shared__ double s_d[MG_THREADS];
  __shared__ uint32_t s_i[MG_THREADS];
  __shared__ uint32_t s_m, s_go;  // thread 0's live entry count, and whether a loop goes on
  __shared__ double s_rmax;       // the label's largest radius: bounds how far in x a candidate can lie

  for (uint32_t q = t; q < cap; q += MG_THREADS) {
    if (q < ne) pe[q] = P.ce[e0 + q];
    alive[q] = q < ne;
  }
  for (uint32_t i = t; i < n; i += MG_THREADS) deg[i] = 0;
  double c = 0.0;
  for (uint32_t q = t; q < ne; q += MG_THREADS) c += (double)mg_len(P.v, P.ce[e0 + q].a, P.ce[e0 + q].b);
  s_d[t] = c;
  __syncthreads();
  for (uint32_t q = t; q < ne; q += MG_THREADS) {
    atomicAdd(&deg[P.ce[e0 + q].a - base], 1u);
    atomicAdd(&deg[P.ce[e0 + q].b - base], 1u);
  }
  for (int s = MG_THREADS / 2; s; s >>= 1) {
    __syncthreads();
    if (t < s) s_d[t] += s_d[t + s];
  }
  __syncthreads();
  if (ne == 0 || s_d[0] > P.max_cable) return;  // written as fused

  if (t == 0) {
    uint32_t m = ne;
    if (P.dust > 0) {
      mg_forest(P, uf, pe, alive, m, n, base);
      for (uint32_t i = 0; i < n; ++i) dv[i] = 0.0;
      for (uint32_t q = 0; q < m; ++q) dv[mg_find(uf, pe[q].a - base)] += (double)mg_len(P.v, pe[q].a, pe[q].b);
      for (uint32_t q = 0; q < m; ++q)
        if (dv[mg_find(uf, pe[q].a - base)] < P.dust) {
          alive[q] = 0;
          deg[pe[q].a - base]--;
          deg[pe[q].b - base]--;
        }
    }
    while (mg_one_loop(P, pe, alive, m, n, base, deg, uf, aux, aux2, off, adj)) {}
    s_m = mg_squeeze(pe, alive, m);
    double rmax = 0.0;
    for (uint32_t i = 0; i < n; ++i) rmax = fmax(rmax, (double)P.r[i + base]);
    s_rmax = rmax;
  }
  __syncthreads();

  // connect pieces: Borůvka rounds over the candidates of DESIGN.md §5h
  for (;;) {
    if (t == 0) {
      mg_forest(P, uf, pe, alive, s_m, n, base);
      uint32_t roots = 0;
      for (uint32_t i = 0; i < n; ++i) {
        uf[i] = mg_find(uf, i);
        roots += deg[i] && uf[i] == i;
      }
      s_go = roots > 1;
    }
    __syncthreads();
    if (!s_go) break;
    // every vertex's best candidate: key (d, min, max), which for a fixed u orders partners as (d, w).
    // A label's vertices ascend in x (the consolidation order) and d >= |dx| up to rounding, so only the w
    // with fl(x_w - x_u) within reach = (r_u + the label's largest radius) * (1 + 1e-12) can be candidates;
    // the factor covers the rounding of d and of r_u + r_w.  dx is computed exactly as mg_dist computes it.
    for (uint32_t u = t; u < n; u += MG_THREADS) {
      double bd = INFINITY;
      uint32_t bv = MG_NONE;
      if (deg[u]) {
        const double ru = (double)P.r[u + base], xu = (double)P.v[3 * (u + base)];
        const double reach = __dmul_rn(__dadd_rn(ru, s_rmax), 1.0 + 1e-12);
        uint32_t w0 = 0, w1 = u;  // the first w with fl(x_u - x_w) <= reach
        while (w0 < w1) {
          const uint32_t mid = (w0 + w1) >> 1;
          if (__dsub_rn(xu, (double)P.v[3 * (mid + base)]) > reach) w0 = mid + 1; else w1 = mid;
        }
        for (uint32_t w = w0; w < n; ++w) {
          if (__dsub_rn((double)P.v[3 * (w + base)], xu) > reach) break;
          if (!deg[w] || uf[w] == uf[u]) continue;
          const double d = mg_dist(P.v, u + base, w + base);
          if (!(d < __dadd_rn(ru, (double)P.r[w + base]))) continue;
          if (bv == MG_NONE || d < bd || (d == bd && w < bv)) {
            bd = d;
            bv = w;
          }
        }
      }
      dv[u] = bd;
      aux2[u] = bv;
    }
    __syncthreads();
    if (t == 0) {
      // per root its best vertex (aux), then one edge per root; distinct keys make these a forest
      for (uint32_t i = 0; i < n; ++i) aux[i] = MG_NONE;
      for (uint32_t u = 0; u < n; ++u) {
        if (aux2[u] == MG_NONE) continue;
        const uint32_t rt = uf[u], cur = aux[rt];
        bool better = cur == MG_NONE;
        if (!better) {
          const uint32_t lo = min(u, aux2[u]), hi = max(u, aux2[u]);
          const uint32_t clo = min(cur, aux2[cur]), chi = max(cur, aux2[cur]);
          better = dv[u] < dv[cur] || (dv[u] == dv[cur] && (lo < clo || (lo == clo && hi < chi)));
        }
        if (better) aux[rt] = u;
      }
      uint32_t m = s_m;
      for (uint32_t i = 0; i < n; ++i) {
        if (aux[i] == MG_NONE) continue;
        const uint32_t u = aux[i], w = aux2[u];
        if (mg_union(uf, u, w)) {
          pe[m] = MgEdge{min(u, w) + base, max(u, w) + base};
          alive[m++] = 1;
          deg[u]++;
          deg[w]++;
        }
      }
      s_go = m > s_m;
      s_m = m;
    }
    __syncthreads();
    if (!s_go) break;
    __syncthreads();  // every thread has read s_go before thread 0 writes it for the next round
  }

  if (!(P.tick > 0)) return;
  // ticks: adjacency of the live edges; per root its count of branch vertices (aux; MG_NONE once done);
  // the leaves of components with a branch vertex (aux2), each with its tick length (dv) and end (tend)
  if (t == 0) {
    const uint32_t m = s_m;
    for (uint32_t i = 0; i <= n; ++i) off[i] = 0;
    for (uint32_t q = 0; q < m; ++q) {
      off[pe[q].a - base + 1]++;
      off[pe[q].b - base + 1]++;
    }
    for (uint32_t i = 0; i < n; ++i) off[i + 1] += off[i];
    for (uint32_t i = 0; i < n; ++i) aux[i] = off[i];
    for (uint32_t q = 0; q < m; ++q) {
      const uint32_t a = pe[q].a - base, b = pe[q].b - base;
      adj[aux[a]] = b;
      eid[aux[a]++] = q;
      adj[aux[b]] = a;
      eid[aux[b]++] = q;
    }
    mg_forest(P, uf, pe, alive, m, n, base);
    for (uint32_t i = 0; i < n; ++i) uf[i] = mg_find(uf, i);
    for (uint32_t i = 0; i < n; ++i) aux[i] = 0;
    for (uint32_t i = 0; i < n; ++i)
      if (deg[i] >= 3) aux[uf[i]]++;
    uint32_t nl = 0;
    for (uint32_t i = 0; i < n; ++i)
      if (deg[i] == 1 && aux[uf[i]]) aux2[nl++] = i;
    s_m = nl;
  }
  __syncthreads();
  const uint32_t nl = s_m;
  for (uint32_t j = t; j < nl; j += MG_THREADS)
    dv[aux2[j]] = mg_walk(P, aux2[j], base, off, adj, eid, alive, deg, false, tend[j]);
  __syncthreads();
  for (;;) {
    // block-wide argmin of (length, leaf) over the leaves of components still being trimmed
    double bd = INFINITY;
    uint32_t bj = MG_NONE;
    for (uint32_t j = t; j < nl; j += MG_THREADS) {
      const uint32_t leaf = aux2[j];
      if (leaf == MG_NONE) continue;
      const uint32_t nb = aux[uf[leaf]];
      if (nb == 0 || nb == MG_NONE) continue;
      if (bj == MG_NONE || dv[leaf] < bd) {  // leaves ascend with j: the first of equal lengths is the lowest
        bd = dv[leaf];
        bj = j;
      }
    }
    s_d[t] = bd;
    s_i[t] = bj;
    for (int s = MG_THREADS / 2; s; s >>= 1) {
      __syncthreads();
      if (t < s) {
        const uint32_t o = s_i[t + s];
        if (o != MG_NONE && (s_i[t] == MG_NONE || s_d[t + s] < s_d[t] || (s_d[t + s] == s_d[t] && o < s_i[t]))) {
          s_d[t] = s_d[t + s];
          s_i[t] = o;
        }
      }
    }
    __syncthreads();
    const uint32_t j = s_i[0];
    if (j == MG_NONE) break;
    if (t == 0) {
      const uint32_t leaf = aux2[j], rt = uf[leaf];
      if (!(s_d[0] < P.tick)) {
        aux[rt] = MG_NONE;  // its shortest tick is long enough: nothing in this component changes again
      } else {
        uint32_t b;
        mg_walk(P, leaf, base, off, adj, eid, alive, deg, true, b);
        aux2[j] = MG_NONE;
        if (deg[b] == 2 && --aux[rt])  // b stopped branching: the ticks that ended there run on
          for (uint32_t q = 0; q < nl; ++q)
            if (aux2[q] != MG_NONE && tend[q] == b)
              dv[aux2[q]] = mg_walk(P, aux2[q], base, off, adj, eid, alive, deg, false, tend[q]);
      }
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------ final consolidate and encode
__global__ void __launch_bounds__(256) k_mg_fkeep(const uint32_t* __restrict__ deg, uint32_t nv,
                                                  uint32_t* __restrict__ keep) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i <= nv) keep[i] = i < nv && deg[i] > 0;
}

__global__ void __launch_bounds__(256) k_mg_fkeys(const MgEdge* __restrict__ pe, const uint8_t* __restrict__ alive,
                                                  uint64_t n, const uint32_t* __restrict__ fnew,
                                                  uint64_t* __restrict__ key, MgCtl* ctl) {
  const uint64_t q = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  bool live = false;
  if (q < n) {
    live = alive[q];
    key[q] = live ? ((uint64_t)fnew[pe[q].a] << 32) | fnew[pe[q].b] : ~0ull;
  }
  const unsigned m = __ballot_sync(0xFFFFFFFFu, live);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(&ctl->ne, (unsigned long long)__popc(m));
}

// the final vertices in order: src[fnew[i]] = i
__global__ void __launch_bounds__(256) k_mg_src(const uint32_t* __restrict__ keep, const uint32_t* __restrict__ fnew,
                                                uint32_t nv, uint32_t* __restrict__ src) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nv && keep[i]) src[fnew[i]] = i;
}

// the rows of skelblob_encode: one per label; final vertex j is compacted vertex src[j]
struct MgSource {
  const uint32_t *vs, *fnew, *src, *clab;
  const float *cv, *cr;
  const uint8_t* ct;
  __device__ uint64_t vstart(uint64_t l) const { return fnew[vs[l]]; }
  __device__ uint64_t label(uint64_t l) const { return l; }
  __device__ uint32_t row(uint64_t j) const { return clab[src[j]]; }
  __device__ void vertex(uint64_t j, float c[3], float& r, uint8_t& t) const {
    const uint32_t i = src[j];
    c[0] = cv[3 * i];
    c[1] = cv[3 * i + 1];
    c[2] = cv[3 * i + 2];
    r = cr[i];
    t = ct[i];
  }
};

uint64_t merge_bound(uint64_t L, uint64_t V, uint64_t E) { return 16 * L + 25 * V + 8 * E; }

int mg_fail_host(const MgCtl& h) {
  IGN_REQUIRE(!(h.err & 1u), IGN_ERR_INVALID,
              "skeleton_merge: the fragment ranges are not ascending from 0 to the vertex / edge / fragment counts "
              "(first bad entry %llu)", h.bad[0]);
  IGN_REQUIRE(!(h.err & 2u), IGN_ERR_INVALID, "skeleton_merge: vertex %llu is not finite", h.bad[1]);
  IGN_REQUIRE(!(h.err & 4u), IGN_ERR_INVALID, "skeleton_merge: edge %llu has an end outside its fragment", h.bad[2]);
  return IGN_OK;
}

}  // namespace
}  // namespace ign

using namespace ign;

extern "C" {

int ign_skeleton_merge_capacity(uint64_t n_labels, uint64_t n_vertices, uint64_t n_edges, uint64_t* bytes) {
  IGN_REQUIRE(bytes, IGN_ERR_INVALID, "skeleton_merge: null bytes");
  IGN_REQUIRE(n_vertices < (1ull << 30) && n_edges < (1ull << 30) && n_labels < (1ull << 31), IGN_ERR_OVERFLOW,
              "skeleton_merge: %llu vertices, %llu edges (each below 2^30), %llu labels (below 2^31)",
              (unsigned long long)n_vertices, (unsigned long long)n_edges, (unsigned long long)n_labels);
  *bytes = merge_bound(n_labels, n_vertices, n_edges);
  return IGN_OK;
}

int ign_skeleton_merge_dev(ign_ctx* ctx, uint64_t n_labels, const uint64_t* label_frag, uint64_t n_frags,
                           const uint64_t* frag_vert, const uint64_t* frag_edge, const double* frag_box,
                           const float* vertices, const float* radius, const uint8_t* vertex_types_in,
                           uint64_t n_vertices, const uint32_t* edges, uint64_t n_edges, double dust_threshold,
                           double tick_threshold, double max_cable_length, int vertex_types, uint8_t* blobs_out,
                           uint64_t capacity, uint64_t* table_out, uint64_t* nbytes) {
  IGN_TRY(activate(ctx));
  IGN_REQUIRE(nbytes, IGN_ERR_INVALID, "skeleton_merge: null nbytes");
  *nbytes = 0;
  const uint64_t L = n_labels, F = n_frags, V = n_vertices, E = n_edges;
  IGN_REQUIRE(V < (1ull << 30) && E < (1ull << 30) && L < (1ull << 31) && F < (1ull << 31), IGN_ERR_OVERFLOW,
              "skeleton_merge: %llu vertices, %llu edges (each below 2^30), %llu labels, %llu fragments "
              "(below 2^31)", (unsigned long long)V, (unsigned long long)E, (unsigned long long)L,
              (unsigned long long)F);
  IGN_REQUIRE(!isnan(dust_threshold) && !isnan(tick_threshold) && !isnan(max_cable_length), IGN_ERR_INVALID,
              "skeleton_merge: a threshold is NaN");
  const uint64_t bound = merge_bound(L, V, E);
  IGN_REQUIRE(capacity >= bound, IGN_ERR_INVALID,
              "skeleton_merge: capacity %llu bytes is below the bound 16 * labels + 25 * vertices + 8 * edges = %llu",
              (unsigned long long)capacity, (unsigned long long)bound);
  if (L == 0) return IGN_OK;
  IGN_REQUIRE(label_frag && frag_vert && frag_edge && frag_box && blobs_out && table_out, IGN_ERR_INVALID,
              "skeleton_merge: null buffer");
  IGN_REQUIRE(V == 0 || (vertices && radius && vertex_types_in), IGN_ERR_INVALID, "skeleton_merge: null vertices");
  IGN_REQUIRE(E == 0 || edges, IGN_ERR_INVALID, "skeleton_merge: null edges");
  IGN_REQUIRE(((uintptr_t)blobs_out & 7) == 0 && ((uintptr_t)table_out & 7) == 0, IGN_ERR_INVALID,
              "skeleton_merge: blobs and table must be aligned to 8 bytes");
  ScratchFrame f(ctx);
  MgCtl* ctl;
  IGN_TRY(f.take(&ctl, 1));
  MgCtl init{};
  for (int b = 0; b < 3; ++b) init.bad[b] = ~0ull;
  IGN_TRY(small_h2d(ctx, ctl, &init, sizeof(MgCtl)));
  MgCtl h{};
  IGN_LAUNCH(ctx, k_mg_ranges, blocks_for(std::max(L, F) + 1, 256), 256, 0, label_frag, L, frag_vert, frag_edge, F, V,
             E, ctl);
  IGN_TRY(small_d2h(ctx, &h, ctl, sizeof(MgCtl)));
  IGN_TRY(small_sync(ctx));
  IGN_TRY(mg_fail_host(h));  // the passes below search the ranges
  if (V) IGN_LAUNCH(ctx, k_mg_verts, blocks_for(V, 256), 256, 0, vertices, V, ctl);
  if (E) IGN_LAUNCH(ctx, k_mg_edges, blocks_for(E, 256), 256, 0, frag_vert, frag_edge, F, edges, E, ctl);
  IGN_TRY(small_d2h(ctx, &h, ctl, sizeof(MgCtl)));
  IGN_TRY(small_sync(ctx));
  IGN_TRY(mg_fail_host(h));

  // ---- fuse and consolidate
  const uint64_t Vs = std::max<uint64_t>(V, 1), Es = std::max<uint64_t>(E, 1);
  uint32_t *kl, *kx, *ky, *kz, *perm, *perm2, *tk, *tk2, *head, *run, *uid, *first, *used, *vnew, *ehead, *enew;
  uint64_t *ekey, *ekey_s;
  IGN_TRY(f.take(&kl, Vs));
  IGN_TRY(f.take(&kx, Vs));
  IGN_TRY(f.take(&ky, Vs));
  IGN_TRY(f.take(&kz, Vs));
  IGN_TRY(f.take(&perm, Vs));
  IGN_TRY(f.take(&perm2, Vs));
  IGN_TRY(f.take(&tk, Vs));
  IGN_TRY(f.take(&tk2, Vs));
  IGN_TRY(f.take(&head, Vs));
  IGN_TRY(f.take(&run, Vs));
  IGN_TRY(f.take(&uid, Vs));
  IGN_TRY(f.take(&first, Vs));
  IGN_TRY(f.take(&used, Vs + 1));
  IGN_TRY(f.take(&vnew, Vs + 1));
  IGN_TRY(f.take(&ekey, Es));
  IGN_TRY(f.take(&ekey_s, Es));
  IGN_TRY(f.take(&ehead, Es + 1));
  IGN_TRY(f.take(&enew, Es + 1));
  // postprocess slices: 2 * ne + nv + 1 entries per label (at most 2 * E + V + L)
  const uint64_t P_cap = 2 * E + V + L;
  float *cv, *cr;
  uint8_t *ct, *alive;
  uint32_t *clab, *vs, *es, *deg, *uf, *aux, *aux2, *off, *adj, *eid, *tend, *keep, *fnew, *src;
  MgEdge *ce, *pe;
  double* dv;
  uint64_t *fkey, *fkey_s;
  IGN_TRY(f.take(&cv, 3 * Vs));
  IGN_TRY(f.take(&cr, Vs));
  IGN_TRY(f.take(&ct, Vs));
  IGN_TRY(f.take(&clab, Vs));
  IGN_TRY(f.take(&ce, Es));
  IGN_TRY(f.take(&vs, L + 1));
  IGN_TRY(f.take(&es, L + 1));
  IGN_TRY(f.take(&pe, P_cap));
  IGN_TRY(f.take(&alive, P_cap));
  IGN_TRY(f.take(&deg, Vs));
  IGN_TRY(f.take(&uf, Vs));
  IGN_TRY(f.take(&aux, Vs));
  IGN_TRY(f.take(&aux2, Vs));
  IGN_TRY(f.take(&off, V + L + 1));
  IGN_TRY(f.take(&adj, 2 * P_cap));
  IGN_TRY(f.take(&eid, 2 * P_cap));
  IGN_TRY(f.take(&dv, Vs));
  IGN_TRY(f.take(&tend, Vs));
  IGN_TRY(f.take(&keep, Vs + 1));
  IGN_TRY(f.take(&fnew, Vs + 1));
  IGN_TRY(f.take(&src, Vs));
  IGN_TRY(f.take(&fkey, P_cap));
  IGN_TRY(f.take(&fkey_s, P_cap));
  size_t tb = 0, t;
  const int vitems = (int)Vs, eitems = (int)Es;
  IGN_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, t, tk, tk2, perm, perm2, vitems, 0, 32, ctx->stream));
  tb = std::max(tb, t);
  IGN_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, t, ekey, ekey_s, eitems, 0, 64, ctx->stream));
  tb = std::max(tb, t);
  IGN_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, t, fkey, fkey_s, (int)P_cap, 0, 64, ctx->stream));
  tb = std::max(tb, t);
  IGN_CUDA(cub::DeviceScan::InclusiveSum(nullptr, t, head, run, vitems, ctx->stream));
  tb = std::max(tb, t);
  IGN_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, t, used, vnew, vitems + 1, ctx->stream));
  tb = std::max(tb, t);
  IGN_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, t, ehead, enew, eitems + 1, ctx->stream));
  tb = std::max(tb, t);
  void* tmp;
  IGN_TRY(f.take(&tmp, tb));

  uint32_t U = 0, nv1 = 0, ne1 = 0;
  if (V) {
    const unsigned vg = blocks_for(V, 256);
    IGN_LAUNCH(ctx, k_mg_keys, vg, 256, 0, label_frag, L, frag_vert, F, frag_box, vertices, V, kl, kx, ky, kz, perm);
    const uint32_t* comp[4] = {kz, ky, kx, kl};
    for (int c = 0; c < 4; ++c) {
      IGN_LAUNCH(ctx, k_mg_gather, vg, 256, 0, comp[c], perm, V, tk);
      // cropped vertices carry label ~0, so the label pass sorts all 32 bits too
      IGN_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tb, tk, tk2, perm, perm2, (int)V, 0, 32, ctx->stream));
      std::swap(perm, perm2);
    }
    IGN_LAUNCH(ctx, k_mg_heads, vg, 256, 0, perm, V, kl, kx, ky, kz, head);
    IGN_CUDA(cub::DeviceScan::InclusiveSum(tmp, tb, head, run, (int)V, ctx->stream));
    IGN_LAUNCH(ctx, k_mg_uid, vg, 256, 0, perm, V, kl, head, run, uid, first);
    IGN_TRY(small_d2h(ctx, &U, run + (V - 1), 4));
    IGN_TRY(small_sync(ctx));
  }
  if (U && E) {
    const unsigned eg = blocks_for(E, 256);
    IGN_LAUNCH(ctx, k_mg_ekeys, eg, 256, 0, frag_vert, frag_edge, F, edges, E, uid, ekey);
    IGN_CUDA(cub::DeviceRadixSort::SortKeys(tmp, tb, ekey, ekey_s, (int)E, 0, 64, ctx->stream));
    IGN_CUDA(cudaMemsetAsync(ehead, 0, (E + 1) * 4, ctx->stream));
    IGN_LAUNCH(ctx, k_mg_eheads, eg, 256, 0, ekey_s, E, ehead);
    IGN_CUDA(cudaMemsetAsync(used, 0, (U + 1) * 4, ctx->stream));
    IGN_LAUNCH(ctx, k_mg_used, eg, 256, 0, ekey_s, ehead, E, used);
    IGN_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tb, used, vnew, (int)U + 1, ctx->stream));
    IGN_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tb, ehead, enew, (int)E + 1, ctx->stream));
    IGN_TRY(small_d2h(ctx, &nv1, vnew + U, 4));
    IGN_TRY(small_d2h(ctx, &ne1, enew + E, 4));
    IGN_TRY(small_sync(ctx));
    IGN_LAUNCH(ctx, k_mg_compact_v, blocks_for(U, 256), 256, 0, used, vnew, first, U, kl, vertices, radius,
               vertex_types_in, cv, cr, ct, clab);
    IGN_LAUNCH(ctx, k_mg_compact_e, eg, 256, 0, ekey_s, ehead, enew, E, vnew, ce);
  }
  IGN_LAUNCH(ctx, k_mg_label_ranges, blocks_for(L + 1, 256), 256, 0, clab, nv1, ce, ne1, L, vs, es);

  // ---- postprocess
  IGN_CUDA(cudaMemsetAsync(alive, 0, 2 * (uint64_t)ne1 + nv1 + L, ctx->stream));
  if (nv1) {
    MgPost P{cv, cr, ce, vs, es, pe, alive, deg, uf, aux, aux2, off, adj, eid, dv, tend, dust_threshold,
             tick_threshold, max_cable_length};
    IGN_LAUNCH(ctx, k_mg_post, (unsigned)L, MG_THREADS, 0, P);
  }

  // ---- final consolidate and encode
  const uint64_t slots = 2 * (uint64_t)ne1 + nv1 + L;
  IGN_LAUNCH(ctx, k_mg_fkeep, blocks_for(nv1 + 1, 256), 256, 0, deg, nv1, keep);
  IGN_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tb, keep, fnew, (int)nv1 + 1, ctx->stream));
  IGN_LAUNCH(ctx, k_mg_fkeys, blocks_for(slots, 256), 256, 0, pe, alive, slots, fnew, fkey, ctl);
  IGN_CUDA(cub::DeviceRadixSort::SortKeys(tmp, tb, fkey, fkey_s, (int)slots, 0, 64, ctx->stream));
  if (nv1) IGN_LAUNCH(ctx, k_mg_src, blocks_for(nv1, 256), 256, 0, keep, fnew, nv1, src);
  const MgSource source{vs, fnew, src, clab, cv, cr, ct};
  IGN_TRY(skelblob_encode(ctx, f, source, L, nv1, fkey_s, slots, &ctl->ne, vertex_types, table_out, blobs_out,
                          &ctl->bytes));
  IGN_TRY(small_d2h(ctx, &h, ctl, sizeof(MgCtl)));
  IGN_TRY(small_sync(ctx));
  *nbytes = h.bytes;
  return IGN_OK;
}

}  // extern "C"
