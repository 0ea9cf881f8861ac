// simplify.cu -- quadric edge-collapse mesh simplification (K10)
//
// Replaces the simplifier inside zmesh.Mesher.get(id, reduction_factor,
// max_error) (igneous/tasks/mesh/mesh.py:376-381) for ALL labels of a task at
// once.  zmesh's simplifier is a sequential heap-ordered collapse per label; a
// GPU needs a data-parallel formulation, so this is a round-based variant:
//
//   init    per-vertex Garland-Heckbert plane quadrics (unit normals, summed in
//           face order), boundary vertices locked (chunk borders must stitch),
//           per-vertex incident-face arrays (half-edge nodes, fixed capacity,
//           merged and compacted on collapse).
//   round   E  every edge of a label still above its face target computes the cheap
//              quadric cost (min over {u, v, midpoint} of p^T (Qu+Qv) p) and, if
//              cost <= max_error^2, posts a (cost, per-round hash of the label-local
//              half-edge id) key to both endpoints (atomic min); labels with at most
//              65536 half-edges use a 32-bit key (16 cost bits | 16-bit id permutation);
//           K2 per vertex: is its key the minimum over its face neighbours' keys?
//           C  an edge WINS iff its key is the minimum of both endpoints' keys and of
//              all their neighbours' -> winners are two edges apart, never touch each
//              other's faces or vertices and are processed concurrently: a winner
//              collapses iff the link condition holds and no incident face flips,
//              otherwise it is parked until one of its endpoints' rings changes.
//   stop    per label: faces <= target, or a round without winners, or four
//           consecutive rounds that each remove < 0.2% of the label's faces.
//   compact scans renumber surviving vertices / faces per label.
//
// Labels are independent, so all rounds of one label run inside ONE CTA with the
// label's topology in shared memory (k_simp_labels below: one launch per MeshTask, one
// CTA per label).
//
// All arithmetic is double precision WITHOUT fused multiply-add (this file is
// compiled with -fmad=false) so that oracle/igneous_oracle.c::orc_simplify
// reproduces it bit for bit.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <type_traits>

#include "mesher.h"

namespace ign {

constexpr uint64_t S_KEYMAX = 0xFFFFFFFFFFFFFFFFull;
constexpr int S_MAXV = 32;
constexpr int S_VCAP = 64;  // two rings of < S_MAXV alive faces always fit after a collapse
constexpr int VB = 11;  // vertex key coordinate bits (mesh.cu V_COORD_BITS)

struct Simp {
  uint64_t U, T;
  double* pos;      // 3U
  double* Q;        // 10U
  uint32_t* face;   // 3T global vertex ids
  uint32_t* flabel; // T dense labels
  uint8_t* falive;
  uint8_t* valive;
  uint8_t* vbound;
  // incident half-edge nodes (3f+c) of every vertex as a fixed-capacity array: ring
  // enumeration is a set of independent loads instead of a linked-list pointer chase
  uint32_t* vf;   // [U * S_VCAP]
  uint32_t* vn;   // [U] entries in use (dead faces are skipped, compacted when the vertex is kept)
  const uint32_t* tri_off;  // [K+2] first face of each label
};

__device__ __forceinline__ uint32_t s_mix(uint32_t x) {
  x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16;
  return x;
}
__device__ __forceinline__ uint32_t s_unmix(uint32_t x) {
  x ^= x >> 16; x *= 0x43021123U; x ^= x >> 15 ^ x >> 30; x *= 0x1d69e2a5U; x ^= x >> 16;
  return x;
}
// 16-bit variant for labels whose half-edge ids fit 16 bits (oracle: simp_mix16 / simp_unmix16)
__device__ __forceinline__ uint32_t s_mix16(uint32_t x) {
  x &= 0xFFFFu;
  x = (x * 0x2F35u) & 0xFFFFu; x ^= x >> 7;
  x = (x * 0x4A6Bu) & 0xFFFFu; x ^= x >> 9;
  x = (x * 0x9E37u) & 0xFFFFu; x ^= x >> 8;
  return x;
}
__device__ __forceinline__ uint32_t s_unmix16(uint32_t x) {
  x &= 0xFFFFu;
  x ^= x >> 8; x = (x * 0x7787u) & 0xFFFFu;
  x ^= x >> 9; x = (x * 0x1243u) & 0xFFFFu;
  x ^= x >> 7; x ^= x >> 14; x = (x * 0xEB1Du) & 0xFFFFu;
  return x;
}
__device__ __forceinline__ unsigned long long s_key(double cost, uint32_t h, uint32_t salt) {
  const float c = __double2float_rn(cost);
  return ((unsigned long long)__float_as_uint(c) << 32) | s_mix(h ^ salt);
}

// Key and cost format of a label of T faces (oracle: simp_key): 32-bit keys when its 3T half-edge ids fit 16
// bits, else 64-bit keys.
__host__ __device__ __forceinline__ bool s_fmt16(uint64_t T) { return 3 * T <= 65536ull; }
// the 16 cost bits of a 32-bit key (8 exponent + 8 mantissa bits of the non-negative float cost)
__device__ __forceinline__ uint32_t s_kfield(float cost) { return (__float_as_uint(cost) >> 15) & 0xFFFFu; }
// Cached costs (ecost: 12 bytes per face of the task, a label's slice [12 tbase, 12 (tbase + T))).  A label
// with 64-bit keys keeps the float cost of half-edge 3i + c at float 3 (tbase + i) + c.  A label with 32-bit
// keys needs only their 16 cost bits: the fields of face i's corners 0..2 (bits 16c.., 16 bits of padding) are
// one 8-byte word, word i from the slice's first 8-byte boundary (it ends in the slice: 8T + 4 <= 12T).
__device__ __forceinline__ unsigned long long* s_cwords(float* ecost, uint32_t tbase) {
  return (unsigned long long*)(ecost + 3 * (uint64_t)tbase + (tbase & 1u));
}
// the field of corner c in word i (the index arithmetic of s_cwords, in 2-byte units)
__device__ __forceinline__ uint16_t* s_cfield(float* ecost, uint32_t tbase, uint32_t i, uint32_t c) {
  return (uint16_t*)ecost + 2 * (3 * (uint64_t)tbase + (tbase & 1u) + 2 * i) + c;
}

__device__ __forceinline__ double s_qeval(const double* q, const double* p) {
  const double x = p[0], y = p[1], z = p[2];
  return q[0] * x * x + 2.0 * q[1] * x * y + 2.0 * q[2] * x * z + 2.0 * q[3] * x + q[4] * y * y +
         2.0 * q[5] * y * z + 2.0 * q[6] * y + q[7] * z * z + 2.0 * q[8] * z + q[9];
}

__device__ int s_twins(const Simp& s, uint32_t f, uint32_t u, uint32_t v, uint32_t* twin) {
  int cnt = 0;
  const uint32_t* lu = s.vf + (uint64_t)u * S_VCAP;
  const uint32_t cu = s.vn[u];
  for (uint32_t j = 0; j < cu; j++) {
    const uint32_t h = lu[j];
    const uint32_t g = h / 3;
    if (g == f || !s.falive[g]) continue;
    const uint32_t* fv = s.face + 3 * (uint64_t)g;
    if (fv[0] == v || fv[1] == v || fv[2] == v) {
      if (cnt == 0) *twin = h;
      cnt++;
    }
  }
  return cnt;
}

struct SEval {
  bool valid;
  double cost;
  uint32_t keep, remove;
  double p[3];
};

// s_cost from the summed quadric q = Qu + Qv and the endpoint positions pu, pv (memory or registers)
__device__ __forceinline__ void s_cost_q(const double* q, const double* pu, const double* pv, double max_err2,
                                         uint32_t u, uint32_t v, bool bu, bool bv, SEval* e) {
  e->valid = false;
  if (bu && bv) return;
  double best[3], cost;
  if (bu) {
    e->keep = u;
    e->remove = v;
    best[0] = pu[0]; best[1] = pu[1]; best[2] = pu[2];
    cost = s_qeval(q, best);
  } else if (bv) {
    e->keep = v;
    e->remove = u;
    best[0] = pv[0]; best[1] = pv[1]; best[2] = pv[2];
    cost = s_qeval(q, best);
  } else {
    e->keep = u < v ? u : v;
    e->remove = u < v ? v : u;
    // (selected per component: a pointer select would put register arrays in local memory)
    const bool uk = u < v;
    const double kk[3] = {uk ? pu[0] : pv[0], uk ? pu[1] : pv[1], uk ? pu[2] : pv[2]};
    const double rr[3] = {uk ? pv[0] : pu[0], uk ? pv[1] : pu[1], uk ? pv[2] : pu[2]};
    const double mid[3] = {(kk[0] + rr[0]) * 0.5, (kk[1] + rr[1]) * 0.5, (kk[2] + rr[2]) * 0.5};
    const double ck = s_qeval(q, kk), cr = s_qeval(q, rr), cm = s_qeval(q, mid);
    cost = ck;
    best[0] = kk[0]; best[1] = kk[1]; best[2] = kk[2];
    if (cr < cost) { cost = cr; best[0] = rr[0]; best[1] = rr[1]; best[2] = rr[2]; }
    if (cm < cost) { cost = cm; best[0] = mid[0]; best[1] = mid[1]; best[2] = mid[2]; }
  }
  if (cost < 0.0) cost = 0.0;
  if (!(cost <= max_err2)) return;
  e->valid = true;
  e->cost = cost;
  e->p[0] = best[0]; e->p[1] = best[1]; e->p[2] = best[2];
}

// collapse cost of the edge (u, v) (min over {u, v, midpoint} of p^T (Qu+Qv) p, boundary endpoints stay
// put): u / v are vertex ids of any one numbering (they pick the kept vertex), gu / gv their rows of Q and
// pos.  Invalid when both endpoints are on the boundary or the cost exceeds max_err2.
__device__ __forceinline__ void s_cost(const double* Q, const double* pos, double max_err2, uint32_t u, uint32_t v,
                                       uint64_t gu, uint64_t gv, bool bu, bool bv, SEval* e) {
  e->valid = false;
  if (bu && bv) return;
  const double* Qu = Q + 10 * gu;
  const double* Qv = Q + 10 * gv;
  double q[10];
#pragma unroll
  for (int i = 0; i < 10; i++) q[i] = Qu[i] + Qv[i];
  s_cost_q(q, pos + 3 * gu, pos + 3 * gv, max_err2, u, v, bu, bv, e);
}

// ------------------------------------------------------------------ kernels
__global__ void __launch_bounds__(256)
    k_simp_init_verts(const uint64_t* __restrict__ vkeys, uint64_t U, double rx, double ry, double rz,
                      double* __restrict__ pos, uint8_t* __restrict__ valive,
                      uint8_t* __restrict__ vbound, uint32_t* __restrict__ vn) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= U) return;
  const uint64_t k = vkeys[i];
  const double x = (double)(k & ((1u << VB) - 1));
  const double y = (double)((k >> VB) & ((1u << VB) - 1));
  const double z = (double)((k >> (2 * VB)) & ((1u << VB) - 1));
  pos[3 * i + 0] = x * 0.5 * rx;
  pos[3 * i + 1] = y * 0.5 * ry;
  pos[3 * i + 2] = z * 0.5 * rz;
  valive[i] = 1;
  vbound[i] = 0;
  vn[i] = 0;
}

// faces: local ids + per-label vertex base -> global ids; flabel by offsets search
__global__ void __launch_bounds__(256)
    k_simp_init_faces(const uint32_t* __restrict__ faces_local, const uint32_t* __restrict__ tri_off,
                      const uint32_t* __restrict__ vert_off, uint32_t K, uint64_t T,
                      uint32_t* __restrict__ face, uint32_t* __restrict__ flabel,
                      uint8_t* __restrict__ falive, uint32_t* __restrict__ node_vertex,
                      uint32_t* __restrict__ node_id) {
  const uint64_t f = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (f >= T) return;
  // largest l in [1,K] with tri_off[l] <= f
  uint32_t lo = 1, hi = K;
  while (lo < hi) {
    const uint32_t mid = (lo + hi + 1) >> 1;
    if (tri_off[mid] <= f) lo = mid;
    else hi = mid - 1;
  }
  flabel[f] = lo;
  falive[f] = 1;
  for (int k = 0; k < 3; k++) {
    const uint32_t g = faces_local[3 * f + k] + vert_off[lo];
    face[3 * f + k] = g;
    node_vertex[3 * f + k] = g;
    node_id[3 * f + k] = (uint32_t)(3 * f + k);
  }
}

// sorted (vertex, node) pairs -> per-vertex arrays in ascending node order
__global__ void __launch_bounds__(256)
    k_simp_link(const uint32_t* __restrict__ sv, const uint32_t* __restrict__ sh, uint64_t n,
                uint32_t* __restrict__ vf, uint32_t* __restrict__ vn, uint32_t* overflow) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t v = sv[i];
  if (i > 0 && sv[i - 1] == v) return;  // the first pair of a run writes the whole run
  uint32_t c = 0;
  for (uint64_t j = i; j < n && sv[j] == v; j++) {
    if (c < S_VCAP) vf[(uint64_t)v * S_VCAP + c] = sh[j];
    c++;
  }
  if (c > S_VCAP) {
    *overflow = 1;
    c = S_VCAP;
  }
  vn[v] = c;
}

__global__ void __launch_bounds__(128) k_simp_quadrics(Simp s) {
  const uint64_t v = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (v >= s.U) return;
  double q[10];
  for (int i = 0; i < 10; i++) q[i] = 0.0;
  for (uint32_t j = 0; j < s.vn[v]; j++) {
    const uint32_t h = s.vf[(uint64_t)v * S_VCAP + j];
    const uint32_t* fv = s.face + 3 * (uint64_t)(h / 3);
    const double* a = s.pos + 3 * (uint64_t)fv[0];
    const double* b = s.pos + 3 * (uint64_t)fv[1];
    const double* c = s.pos + 3 * (uint64_t)fv[2];
    const double ux = b[0] - a[0], uy = b[1] - a[1], uz = b[2] - a[2];
    const double vx = c[0] - a[0], vy = c[1] - a[1], vz = c[2] - a[2];
    double nx = uy * vz - uz * vy, ny = uz * vx - ux * vz, nz = ux * vy - uy * vx;
    const double len = sqrt(nx * nx + ny * ny + nz * nz);
    if (!(len > 0.0)) continue;
    nx = nx / len; ny = ny / len; nz = nz / len;
    const double d = -(nx * a[0] + ny * a[1] + nz * a[2]);
    q[0] += nx * nx; q[1] += nx * ny; q[2] += nx * nz; q[3] += nx * d;
    q[4] += ny * ny; q[5] += ny * nz; q[6] += ny * d;
    q[7] += nz * nz; q[8] += nz * d; q[9] += d * d;
  }
  for (int i = 0; i < 10; i++) s.Q[10 * v + i] = q[i];
}

__global__ void __launch_bounds__(256) k_simp_boundary(Simp s) {
  const uint64_t h = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (h >= 3 * s.T) return;
  const uint32_t f = (uint32_t)(h / 3), c = (uint32_t)(h % 3);
  const uint32_t u = s.face[3 * (uint64_t)f + c], v = s.face[3 * (uint64_t)f + (c + 1) % 3];
  uint32_t tw;
  if (s_twins(s, f, u, v, &tw) != 1) {
    s.vbound[u] = 1;
    s.vbound[v] = 1;
  }
}

// Initial cost of every canonical half-edge (u < v; label-local order is the global one): the cost in ecost,
// in the label's format (s_cwords), and the memo of the half-edge in the face's state byte (2 cached, 3 exceeds
// max_error), which the label kernel's load takes over.  One thread per face, so that the byte has a single
// writer.  counts[0] += evaluations.
__global__ void __launch_bounds__(256)
    k_simp_ecost(Simp s, double max_err2, float* __restrict__ ecost, uint8_t* __restrict__ fstate,
                 uint32_t* counts) {
  const uint64_t f = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  uint32_t n = 0;
  if (f < s.T) {
    const uint32_t* fv = s.face + 3 * f;
    const uint32_t l = s.flabel[f], tbase = s.tri_off[l];
    const bool fmt16 = s_fmt16(s.tri_off[l + 1] - tbase);
    uint32_t st = 0;
    unsigned long long word = 0;
#pragma unroll
    for (int c = 0; c < 3; c++) {
      const uint32_t u = fv[c], v = fv[(c + 1) % 3];
      if (!(u < v)) continue;
      SEval ev;
      s_cost(s.Q, s.pos, max_err2, u, v, u, v, s.vbound[u] != 0, s.vbound[v] != 0, &ev);
      uint32_t es = 3;
      if (ev.valid) {
        const float cf = __double2float_rn(ev.cost);
        if (fmt16) word |= (unsigned long long)s_kfield(cf) << (16 * c);
        else ecost[3 * f + c] = cf;
        es = 2;
      }
      st |= es << (2 * c);
      n++;
    }
    if (fmt16) s_cwords(ecost, tbase)[f - tbase] = word;
    fstate[f] = (uint8_t)st;
  }
  const int tot = __syncthreads_count(n & 1u) + 2 * __syncthreads_count(n >> 1);
  if (threadIdx.x == 0 && tot) atomicAdd(counts, (uint32_t)tot);
}

// ------------------------------------------------------------------ per-label rounds
// One CTA owns one label for ALL of its rounds (labels are independent: keys use
// label-local half-edge ids and the stop rules are per label).  The topology of the
// label -- faces as label-local vertex ids (u16 SoA), one state byte per face (alive bit
// + a 2-bit memo per half-edge), a flag byte and a "lose" byte per vertex, the 32-bit round
// keys and the ring lists of the round's winners -- lives in SHARED MEMORY for the whole
// run; only the double-precision data that a round touches sparsely (positions, quadrics,
// cached costs) stays in global memory (L2).  A round is a handful of
// __syncthreads() phases instead of five launches and a host round trip:
//
//   P1  key1[v] = MAX, lose[v] = 0                             (vertex parallel)
//   P2  every canonical half-edge (u < v) of an alive face posts its cached key to both
//       endpoints with a shared-memory min reduction (the cached costs come from k_simp_ecost
//       and E2; P2 evaluates none)                                 (face parallel)
//   P3  a vertex LOSEs if a face neighbour holds a smaller key1 (== key2 test of the
//       round formulation: key2[w] == key1[w] <=> !LOSE[w]); plain byte stores
//                                                               (face parallel)
//   P4  a vertex a WINs iff its key's half-edge starts at a, both endpoints hold that
//       key and neither LOSEs; at most L.wcap winners per pass   (vertex parallel)
//   E1  the faces that touch a winner's endpoints append themselves to the winner's
//       two ring lists; the first warps compute the winners' placement and cost (E2a)
//       at the same time                                         (face parallel)
//   E2  one group of 8 lanes per winner (16 / 32 for rings over 8 / 16 faces), a lane per ring
//       face of each endpoint: flip tests, link condition by ballots / shuffles, the collapse
//       itself and the re-costs of the kept vertex's canonical half-edges, with no barrier
//       between them                                             (winner parallel)
//
// Labels that do not fit (more than 16384 faces, or 6U + 9T + 23 KB over the CTA's shared
// memory) keep faces and lists in global memory, with keys / flags / states still in
// shared memory when those fit ("hybrid"), else everything global (SM = false, 64-bit
// key slots).
// vertex flags: RDIRTY the vertex's ring changed (parked edges around it may be valid now)
constexpr uint32_t VF_ALIVE = 1, VF_BOUND = 2, VF_DONE = 16, VF_END = 32, VF_RDIRTY = 64;
constexpr int SL_THREADS = 1024;
// winners validated per selection pass (a round runs as many passes as it needs): every label that fits a
// class has room for SL_WCAP; a shared-memory label takes more where the class's shared memory leaves room
// (sl_wcap), since each further pass rescans the vertices (P4) and the alive faces (E1)
constexpr int SL_WCAP = 128;
constexpr uint32_t WF_BAD = 1;  // winner flag: E2a found no valid placement (both endpoints locked, or over max_error)
constexpr int SL_LIST_PER = 16;  // list entries per thread held in registers while a list is compacted in place

// Size classes of k_simp_labels: CTA size and CTAs per SM.  A label runs in the smallest class whose
// shared-memory budget holds it, so labels that need less than half (a quarter) of an SM's shared
// memory run two (four) to an SM and overlap each other's barrier and latency phases.
constexpr int SL_NCLASS = 3;
constexpr int SL_CLASS_THREADS[SL_NCLASS] = {1024, 512, 256};

// a winner of a selection pass: its edge, ring lengths, flags and placement (dynamic shared memory)
struct SlWin {
  double best[3];
  uint32_t u, v, h, cnt[2], keep, flags;
  uint32_t order;  // E2 takes the winners in the order win[0].order, win[1].order, ... (8-lane groups first)
};
// shared memory a shared-memory label needs per winner of a pass: the record and two 16-bit ring lists
constexpr size_t SL_WIN_BYTES = sizeof(SlWin) + 2 * S_MAXV * 2;

// dynamic shared-memory layout of a label at `threads` threads with `wcap` winners per pass:
// winners | ring lists | key1 | faces SoA | face list | face state | vertex flags | lose marks
// [| original face ids | original vertex ids: a label resumed in a smaller class after migrating]
struct SlLayout {
  size_t o_ring, o_key, o_f0, o_fl, o_fs, o_vf, o_vl, o_fm, o_vm, need;
};
__host__ __device__ inline SlLayout sl_layout(uint32_t T, uint32_t U, bool resumed = false,
                                              uint32_t wcap = SL_WCAP) {
  SlLayout y;
  y.o_ring = (size_t)wcap * sizeof(SlWin);
  y.o_key = y.o_ring + (size_t)wcap * 2 * S_MAXV * 2;  // shared-memory class: 16-bit face ids in the rings
  y.o_f0 = y.o_key + 4 * (size_t)U;                    // 32-bit keys
  y.o_fl = y.o_f0 + 6 * (size_t)T;
  y.o_fs = y.o_fl + 2 * (size_t)T;
  y.o_vf = (y.o_fs + T + 3) & ~(size_t)3;
  y.o_vl = (y.o_vf + U + 3) & ~(size_t)3;
  y.o_fm = (y.o_vl + U + 3) & ~(size_t)3;
  y.o_vm = y.o_fm + 2 * (size_t)T;
  y.need = resumed ? y.o_vm + 2 * (size_t)U + 4 : y.o_vl + U + 4;
  return y;
}
// the shared-memory class also needs 16-bit keys and lists that a compaction holds in registers
__host__ __device__ inline bool sl_fits_smem(uint32_t T, uint32_t U, uint32_t threads, size_t smem_bytes,
                                             bool resumed = false) {
  const uint32_t cap = (uint32_t)SL_LIST_PER * threads;
  return s_fmt16(T) && T <= cap && U <= cap && sl_layout(T, U, resumed).need <= smem_bytes;
}
// winners per pass of a label that sl_fits_smem accepts: SL_WCAP plus what the rest of the budget holds, at
// most one per thread (E2a gives each winner a thread) and at most `limit` (IGN_SIMP_WCAP)
__host__ __device__ inline uint32_t sl_wcap(uint32_t T, uint32_t U, uint32_t threads, size_t smem_bytes,
                                            bool resumed, uint32_t limit) {
  const size_t w = SL_WCAP + (smem_bytes - sl_layout(T, U, resumed).need) / SL_WIN_BYTES;
  const size_t m = threads < limit ? threads : limit;
  return (uint32_t)(w < m ? w : m);
}

struct SlArgs {
  double* pos;            // 3U
  double* Q;              // 10U
  uint32_t* face;         // 3T global vertex ids
  uint8_t* falive;        // T   (out)
  uint8_t* valive;        // U   (out)
  const uint8_t* vbound;  // U
  float* ecost;           // 3T  memoised cost per half-edge, in the label's key format (s_cwords)
  // global-memory class only (labels that do not fit shared memory)
  unsigned long long* key1;  // U
  uint8_t* fstate;           // T
  uint8_t* vflag;            // U
  uint8_t* vlose;            // U  LOSE marks of the round (plain byte stores)
  uint32_t *flist, *flist2;  // T  alive-face lists (ping-pong)
  uint32_t *vlist, *vlist2;  // U
  const uint32_t* tri_off;   // [K+2]
  const uint32_t* vert_off;  // [K+2]
  const uint32_t* target;    // [K+2]
  const uint32_t* order;     // [K] dense labels of this launch's size class, largest first
  uint32_t K;
  uint32_t base;       // position of order[0] in the task's work order (all classes)
  uint32_t cls;        // size class of the launch
  uint32_t* counters;  // [1] max rounds  [2] labels run in shared memory  [3] in global memory
                       // [4 + class] next work item  [8 + class] labels run in the class
                       // [16 + class] labels migrated into the class  [20 + class] next migrated label to resume
                       // [24] multi-pass label-rounds  [25] winners with a ring over S_MAXV faces
                       // [26] initial cost evaluations (k_simp_ecost)  [27] re-costs after collapses (E2)
                       // [28] canonical half-edges without a cost met by the key pass (always 0)
                       // [29..31] winners taken by E2 groups of 8, 16 and 32 lanes
  double max_err2;
  int max_rounds;
  uint32_t smem_bytes;  // dynamic shared memory of the launch
  // migration into the next smaller class (shared-memory labels only).  A migrated label's state goes to
  // its own slices of the global-memory class's arrays, which shared-memory labels do not use otherwise:
  // flist[tbase + i] = vertices 0 | 1 << 16 and flist2[tbase + i] = vertex 2 | original face << 16 of
  // alive face i, fstate[tbase + i] its state; vlist[vbase + j] = original vertex | flags << 16 of alive
  // vertex j (in vertex order); finv[tbase + original face] = i.  The header goes to a queue of the class.
  uint32_t* mq_next;     // [labels][SL_MREC] headers of labels migrating out of this launch (null: no migration)
  uint32_t smem_next;    // dynamic shared memory of the next smaller class
  const uint32_t* mq;    // resume launches: headers of the labels migrated into the class
  uint16_t* finv;        // [T] compacted face of an original face (read when a resumed label decodes a key)
  int persist;          // 1: a CTA keeps taking labels until the list is empty (IGN_SIMP_PERSIST=1)
  uint32_t* lrec;       // IGN_SIMP_TRACE=1: [base + work item][SL_LREC] = faces, rounds, kilocycles, face visits
                        // (sum of list lengths), winners, memory class | size class << 2, SM kilocycles
                        // (kilocycles / CTAs per SM); a migrated label sums its segments
  uint32_t* trace;      // IGN_SIMP_TRACE=1: [round][4] = winners, collapses, alive faces, list length of the largest label
                        // [SL_HIST +] per size class: selection passes, winners, ring lengths per round (SL_H*)
  uint32_t wcap_max;    // most winners per pass (IGN_SIMP_WCAP; default: no limit beyond the budget)
  uint32_t group_min;   // narrowest lane group of E2: 8, 16 or 32 (IGN_SIMP_GROUP; default 8)
};

// IGN_SIMP_TRACE histograms, per size class the segment runs in: passes per round (1..SL_HP, last bin more),
// winners per round before capping (bins of 16, last bin more), ring length per winner side (0..S_MAXV, more)
constexpr int SL_HIST = 1664, SL_HP = 16, SL_HW = 64, SL_HR = S_MAXV + 2, SL_HCLS = SL_HP + SL_HW + SL_HR;

// header of a migrated label: dense label, trace record, next round, slow rounds, alive faces, alive vertices
constexpr int SL_MREC = 8;
constexpr int SL_LREC = 7;  // words of a label's IGN_SIMP_TRACE record (SlArgs::lrec)
constexpr int SL_NPH = 9;  // IGN_SIMP_TRACE phase timers (trace words 1600.., 64 bits each)
// IGN_SIMP_TRACE E2 flip tests (trace words SL_TFLIP..): winners rejected by flips on the u side only, on the
// v side only, on both sides
constexpr int SL_TFLIP = 1624;

struct SlShared {
  uint32_t work, alive, progress, ncol, nwin, stop, slow, counter, npass;
  uint32_t ring8, ring16;  // E1 saw a ring of more than 8 / 16 faces in this pass
  uint32_t nnarrow, nwide;  // winners of the pass that 8-lane groups take, and the others
  uint32_t rec, valive;  // trace record of the label; alive vertices (one dies per collapse)
  unsigned long long visits, wins;  // IGN_SIMP_TRACE
  long long t_label;
  uint32_t nrecost;    // half-edges re-costed after collapses (E2)
  uint32_t ngroup[3];  // winners taken by groups of 8, 16 and 32 lanes (E2)
  unsigned long long ph[SL_NPH];  // phase timers (IGN_SIMP_TRACE)
  long long t_prev;
};

template <bool SM>
struct SlLab {
  typedef typename std::conditional<SM, uint16_t, uint32_t>::type idx_t;
  uint32_t T, U, tbase, vbase, target, label;
  idx_t *fc0, *fc1, *fc2;  // SM: label-local ids, SoA in shared memory
  idx_t *fmap, *vmap;      // resumed labels: original label-local face / vertex id of each compacted one
  uint32_t* gface;         // !SM: AoS global ids in place
  uint8_t* fstate;         // bit 7 alive, bits 2c..2c+1 memo of half-edge c
  uint8_t* vflag;
  uint8_t* vlose;  // a face neighbour holds a smaller key this round (written with plain byte stores: every writer stores 1)
  // key format (oracle: simp_key): labels with 3T <= 65536 use 32-bit keys (bf16-like cost | 16-bit id
  // permutation).  The shared-memory class only takes such labels and stores them in 32 bits (native
  // shared-memory min); the other classes keep 64-bit slots for both formats.
  typedef typename std::conditional<SM, uint32_t, unsigned long long>::type key_t;
  key_t* key1;
  bool fmt16;
  uint32_t wcap;   // winners per selection pass (their records are at the start of the dynamic shared memory)
  idx_t* ring;     // [wcap][2][S_MAXV] face ids of the winners' rings (shared memory)
  idx_t *flist, *flist2, *vlist, *vlist2;  // alive lists (flist2 / vlist2: global-memory class only)
};

template <bool SM>
__device__ __forceinline__ uint32_t sl_fget(const SlLab<SM>& L, uint32_t f, int c) {
  if (SM) return c == 0 ? L.fc0[f] : (c == 1 ? L.fc1[f] : L.fc2[f]);
  return L.gface[3 * (uint64_t)f + c] - L.vbase;
}
template <bool SM>
__device__ __forceinline__ void sl_fset(const SlLab<SM>& L, uint32_t f, int c, uint32_t x) {
  typedef typename SlLab<SM>::idx_t idx_t;
  if (SM) {
    if (c == 0) L.fc0[f] = (idx_t)x;
    else if (c == 1) L.fc1[f] = (idx_t)x;
    else L.fc2[f] = (idx_t)x;
  } else {
    L.gface[3 * (uint64_t)f + c] = x + L.vbase;
  }
}
// task-wide index of a label-local vertex (positions and quadrics) and label-local id of a face (keys,
// cached costs): a resumed label maps its compacted ids back to the original ones
template <bool SM, bool R>
__device__ __forceinline__ uint64_t sl_vg(const SlLab<SM>& L, uint32_t v) {
  return L.vbase + (uint64_t)(R ? (uint32_t)L.vmap[v] : v);
}
template <bool SM, bool R>
__device__ __forceinline__ uint32_t sl_fo(const SlLab<SM>& L, uint32_t f) {
  return R ? (uint32_t)L.fmap[f] : f;
}
// flag bytes are modified with word atomics whenever two threads may touch the same word
// (SM: the flags are in shared memory for sure -> shared-space reductions instead of generic atomics)
template <bool SM>
__device__ __forceinline__ void sl_vor(uint8_t* vflag, uint32_t v, uint32_t bits) {
  const uintptr_t a = (uintptr_t)(vflag + v);
  if ((*(volatile uint8_t*)a & bits) == bits) return;
  const uint32_t word = bits << (8 * (a & 3));
  if (SM) {
    asm volatile("red.shared.or.b32 [%0], %1;" ::"r"((uint32_t)__cvta_generic_to_shared((void*)(a & ~(uintptr_t)3))), "r"(word) : "memory");
  } else {
    atomicOr((uint32_t*)(a & ~(uintptr_t)3), word);
  }
}
template <bool SM>
__device__ __forceinline__ void sl_vclear(uint8_t* vflag, uint32_t v, uint32_t bits) {
  const uintptr_t a = (uintptr_t)(vflag + v);
  const uint32_t word = ~(bits << (8 * (a & 3)));
  if (SM) {
    asm volatile("red.shared.and.b32 [%0], %1;" ::"r"((uint32_t)__cvta_generic_to_shared((void*)(a & ~(uintptr_t)3))), "r"(word) : "memory");
  } else {
    atomicAnd((uint32_t*)(a & ~(uintptr_t)3), word);
  }
}
__device__ __forceinline__ void sl_post(unsigned long long* key1, uint32_t u, uint32_t v, unsigned long long key) {
  if (key < *(volatile unsigned long long*)&key1[u]) atomicMin(&key1[u], key);
  if (key < *(volatile unsigned long long*)&key1[v]) atomicMin(&key1[v], key);
}
__device__ __forceinline__ void sl_post(uint32_t* key1, uint32_t u, uint32_t v, uint32_t key) {  // shared memory only
  if (key < *(volatile uint32_t*)&key1[u])
    asm volatile("red.shared.min.u32 [%0], %1;" ::"r"((uint32_t)__cvta_generic_to_shared(key1 + u)), "r"(key) : "memory");
  if (key < *(volatile uint32_t*)&key1[v])
    asm volatile("red.shared.min.u32 [%0], %1;" ::"r"((uint32_t)__cvta_generic_to_shared(key1 + v)), "r"(key) : "memory");
}
// 32-bit key from the cost field s_kfield(cost) (as cached for labels with 32-bit keys, s_cwords)
__device__ __forceinline__ uint32_t sl_key(uint32_t field, uint32_t hl, uint32_t salt) {
  return (field << 16) | s_mix16((hl ^ salt) & 0xFFFFu);
}
template <bool SM>
__device__ __forceinline__ typename SlLab<SM>::key_t sl_key(const SlLab<SM>& L, float cost, uint32_t hl, uint32_t salt) {
  typedef typename SlLab<SM>::key_t key_t;
  if (SM || L.fmt16) return (key_t)sl_key(s_kfield(cost), hl, salt);
  return (key_t)(((unsigned long long)__float_as_uint(cost) << 32) | s_mix(hl ^ salt));
}
template <bool SM>
__device__ __forceinline__ uint32_t sl_key_edge(const SlLab<SM>& L, typename SlLab<SM>::key_t key, uint32_t salt) {
  if (SM || L.fmt16) return s_unmix16((uint32_t)key & 0xFFFFu) ^ (salt & 0xFFFFu);
  return s_unmix((uint32_t)((unsigned long long)key & 0xFFFFFFFFull)) ^ salt;
}

// s_cost on label-local ids
template <bool SM, bool R>
__device__ __forceinline__ void sl_cost(const SlArgs& A, const SlLab<SM>& L, uint32_t u, uint32_t v, SEval* e) {
  s_cost(A.Q, A.pos, A.max_err2, u, v, sl_vg<SM, R>(L, u), sl_vg<SM, R>(L, v), (L.vflag[u] & VF_BOUND) != 0,
         (L.vflag[v] & VF_BOUND) != 0, e);
}

// The two half-edges of face f that hold the kept vertex k of a collapse: t = 0 is k -> o1, t = 1 is o2 -> k.
// sl_kcorner gives k's corner, sl_kcorner(..) + 2 * t (mod 3) the corner that starts half-edge t.
template <bool SM>
__device__ __forceinline__ uint32_t sl_kcorner(const SlLab<SM>& L, uint32_t f, uint32_t k) {
  return sl_fget<SM>(L, f, 0) == k ? 0u : (sl_fget<SM>(L, f, 1) == k ? 1u : 2u);
}
// Re-cost the half-edge that starts at corner c of face f (if `has`), one of whose endpoints is the vertex k
// that a collapse of the lane's group has just moved: cached float cost, and the memo to store (2 cached,
// 3 exceeds max_error).  k's new quadric comes by shuffles from the group lanes that summed it (component i
// in lane i; with 8 lanes, components 8-9 in qs2 of lanes 0-1) and its new position is the winner's
// placement pk, so only the other endpoint's rows of Q and pos are loaded.  Every lane of the warp calls it.
template <bool SM, bool R, int W>
__device__ __forceinline__ uint32_t sl_recost_k(const SlArgs& A, const SlLab<SM>& L, bool has, uint32_t f,
                                                uint32_t c, uint32_t k, double qs, double qs2, const double* pk) {
  uint32_t u = k, v = k;
  if (has) { u = sl_fget<SM>(L, f, (int)c); v = sl_fget<SM>(L, f, (int)((c + 1) % 3)); }
  const bool ku = (u == k);
  const uint64_t go = sl_vg<SM, R>(L, ku ? v : u);
  double q[10], po[3] = {0.0, 0.0, 0.0};
#pragma unroll
  for (int i = 0; i < 10; i++) q[i] = has ? A.Q[10 * go + i] : 0.0;
  if (has) { po[0] = A.pos[3 * go]; po[1] = A.pos[3 * go + 1]; po[2] = A.pos[3 * go + 2]; }
#pragma unroll
  for (int i = 0; i < 10; i++)  // Q[k] + Q[o]: IEEE addition is commutative, so the sum has s_cost's bits
    q[i] += __shfl_sync(0xFFFFFFFFu, (W == 8 && i >= 8) ? qs2 : qs, (W == 8 && i >= 8) ? i - 8 : i, W);
  if (!has) return 0;
  double pu[3], pv[3];
#pragma unroll
  for (int i = 0; i < 3; i++) {
    const double b = pk[i];
    pu[i] = ku ? b : po[i];
    pv[i] = ku ? po[i] : b;
  }
  SEval ev;
  s_cost_q(q, pu, pv, A.max_err2, u, v, (L.vflag[u] & VF_BOUND) != 0, (L.vflag[v] & VF_BOUND) != 0, &ev);
  if (!ev.valid) return 3;
  const float cf = __double2float_rn(ev.cost);
  const uint32_t fo = sl_fo<SM, R>(L, f);
  if (SM || L.fmt16) *s_cfield(A.ecost, L.tbase, fo, c) = (uint16_t)s_kfield(cf);
  else A.ecost[3 * (uint64_t)(L.tbase + fo) + c] = cf;
  return 2;
}

// does face (a0,a1,a2) flip when vertex w moves to `best`?  (the validation's flip test)
template <bool SM, bool R>
__device__ __forceinline__ bool sl_flips(const SlArgs& A, const SlLab<SM>& L, const uint32_t* a, uint32_t w,
                                         const double* best) {
  double P[3][3], N[3][3];
#pragma unroll
  for (int k = 0; k < 3; k++) {
    const double* p = A.pos + 3 * sl_vg<SM, R>(L, a[k]);
    P[k][0] = p[0]; P[k][1] = p[1]; P[k][2] = p[2];
  }
#pragma unroll
  for (int k = 0; k < 3; k++) {
    const bool mv = (a[k] == w);
    N[k][0] = mv ? best[0] : P[k][0];
    N[k][1] = mv ? best[1] : P[k][1];
    N[k][2] = mv ? best[2] : P[k][2];
  }
  const double ax = P[1][0] - P[0][0], ay = P[1][1] - P[0][1], az = P[1][2] - P[0][2];
  const double bx = P[2][0] - P[0][0], by = P[2][1] - P[0][1], bz = P[2][2] - P[0][2];
  const double n0x = ay * bz - az * by, n0y = az * bx - ax * bz, n0z = ax * by - ay * bx;
  const double cx = N[1][0] - N[0][0], cy = N[1][1] - N[0][1], cz = N[1][2] - N[0][2];
  const double dx = N[2][0] - N[0][0], dy = N[2][1] - N[0][1], dz = N[2][2] - N[0][2];
  const double n1x = cy * dz - cz * dy, n1y = cz * dx - cx * dz, n1z = cx * dy - cy * dx;
  const double dot = n0x * n1x + n0y * n1y + n0z * n1z;
  return !(dot > 0.0);
}

// the two corners of a ring face other than w, in cyclic order after w
__device__ __forceinline__ void sl_others(const uint32_t* a, uint32_t w, uint32_t* o1, uint32_t* o2) {
  if (a[0] == w) { *o1 = a[1]; *o2 = a[2]; }
  else if (a[1] == w) { *o1 = a[2]; *o2 = a[0]; }
  else { *o1 = a[0]; *o2 = a[1]; }
}

// distinct values among the (x1, x2) of the first n lanes; f1 / f2 flag the first occurrences
__device__ __forceinline__ uint32_t sl_distinct(uint32_t x1, uint32_t x2, uint32_t n, uint32_t lane, bool* f1,
                                                bool* f2) {
  const uint32_t FULL = 0xFFFFFFFFu;
  const bool have = lane < n;
  const uint32_t m1 = __match_any_sync(FULL, x1);
  const uint32_t m2 = __match_any_sync(FULL, x2);
  *f1 = have && ((int)lane == __ffs(m1) - 1);
  bool in1 = false;
  for (uint32_t j = 0; j < n; j++) in1 |= (__shfl_sync(FULL, x1, j) == x2);
  *f2 = have && ((int)lane == __ffs(m2) - 1) && !in1;
  return __popc(__ballot_sync(FULL, *f1)) + __popc(__ballot_sync(FULL, *f2));
}

// drop the dead entries of an alive list (order is irrelevant).  SM: in place, the entries
// pass through registers; global-memory class: into the second buffer, then swap.
template <bool SM, typename IDX, typename PRED>
__device__ __forceinline__ uint32_t sl_compact(IDX*& list, IDX*& list2, uint32_t n, uint32_t* counter, PRED alive) {
  const uint32_t FULL = 0xFFFFFFFFu;
  const uint32_t tid = threadIdx.x, lane = tid & 31u;
  if (tid == 0) *counter = 0;
  __syncthreads();
  if (SM) {
    IDX keep[SL_LIST_PER];
    uint32_t m = 0;
#pragma unroll
    for (int k = 0; k < SL_LIST_PER; k++) {
      const uint32_t i = tid + k * blockDim.x;
      keep[k] = 0;
      if (i < n) {
        const IDX e = list[i];
        keep[k] = e;
        if (alive((uint32_t)e)) m |= 1u << k;
      }
    }
    __syncthreads();
    const uint32_t cnt = __popc(m);
    uint32_t inc = cnt;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t o = __shfl_up_sync(FULL, inc, d);
      if ((int)lane >= d) inc += o;
    }
    uint32_t base = 0;
    if (lane == 31 && inc) base = atomicAdd(counter, inc);
    base = __shfl_sync(FULL, base, 31) + inc - cnt;
#pragma unroll
    for (int k = 0; k < SL_LIST_PER; k++)
      if ((m >> k) & 1u) list[base++] = keep[k];
  } else {
    for (uint32_t i0 = (tid & ~31u); i0 < n; i0 += blockDim.x) {
      const uint32_t i = i0 + lane;
      IDX e = 0;
      bool al = false;
      if (i < n) {
        e = list[i];
        al = alive((uint32_t)e);
      }
      const uint32_t bal = __ballot_sync(FULL, al);
      if (!bal) continue;
      uint32_t base = 0;
      const int leader = __ffs(bal) - 1;
      if ((int)lane == leader) base = atomicAdd(counter, (uint32_t)__popc(bal));
      base = __shfl_sync(FULL, base, leader);
      if (al) list2[base + __popc(bal & ((1u << lane) - 1u))] = e;
    }
    IDX* t = list;
    list = list2;
    list2 = t;
  }
  __syncthreads();
  const uint32_t kept = *counter;
  __syncthreads();  // everyone has read the count: the counter may be reused by the next call
  return kept;
}

// phase timers (IGN_SIMP_TRACE=1): thread 0 attributes the cycles since the previous mark to a phase
#define SL_MARK(id)                                   \
  do {                                                \
    if (A.trace != nullptr && tid == 0) {             \
      const long long _t = clock64();                 \
      sh.ph[id] += (unsigned long long)(_t - sh.t_prev); \
      sh.t_prev = _t;                                 \
    }                                                 \
  } while (0)

extern __shared__ __align__(16) unsigned char sl_smem[];

// the winner records of the pass (SlLayout: first in the dynamic shared memory)
__device__ __forceinline__ SlWin* sl_win() { return (SlWin*)sl_smem; }

// group width that E2 gives a winner whose rings hold nfu and nfv faces: 8, 16 or 32 lanes, at least
// `wmin` (IGN_SIMP_GROUP).  Rings over S_MAXV faces take 32 lanes and are parked there.
__device__ __forceinline__ uint32_t sl_width(uint32_t nfu, uint32_t nfv, uint32_t wmin) {
  const uint32_t n = nfu > nfv ? nfu : nfv;
  const uint32_t w = n <= 8u ? 8u : (n <= 16u ? 16u : 32u);
  return w > wmin ? w : wmin;
}

// One sweep of E2 with groups of W lanes (32 / W winners per warp side by side), each group taking the
// winners whose width (sl_width) is W.  A group owns its winner from the flip tests to the re-costs, with
// no barrier in between: that is safe because winners are two apart (§5 of DESIGN.md), so no other
// group writes a face, a state byte, a quadric or a position that this group reads or writes.  Lane gl
// holds ring entry gl of each side.  The groups of a warp run the same instructions; everything that
// differs between them is predicated and loop counts are made warp uniform.  Warp w0 takes the first G
// winners and the warps after it (cyclically) the next ones, so that a sweep starts on the warps that the
// previous sweep's last round left idle.  *nev counts the re-costed half-edges.
template <bool SM, bool R, int W>
__device__ __forceinline__ void sl_group_pass(const SlArgs& A, const SlLab<SM>& L, SlShared& sh, uint32_t first,
                                              uint32_t last, uint32_t w0, uint32_t* nev) {
  static_assert(W == 8 || W == 16 || W == 32, "group width");
  const uint32_t FULL = 0xFFFFFFFFu;
  const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5, NW = blockDim.x >> 5;
  constexpr uint32_t G = 32 / W;                       // groups per warp
  const uint32_t gl = lane & (W - 1), goff = lane & ~(uint32_t)(W - 1);
  const uint32_t wmask = W == 32 ? FULL : (1u << W) - 1u;
  const uint32_t gmask = wmask << goff;
  const uint32_t gidx = lane / W;
  SlWin* const win = sl_win();
  for (uint32_t base = first + ((warp + NW - w0) % NW) * G; base < last; base += NW * G) {  // warp uniform
    bool act = base + gidx < last;
    uint32_t slot = 0, nfu = 0, nfv = 0;
    if (act) {
      slot = win[base + gidx].order;
      nfu = win[slot].cnt[0]; nfv = win[slot].cnt[1];
    }
    act = act && sl_width(nfu, nfv, A.group_min) == (uint32_t)W;
    const uint32_t b_act = __ballot_sync(FULL, act && gl == 0);
    if (!b_act) continue;  // no winner of this width in the warp's slots
    if (lane == 0) atomicAdd(&sh.ngroup[W == 8 ? 0 : (W == 16 ? 1 : 2)], (uint32_t)__popc(b_act));
    if (W == 32 && act && gl == 0 && (nfu > (uint32_t)S_MAXV || nfv > (uint32_t)S_MAXV)) atomicAdd(&A.counters[25], 1u);
    uint32_t fu = 0, fv = 0, u = 0, v = 0, k = 0;
    bool ok = false;
    if (act) {
      if (gl < nfu) fu = L.ring[(2 * slot) * S_MAXV + gl];
      if (gl < nfv) fv = L.ring[(2 * slot + 1) * S_MAXV + gl];
      u = win[slot].u; v = win[slot].v; k = win[slot].keep;
      ok = !(win[slot].flags & WF_BAD) && nfu <= (uint32_t)S_MAXV && nfv <= (uint32_t)S_MAXV;
    }
    uint32_t au[3] = {0, 0, 0}, av[3] = {0, 0, 0};
    if (ok && gl < nfu) { au[0] = sl_fget<SM>(L, fu, 0); au[1] = sl_fget<SM>(L, fu, 1); au[2] = sl_fget<SM>(L, fu, 2); }
    if (ok && gl < nfv) { av[0] = sl_fget<SM>(L, fv, 0); av[1] = sl_fget<SM>(L, fv, 1); av[2] = sl_fget<SM>(L, fv, 2); }
    // flip tests of the faces that survive the collapse (those holding the other endpoint die with the
    // edge), one side after the other; one flipping face rejects the winner
    uint32_t flip = 0;  // bit 0: the lane's u-side face flips, bit 1: its v-side face
    if (ok && gl < nfu && au[0] != v && au[1] != v && au[2] != v && sl_flips<SM, R>(A, L, au, u, win[slot].best)) flip = 1u;
    if (ok && gl < nfv && av[0] != u && av[1] != u && av[2] != u && sl_flips<SM, R>(A, L, av, v, win[slot].best)) flip |= 2u;
    if (__ballot_sync(FULL, flip != 0) & gmask) ok = false;
    if (A.trace != nullptr) {
      const uint32_t b_u = __ballot_sync(FULL, flip & 1u) & gmask, b_v = __ballot_sync(FULL, flip & 2u) & gmask;
      if (act && gl == 0 && (b_u || b_v)) atomicAdd(&A.trace[SL_TFLIP + (b_u && b_v ? 2 : (b_u ? 0 : 1))], 1u);
    }
    const uint32_t rm = (k == u) ? v : u;
    // the quadrics of the two endpoints are needed only if the collapse happens, but the L2 round
    // trip is as long as the whole link test: request them now
    const uint64_t gk = sl_vg<SM, R>(L, k), gr = sl_vg<SM, R>(L, rm);
    double* Qk = A.Q + 10 * gk;
    const double* Qr = A.Q + 10 * gr;
    // lane gl sums component gl of the quadrics and lanes 10-12 write the position; with 8 lanes, lanes
    // 0-1 also sum components 8-9 and lanes 2-4 write the position
    double qk = 0.0, qr = 0.0, qk2 = 0.0, qr2 = 0.0;
    if (ok && gl < 10) { qk = Qk[gl]; qr = Qr[gl]; }
    if (W == 8 && ok && gl < 2) { qk2 = Qk[gl + 8]; qr2 = Qr[gl + 8]; }
    const bool hu = ok && gl < nfu, hv = ok && gl < nfv;
    uint32_t x1 = 0xF0000000u + lane, x2 = 0xF1000000u + lane, y1 = 0xF2000000u + lane, y2 = 0xF3000000u + lane;
    if (hu) sl_others(au, u, &x1, &x2);
    if (hv) sl_others(av, v, &y1, &y2);
    const bool rm_is_u = (rm == u);
    // rm's corner of the lane's face of rm (the collapse writes k there)
    const uint32_t crm = rm_is_u ? (au[0] == u ? 0u : (au[1] == u ? 1u : 2u)) : (av[0] == v ? 0u : (av[1] == v ? 1u : 2u));
    // (every lane of the warp takes part in the collectives below; n = 0 for groups without a winner)
    const uint32_t nu = ok ? nfu : 0u, nv = ok ? nfv : 0u;
    uint32_t nmax = nu > nv ? nu : nv;
#pragma unroll
    for (uint32_t d = W; d < 32u; d <<= 1) {
      const uint32_t o = __shfl_xor_sync(FULL, nmax, d);
      nmax = o > nmax ? o : nmax;
    }
    // distinct neighbours of u (first occurrences f1 among x1, f2 among x2 not in x1), same for v
    const uint32_t mu1 = __match_any_sync(FULL, x1) & gmask, mu2 = __match_any_sync(FULL, x2) & gmask;
    const uint32_t mv1 = __match_any_sync(FULL, y1) & gmask, mv2 = __match_any_sync(FULL, y2) & gmask;
    // coinc: the lane's face {u, x1, x2} and a face {v, x1, x2} would both become {k, x1, x2}
    bool inu = false, inv = false, c1 = false, c2 = false, coinc = false;
    for (uint32_t j = 0; j < nmax; j++) {
      const uint32_t sx1 = __shfl_sync(FULL, x1, j, W), sy1 = __shfl_sync(FULL, y1, j, W), sy2 = __shfl_sync(FULL, y2, j, W);
      if (j < nu) inu |= (sx1 == x2);
      if (j < nv) {
        inv |= (sy1 == y2);
        c1 |= (x1 == sy1) | (x1 == sy2);
        c2 |= (x2 == sy1) | (x2 == sy2);
        coinc |= ((x1 == sy1) & (x2 == sy2)) | ((x1 == sy2) & (x2 == sy1));
      }
    }
    const bool f1 = hu && ((int)lane == __ffs(mu1) - 1);
    const bool f2 = hu && ((int)lane == __ffs(mu2) - 1) && !inu;
    const bool g1 = hv && ((int)lane == __ffs(mv1) - 1);
    const bool g2 = hv && ((int)lane == __ffs(mv2) - 1) && !inv;
    const uint32_t b_f1 = __ballot_sync(FULL, f1), b_f2 = __ballot_sync(FULL, f2);
    const uint32_t b_g1 = __ballot_sync(FULL, g1), b_g2 = __ballot_sync(FULL, g2);
    const uint32_t b_c1 = __ballot_sync(FULL, f1 && c1), b_c2 = __ballot_sync(FULL, f2 && c2);
    const uint32_t b_sh = __ballot_sync(FULL, hu && (x1 == v || x2 == v));
    const uint32_t nnu = __popc(b_f1 & gmask) + __popc(b_f2 & gmask), nnv = __popc(b_g1 & gmask) + __popc(b_g2 & gmask);
    const uint32_t common = __popc(b_c1 & gmask) + __popc(b_c2 & gmask), shared = __popc(b_sh & gmask);
    // link condition for an interior edge, except on a tetrahedron (two faces on the wings would coincide)
    const uint32_t b_co = __ballot_sync(FULL, hu && coinc) & gmask;
    const bool go = ok && nnu <= (uint32_t)S_MAXV && nnv <= (uint32_t)S_MAXV && shared == 2 && common == 2 && !b_co;
    if (act && !go && gl == 0) {  // park the edge until one of its endpoints' rings changes
      const uint32_t hl = win[slot].h, f = hl / 3, c = hl - 3 * f;
      const uint32_t st = L.fstate[f];  // (winners of one pass never share a face: byte accesses are disjoint)
      L.fstate[f] = (uint8_t)((st & ~(3u << (2 * c))) | (1u << (2 * c)));
      sl_vclear<SM>(L.vflag, u, VF_END);
      sl_vclear<SM>(L.vflag, v, VF_END);
      atomicOr(&sh.progress, 1u);
    }
    const bool hr = go && (rm_is_u ? hu : hv);
    const uint32_t rf = rm_is_u ? fu : fv;
    // faces of rm: those that also hold k die, the others get k in rm's corner
    const bool dies = hr && (rm_is_u ? (x1 == k || x2 == k) : (y1 == k || y2 == k));
    if (hr) {
      if (dies) L.fstate[rf] = (uint8_t)(L.fstate[rf] & 0x7Fu);
      else sl_fset<SM>(L, rf, (int)crm, k);
    }
    const uint32_t dead = __popc(__ballot_sync(FULL, dies) & gmask);
    const double qs = qk + qr, qs2 = qk2 + qr2;  // k's new quadric: component gl (8-lane groups: gl + 8 in qs2)
    if (go) {
      // the new ring of k: parked edges around it may be valid now
      if (hu && x1 != v && x2 != v) { sl_vor<SM>(L.vflag, x1, VF_RDIRTY); sl_vor<SM>(L.vflag, x2, VF_RDIRTY); }
      if (hv && y1 != u && y2 != u) { sl_vor<SM>(L.vflag, y1, VF_RDIRTY); sl_vor<SM>(L.vflag, y2, VF_RDIRTY); }
      if (gl < 10) Qk[gl] = qs;
      if (gl >= 10 && gl < 13) A.pos[3 * gk + (gl - 10)] = win[slot].best[gl - 10];
      if (W == 8) {
        if (gl < 2) Qk[gl + 8] = qs2;
        else if (gl < 5) A.pos[3 * gk + (gl - 2)] = win[slot].best[gl - 2];
      }
      if (gl == 0) {
        sl_vclear<SM>(L.vflag, k, VF_END);
        sl_vclear<SM>(L.vflag, rm, 0xFFu);
        atomicSub(&sh.alive, dead);
        atomicAdd(&sh.ncol, 1u);
        atomicOr(&sh.progress, 1u);
      }
    }
    // k has its final quadric and position, and so do its neighbours (winners are two apart, in this pass
    // and in the later passes of the round), so the costs of k's edges are final until the next round:
    // re-cost them now.  Every alive face of the two ring lists holds k, and each is in one list (so its
    // state byte has one writer: the lane that holds it).  The canonical half-edges of k (bit 2 side + t of
    // m, sl_kcorner) are dealt out to the group's lanes, item i to lane i mod W, so that a lane evaluates
    // about one cost instead of up to four one after the other; the memos go back to the lanes that hold
    // the faces.  k's quadric and position come from the group's registers (sl_recost_k).
    __syncwarp();  // the rewritten faces and state bytes are visible to the group
    uint32_t m = 0, ck = 0, st0 = 0, st1 = 0;
    if (go && gl < nfu) {
      st0 = L.fstate[fu];
      if (st0 & 0x80u) {
        const uint32_t c = sl_kcorner<SM>(L, fu, k);
        ck = c;
        m |= (k < sl_fget<SM>(L, fu, (int)((c + 1) % 3)) ? 1u : 0u) | (sl_fget<SM>(L, fu, (int)((c + 2) % 3)) < k ? 2u : 0u);
      }
    }
    if (go && gl < nfv) {
      st1 = L.fstate[fv];
      if (st1 & 0x80u) {
        const uint32_t c = sl_kcorner<SM>(L, fv, k);
        ck |= c << 2;
        m |= (k < sl_fget<SM>(L, fv, (int)((c + 1) % 3)) ? 4u : 0u) | (sl_fget<SM>(L, fv, (int)((c + 2) % 3)) < k ? 8u : 0u);
      }
    }
    const uint32_t cnt = __popc(m);
    uint32_t inc = cnt;
#pragma unroll
    for (uint32_t d = 1; d < W; d <<= 1) {
      const uint32_t o = __shfl_up_sync(FULL, inc, d, W);
      if (gl >= d) inc += o;
    }
    const uint32_t P = inc - cnt, N = __shfl_sync(FULL, inc, W - 1, W);  // first item of the lane, items of the group
    uint32_t rounds = (N + W - 1) / W;
#pragma unroll
    for (uint32_t d = W; d < 32u; d <<= 1) {
      const uint32_t o = __shfl_xor_sync(FULL, rounds, d);
      rounds = o > rounds ? o : rounds;
    }
    uint32_t res = 0;  // memo of this lane's item of round r in bits 2r..2r+1
    for (uint32_t r = 0; r < rounds; r++) {  // warp uniform
      const uint32_t idx = r * W + gl;
      uint32_t own = 0;  // the lane that holds item idx: the last one whose first item is at most idx
      for (uint32_t j = 1; j < W; j++)
        if (__shfl_sync(FULL, P, j, W) <= idx) own = j;
      const uint32_t mo = __shfl_sync(FULL, m, own, W), po = __shfl_sync(FULL, P, own, W);
      const uint32_t fuo = __shfl_sync(FULL, fu, own, W), fvo = __shfl_sync(FULL, fv, own, W);
      const uint32_t cko = __shfl_sync(FULL, ck, own, W);
      const bool has = idx < N;
      uint32_t f = 0, c = 0;
      if (has) {
        uint32_t b = mo;
        for (uint32_t q = idx - po; q; q--) b &= b - 1;  // the (idx - po)-th item of the owner
        const uint32_t bit = (uint32_t)__ffs(b) - 1, side = bit >> 1;
        c = (((cko >> (2 * side)) & 3u) + 2u * (bit & 1u)) % 3u;
        f = side ? fvo : fuo;
        (*nev)++;
      }
      res |= sl_recost_k<SM, R, W>(A, L, has, f, c, k, qs, qs2, win[slot].best) << (2 * r);
    }
    uint32_t q = P;
#pragma unroll
    for (uint32_t bit = 0; bit < 4; bit++) {  // the memos of this lane's items
      const uint32_t val = __shfl_sync(FULL, res, q % W, W);
      if ((m >> bit) & 1u) {
        const uint32_t side = bit >> 1, es = (val >> (2 * (q / W))) & 3u;
        const uint32_t c = (((ck >> (2 * side)) & 3u) + 2u * (bit & 1u)) % 3u;
        if (side) st1 = (st1 & ~(3u << (2 * c))) | (es << (2 * c));
        else st0 = (st0 & ~(3u << (2 * c))) | (es << (2 * c));
        q++;
      }
    }
    if (m & 3u) L.fstate[fu] = (uint8_t)st0;
    if (m & 12u) L.fstate[fv] = (uint8_t)st1;
  }
}

// Hand a shared-memory label over to the next smaller class at the end of round r (right after a face-list
// compaction: flist[0, nF) are exactly the alive faces).  Alive vertices are renumbered in vertex order, so
// keep = min(u, v) and the canonical u < v half-edge of every edge stay what they were.
template <bool R>
__device__ void sl_migrate(const SlArgs& A, const SlLab<true>& L, SlShared& sh, const uint16_t* flist, uint32_t nF,
                           int r) {
  const uint32_t FULL = 0xFFFFFFFFu;
  const uint32_t tid = threadIdx.x, NT = blockDim.x, lane = tid & 31u, warp = tid >> 5, NW = NT >> 5;
  // block-wide exclusive scan of the alive vertices over contiguous chunks (the winner records and ring
  // lists are free between rounds and hold the warp totals: 184 bytes or more, 4 per warp)
  uint32_t* const wsum = (uint32_t*)sl_win();
  const uint32_t per = (L.U + NT - 1) / NT, v0 = min(tid * per, L.U), v1 = min(v0 + per, L.U);
  uint32_t cnt = 0;
  for (uint32_t v = v0; v < v1; v++) cnt += L.vflag[v] & VF_ALIVE;
  uint32_t inc = cnt;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t o = __shfl_up_sync(FULL, inc, d);
    if ((int)lane >= d) inc += o;
  }
  if (lane == 31) wsum[warp] = inc;
  __syncthreads();
  if (warp == 0) {
    const uint32_t t = lane < NW ? wsum[lane] : 0u;
    uint32_t x = t;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t o = __shfl_up_sync(FULL, x, d);
      if ((int)lane >= d) x += o;
    }
    if (lane < NW) wsum[lane] = x - t;
  }
  __syncthreads();
  uint32_t j = wsum[warp] + inc - cnt;
  for (uint32_t v = v0; v < v1; v++) {
    const uint32_t fl = L.vflag[v];
    if (!(fl & VF_ALIVE)) continue;
    A.vlist[L.vbase + j] = (uint32_t)(R ? L.vmap[v] : v) | (fl << 16);
    L.key1[v] = j++;  // key1 is dead until the next round's P1: it holds the new vertex ids
  }
  __syncthreads();
  for (uint32_t i = tid; i < nF; i += NT) {
    const uint32_t f = flist[i], fo = sl_fo<true, R>(L, f);
    A.flist[L.tbase + i] = L.key1[L.fc0[f]] | (L.key1[L.fc1[f]] << 16);
    A.flist2[L.tbase + i] = L.key1[L.fc2[f]] | (fo << 16);
    A.fstate[L.tbase + i] = L.fstate[f];
    A.finv[L.tbase + fo] = (uint16_t)i;
  }
  if (tid == 0) {
    uint32_t* h = A.mq_next + SL_MREC * (size_t)atomicAdd(&A.counters[16 + A.cls + 1], 1u);
    h[0] = L.label;
    h[1] = sh.rec;
    h[2] = (uint32_t)r + 1;
    h[3] = sh.slow;
    h[4] = nF;
    h[5] = sh.valive;
  }
}

// P2: every canonical half-edge (u < v) of an alive face posts its cached key to both endpoints.  A warp takes
// 32 alive faces per iteration.  The cached costs are the only global loads: PK (32-bit keys) one packed word
// per face (s_cwords), requested two iterations ahead; else three floats, one iteration ahead.  A resumed label
// addresses them by the original face id.
template <bool SM, bool R, bool PK>
__device__ __forceinline__ void sl_keys(const SlArgs& A, const SlLab<SM>& L, const typename SlLab<SM>::idx_t* flist,
                                        uint32_t nF, uint32_t salt) {
  typedef typename SlLab<SM>::key_t key_t;
  constexpr int D = PK ? 2 : 1;
  const uint32_t tid = threadIdx.x, NT = blockDim.x, lane = tid & 31u, warp = tid >> 5;
  const unsigned long long* cw = s_cwords(A.ecost, L.tbase);
  const float* ecb = A.ecost + 3 * (uint64_t)L.tbase;
  // stage s: face id, original face id and cached costs of the lane's face s iterations after the current one
  uint32_t f_n[D], fo_n[D];
  unsigned long long w_n[D];
  float ec_n[D][3];
#pragma unroll
  for (int s = 0; s < D; s++) {
    const uint32_t i = warp * 32 + lane + s * NT;
    f_n[s] = fo_n[s] = 0;
    w_n[s] = 0;
    ec_n[s][0] = ec_n[s][1] = ec_n[s][2] = 0.f;
    if (i < nF) {
      f_n[s] = flist[i];
      fo_n[s] = sl_fo<SM, R>(L, f_n[s]);
      if (PK) w_n[s] = cw[fo_n[s]];
      else { ec_n[s][0] = ecb[3 * (uint64_t)fo_n[s]]; ec_n[s][1] = ecb[3 * (uint64_t)fo_n[s] + 1]; ec_n[s][2] = ecb[3 * (uint64_t)fo_n[s] + 2]; }
    }
  }
  for (uint32_t base = warp * 32; base < nF; base += NT) {
    const uint32_t i = base + lane;
    const uint32_t f = f_n[0], fo = fo_n[0];
    const unsigned long long w = w_n[0];
    const float ec[3] = {ec_n[0][0], ec_n[0][1], ec_n[0][2]};
#pragma unroll
    for (int s = 0; s + 1 < D; s++) {
      f_n[s] = f_n[s + 1]; fo_n[s] = fo_n[s + 1]; w_n[s] = w_n[s + 1];
      ec_n[s][0] = ec_n[s + 1][0]; ec_n[s][1] = ec_n[s + 1][1]; ec_n[s][2] = ec_n[s + 1][2];
    }
    if (i + D * NT < nF) {
      f_n[D - 1] = flist[i + D * NT];
      fo_n[D - 1] = sl_fo<SM, R>(L, f_n[D - 1]);
      if (PK) w_n[D - 1] = cw[fo_n[D - 1]];
      else {
        const float* e = ecb + 3 * (uint64_t)fo_n[D - 1];
        ec_n[D - 1][0] = e[0]; ec_n[D - 1][1] = e[1]; ec_n[D - 1][2] = e[2];
      }
    }
    uint32_t st = 0, a[3] = {0, 0, 0}, fl[3] = {0, 0, 0};
    if (i < nF) st = L.fstate[f];
    bool act = (st & 0x80u) != 0;
    if (act) {
      a[0] = sl_fget<SM>(L, f, 0); a[1] = sl_fget<SM>(L, f, 1); a[2] = sl_fget<SM>(L, f, 2);
      fl[0] = L.vflag[a[0]]; fl[1] = L.vflag[a[1]]; fl[2] = L.vflag[a[2]];
    }
    if (act) {
      uint32_t nst = st;
#pragma unroll
      for (int c = 0; c < 3; c++) {
        const uint32_t u = a[c], v = a[(c + 1) % 3];
        const uint32_t fe = fl[c] | fl[(c + 1) % 3];
        if (!(u < v)) continue;  // one key per edge
        // memo: 1 parked (won a round, failed validation), 2 cost cached in ecost, 3 known to
        // exceed max_error.  A parked edge is un-parked when an endpoint's ring changed (RDIRTY):
        // its cost was cached when it won, and an endpoint that moved since would have re-costed it.
        uint32_t es = (st >> (2 * c)) & 3u;
        if (es == 1 && (fe & VF_RDIRTY)) es = 2;
        if (es == 2) {
          const uint32_t hl = 3u * fo + (uint32_t)c;
          const key_t key = PK ? (key_t)sl_key((uint32_t)(w >> (16 * c)) & 0xFFFFu, hl, salt)
                               : sl_key<SM>(L, ec[c], hl, salt);
          sl_post(L.key1, u, v, key);
        } else if (es == 0) {
          atomicAdd(&A.counters[28], 1u);  // a half-edge without a cost: a bug
        }
        nst = (nst & ~(3u << (2 * c))) | (es << (2 * c));
      }
      if (nst != st) L.fstate[f] = (uint8_t)nst;
    }
  }
}

// All rounds of one label (R: a label resumed from the header `hdr` after it migrated from a larger class)
template <bool SM, bool R>
__device__ void sl_run(const SlArgs& A, const SlLab<SM>& L, SlShared& sh, const uint32_t* hdr) {
  if (threadIdx.x == 0) sh.nrecost = sh.ngroup[0] = sh.ngroup[1] = sh.ngroup[2] = 0;
  if (A.trace != nullptr && threadIdx.x == 0) {
    for (int q = 0; q < SL_NPH; q++) sh.ph[q] = 0;
    sh.t_prev = clock64();
    sh.t_label = sh.t_prev;
    sh.visits = 0;
    sh.wins = 0;
  }
  typedef typename SlLab<SM>::idx_t idx_t;
  typedef typename SlLab<SM>::key_t key_t;
  const uint32_t FULL = 0xFFFFFFFFu;
  const uint32_t tid = threadIdx.x, NT = blockDim.x, lane = tid & 31u, warp = tid >> 5, NW = NT >> 5;
  const uint32_t T = L.T, U = L.U;
  idx_t *flist = L.flist, *flist2 = L.flist2, *vlist = L.vlist, *vlist2 = L.vlist2;
  // ---- load the label
  int r = 0;
  if (R) {  // the migrated state (see SlArgs::mq_next)
    for (uint32_t f = tid; f < T; f += NT) {
      const uint32_t w0 = A.flist[L.tbase + f], w1 = A.flist2[L.tbase + f];
      sl_fset<SM>(L, f, 0, w0 & 0xFFFFu);
      sl_fset<SM>(L, f, 1, w0 >> 16);
      sl_fset<SM>(L, f, 2, w1 & 0xFFFFu);
      L.fmap[f] = (idx_t)(w1 >> 16);
      L.fstate[f] = A.fstate[L.tbase + f];
      flist[f] = (idx_t)f;
    }
    for (uint32_t v = tid; v < U; v += NT) {
      const uint32_t w = A.vlist[L.vbase + v];
      L.vmap[v] = (idx_t)(w & 0xFFFFu);
      L.vflag[v] = (uint8_t)(w >> 16);
    }
    r = (int)hdr[2];
    if (tid == 0) {
      sh.rec = hdr[1];
      sh.slow = hdr[3];
      sh.alive = hdr[4];
    }
  } else {
    for (uint32_t f = tid; f < T; f += NT) {
      if (SM) {
        const uint32_t* g = A.face + 3 * (uint64_t)(L.tbase + f);
        sl_fset<SM>(L, f, 0, g[0] - L.vbase);
        sl_fset<SM>(L, f, 1, g[1] - L.vbase);
        sl_fset<SM>(L, f, 2, g[2] - L.vbase);
      }
      L.fstate[f] = (uint8_t)(0x80u | A.fstate[L.tbase + f]);  // alive, memos of k_simp_ecost
      flist[f] = (idx_t)f;
    }
    for (uint32_t v = tid; v < U; v += NT) {
      L.vflag[v] = (uint8_t)(VF_ALIVE | (A.vbound[L.vbase + v] ? VF_BOUND : 0u));
      if (!SM) vlist[v] = (idx_t)v;  // the shared-memory class scans its vertices directly (no list: 2 B / vertex saved)
    }
    if (tid == 0) {
      sh.rec = A.base + sh.work;
      sh.alive = T;
      sh.slow = 0;
    }
  }
  if (tid == 0) {
    sh.valive = U;
    sh.stop = 0;
  }
  __syncthreads();
  uint32_t nF = T, nV = U;
  bool migrated = false;

  for (; r < A.max_rounds; r++) {
    if (sh.alive <= L.target) break;  // reached the target before this round
    // per-round salt: equal-cost edges get a fresh pseudo-random priority every round (a fixed
    // one lets the same validation failures win again and again: 8738 instead of 454 faces on the
    // reference's box volume)
    const uint32_t salt = (uint32_t)r * 0x9E3779B9u;
    // ---- P1
    for (uint32_t i = tid; i < nV; i += NT) {
      const uint32_t v = SM ? i : (uint32_t)vlist[i];
      L.key1[v] = (key_t)S_KEYMAX;
      L.vlose[v] = 0;
      const uint8_t b = L.vflag[v];
      if (b & VF_DONE) L.vflag[v] = (uint8_t)(b & ~VF_DONE);
    }
    if (tid == 0) {
      sh.progress = 0;
      sh.ncol = 0;
      sh.npass = 0;
    }
    __syncthreads();
    SL_MARK(0);
    // ---- P2: keys of the canonical half-edges.  No cost is evaluated here: k_simp_ecost costs every
    // half-edge before the first round and E2 re-costs the edges of every vertex that moved right after
    // its collapse.
    if (SM || L.fmt16) sl_keys<SM, R, true>(A, L, flist, nF, salt);
    else sl_keys<SM, R, false>(A, L, flist, nF, salt);
    __syncthreads();
    SL_MARK(1);
    // ---- P3: dirty flags consumed; LOSE = a face neighbour holds a smaller key
    for (uint32_t i = tid; i < nV; i += NT) {
      const uint32_t v = SM ? i : (uint32_t)vlist[i];
      if (L.vflag[v] & VF_RDIRTY) sl_vclear<SM>(L.vflag, v, VF_RDIRTY);
    }
    // two faces per thread and iteration, the loads of both issued before anything depends on them
    for (uint32_t i = tid; i < nF; i += 2 * NT) {
      const uint32_t i2 = i + NT;
      const bool two = i2 < nF;
      const uint32_t fa = flist[i], fb = two ? (uint32_t)flist[i2] : fa;
      const bool la = (L.fstate[fa] & 0x80u) != 0, lb = two && (L.fstate[fb] & 0x80u) != 0;
      uint32_t a0 = 0, a1 = 0, a2 = 0, b0 = 0, b1 = 0, b2 = 0;
      if (la) { a0 = sl_fget<SM>(L, fa, 0); a1 = sl_fget<SM>(L, fa, 1); a2 = sl_fget<SM>(L, fa, 2); }
      if (lb) { b0 = sl_fget<SM>(L, fb, 0); b1 = sl_fget<SM>(L, fb, 1); b2 = sl_fget<SM>(L, fb, 2); }
      key_t ka0 = 0, ka1 = 0, ka2 = 0, kb0 = 0, kb1 = 0, kb2 = 0;
      if (la) { ka0 = L.key1[a0]; ka1 = L.key1[a1]; ka2 = L.key1[a2]; }
      if (lb) { kb0 = L.key1[b0]; kb1 = L.key1[b1]; kb2 = L.key1[b2]; }
      if (la) {
        key_t m = ka0 < ka1 ? ka0 : ka1;
        m = ka2 < m ? ka2 : m;
        if (ka0 > m) L.vlose[a0] = 1;
        if (ka1 > m) L.vlose[a1] = 1;
        if (ka2 > m) L.vlose[a2] = 1;
      }
      if (lb) {
        key_t m = kb0 < kb1 ? kb0 : kb1;
        m = kb2 < m ? kb2 : m;
        if (kb0 > m) L.vlose[b0] = 1;
        if (kb1 > m) L.vlose[b1] = 1;
        if (kb2 > m) L.vlose[b2] = 1;
      }
    }
    __syncthreads();
    SL_MARK(2);
    // ---- P4 + E: the round's winners (marked DONE on both endpoints), L.wcap per pass
    SlWin* const win = sl_win();
    for (;;) {
      if (tid == 0) { sh.nwin = 0; sh.ring8 = 0; sh.ring16 = 0; sh.nnarrow = 0; sh.nwide = 0; sh.npass++; }
      __syncthreads();
      for (uint32_t i = tid; i < nV; i += NT) {
        const uint32_t a = SM ? i : (uint32_t)vlist[i];
        const uint32_t fl = L.vflag[a];
        if (!(fl & VF_ALIVE) || (fl & VF_DONE) || L.vlose[a]) continue;
        const key_t key = L.key1[a];
        if (key == (key_t)S_KEYMAX) continue;
        const uint32_t hl = sl_key_edge<SM>(L, key, salt);
        const uint32_t fo = hl / 3, c = hl - 3 * fo;
        const uint32_t f = R ? (uint32_t)A.finv[L.tbase + fo] : fo;
        if (sl_fget<SM>(L, f, (int)c) != a) continue;
        const uint32_t v = sl_fget<SM>(L, f, (int)((c + 1) % 3));
        if (L.key1[v] != key || (L.vflag[v] & VF_DONE) || L.vlose[v]) continue;
        const uint32_t slot = atomicAdd(&sh.nwin, 1u);
        if (slot < L.wcap) {
          win[slot].u = a;
          win[slot].v = v;
          win[slot].h = 3 * f + c;
          win[slot].cnt[0] = 0;
          win[slot].cnt[1] = 0;
          win[slot].flags = 0;
          sl_vor<SM>(L.vflag, a, VF_DONE | VF_END);
          sl_vor<SM>(L.vflag, v, VF_DONE | VF_END);
        }
      }
      __syncthreads();
      SL_MARK(3);
      const uint32_t total = sh.nwin;
      const uint32_t nb = total < L.wcap ? total : L.wcap;
      if (A.trace != nullptr && tid == 0 && sh.npass == 1) {
        const uint32_t b = total / 16 < (uint32_t)SL_HW - 1 ? total / 16 : (uint32_t)SL_HW - 1;
        atomicAdd(&A.trace[SL_HIST + SL_HCLS * A.cls + SL_HP + b], 1u);
      }
      if (nb == 0) break;
      if (A.trace != nullptr && tid == 0) sh.wins += nb;
      // key1 is dead until the next P1: the winners' entries now name their ring lists
      for (uint32_t i = tid; i < nb; i += NT) {
        L.key1[win[i].u] = (key_t)(2u * i);
        L.key1[win[i].v] = (key_t)(2u * i + 1u);
      }
      __syncthreads();
      SL_MARK(4);
      // ---- E1 + E2a in one barrier interval (they do not depend on each other): the first warps
      // compute placement and cost of the winners (one thread each, double precision, L2 latency)
      // while the others build the ring lists with one pass over the alive faces.
      {
        const uint32_t nbt = (nb + 31u) & ~31u;
        const bool split = NT - nbt >= NT / 2;
        if (tid < nb) {
          const uint32_t i = tid;
          SEval e;
          sl_cost<SM, R>(A, L, win[i].u, win[i].v, &e);
          win[i].keep = e.valid ? e.keep : win[i].u;
          win[i].flags = e.valid ? 0u : WF_BAD;
          if (e.valid) {
            win[i].best[0] = e.p[0]; win[i].best[1] = e.p[1]; win[i].best[2] = e.p[2];
          }
        }
        if (!split || tid >= nbt) {
          const uint32_t first = split ? tid - nbt : tid, step = split ? NT - nbt : NT;
          for (uint32_t i = first; i < nF; i += 2 * step) {
            const uint32_t i2 = i + step;
            const bool two = i2 < nF;
            const uint32_t fa = flist[i], fb = two ? (uint32_t)flist[i2] : fa;
            const bool la = (L.fstate[fa] & 0x80u) != 0, lb = two && (L.fstate[fb] & 0x80u) != 0;
            uint32_t x[6] = {0, 0, 0, 0, 0, 0}, fl[6] = {0, 0, 0, 0, 0, 0};
            if (la) { x[0] = sl_fget<SM>(L, fa, 0); x[1] = sl_fget<SM>(L, fa, 1); x[2] = sl_fget<SM>(L, fa, 2); }
            if (lb) { x[3] = sl_fget<SM>(L, fb, 0); x[4] = sl_fget<SM>(L, fb, 1); x[5] = sl_fget<SM>(L, fb, 2); }
            if (la) { fl[0] = L.vflag[x[0]]; fl[1] = L.vflag[x[1]]; fl[2] = L.vflag[x[2]]; }
            if (lb) { fl[3] = L.vflag[x[3]]; fl[4] = L.vflag[x[4]]; fl[5] = L.vflag[x[5]]; }
#pragma unroll
            for (int c = 0; c < 6; c++) {
              if (!(fl[c] & VF_END)) continue;
              const uint32_t sl = (uint32_t)L.key1[x[c]];
              const uint32_t p = atomicAdd(&win[sl >> 1].cnt[sl & 1u], 1u);
              if (p < (uint32_t)S_MAXV) L.ring[sl * S_MAXV + p] = (idx_t)(c < 3 ? fa : fb);
              if (p == 8u) sh.ring8 = 1;  // (every writer stores 1)
              if (p == 16u) sh.ring16 = 1;
            }
          }
        }
      }
      __syncthreads();
      SL_MARK(5);
      SL_MARK(6);
      if (A.trace != nullptr) {
        for (uint32_t i = tid; i < 2 * nb; i += NT) {
          const uint32_t n = win[i >> 1].cnt[i & 1u];
          atomicAdd(&A.trace[SL_HIST + SL_HCLS * A.cls + SL_HP + SL_HW + (n <= (uint32_t)S_MAXV ? n : S_MAXV + 1)], 1u);
        }
      }
      // E2: flip tests, link condition by ballots / shuffles over the ring lists, the collapse and the
      // re-costs of the kept vertex's edges, one group of lanes per winner from start to end (a lane holds
      // one ring face of each endpoint).  Rings hold 5-6 faces typically, so most winners take 8 lanes,
      // four per warp; the duration of the phase is the number of winners a warp handles one after the
      // other, each a chain of dependent loads.  Wider rings take 16 or 32 lanes in further sweeps, only
      // in passes where E1 saw one.  The winners are first ordered by width (8-lane winners to the front,
      // the others to the back), so that each sweep hands out only its own winners; no barrier between
      // the sweeps: groups never touch each other's data.
      for (uint32_t i0 = warp * 32; i0 < nb; i0 += NT) {  // warp uniform
        const uint32_t i = i0 + lane;
        const bool have = i < nb;
        const bool narrow = have && sl_width(win[i].cnt[0], win[i].cnt[1], A.group_min) == 8u;
        const uint32_t bn = __ballot_sync(FULL, narrow), bw = __ballot_sync(FULL, have && !narrow);
        uint32_t pn = 0, pw = 0;
        if (lane == 0) {
          if (bn) pn = atomicAdd(&sh.nnarrow, (uint32_t)__popc(bn));
          if (bw) pw = atomicAdd(&sh.nwide, (uint32_t)__popc(bw));
        }
        pn = __shfl_sync(FULL, pn, 0);
        pw = __shfl_sync(FULL, pw, 0);
        const uint32_t below = (1u << lane) - 1u;
        if (narrow) win[pn + __popc(bn & below)].order = i;
        else if (have) win[nb - 1 - (pw + __popc(bw & below))].order = i;
      }
      __syncthreads();
      {
        uint32_t nev = 0;
        const uint32_t wmin = A.group_min, n8 = sh.nnarrow;
        // each sweep continues the deal of winners to warps where the previous one stopped: the wide
        // winners go to the warps that the 8-lane sweep's last round left without a winner
        uint32_t w0 = 0;
        if (n8) {
          sl_group_pass<SM, R, 8>(A, L, sh, 0, n8, w0, &nev);
          w0 = (w0 + (n8 + 3u) / 4u) % NW;
        }
        if (wmin == 16u || (wmin == 8u && sh.ring8)) {
          sl_group_pass<SM, R, 16>(A, L, sh, n8, nb, w0, &nev);
          w0 = (w0 + (nb - n8 + 1u) / 2u) % NW;
        }
        if (wmin == 32u || sh.ring16) sl_group_pass<SM, R, 32>(A, L, sh, n8, nb, w0, &nev);
        if (nev) atomicAdd(&sh.nrecost, nev);
      }
      __syncthreads();  // (the next pass resets the ring flags and the winner records)
      SL_MARK(7);
      if (total <= L.wcap) break;
    }
    if (tid == 0) {
      const uint32_t passes = sh.npass;
      if (passes > 1) atomicAdd(&A.counters[24], 1u);
      if (A.trace != nullptr) atomicAdd(&A.trace[SL_HIST + SL_HCLS * A.cls + (passes < (uint32_t)SL_HP ? passes : SL_HP) - 1], 1u);
    }
    // ---- stop rules of the label
    if (tid == 0 && A.trace != nullptr && sh.rec == 0 && r < 400) {
      A.trace[4 * r + 0] = sh.progress;
      A.trace[4 * r + 1] = sh.ncol;
      A.trace[4 * r + 2] = sh.alive;
      A.trace[4 * r + 3] = nF;
    }
    if (A.trace != nullptr && tid == 0) sh.visits += nF;
    if (tid == 0) {
      sh.valive -= sh.ncol;
      uint32_t stop = 0;
      if (!sh.progress) {
        stop = 1;  // nothing collapsed or parked: fixed point
      } else {
        // four consecutive rounds that each remove fewer than 0.2% of the remaining faces
        if ((uint64_t)sh.ncol * 1000 < (uint64_t)sh.alive) sh.slow++;
        else sh.slow = 0;
        if (sh.slow >= 4) stop = 1;
      }
      sh.stop = stop;
    }
    __syncthreads();
    SL_MARK(8);
    if (sh.stop) {
      r++;
      break;
    }
    // ---- dead entries leave the lists every second round
    if (r & 1) {
      nF = sl_compact<SM>(flist, flist2, nF, &sh.counter, [&](uint32_t f) { return (L.fstate[f] & 0x80u) != 0; });
      if (!SM) nV = sl_compact<SM>(vlist, vlist2, nV, &sh.counter, [&](uint32_t v) { return (L.vflag[v] & VF_ALIVE) != 0; });
      // a label that has shrunk enough continues in the next smaller class and returns its SM share (the
      // header's queue is resumed by a later launch); alive counts only fall, so it never moves back up
      if (SM && A.mq_next != nullptr && sl_fits_smem(nF, sh.valive, NT / 2, A.smem_next, true)) {
        if constexpr (SM) sl_migrate<R>(A, L, sh, flist, nF, r);
        migrated = true;
        r++;
        break;
      }
    }
  }
  // ---- write the label back to the whole-task arrays (a migrating label writes its dead faces and
  // vertices; the class that resumes it writes the others when it finishes)
  for (uint32_t f = tid; f < T; f += NT) {
    const bool al = L.fstate[f] & 0x80u;
    const uint32_t fo = sl_fo<SM, R>(L, f);
    if (migrated && al) continue;
    A.falive[L.tbase + fo] = al ? 1 : 0;
    if (SM && al) {
      uint32_t* g = A.face + 3 * (uint64_t)(L.tbase + fo);
      g[0] = (uint32_t)sl_vg<SM, R>(L, sl_fget<SM>(L, f, 0));
      g[1] = (uint32_t)sl_vg<SM, R>(L, sl_fget<SM>(L, f, 1));
      g[2] = (uint32_t)sl_vg<SM, R>(L, sl_fget<SM>(L, f, 2));
    }
  }
  for (uint32_t v = tid; v < U; v += NT) {
    const bool al = L.vflag[v] & VF_ALIVE;
    if (!(migrated && al)) A.valive[sl_vg<SM, R>(L, v)] = al ? 1 : 0;
  }
  if (tid == 0 && A.trace != nullptr) {
    // a migrated label's record sums the cycles, visits and winners of all its segments
    for (int q = 0; q < SL_NPH; q++) atomicAdd((unsigned long long*)(A.trace + 1600) + q, sh.ph[q]);
    uint32_t* rec = A.lrec + SL_LREC * (size_t)sh.rec;
    const unsigned long long vis = rec[3] + sh.visits;
    const uint32_t kc = (uint32_t)((clock64() - sh.t_label) >> 10);
    if (!R) rec[0] = T;
    rec[1] = (uint32_t)r;
    rec[2] += kc;
    rec[6] += kc / (SL_THREADS / NT);
    rec[3] = (uint32_t)(vis > 0xFFFFFFFFull ? 0xFFFFFFFFull : vis);
    rec[4] += (uint32_t)sh.wins;
    if (!R) rec[5] = (SM ? 1u : ((const void*)L.key1 == (const void*)(A.key1 + L.vbase) ? 3u : 2u)) | (A.cls << 2);
  }
  if (tid == 0) {
    if (sh.nrecost) atomicAdd(&A.counters[27], sh.nrecost);
    for (int w = 0; w < 3; w++)
      if (sh.ngroup[w]) atomicAdd(&A.counters[29 + w], sh.ngroup[w]);
    if (!migrated) atomicMax(&A.counters[1], (uint32_t)r);
    if (!R) {  // a label counts in the class it started in
      atomicAdd(&A.counters[SM ? 2 : 3], 1u);
      atomicAdd(&A.counters[8 + A.cls], 1u);
    }
  }
}

// A shared-memory label of T faces and U vertices laid out as y, with wcap winners per pass; a resumed
// label also has the maps of its compacted faces and vertices.  The caller sets tbase, vbase, target, label.
__device__ __forceinline__ SlLab<true> sl_lab_smem(uint32_t T, uint32_t U, uint32_t wcap, const SlLayout& y,
                                                   bool resumed) {
  SlLab<true> L;
  L.T = T; L.U = U;
  L.wcap = wcap;
  L.ring = (uint16_t*)(sl_smem + y.o_ring);
  L.key1 = (uint32_t*)(sl_smem + y.o_key);
  L.fmt16 = true;
  L.fc0 = (uint16_t*)(sl_smem + y.o_f0);
  L.fc1 = L.fc0 + T;
  L.fc2 = L.fc1 + T;
  L.flist = (uint16_t*)(sl_smem + y.o_fl);
  L.vlist = nullptr;
  L.flist2 = L.vlist2 = nullptr;
  L.gface = nullptr;
  L.fstate = sl_smem + y.o_fs;
  L.vflag = sl_smem + y.o_vf;
  L.vlose = sl_smem + y.o_vl;
  L.fmap = resumed ? (uint16_t*)(sl_smem + y.o_fm) : nullptr;
  L.vmap = resumed ? (uint16_t*)(sl_smem + y.o_vm) : nullptr;
  return L;
}

// One label per CTA (the launch has one CTA per label of its size class; a CTA takes the next label of
// the size-sorted order from a counter, so big labels start first whatever order the hardware dispatches
// CTAs in).  The block size is the class's (1024, 512 or 256 threads); 64 registers per thread let two
// 512-thread or four 256-thread CTAs share an SM.
// CTAs that end after one label keep returning their SM to the block scheduler: kernels of
// other streams -- the CCL passes of the volume pipeline run on a higher-priority stream while
// MeshTasks are in flight -- get SMs within a label's run time instead of a whole task's.
__global__ void __launch_bounds__(SL_THREADS, 1) k_simp_labels(SlArgs A) {
  __shared__ SlShared sh;
  do {
    __syncthreads();  // (persistent mode) the previous label is completely written back; sh.work may be reused
    if (threadIdx.x == 0) sh.work = atomicAdd(&A.counters[4 + A.cls], 1u);
    __syncthreads();
    const uint32_t wi = sh.work;
    if (wi >= A.K) break;
    const uint32_t l = A.order[wi];
    const uint32_t tbase = A.tri_off[l], T = A.tri_off[l + 1] - tbase;
    const uint32_t vbase = A.vert_off[l], U = A.vert_off[l + 1] - vbase;
    const uint32_t target = A.target[l];
    if (T == 0 || T <= target) continue;  // init left every face / vertex alive
    const bool fmt16 = s_fmt16(T);
    if (sl_fits_smem(T, U, blockDim.x, A.smem_bytes)) {
      const uint32_t wcap = sl_wcap(T, U, blockDim.x, A.smem_bytes, false, A.wcap_max);
      SlLab<true> L = sl_lab_smem(T, U, wcap, sl_layout(T, U, false, wcap), false);
      L.tbase = tbase; L.vbase = vbase; L.target = target; L.label = l;
      sl_run<true, false>(A, L, sh, nullptr);
    } else {
      const SlLayout y = sl_layout(T, U);
      const size_t o_keyg = y.o_ring + (size_t)SL_WCAP * 2 * S_MAXV * 4;  // 32-bit face ids in the rings
      SlLab<false> L;
      L.T = T; L.U = U; L.tbase = tbase; L.vbase = vbase; L.target = target;
      L.label = l;
      L.fmap = L.vmap = nullptr;
      L.wcap = SL_WCAP < A.wcap_max ? SL_WCAP : A.wcap_max;
      L.ring = (uint32_t*)(sl_smem + y.o_ring);  // the winners and the ring lists always fit
      L.fc0 = L.fc1 = L.fc2 = nullptr;
      L.flist = A.flist + tbase; L.flist2 = A.flist2 + tbase;
      L.vlist = A.vlist + vbase; L.vlist2 = A.vlist2 + vbase;
      L.gface = A.face + 3 * (uint64_t)tbase;
      L.fmt16 = fmt16;
      // the arrays that take the atomics (keys, vertex flags) and the face states stay in shared
      // memory whenever they fit; only the faces and the alive lists are read from global memory
      const size_t h_fs = o_keyg + 8 * (size_t)U;
      const size_t h_vf = (h_fs + T + 3) & ~(size_t)3;
      const size_t h_vl = (h_vf + U + 3) & ~(size_t)3;
      if (h_vl + U + 4 <= A.smem_bytes) {
        L.key1 = (unsigned long long*)(sl_smem + o_keyg);
        L.fstate = sl_smem + h_fs;
        L.vflag = sl_smem + h_vf;
        L.vlose = sl_smem + h_vl;
      } else {
        L.key1 = A.key1 + vbase;
        L.fstate = A.fstate + tbase;
        L.vflag = A.vflag + vbase;
        L.vlose = A.vlose + vbase;
      }
      sl_run<false, false>(A, L, sh, nullptr);
    }
  } while (A.persist);
}

// Labels that migrated into the launch's class (A.mq), in the order they migrated; the grid is an upper
// bound on their number and surplus CTAs exit at once.  Its own kernel, so that the maps of the resumed
// path cost k_simp_labels no registers.
__global__ void __launch_bounds__(SL_THREADS / 2, 2) k_simp_resume(SlArgs A) {
  __shared__ SlShared sh;
  do {
    __syncthreads();
    if (threadIdx.x == 0) {
      sh.work = atomicAdd(&A.counters[20 + A.cls], 1u);
      sh.counter = A.counters[16 + A.cls];  // written by earlier launches only
    }
    __syncthreads();
    const uint32_t wi = sh.work;
    if (wi >= sh.counter) break;
    const uint32_t* hdr = A.mq + SL_MREC * (size_t)wi;
    const uint32_t l = hdr[0];
    const uint32_t T = hdr[4], U = hdr[5];
    const uint32_t wcap = sl_wcap(T, U, blockDim.x, A.smem_bytes, true, A.wcap_max);
    SlLab<true> L = sl_lab_smem(T, U, wcap, sl_layout(T, U, true, wcap), true);
    L.tbase = A.tri_off[l]; L.vbase = A.vert_off[l]; L.target = A.target[l]; L.label = l;
    sl_run<true, true>(A, L, sh, hdr);
  } while (A.persist);
}

__global__ void __launch_bounds__(256)
    k_simp_flags_u32(const uint8_t* __restrict__ a, uint64_t n, uint32_t* __restrict__ out) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i < n) out[i] = a[i];
}

__global__ void __launch_bounds__(256)
    k_simp_new_offsets(const uint32_t* __restrict__ old_off, const uint32_t* __restrict__ scan,
                       uint32_t K2, uint64_t n, uint32_t total, uint32_t* __restrict__ new_off) {
  const uint32_t l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l < K2) new_off[l] = (old_off[l] < n) ? scan[old_off[l]] : total;
}

__global__ void __launch_bounds__(256)
    k_simp_compact_verts(Simp s, const uint32_t* __restrict__ vscan, float* __restrict__ pos_f) {
  const uint64_t v = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (v >= s.U || !s.valive[v]) return;
  const uint32_t n = vscan[v];
  pos_f[3 * (uint64_t)n + 0] = __double2float_rn(s.pos[3 * v + 0]);
  pos_f[3 * (uint64_t)n + 1] = __double2float_rn(s.pos[3 * v + 1]);
  pos_f[3 * (uint64_t)n + 2] = __double2float_rn(s.pos[3 * v + 2]);
}

__global__ void __launch_bounds__(256)
    k_simp_compact_faces(Simp s, const uint32_t* __restrict__ vscan, const uint32_t* __restrict__ fscan,
                         const uint32_t* __restrict__ new_vert_off, uint32_t* __restrict__ faces_out) {
  const uint64_t f = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (f >= s.T || !s.falive[f]) return;
  const uint32_t n = fscan[f];
  const uint32_t base = new_vert_off[s.flabel[f]];
  for (int k = 0; k < 3; k++) faces_out[3 * (uint64_t)n + k] = vscan[s.face[3 * f + k]] - base;
}

__global__ void __launch_bounds__(256)
    k_simp_export(const float* __restrict__ pos_f, uint64_t first, uint64_t count, float sx, float sy,
                  float sz, float* __restrict__ out) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= count) return;
  out[3 * i + 0] = __fadd_rn(pos_f[3 * (first + i) + 0], sx);
  out[3 * i + 1] = __fadd_rn(pos_f[3 * (first + i) + 1], sy);
  out[3 * i + 2] = __fadd_rn(pos_f[3 * (first + i) + 2], sz);
}

// exposed to mesh.cu for export of simplified positions
int simp_export_positions(ign_ctx* ctx, const float* pos_f, uint64_t first, uint64_t count,
                          const float shift[3], float* d_out) {
  if (count == 0) return IGN_OK;
  IGN_LAUNCH(ctx, k_simp_export, blocks_for(count, 256), 256, 0, pos_f, first, count, shift[0], shift[1],
             shift[2], d_out);
  return IGN_OK;
}

}  // namespace ign

using namespace ign;

extern "C" int ign_mesh_simplify(ign_mesher* m, const float resolution[3], int reduction_factor,
                                 float max_error) {
  IGN_REQUIRE(m && resolution, IGN_ERR_INVALID, "null argument");
  ign_ctx* ctx = m->ctx;
  IGN_TRY(activate(ctx));
  IGN_REQUIRE(!m->simplified, IGN_ERR_INVALID, "mesher is already simplified; call mesh() again");
  IGN_REQUIRE(reduction_factor >= 1, IGN_ERR_INVALID, "reduction_factor must be >= 1");
  m->res[0] = resolution[0];
  m->res[1] = resolution[1];
  m->res[2] = resolution[2];
  m->simp_factor = reduction_factor;
  m->simp_max_error = max_error;
  memset(m->simp_counters, 0, sizeof(m->simp_counters));
  const uint64_t U = m->U, T = m->T, K = m->K;
  if (T == 0 || U == 0) {
    m->simplified = true;
    m->d_pos_f = nullptr;
    return IGN_OK;
  }
  size_t sortb = 0, scanb = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, sortb, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                  (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)(3 * T));
  cub::DeviceScan::ExclusiveSum(nullptr, scanb, (const uint32_t*)nullptr, (uint32_t*)nullptr,
                                (int)(3 * T));
  const size_t tmpb = (sortb > scanb ? sortb : scanb) + 256;
  ScratchFrame f(ctx);
  Simp s;
  s.U = U;
  s.T = T;
  uint32_t *node_v, *node_h, *vscan, *vflag32, *d_target, *d_tri_off, *d_vert_off, *d_new_tri_off, *d_new_vert_off;
  uint32_t *d_order, *flags, *gl_f[2], *gl_v[2], *sorted_v, *sorted_h, *d_mq;
  uint16_t* finv;
  uint8_t *fstate, *vflag, *vlose;
  unsigned long long* key1;
  float* ecost;
  void* tmp;
  IGN_TRY(f.take(&s.pos, U * 3));
  IGN_TRY(f.take(&s.Q, U * 10));
  IGN_TRY(f.take(&s.face, 3 * T));
  IGN_TRY(f.take(&s.vf, U * S_VCAP));
  IGN_TRY(f.take(&node_v, 3 * T));  // reused as face scan later
  IGN_TRY(f.take(&node_h, 3 * T));
  IGN_TRY(f.take(&s.flabel, T));
  IGN_TRY(f.take(&s.falive, T));
  IGN_TRY(f.take(&fstate, T));
  IGN_TRY(f.take(&s.valive, U));
  IGN_TRY(f.take(&s.vbound, U));
  IGN_TRY(f.take(&vflag, U));
  IGN_TRY(f.take(&vlose, U));
  IGN_TRY(f.take(&s.vn, U));
  IGN_TRY(f.take(&vscan, U));
  IGN_TRY(f.take(&vflag32, U));
  IGN_TRY(f.take(&key1, U));
  IGN_TRY(f.take(&d_target, K + 2));
  IGN_TRY(f.take(&d_tri_off, K + 2));
  IGN_TRY(f.take(&d_vert_off, K + 2));
  IGN_TRY(f.take(&d_new_tri_off, K + 2));
  IGN_TRY(f.take(&d_new_vert_off, K + 2));
  IGN_TRY(f.take(&d_order, K + 2));
  IGN_TRY(f.take(&flags, 64));
  IGN_TRY(f.take(&ecost, 3 * T));
  // alive lists of the global-memory class (ping-pong); the init scratch is free by then
  IGN_TRY(f.take(&gl_f[0], T));
  IGN_TRY(f.take(&gl_f[1], T));
  IGN_TRY(f.take(&gl_v[0], U));
  IGN_TRY(f.take(&gl_v[1], U));
  // labels migrating to a smaller size class: headers (one queue per destination class) and the
  // original-to-compacted face map
  IGN_TRY(f.take(&d_mq, (size_t)SL_MREC * K * (SL_NCLASS - 1)));
  IGN_TRY(f.take(&finv, T));
  IGN_TRY(f.take(&tmp, tmpb));
  IGN_TRY(f.take(&sorted_v, 3 * T));
  IGN_TRY(f.take(&sorted_h, 3 * T));
  s.tri_off = d_tri_off;

  std::vector<uint32_t> target(K + 2, 0);
  for (uint64_t l = 1; l <= K; l++)
    target[l] = (m->tri_off[l + 1] - m->tri_off[l]) / (uint32_t)reduction_factor;
  // dynamic shared memory of a CTA of each size class: the SM's 227 KB split between its CTAs, less
  // the static SlShared and the 1 KB the SM reserves per CTA
  const size_t sl_static = ((sizeof(SlShared) + 255) / 256) * 256 + 1024;
  size_t sl_dyn[SL_NCLASS];
  for (int c = 0; c < SL_NCLASS; c++) sl_dyn[c] = (232448 / (size_t)(1024 / SL_CLASS_THREADS[c]) - sl_static) & ~(size_t)255;
  // size class of every label: the smallest whose shared-memory budget holds the label (labels that fit
  // no class run in the 1024-thread class on global memory)
  std::vector<uint32_t> lcls(K + 2, 0);
  uint32_t ccount[SL_NCLASS] = {0, 0, 0};
  for (uint64_t l = 1; l <= K; l++) {
    const uint32_t tl = m->tri_off[l + 1] - m->tri_off[l], ul = m->vert_off[l + 1] - m->vert_off[l];
    int c = SL_NCLASS - 1;
    while (c > 0 && !sl_fits_smem(tl, ul, SL_CLASS_THREADS[c], sl_dyn[c])) c--;
    lcls[l] = (uint32_t)c;
    ccount[c]++;
  }
  // work order of the label kernel: class by class, largest labels first within a class (the tail of
  // each launch is made of its small labels)
  std::vector<uint32_t> order(K);
  for (uint64_t l = 0; l < K; l++) order[l] = (uint32_t)(l + 1);
  std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) {
    const uint32_t ta = m->tri_off[a + 1] - m->tri_off[a], tb = m->tri_off[b + 1] - m->tri_off[b];
    if (lcls[a] != lcls[b]) return lcls[a] < lcls[b];
    return ta != tb ? ta > tb : a < b;
  });
  IGN_TRY(small_h2d(ctx, d_target, target.data(), (K + 2) * 4));
  IGN_TRY(small_h2d(ctx, d_tri_off, m->tri_off.data(), (K + 2) * 4));
  IGN_TRY(small_h2d(ctx, d_vert_off, m->vert_off.data(), (K + 2) * 4));
  IGN_TRY(small_h2d(ctx, d_order, order.data(), K * 4));
  IGN_LAUNCH(ctx, k_simp_init_verts, blocks_for(U, 256), 256, 0, m->d_uniq_vkeys, U, (double)resolution[0],
             (double)resolution[1], (double)resolution[2], s.pos, s.valive, s.vbound, s.vn);
  IGN_LAUNCH(ctx, k_simp_init_faces, blocks_for(T, 256), 256, 0, m->d_faces, d_tri_off, d_vert_off, (uint32_t)K, T,
             s.face, s.flabel, s.falive, node_v, node_h);
  {
    int bits = 1;
    while (bits < 32 && (1ull << bits) < U) bits++;
    size_t tb = tmpb;
    IGN_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tb, node_v, sorted_v, node_h, sorted_h, (int)(3 * T), 0, bits,
                                             ctx->stream));
    ctx->launches += 3;
  }
  IGN_CUDA(cudaMemsetAsync(flags, 0, 32 * 4, ctx->stream));
  IGN_LAUNCH(ctx, k_simp_link, blocks_for(3 * T, 256), 256, 0, sorted_v, sorted_h, (uint64_t)(3 * T), s.vf, s.vn,
             flags + 12);
  IGN_LAUNCH(ctx, k_simp_quadrics, blocks_for(U, 128), 128, 0, s);
  IGN_LAUNCH(ctx, k_simp_boundary, blocks_for(3 * T, 256), 256, 0, s);
  const double max_err2 = (double)max_error * (double)max_error;
  IGN_LAUNCH(ctx, k_simp_ecost, blocks_for(T, 256), 256, 0, s, max_err2, ecost, fstate, flags + 26);

  // ---- all rounds of every label: one launch per size class, one CTA per label.  The kernel is
  // latency and barrier bound, so labels that fit half (a quarter) of an SM's shared memory run two
  // (four) CTAs to an SM, which overlap each other's stalls; larger labels keep the whole SM.
  IGN_CUDA(cudaFuncSetAttribute(k_simp_labels, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sl_dyn[0]));
  IGN_CUDA(cudaFuncSetAttribute(k_simp_resume, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sl_dyn[1]));
  SlArgs A;
  A.pos = s.pos; A.Q = s.Q; A.face = s.face; A.falive = s.falive; A.valive = s.valive; A.vbound = s.vbound;
  A.ecost = ecost; A.key1 = key1; A.fstate = fstate; A.vflag = vflag; A.vlose = vlose; A.finv = finv;
  A.flist = gl_f[0]; A.flist2 = gl_f[1]; A.vlist = gl_v[0]; A.vlist2 = gl_v[1];
  A.tri_off = d_tri_off; A.vert_off = d_vert_off; A.target = d_target;
  A.counters = flags;
  A.max_err2 = max_err2;
  A.max_rounds = 400;
  // IGN_SIMP_GMEM=1 (test knob): run every label on the global-memory arrays, the path of
  // labels that do not fit shared memory (only the winners' ring lists stay in smem)
  A.trace = nullptr;
  A.lrec = nullptr;
  if (getenv("IGN_SIMP_TRACE") != nullptr) {
    IGN_TRY(f.take(&A.trace, SL_HIST + SL_NCLASS * SL_HCLS));
    IGN_TRY(f.take(&A.lrec, (size_t)K * SL_LREC + 16));
    IGN_CUDA(cudaMemsetAsync(A.trace, 0, (SL_HIST + SL_NCLASS * SL_HCLS) * 4, ctx->stream));
    IGN_CUDA(cudaMemsetAsync(A.lrec, 0, ((size_t)K * SL_LREC + 16) * 4, ctx->stream));
  }
  const char* force_gmem = getenv("IGN_SIMP_GMEM");
  const bool gmem_only = force_gmem && force_gmem[0] == '1';
  // IGN_SIMP_WCAP=n (test knob): at most n winners per selection pass, so that rounds take several passes
  const char* wcap_env = getenv("IGN_SIMP_WCAP");
  A.wcap_max = wcap_env && atoi(wcap_env) > 0 ? (uint32_t)atoi(wcap_env) : 0xFFFFFFFFu;
  // IGN_SIMP_GROUP=16|32 (test knob): the narrowest lane group E2 gives a winner, so that the wider sweeps
  // take the winners with small rings too
  const char* group_env = getenv("IGN_SIMP_GROUP");
  const int group = group_env ? atoi(group_env) : 0;
  A.group_min = group == 16 || group == 32 ? (uint32_t)group : 8u;
  {
    const int slot = prof_begin(ctx, IGN_PROF_SIMP);
    // default: one CTA per label (SMs are handed back to the block scheduler after every label, so
    // higher-priority streams get them quickly); IGN_SIMP_PERSIST=1: one CTA per SM slot loops over labels
    const char* pe = getenv("IGN_SIMP_PERSIST");
    A.persist = (pe && pe[0] == '1') ? 1 : 0;
    // The classes run side by side on streams forked from the task's stream, launched largest class
    // first: the block scheduler dispatches the CTAs of earlier launches first, so the smaller classes
    // fill the SMs that the end of a larger class leaves idle instead of waiting for its last label.
    // (Streams and events are released by the runtime once their work is done.)
    //
    // A shared-memory label whose alive faces and vertices come to fit the next smaller class migrates
    // there (SlArgs::mq_next).  After the fresh launches, a resume launch of the 512-thread class takes the
    // labels that left the 1024-thread class once that launch is over, and one of the 256-thread class
    // those that left the 512-thread class once both of its launches are over: stream and event order
    // only, no CTA waits for another.
    // resume[c]: most labels that can migrate into class c (the grid of its resume launch)
    uint32_t resume[SL_NCLASS] = {0, 0, 0};
    if (!gmem_only)
      for (int c = 1; c < SL_NCLASS; c++) resume[c] = resume[c - 1] + ccount[c - 1];
    int prio = 0;
    IGN_CUDA(cudaStreamGetPriority(ctx->stream, &prio));
    cudaStream_t cs[SL_NCLASS] = {ctx->stream, nullptr, nullptr};
    cudaEvent_t ev[SL_NCLASS] = {nullptr, nullptr, nullptr};  // [0] fork, [c] end of class c's launches
    cudaError_t err = cudaEventCreateWithFlags(&ev[0], cudaEventDisableTiming);
    if (err == cudaSuccess) err = cudaEventRecord(ev[0], ctx->stream);
    for (int c = 1; c < SL_NCLASS && err == cudaSuccess; c++) {
      if (ccount[c] == 0 && resume[c] == 0) continue;
      err = cudaStreamCreateWithPriority(&cs[c], cudaStreamNonBlocking, prio);
      if (err == cudaSuccess) err = cudaStreamWaitEvent(cs[c], ev[0], 0);
      if (err == cudaSuccess) err = cudaEventCreateWithFlags(&ev[c], cudaEventDisableTiming);
    }
    cudaEvent_t ev_full = nullptr;  // end of the 1024-thread class
    if (err == cudaSuccess && resume[1]) err = cudaEventCreateWithFlags(&ev_full, cudaEventDisableTiming);
    uint32_t base = 0;
    for (int c = 0; c < SL_NCLASS && err == cudaSuccess; c++) {  // largest class first
      const uint32_t n = ccount[c], nt = (uint32_t)SL_CLASS_THREADS[c];
      A.cls = (uint32_t)c;
      // 0: every label takes the global-memory path (only the cost queues and ring lists stay in smem)
      A.smem_bytes = gmem_only ? 0u : (uint32_t)sl_dyn[c];
      A.smem_next = c + 1 < SL_NCLASS ? (uint32_t)sl_dyn[c + 1] : 0u;
      A.mq_next = (c + 1 < SL_NCLASS && resume[c + 1]) ? d_mq + (size_t)SL_MREC * K * c : nullptr;
      A.mq = nullptr;
      const uint64_t slots = (uint64_t)ctx->sm_count * (1024 / nt);
      if (n) {
        A.order = d_order + base; A.K = n; A.base = base;
        const unsigned grid = A.persist ? (unsigned)(n < slots ? n : slots) : n;
        k_simp_labels<<<grid, nt, sl_dyn[c], cs[c]>>>(A);
        ctx->launches++;
        err = cudaGetLastError();
        base += n;
      }
      if (c == 0 && ev_full && err == cudaSuccess) err = cudaEventRecord(ev_full, cs[0]);
    }
    for (int c = 1; c < SL_NCLASS && err == cudaSuccess; c++) {
      if (resume[c]) {
        const uint32_t nt = (uint32_t)SL_CLASS_THREADS[c];
        err = cudaStreamWaitEvent(cs[c], c == 1 ? ev_full : ev[c - 1], 0);
        if (err != cudaSuccess) break;
        A.cls = (uint32_t)c;
        A.smem_bytes = (uint32_t)sl_dyn[c];
        A.smem_next = c + 1 < SL_NCLASS ? (uint32_t)sl_dyn[c + 1] : 0u;
        A.mq_next = (c + 1 < SL_NCLASS) ? d_mq + (size_t)SL_MREC * K * c : nullptr;
        A.mq = d_mq + (size_t)SL_MREC * K * (c - 1);
        const uint64_t slots = (uint64_t)ctx->sm_count * (1024 / nt);
        const unsigned grid = A.persist ? (unsigned)(resume[c] < slots ? resume[c] : slots) : resume[c];
        k_simp_resume<<<grid, nt, sl_dyn[c], cs[c]>>>(A);
        ctx->launches++;
        err = cudaGetLastError();
      }
      if (ev[c] && err == cudaSuccess) err = cudaEventRecord(ev[c], cs[c]);
    }
    for (int c = 1; c < SL_NCLASS && err == cudaSuccess; c++)
      if (ev[c]) err = cudaStreamWaitEvent(ctx->stream, ev[c], 0);
    if (ev_full) cudaEventDestroy(ev_full);
    for (int c = 0; c < SL_NCLASS; c++) {
      if (ev[c]) cudaEventDestroy(ev[c]);
      if (c > 0 && cs[c]) cudaStreamDestroy(cs[c]);
    }
    prof_end(ctx, slot);
    IGN_CUDA(err);
  }

  // ---- compaction
  uint32_t* fscan = node_v;   // 3T u32 >= T
  uint32_t* fflag = node_h;
  size_t tb = tmpb;
  IGN_LAUNCH(ctx, k_simp_flags_u32, blocks_for(U, 256), 256, 0, s.valive, U, vflag32);
  IGN_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tb, vflag32, vscan, (int)U, ctx->stream));
  IGN_LAUNCH(ctx, k_simp_flags_u32, blocks_for(T, 256), 256, 0, s.falive, T, fflag);
  tb = tmpb;
  IGN_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tb, fflag, fscan, (int)T, ctx->stream));
  ctx->launches += 4;
  uint32_t last[4], hflags[32];
  IGN_TRY(small_d2h(ctx, &last[0], vscan + (U - 1), 4));
  IGN_TRY(small_d2h(ctx, &last[1], vflag32 + (U - 1), 4));
  IGN_TRY(small_d2h(ctx, &last[2], fscan + (T - 1), 4));
  IGN_TRY(small_d2h(ctx, &last[3], fflag + (T - 1), 4));
  IGN_TRY(small_d2h(ctx, hflags, flags, sizeof(hflags)));
  IGN_TRY(small_sync(ctx));
  if (hflags[12] != 0) {
    set_error("simplify: a vertex has more than %d incident faces", S_VCAP);
    return IGN_ERR_UNSUPPORTED;
  }
  if (A.trace) {
    std::vector<uint32_t> tr(SL_HIST);
    IGN_CUDA(cudaMemcpy(tr.data(), A.trace, SL_HIST * 4, cudaMemcpyDeviceToHost));
    unsigned long long phs[SL_NPH];
    IGN_CUDA(cudaMemcpy(phs, A.trace + 1600, sizeof(phs), cudaMemcpyDeviceToHost));
    static const char* names[SL_NPH] = {"P1", "P2 keys", "P3 lose", "P4 select", "setup", "E1 rings", "E2a cost", "E2 validate+collapse+recost", "stop+compact"};
    unsigned long long tot = 0;
    for (int q = 0; q < SL_NPH; q++) tot += phs[q];
    for (int q = 0; q < SL_NPH; q++)
      fprintf(stderr, "phase %-27s %6.2f %%  %10.3f Mcycles\n", names[q], 100.0 * phs[q] / (tot ? tot : 1), phs[q] / 1e6);
    fprintf(stderr, "cost evaluations: %u initial (k_simp_ecost), %u after collapses (E2), %u half-edges without a cost in P2\n",
            hflags[26], hflags[27], hflags[28]);
    fprintf(stderr, "winners by E2 group width: %u of 8 lanes, %u of 16, %u of 32\n", hflags[29], hflags[30], hflags[31]);
    fprintf(stderr, "winners rejected by E2 flip tests: %u on the u side only, %u on the v side only, %u on both\n",
            tr[SL_TFLIP], tr[SL_TFLIP + 1], tr[SL_TFLIP + 2]);
    {
      // per-label records: where do the cycles go -- per round (fixed latency) or per face visit?
      std::vector<uint32_t> rec(SL_LREC * (size_t)K);
      IGN_CUDA(cudaMemcpy(rec.data(), A.lrec, rec.size() * 4, cudaMemcpyDeviceToHost));
      static const uint32_t edges[] = {0, 500, 1000, 2000, 3000, 4000, 6000, 8000, 10000, 12000, 16000, 32000, 64000, 0xFFFFFFFFu};
      const int nedges = (int)(sizeof(edges) / sizeof(edges[0]));
      // kilocycles are wall cycles of the label's CTA, which shares its SM with the other CTAs of its class;
      // SM Mcycles divide each segment's wall cycles by the CTAs per SM of the class it ran in.  A label
      // that migrated sums all its segments and is listed under the class it started in.
      for (int c = 0; c < SL_NCLASS; c++) {
        int per_sm = 0;
        IGN_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_simp_labels, SL_CLASS_THREADS[c], sl_dyn[c]));
        fprintf(stderr, "size class %d: %4d threads, %6zu B dynamic shared memory, %d CTAs per SM, %u labels\n", c,
                SL_CLASS_THREADS[c], sl_dyn[c], per_sm, ccount[c]);
      }
      fprintf(stderr, "%7s %12s %7s %8s %10s %10s %10s %9s %9s  class(sm/hy/gl)\n", "threads", "faces<", "labels", "rounds", "Mcycles", "SM Mcyc", "Mvisits", "kwins", "cyc/round");
      double sr = 0, sv = 0, sc = 0, srr = 0, svv = 0, srv = 0, src = 0, svc = 0;
      uint64_t sm_total[SL_NCLASS] = {0, 0, 0};
      for (int szc = 0; szc < SL_NCLASS; szc++) {
        for (int b = 0; b + 1 < nedges; b++) {
          uint64_t n = 0, rounds = 0, kc = 0, ksm = 0, vis = 0, wins = 0, cls[4] = {0, 0, 0, 0};
          for (uint64_t i = 0; i < K; i++) {
            const uint32_t* q = &rec[SL_LREC * i];
            if (q[1] == 0 || (int)(q[5] >> 2) != szc || q[0] < edges[b] || q[0] >= edges[b + 1]) continue;
            n++; rounds += q[1]; kc += q[2]; ksm += q[6]; vis += q[3]; wins += q[4]; cls[q[5] & 3]++;
            const double R = q[1], V = q[3], C = q[2] * 1024.0;
            sr += R; sv += V; sc += C; srr += R * R; svv += V * V; srv += R * V; src += R * C; svc += V * C;
          }
          sm_total[szc] += ksm;
          if (n) fprintf(stderr, "%7d %12u %7llu %8.1f %10.2f %10.2f %10.3f %9.1f %9.0f  %llu/%llu/%llu\n", SL_CLASS_THREADS[szc], edges[b + 1],
                         (unsigned long long)n, (double)rounds / n, kc * 1024.0 / 1e6, ksm * 1024.0 / 1e6, vis / 1e6, wins / 1e3,
                         rounds ? kc * 1024.0 / rounds : 0.0, (unsigned long long)cls[1], (unsigned long long)cls[2],
                         (unsigned long long)cls[3]);
        }
      }
      fprintf(stderr, "SM Mcycles by starting class: %.0f + %.0f + %.0f = %.0f; labels resumed in the 512- / 256-thread class: %u / %u\n",
              sm_total[0] * 1024.0 / 1e6, sm_total[1] * 1024.0 / 1e6, sm_total[2] * 1024.0 / 1e6,
              (sm_total[0] + sm_total[1] + sm_total[2]) * 1024.0 / 1e6, hflags[17], hflags[18]);
      // per class the label-rounds ran in: selection passes per round, winners per round (before capping,
      // bins of 16), ring length per winner side (the last bin of each: more)
      std::vector<uint32_t> hist(SL_NCLASS * SL_HCLS);
      IGN_CUDA(cudaMemcpy(hist.data(), A.trace + SL_HIST, hist.size() * 4, cudaMemcpyDeviceToHost));
      for (int c = 0; c < SL_NCLASS; c++) {
        const uint32_t* h = &hist[SL_HCLS * c];
        fprintf(stderr, "class %d passes/round (1..%d+):", SL_CLASS_THREADS[c], SL_HP);
        for (int b = 0; b < SL_HP; b++) fprintf(stderr, " %u", h[b]);
        fprintf(stderr, "\nclass %d winners/round (bins of 16, last %d+):", SL_CLASS_THREADS[c], 16 * (SL_HW - 1));
        for (int b = 0; b < SL_HW; b++) fprintf(stderr, " %u", h[SL_HP + b]);
        fprintf(stderr, "\nclass %d ring length per winner side (0..%d, more):", SL_CLASS_THREADS[c], S_MAXV);
        for (int b = 0; b < SL_HR; b++) fprintf(stderr, " %u", h[SL_HP + SL_HW + b]);
        fprintf(stderr, "\n");
      }
      // least squares cycles = a * rounds + b * visits (no intercept)
      const double det = srr * svv - srv * srv;
      if (det != 0) fprintf(stderr, "fit: cycles ~= %.0f * rounds + %.2f * face visits   (totals: %.0f rounds, %.3g visits, %.3g cycles)\n",
                            (src * svv - svc * srv) / det, (svc * srr - src * srv) / det, sr, sv, sc);
    }
    for (int r = 0; r < 400 && getenv("IGN_SIMP_TRACE_ROUNDS") && (tr[4 * r + 2] || tr[4 * r + 3]); r++)
      fprintf(stderr, "gpu round %d progress %u collapses %u alive %u list %u\n", r, tr[4 * r], tr[4 * r + 1], tr[4 * r + 2], tr[4 * r + 3]);
  }
  // the SlArgs::counters words that ign_mesh_simplify_counters returns, in its order
  static const int word[17] = {1, 2, 3, 8, 9, 10, 16, 17, 18, 24, 25, 26, 27, 28, 29, 30, 31};
  for (int i = 0; i < 17; i++) m->simp_counters[i] = hflags[word[i]];
  const uint32_t U2 = last[0] + last[1], T2 = last[2] + last[3];
  IGN_LAUNCH(ctx, k_simp_new_offsets, blocks_for(K + 2, 256), 256, 0, d_vert_off, vscan, (uint32_t)(K + 2), U, U2,
                   d_new_vert_off);
  IGN_LAUNCH(ctx, k_simp_new_offsets, blocks_for(K + 2, 256), 256, 0, d_tri_off, fscan, (uint32_t)(K + 2), T, T2,
                   d_new_tri_off);
  // results overwrite the mesher's buffers (inputs were copied into the arena; the vertex buffer holds 12 B / vertex)
  float* pos_f = (float*)m->d_uniq_vkeys;
  IGN_LAUNCH(ctx, k_simp_compact_verts, blocks_for(U, 256), 256, 0, s, vscan, pos_f);
  IGN_LAUNCH(ctx, k_simp_compact_faces, blocks_for(T, 256), 256, 0, s, vscan, fscan, d_new_vert_off, m->d_faces);
  IGN_TRY(small_d2h(ctx, m->tri_off.data(), d_new_tri_off, (K + 2) * 4));
  IGN_TRY(small_d2h(ctx, m->vert_off.data(), d_new_vert_off, (K + 2) * 4));
  IGN_TRY(small_sync(ctx));
  m->U = U2;
  m->T = T2;
  m->d_pos_f = pos_f;
  m->simplified = true;
  m->present.clear();
  for (uint64_t l = 1; l <= K; l++)
    if (m->tri_off[l + 1] > m->tri_off[l]) m->present.push_back(m->ids[l - 1]);
  return IGN_OK;
}

extern "C" int ign_mesh_simplify_counters(ign_mesher* m, uint32_t counters[17]) {
  IGN_REQUIRE(m && counters, IGN_ERR_INVALID, "null argument");
  IGN_REQUIRE(m->simplified, IGN_ERR_INVALID, "mesher is not simplified");
  memcpy(counters, m->simp_counters, sizeof(m->simp_counters));
  return IGN_OK;
}
