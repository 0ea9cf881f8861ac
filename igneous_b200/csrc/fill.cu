// fill.cu -- hole filling for MeshTask(fill_holes=N) and the multilabel dilation before it
//
// Replaces fastmorph.dilate(data, mode=multilabel, background_only=True) and
// fastmorph.fill_holes_v2(data, fix_borders, merge_threshold) as called from
// igneous/tasks/mesh/mesh.py:211-228.  fastmorph is not available offline, so the rule
// below is this library's own (DESIGN.md "Hole filling"); it is integer-only and
// tests/fillref.py restates it in numpy, oracle_fill/fill_oracle.c serially in C.
//
//   dilate   k_fill_dilate: 32x4x4 output tiles staged with their 1-voxel halo in shared
//            memory; a 0 voxel with a non-zero 26-neighbour takes the most frequent non-zero
//            neighbour label, ties to the smaller label.  One Jacobi pass.
//   fill     per pass (each face plane for fix_borders, then the volume):
//     key      k_fill_key: value + 1, so that 0 is an ordinary label for the CCL (ccl.cu,
//              unchanged): components are maximal 6-connected sets of equal value, 0 included,
//              numbered 1..N by first voxel in Fortran order.
//     labels   k_fill_comp_label: value of every component (written at x-run starts).
//     contacts k_fill_contacts: a count pass and an emit pass over the voxels; every +x/+y/+z
//              pair of different components emits its (min, max) key and every voxel face on
//              the box surface emits (0, c); warp-aggregated appends.  Radix sort + run-length
//              encode turns the keys into the weighted contact graph (node 0 = outside).
//     solve    on the host after one readback (O(components + edges), as ign_ccl6_solve):
//              merge-threshold rounds, then an iterative DFS with Tarjan low-links gives each
//              region the non-zero separator nearest the outside (its filler).
//     apply    k_fill_apply: filled = table[component]; holes = input where filled differs.
//   The host solve makes ign_fill_holes_dev synchronous: each pass waits on the stream four times
//   (2^64-1 check + component count, contact count, run count, table upload); its buffers are
//   taken from the context's scratch arena.
//   A face plane is gathered into an (a, b, 1) volume (6-connectivity there is 4-connectivity),
//   solved with only its in-plane edges as the outside, and scattered back.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_run_length_encode.cuh>

#include <algorithm>
#include <set>
#include <unordered_map>
#include <vector>

#include "common.cuh"

namespace ign {

// ------------------------------------------------------------------ dilation
constexpr int DL_BX = 32, DL_BY = 4, DL_BZ = 4;
constexpr int DL_PX = DL_BX + 2, DL_PY = DL_BY + 2, DL_PZ = DL_BZ + 2;

template <typename T>
__global__ void __launch_bounds__(DL_BX * DL_BY * DL_BZ)
    k_fill_dilate(const T* __restrict__ in, uint32_t sx, uint32_t sy, uint32_t sz, uint32_t ntx, uint32_t nty,
                  T* __restrict__ out) {
  __shared__ T tile[DL_PZ][DL_PY][DL_PX];
  const uint32_t tid = threadIdx.x;
  const uint32_t bx = blockIdx.x % ntx, by = (blockIdx.x / ntx) % nty, bz = blockIdx.x / ntx / nty;
  const int64_t x0 = (int64_t)bx * DL_BX - 1, y0 = (int64_t)by * DL_BY - 1, z0 = (int64_t)bz * DL_BZ - 1;
  // out-of-box halo reads as 0, which the rule ignores: only in-box neighbours count
  for (uint32_t e = tid; e < (uint32_t)(DL_PX * DL_PY * DL_PZ); e += blockDim.x) {
    const uint32_t ix = e % DL_PX, iy = (e / DL_PX) % DL_PY, iz = e / (DL_PX * DL_PY);
    const int64_t gx = x0 + ix, gy = y0 + iy, gz = z0 + iz;
    const bool ok = gx >= 0 && gy >= 0 && gz >= 0 && gx < sx && gy < sy && gz < sz;
    tile[iz][iy][ix] = ok ? in[((uint64_t)gz * sy + (uint64_t)gy) * sx + (uint64_t)gx] : (T)0;
  }
  __syncthreads();
  const uint32_t lx = tid % DL_BX, ly = (tid / DL_BX) % DL_BY, lz = tid / (DL_BX * DL_BY);
  const uint64_t gx = (uint64_t)bx * DL_BX + lx, gy = (uint64_t)by * DL_BY + ly, gz = (uint64_t)bz * DL_BZ + lz;
  if (gx >= sx || gy >= sy || gz >= sz) return;
  const T c = tile[lz + 1][ly + 1][lx + 1];
  T best = c;
  if (c == (T)0) {
    T nb[26];
    int k = 0;
#pragma unroll
    for (int dz = 0; dz < 3; dz++)
#pragma unroll
      for (int dy = 0; dy < 3; dy++)
#pragma unroll
        for (int dx = 0; dx < 3; dx++)
          if (dx != 1 || dy != 1 || dz != 1) nb[k++] = tile[lz + dz][ly + dy][lx + dx];
    int bestc = 0;
#pragma unroll
    for (int i = 0; i < 26; i++) {
      const T v = nb[i];
      int cnt = 0;
#pragma unroll
      for (int j = 0; j < 26; j++) cnt += (nb[j] == v);
      if (v != (T)0 && (cnt > bestc || (cnt == bestc && v < best))) {
        best = v;
        bestc = cnt;
      }
    }
  }
  out[(gz * sy + gy) * sx + gx] = best;
}

template <typename T>
static int dilate_typed(ign_ctx* ctx, const void* in, uint64_t sx, uint64_t sy, uint64_t sz, void* out) {
  const uint64_t nty = (sy + DL_BY - 1) / DL_BY, ntz = (sz + DL_BZ - 1) / DL_BZ, ntx = (sx + DL_BX - 1) / DL_BX;
  IGN_REQUIRE(ntx * nty * ntz < 0x7FFFFFFFull, IGN_ERR_OVERFLOW, "dilate: volume too large");
  IGN_LAUNCH(ctx, k_fill_dilate<T>, (unsigned)(ntx * nty * ntz), DL_BX * DL_BY * DL_BZ, 0, (const T*)in, (uint32_t)sx,
             (uint32_t)sy, (uint32_t)sz, (uint32_t)ntx, (uint32_t)nty, (T*)out);
  return IGN_OK;
}

// ------------------------------------------------------------------ fill passes
template <typename T, typename K>
__global__ void __launch_bounds__(256) k_fill_key(const T* __restrict__ in, uint64_t n, K* __restrict__ key,
                                                  uint32_t* __restrict__ flag) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const T v = in[i];
  if (sizeof(T) == 8 && v == (T)~0ull) *flag = 1;  // no key for 2^64-1
  key[i] = (K)v + 1;
}

template <typename T>
__global__ void __launch_bounds__(256) k_fill_comp_label(const uint32_t* __restrict__ comp, const T* __restrict__ in,
                                                         uint64_t n, uint64_t sx, uint64_t* __restrict__ clabel) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const uint32_t c = comp[i];
  if (i % sx == 0 || comp[i - 1] != c) clabel[c] = (uint64_t)in[i];  // equal values within a component
}

// keys of voxel i: up to 3 neighbour contacts and 6 box faces
__device__ __forceinline__ int fill_voxel_keys(const uint32_t* __restrict__ comp, uint64_t i, uint64_t sx, uint64_t sy,
                                               uint64_t sz, uint32_t axes, uint64_t* k) {
  const uint64_t x = i % sx, r = i / sx, y = r % sy, z = r / sy;
  const uint32_t c = comp[i];
  int m = 0;
  auto pair = [&](uint32_t d) {
    if (d != c) k[m++] = c < d ? ((uint64_t)c << 32 | d) : ((uint64_t)d << 32 | c);
  };
  if (x + 1 < sx) pair(comp[i + 1]);
  if (y + 1 < sy) pair(comp[i + sx]);
  if (z + 1 < sz) pair(comp[i + sx * sy]);
  const uint64_t co[3] = {x, y, z}, ext[3] = {sx, sy, sz};
#pragma unroll
  for (int a = 0; a < 3; a++) {
    if (!(axes >> a & 1u)) continue;
    if (co[a] == 0) k[m++] = c;            // (outside, c)
    if (co[a] + 1 == ext[a]) k[m++] = c;   // both faces when the extent is 1
  }
  return m;
}

template <bool EMIT>
__global__ void __launch_bounds__(256)
    k_fill_contacts(const uint32_t* __restrict__ comp, uint64_t sx, uint64_t sy, uint64_t sz, uint32_t axes,
                    unsigned long long* __restrict__ counter, uint64_t* __restrict__ keys) {
  const uint64_t n = sx * sy * sz;
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  const uint32_t lane = threadIdx.x & 31u;
  uint64_t k[9];
  const int m = i < n ? fill_voxel_keys(comp, i, sx, sy, sz, axes, k) : 0;
  // warp-aggregated append: inclusive scan of m, one atomic per warp
  int incl = m;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const int t = __shfl_up_sync(0xFFFFFFFFu, incl, d);
    if ((int)lane >= d) incl += t;
  }
  const int total = __shfl_sync(0xFFFFFFFFu, incl, 31);
  unsigned long long base = 0;
  if (lane == 31 && total) base = atomicAdd(counter, (unsigned long long)total);
  if (!EMIT) return;
  base = __shfl_sync(0xFFFFFFFFu, base, 31);
  const uint64_t at = base + (uint64_t)(incl - m);
  for (int j = 0; j < m; j++) keys[at + j] = k[j];
}

template <typename T>
__global__ void __launch_bounds__(256)
    k_fill_apply(const uint32_t* __restrict__ comp, const T* __restrict__ lut, uint64_t n, const T* __restrict__ x0,
                 T* __restrict__ filled, T* __restrict__ holes) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= n) return;
  const T f = lut[comp[i]];
  filled[i] = f;
  if (holes) {
    const T v = x0[i];
    holes[i] = (f != v && v != (T)0) ? v : (T)0;
  }
}

// plane `idx` normal to `axis`, as an (a, b, 1) volume: a, b = the other two axes in x, y, z order
template <typename T, bool GATHER>
__global__ void __launch_bounds__(256) k_fill_plane(T* __restrict__ vol, uint64_t sx, uint64_t sy, uint64_t sz, int axis,
                                                    uint64_t idx, T* __restrict__ plane) {
  const uint64_t na = axis == 0 ? sy : sx, nb = axis == 2 ? sy : sz;
  const uint64_t j = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (j >= na * nb) return;
  const uint64_t ia = j % na, ib = j / na;
  const uint64_t x = axis == 0 ? idx : ia, y = axis == 0 ? ia : (axis == 1 ? idx : ib), z = axis == 2 ? idx : ib;
  const uint64_t v = (z * sy + y) * sx + x;
  if (GATHER) plane[j] = vol[v];
  else vol[v] = plane[j];
}

// ------------------------------------------------------------------ host solve
// Contact graph of one pass -> for every component the label it takes in `filled`.
//   keys/cnt: unique (min, max) component pairs with their face counts; min 0 = outside.
//   clabel[c]: value of component c (1..N).  p = 100 - merge_threshold_pct.
static void fill_solve(uint32_t N, const uint64_t* keys, const uint32_t* cnt, uint64_t nk, int p,
                       const uint64_t* clabel, std::vector<uint64_t>& out) {
  std::vector<uint32_t> rep(N + 1);
  for (uint32_t i = 0; i <= N; i++) rep[i] = i;
  std::vector<uint64_t> wO(N + 1, 0), A(N + 1, 0);
  std::vector<std::pair<uint32_t, uint32_t>> edges;  // region graph for the enclosure step (0 = outside)
  for (uint64_t e = 0; e < nk; e++) {
    const uint32_t a = (uint32_t)(keys[e] >> 32), b = (uint32_t)keys[e];
    A[b] += cnt[e];
    if (a == 0) wO[b] += cnt[e];
    else A[a] += cnt[e];
  }
  if (p > 0) {
    // ---- merge threshold: regions absorbed into their dominant neighbour (DESIGN.md "Hole filling")
    std::vector<std::unordered_map<uint32_t, uint64_t>> adj(N + 1);
    for (uint64_t e = 0; e < nk; e++) {
      const uint32_t a = (uint32_t)(keys[e] >> 32), b = (uint32_t)keys[e];
      if (a == 0) continue;
      adj[a][b] += cnt[e];
      adj[b][a] += cnt[e];
    }
    std::vector<uint32_t> tgt(N + 1, 0);  // candidate -> target root, 0 = not a candidate
    std::set<uint32_t> cands;
    auto eval = [&](uint32_t r) {
      tgt[r] = 0;
      if (wO[r] == 0 && !adj[r].empty()) {
        uint32_t best = 0;
        uint64_t bw = 0;
        for (const auto& kv : adj[r])
          if (kv.second > bw || (kv.second == bw && kv.first < best)) {
            best = kv.first;
            bw = kv.second;
          }
        if (100 * bw >= (uint64_t)(100 - p) * A[r]) tgt[r] = best;
      }
      if (tgt[r]) cands.insert(r);
      else cands.erase(r);
    };
    for (uint32_t r = 1; r <= N; r++) eval(r);
    std::vector<std::pair<uint32_t, uint32_t>> absorb;
    std::vector<uint32_t> dirty;
    while (!cands.empty()) {
      absorb.clear();
      for (uint32_t r : cands) {
        const uint32_t T = tgt[r];
        const bool loses = A[r] < A[T] || (A[r] == A[T] && r > T);
        if (tgt[T] == 0 || (tgt[T] == r && loses)) absorb.emplace_back(r, T);
      }
      if (absorb.empty()) {  // a longer cycle (cannot arise with symmetric weights; kept for progress)
        uint32_t pick = 0;
        for (uint32_t r : cands)
          if (pick == 0 || A[r] < A[pick] || (A[r] == A[pick] && r > pick)) pick = r;
        absorb.emplace_back(pick, tgt[pick]);
      }
      dirty.clear();
      for (const auto& rt : absorb) {  // targets are never absorbed in the same round: order-free
        const uint32_t r = rt.first, T = rt.second;
        const uint64_t wrt = adj[r][T];
        for (const auto& kv : adj[r]) {
          const uint32_t U = kv.first;
          if (U == T) continue;
          adj[T][U] += kv.second;
          adj[U][T] += kv.second;
          adj[U].erase(r);
          dirty.push_back(U);
        }
        adj[T].erase(r);
        A[T] = A[T] + A[r] - 2 * wrt;
        wO[T] += wO[r];
        rep[r] = T;
        adj[r].clear();
        tgt[r] = 0;
        cands.erase(r);
        dirty.push_back(T);
      }
      for (uint32_t d : dirty)
        if (rep[d] == d) eval(d);
    }
    for (uint32_t r = 1; r <= N; r++)
      if (rep[r] == r) {
        if (wO[r]) edges.emplace_back(0, r);
        for (const auto& kv : adj[r])
          if (r < kv.first) edges.emplace_back(r, kv.first);
      }
    for (uint32_t c = 1; c <= N; c++) {  // region of every component (absorbed roots point at their target)
      uint32_t r = c;
      while (rep[r] != r) r = rep[r];
      rep[c] = r;
    }
  } else {
    edges.reserve(nk);
    for (uint64_t e = 0; e < nk; e++) edges.emplace_back((uint32_t)(keys[e] >> 32), (uint32_t)keys[e]);
  }
  // ---- enclosure: DFS from the outside, Tarjan low-links; a child c of v is cut off from the
  // outside by v exactly when low(c) >= disc(v), and inherits every separator of v
  std::vector<uint32_t> deg(N + 2, 0);
  for (const auto& e : edges) {
    deg[e.first + 1]++;
    deg[e.second + 1]++;
  }
  for (uint32_t i = 1; i <= N + 1; i++) deg[i] += deg[i - 1];
  std::vector<uint32_t> nbr(deg[N + 1]), fillp(deg.begin(), deg.end() - 1);
  for (const auto& e : edges) {
    nbr[fillp[e.first]++] = e.second;
    nbr[fillp[e.second]++] = e.first;
  }
  const uint32_t UNSEEN = 0xFFFFFFFFu;
  std::vector<uint32_t> disc(N + 1, UNSEEN), low(N + 1, 0), parent(N + 1, UNSEEN), order, it(N + 1, 0);
  std::vector<uint32_t> stack;
  uint32_t t = 0;
  disc[0] = low[0] = t++;
  stack.push_back(0);
  it[0] = deg[0];
  while (!stack.empty()) {
    const uint32_t v = stack.back();
    if (it[v] < deg[v + 1]) {
      const uint32_t u = nbr[it[v]++];
      if (disc[u] == UNSEEN) {
        parent[u] = v;
        disc[u] = low[u] = t++;
        it[u] = deg[u];
        order.push_back(u);
        stack.push_back(u);
      } else if (u != parent[v]) {
        low[v] = std::min(low[v], disc[u]);
      }
    } else {
      stack.pop_back();
      if (v != 0) low[parent[v]] = std::min(low[parent[v]], low[v]);
    }
  }
  std::vector<uint32_t> filler(N + 1, 0);  // region -> its filler region, 0 = none
  for (uint32_t c : order) {
    const uint32_t v = parent[c];
    if (v == 0) continue;
    filler[c] = filler[v] ? filler[v] : ((low[c] >= disc[v] && clabel[v] != 0) ? v : 0);
  }
  out.assign(N + 1, 0);
  for (uint32_t c = 1; c <= N; c++) {
    const uint32_t r = rep[c];
    out[c] = filler[r] ? clabel[filler[r]] : (clabel[r] != 0 ? clabel[r] : clabel[c]);
  }
}

template <typename T>
struct KeyOf { using type = typename std::conditional<(sizeof(T) <= 2), uint32_t, uint64_t>::type; };

// One pass of steps 2-5 on `cur` (device, s = sx*sy*sz voxels; axes = bit mask of the axes whose
// box faces are the outside).  Writes filled (may alias cur) and, when holes != null, holes against x0.
template <typename T>
static int fill_pass(ign_ctx* ctx, const T* cur, uint64_t sx, uint64_t sy, uint64_t sz, uint32_t axes, int p,
                     const T* x0, T* filled, T* holes) {
  using K = typename KeyOf<T>::type;
  const uint64_t n = sx * sy * sz;
  ScratchFrame f(ctx);
  K* key;
  uint32_t *comp, *flag;
  IGN_TRY(f.take(&key, n));
  IGN_TRY(f.take(&comp, n));
  IGN_TRY(f.take(&flag, 4));
  IGN_CUDA(cudaMemsetAsync(flag, 0, 16, ctx->stream));
  IGN_LAUNCH(ctx, (k_fill_key<T, K>), blocks_for(n, 256), 256, 0, cur, n, key, flag);
  uint64_t N = 0;
  IGN_TRY(ign_ccl6_dev(ctx, key, sizeof(K) == 4 ? IGN_U32 : IGN_U64, sx, sy, sz, comp, IGN_U32, &N));
  unsigned long long* hcnt = (unsigned long long*)ctx->pinned;
  IGN_CUDA(cudaMemcpyAsync(hcnt, flag, 4, cudaMemcpyDeviceToHost, ctx->stream));
  IGN_CUDA(cudaStreamSynchronize(ctx->stream));
  IGN_REQUIRE(((uint32_t*)hcnt)[0] == 0, IGN_ERR_UNSUPPORTED, "fill_holes: label 2^64-1 is not supported");
  uint64_t* clabel;
  unsigned long long* counter;
  IGN_TRY(f.take(&clabel, N + 1));
  IGN_TRY(f.take(&counter, 1));
  IGN_CUDA(cudaMemsetAsync(clabel, 0, 8, ctx->stream));
  IGN_LAUNCH(ctx, k_fill_comp_label<T>, blocks_for(n, 256), 256, 0, comp, cur, n, sx, clabel);
  IGN_CUDA(cudaMemsetAsync(counter, 0, 8, ctx->stream));
  IGN_LAUNCH(ctx, k_fill_contacts<false>, blocks_for(n, 256), 256, 0, comp, sx, sy, sz, axes, counter,
             (uint64_t*)nullptr);
  IGN_CUDA(cudaMemcpyAsync(hcnt, counter, 8, cudaMemcpyDeviceToHost, ctx->stream));
  IGN_CUDA(cudaStreamSynchronize(ctx->stream));
  const uint64_t M = hcnt[0];
  IGN_REQUIRE(M > 0 && M < 0x7FFFFFFFull, IGN_ERR_OVERFLOW, "fill_holes: %llu contacts", (unsigned long long)M);
  uint64_t *keys, *sorted, *uniq;
  uint32_t* counts;
  int* nruns;
  void* tmp;
  IGN_TRY(f.take(&keys, M));
  IGN_TRY(f.take(&sorted, M));
  IGN_TRY(f.take(&uniq, M));
  IGN_TRY(f.take(&counts, M));
  IGN_TRY(f.take(&nruns, 2));
  IGN_CUDA(cudaMemsetAsync(counter, 0, 8, ctx->stream));
  IGN_LAUNCH(ctx, k_fill_contacts<true>, blocks_for(n, 256), 256, 0, comp, sx, sy, sz, axes, counter, keys);
  int hi_bits = 1;
  while (hi_bits < 32 && (N >> hi_bits)) hi_bits++;
  const int end_bit = 32 + hi_bits;
  size_t sort_b = 0, rle_b = 0;
  cub::DeviceRadixSort::SortKeys(nullptr, sort_b, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int)M, 0, end_bit);
  cub::DeviceRunLengthEncode::Encode(nullptr, rle_b, (const uint64_t*)nullptr, (uint64_t*)nullptr, (uint32_t*)nullptr,
                                     (int*)nullptr, (int)M);
  IGN_TRY(f.take(&tmp, std::max(sort_b, rle_b)));
  IGN_CUDA(cub::DeviceRadixSort::SortKeys(tmp, sort_b, keys, sorted, (int)M, 0, end_bit, ctx->stream));
  IGN_CUDA(cub::DeviceRunLengthEncode::Encode(tmp, rle_b, sorted, uniq, counts, nruns, (int)M, ctx->stream));
  ctx->launches += 4;
  int* hruns = (int*)ctx->pinned;
  IGN_CUDA(cudaMemcpyAsync(hruns, nruns, 4, cudaMemcpyDeviceToHost, ctx->stream));
  IGN_CUDA(cudaStreamSynchronize(ctx->stream));
  const uint64_t nk = (uint64_t)hruns[0];
  std::vector<uint64_t> hkeys(nk), hlab(N + 1);
  std::vector<uint32_t> hcnts(nk);
  IGN_CUDA(cudaMemcpyAsync(hkeys.data(), uniq, nk * 8, cudaMemcpyDeviceToHost, ctx->stream));
  IGN_CUDA(cudaMemcpyAsync(hcnts.data(), counts, nk * 4, cudaMemcpyDeviceToHost, ctx->stream));
  IGN_CUDA(cudaMemcpyAsync(hlab.data(), clabel, (N + 1) * 8, cudaMemcpyDeviceToHost, ctx->stream));
  IGN_CUDA(cudaStreamSynchronize(ctx->stream));
  std::vector<uint64_t> table;
  fill_solve((uint32_t)N, hkeys.data(), hcnts.data(), nk, p, hlab.data(), table);
  std::vector<T> lut(N + 1);
  for (uint64_t c = 0; c <= N; c++) lut[c] = (T)table[c];
  T* dlut;
  IGN_TRY(f.take(&dlut, N + 1));
  IGN_CUDA(cudaMemcpyAsync(dlut, lut.data(), (N + 1) * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
  IGN_LAUNCH(ctx, k_fill_apply<T>, blocks_for(n, 256), 256, 0, comp, dlut, n, x0, filled, holes);
  // lut is a host vector: the copy must complete before it goes out of scope
  IGN_CUDA(cudaStreamSynchronize(ctx->stream));
  return IGN_OK;
}

template <typename T>
static int fill_typed(ign_ctx* ctx, const T* in, uint64_t sx, uint64_t sy, uint64_t sz, int fix_borders, int p,
                      T* filled, T* holes) {
  const uint64_t n = sx * sy * sz;
  if (fix_borders) {
    IGN_CUDA(cudaMemcpyAsync(filled, in, n * sizeof(T), cudaMemcpyDeviceToDevice, ctx->stream));
    const uint64_t ext[3] = {sx, sy, sz};
    ScratchFrame f(ctx);
    T* plane;
    IGN_TRY(f.take(&plane, std::max({sx * sy, sx * sz, sy * sz})));
    for (int axis = 0; axis < 3; axis++) {
      const uint64_t na = axis == 0 ? sy : sx, nb = axis == 2 ? sy : sz;
      for (int side = 0; side < 2; side++) {
        const uint64_t idx = side ? ext[axis] - 1 : 0;
        if (side && idx == 0) continue;  // extent 1: the plane was done already
        IGN_LAUNCH(ctx, (k_fill_plane<T, true>), blocks_for(na * nb, 256), 256, 0, filled, sx, sy, sz, axis, idx, plane);
        IGN_TRY(fill_pass<T>(ctx, plane, na, nb, 1, 3u, p, nullptr, plane, nullptr));
        IGN_LAUNCH(ctx, (k_fill_plane<T, false>), blocks_for(na * nb, 256), 256, 0, filled, sx, sy, sz, axis, idx, plane);
      }
    }
    return fill_pass<T>(ctx, filled, sx, sy, sz, 7u, p, in, filled, holes);
  }
  return fill_pass<T>(ctx, in, sx, sy, sz, 7u, p, in, filled, holes);
}

static int fill_check(uint64_t sx, uint64_t sy, uint64_t sz, int dtype, int pct) {
  IGN_REQUIRE(sx > 0 && sy > 0 && sz > 0, IGN_ERR_INVALID, "empty volume");
  IGN_REQUIRE(pct >= 0 && pct <= 100, IGN_ERR_INVALID, "merge_threshold_pct %d outside 0..100", pct);
  IGN_REQUIRE(dtype >= IGN_U8 && dtype <= IGN_U64, IGN_ERR_UNSUPPORTED, "fill_holes: unsupported dtype %d", dtype);
  return IGN_OK;
}

}  // namespace ign

using namespace ign;

extern "C" {

int ign_dilate_multilabel_dev(ign_ctx* ctx, const void* in, int dtype, uint64_t sx, uint64_t sy, uint64_t sz,
                              void* out) {
  IGN_TRY(activate(ctx));
  IGN_REQUIRE(in && out && in != out, IGN_ERR_INVALID, "null or aliased buffer");
  IGN_REQUIRE(sx > 0 && sy > 0 && sz > 0, IGN_ERR_INVALID, "empty volume");
  IGN_REQUIRE(sx < (1ull << 31) && sy < (1ull << 31) && sz < (1ull << 31), IGN_ERR_OVERFLOW, "extent too large");
  return dispatch_label(dtype, "dilate",
                        [&](auto v) { return dilate_typed<decltype(v)>(ctx, in, sx, sy, sz, out); });
}

int ign_fill_holes_dev(ign_ctx* ctx, const void* in, int dtype, uint64_t sx, uint64_t sy, uint64_t sz,
                       int fix_borders, int merge_threshold_pct, void* filled, void* holes) {
  IGN_TRY(activate(ctx));
  IGN_REQUIRE(in && filled && holes && in != filled && in != holes && filled != holes, IGN_ERR_INVALID,
              "null or aliased buffer");
  IGN_TRY(fill_check(sx, sy, sz, dtype, merge_threshold_pct));
  const int p = 100 - merge_threshold_pct;
  return dispatch_label(dtype, "fill_holes", [&](auto v) {
    using T = decltype(v);
    return fill_typed(ctx, (const T*)in, sx, sy, sz, fix_borders, p, (T*)filled, (T*)holes);
  });
}

// ---- host-buffer wrappers
int ign_dilate_multilabel(ign_ctx* ctx, const void* in, int dtype, uint64_t sx, uint64_t sy, uint64_t sz, void* out) {
  const uint64_t bytes = sx * sy * sz * dtype_size(dtype);
  return staged(ctx, {{in, nullptr, bytes}, {nullptr, out, bytes}},
                [&](void* const* d) { return ign_dilate_multilabel_dev(ctx, d[0], dtype, sx, sy, sz, d[1]); });
}

int ign_fill_holes(ign_ctx* ctx, const void* in, int dtype, uint64_t sx, uint64_t sy, uint64_t sz, int fix_borders,
                   int merge_threshold_pct, void* filled, void* holes) {
  IGN_TRY(fill_check(sx, sy, sz, dtype, merge_threshold_pct));
  const uint64_t bytes = sx * sy * sz * dtype_size(dtype);
  return staged(ctx, {{in, nullptr, bytes}, {nullptr, filled, bytes}, {nullptr, holes, bytes}}, [&](void* const* d) {
    return ign_fill_holes_dev(ctx, d[0], dtype, sx, sy, sz, fix_borders, merge_threshold_pct, d[1], d[2]);
  });
}

}  // extern "C"
