// edt.cu -- multi-label anisotropic Euclidean distance transform (the `edt` wheel that
// kimimaro.skeletonize reads its distance-to-boundary field from, igneous/tasks/skeleton.py:54,
// :312), sm_90a.  The rule is DESIGN.md §5d: edtsq[p] = 0 where label 0, else the least
// sum_i (a_i (p_i - q_i))^2 over voxels q of another label (and the one-voxel shell of label 0
// around the volume with black_border); +inf when there is none.
//
//   k_edt_x      pass 1, along x: one warp per row.  A forward sweep over 32-voxel chunks finds
//                the start of each voxel's run (max-scan of run starts) and parks the distance to
//                the voxel before it in `out`; a backward sweep finds the run's end (min-scan) and
//                writes a_x^2 * min(both)^2.  The row's second read mostly hits L2.
//   k_edt_line   passes 2 and 3, along y and z: one thread per line, lanes over consecutive x, so
//                every load and store of a warp is one coalesced row.  Along the line, each run
//                of one label gets its own lower envelope of parabolas f(q) + a^2 (p - q)^2
//                (Felzenszwalb-Huttenlocher) over its voxels of finite f; the voxels bounding
//                the run (and the shell with black_border) are zero-valued sites, applied in
//                closed form.  Nothing beyond a run boundary can be nearer than the boundary
//                voxel itself, so restricting the envelope to the run is exact.  A run is
//                evaluated as soon as it ends, so its stack (from a ScratchFrame, one slot of
//                n entries per line in flight) is read back while it is still in cache.
//
// The envelope's pop test is the division-free three-parabola test in double precision, and the
// evaluation walks the envelope by comparing values, not breakpoints: with integer anisotropy
// every value below 2^24 is computed exactly, and float32 rounding happens once per pass.
#include <math.h>

#include <algorithm>

#include "common.cuh"

namespace ign {

namespace {

constexpr int X_THREADS = 256;
constexpr int LN_THREADS = 128;
constexpr int LN_BATCH = 8;                        // line elements whose loads are issued together
constexpr uint64_t EDT_STACK_BYTES = 1ull << 30;   // envelope stacks of the lines of one launch
constexpr uint32_t FULL = 0xFFFFFFFFu;
constexpr uint32_t DINF = 0xFFFFFFFFu;  // pass 1: no run boundary on that side

template <typename T>
__device__ __forceinline__ T shfl_up_t(T v, int d) {
  if constexpr (sizeof(T) == 8) return (T)__shfl_up_sync(FULL, (unsigned long long)v, d);
  return (T)__shfl_up_sync(FULL, (unsigned)v, d);
}
template <typename T>
__device__ __forceinline__ T shfl_down_t(T v, int d) {
  if constexpr (sizeof(T) == 8) return (T)__shfl_down_sync(FULL, (unsigned long long)v, d);
  return (T)__shfl_down_sync(FULL, (unsigned)v, d);
}
template <typename T>
__device__ __forceinline__ T shfl_t(T v, int src) {
  if constexpr (sizeof(T) == 8) return (T)__shfl_sync(FULL, (unsigned long long)v, src);
  return (T)__shfl_sync(FULL, (unsigned)v, src);
}

// a2 * d^2 with 0 for d == 0 (a2 is +inf on an axis of extent 1 that the caller's array lacks)
__device__ __forceinline__ double sqdist(double a2, double d) { return d == 0.0 ? 0.0 : a2 * d * d; }

template <typename T>
__global__ void __launch_bounds__(X_THREADS) k_edt_x(const T* __restrict__ lab, float* __restrict__ out, uint64_t sx,
                                                     uint64_t nrows, double a2, int border) {
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t nw = (uint64_t)gridDim.x * (X_THREADS / 32);
  for (uint64_t r = blockIdx.x * (uint64_t)(X_THREADS / 32) + (threadIdx.x >> 5); r < nrows; r += nw) {
    const T* L = lab + r * sx;
    float* O = out + r * sx;
    uint32_t* D = (uint32_t*)O;
    // forward: distance to the voxel before the run (x + 1 from the shell at -1)
    T carry = 0;
    uint64_t cs = 0;
    for (uint64_t c0 = 0; c0 < sx; c0 += 32) {
      const uint64_t x = c0 + lane;
      const bool valid = x < sx;
      const T v = valid ? L[x] : T(0);
      T prev = shfl_up_t(v, 1);
      if (lane == 0) prev = carry;
      uint64_t st = (valid && (x == 0 || v != prev)) ? x : (lane == 0 ? cs : 0);
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint64_t u = shfl_up_t(st, o);
        if (lane >= (uint32_t)o) st = max(st, u);
      }
      if (valid) D[x] = (st == 0 && !border) ? DINF : (uint32_t)(x - st + 1);
      carry = shfl_t(v, 31);
      cs = shfl_t(st, 31);
    }
    // backward: distance to the voxel after the run (sx - x to the shell at sx)
    carry = 0;
    uint64_t ce = sx - 1;
    for (int64_t c0 = (int64_t)((sx - 1) / 32 * 32); c0 >= 0; c0 -= 32) {
      const uint64_t x = (uint64_t)c0 + lane;
      const bool valid = x < sx;
      const T v = valid ? L[x] : T(0);
      T next = shfl_down_t(v, 1);
      if (lane == 31) next = carry;
      uint64_t en = (valid && (x == sx - 1 || v != next)) ? x : (lane == 31 ? ce : ~0ull);
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint64_t u = shfl_down_t(en, o);
        if (lane + o < 32) en = min(en, u);
      }
      if (valid) {
        const uint32_t db = (en == sx - 1 && !border) ? DINF : (uint32_t)(en + 1 - x);
        const uint32_t d = min(D[x], db);
        O[x] = v == T(0) ? 0.f : d == DINF ? __int_as_float(0x7f800000) : (float)sqdist(a2, (double)d);
      }
      carry = shfl_t(v, 0);
      ce = shfl_t(en, 0);
    }
  }
}

// Writes the run [s, s + len) of one line from its envelope stack (k entries (q - s, f(q)) at
// S[j * nl]) and the zero-valued sites at s - 1 (lb) and s + len (rb); sqrt of it when ROOT.
template <bool ROOT>
__device__ __noinline__ void run_out(const uint2* __restrict__ S, uint64_t nl, uint32_t k, float* __restrict__ F,
                                     uint64_t stride, uint64_t s, uint64_t len, bool lb, bool rb, double a2) {
  uint32_t c = 0;
  double cv = 0, cf = 0, nv = 0, nf = 0;
  if (k > 0) {
    const uint2 e = S[0];
    cv = e.x;
    cf = __uint_as_float(e.y);
  }
  if (k > 1) {
    const uint2 e = S[nl];
    nv = e.x;
    nf = __uint_as_float(e.y);
  }
  const double inf = __longlong_as_double(0x7ff0000000000000ll);
  for (uint64_t p = 0; p < len; ++p) {
    const double dp = (double)p;
    double best = inf;
    if (k > 0) {
      double cval = cf + sqdist(a2, dp - cv);
      while (c + 1 < k) {
        const double nval = nf + sqdist(a2, dp - nv);
        if (nval > cval) break;
        ++c;
        cv = nv;
        cf = nf;
        cval = nval;
        if (c + 1 < k) {
          const uint2 e = S[(uint64_t)(c + 1) * nl];
          nv = e.x;
          nf = __uint_as_float(e.y);
        }
      }
      best = cval;
    }
    if (lb) best = min(best, sqdist(a2, dp + 1.0));
    if (rb) best = min(best, sqdist(a2, (double)len - dp));
    float r = (float)best;
    if (ROOT) r = sqrtf(r);
    F[(s + p) * stride] = r;
  }
}

// One thread per line of n elements `stride` apart; line l of the launch starts at element
// (line0 + l) % sx + ((line0 + l) / sx) * ostride.  f holds the previous pass and is overwritten.
template <typename T, bool ROOT>
__global__ void __launch_bounds__(LN_THREADS) k_edt_line(const T* __restrict__ lab, float* __restrict__ f, uint64_t n,
                                                         uint64_t stride, uint64_t sx, uint64_t ostride,
                                                         uint64_t line0, uint64_t nl, double a2, int border,
                                                         uint2* __restrict__ stk) {
  const uint64_t t = blockIdx.x * (uint64_t)LN_THREADS + threadIdx.x;
  if (t >= nl) return;
  const uint64_t l = line0 + t;
  const uint64_t base = l % sx + (l / sx) * ostride;
  const T* L = lab + base;
  float* F = f + base;
  uint2* S = stk + t;
  T run = 0;
  uint64_t s = 0;
  bool lb = border;
  uint32_t k = 0;                     // entries on the run's stack
  double v0 = 0, F0 = 0, v1 = 0, F1 = 0;  // the two top entries: position and f + a2 v^2
  for (uint64_t i0 = 0; i0 < n; i0 += LN_BATCH) {
    T lv[LN_BATCH];
    float fv[LN_BATCH];
#pragma unroll
    for (int b = 0; b < LN_BATCH; ++b) {
      if (i0 + b < n) {
        lv[b] = L[(i0 + b) * stride];
        fv[b] = F[(i0 + b) * stride];
      }
    }
#pragma unroll
    for (int b = 0; b < LN_BATCH; ++b) {
      const uint64_t i = i0 + b;
      if (i < n) {
        if (i == 0) {
          run = lv[b];
        } else if (lv[b] != run) {
          if (run != T(0)) run_out<ROOT>(S, nl, k, F, stride, s, i - s, lb, true, a2);
          s = i;
          k = 0;
          lb = true;
          run = lv[b];
        }
        if (run != T(0) && fv[b] < __int_as_float(0x7f800000)) {
          const double dq = (double)(i - s), Fq = fv[b] + sqdist(a2, dq);
          while (k >= 2 && (Fq - F1) * (v1 - v0) <= (F1 - F0) * (dq - v1)) {  // top is under the envelope
            --k;
            v1 = v0;
            F1 = F0;
            if (k >= 2) {
              const uint2 e = S[(uint64_t)(k - 2) * nl];
              v0 = e.x;
              F0 = __uint_as_float(e.y) + sqdist(a2, v0);
            }
          }
          S[(uint64_t)k * nl] = make_uint2((uint32_t)(i - s), __float_as_uint(fv[b]));
          v0 = v1;
          F0 = F1;
          v1 = dq;
          F1 = Fq;
          ++k;
        }
      }
    }
  }
  if (run != T(0)) run_out<ROOT>(S, nl, k, F, stride, s, n - s, lb, border != 0, a2);
}

template <typename T, bool ROOT>
int line_pass(ign_ctx* ctx, const T* lab, float* out, uint64_t n, uint64_t stride, uint64_t sx, uint64_t ostride,
              uint64_t lines, double a2, int border) {
  ScratchFrame f(ctx);
  const uint64_t per = n * sizeof(uint2);
  const uint64_t L = std::min<uint64_t>(lines, std::max<uint64_t>(1, EDT_STACK_BYTES / per));
  uint2* S;
  IGN_TRY(f.take(&S, L * n));
  for (uint64_t l0 = 0; l0 < lines; l0 += L) {
    const uint64_t m = std::min(L, lines - l0);
    IGN_LAUNCH(ctx, (k_edt_line<T, ROOT>), blocks_for(m, LN_THREADS), LN_THREADS, 0, lab, out, n, stride, sx,
               ostride, l0, m, a2, border, S);
  }
  return IGN_OK;
}

template <typename T>
int edt_run(ign_ctx* ctx, const void* labels, uint64_t sx, uint64_t sy, uint64_t sz, const float* a, int border,
            int squared, float* out) {
  const T* lab = (const T*)labels;
  const double ax = a[0], ay = a[1], az = a[2];
  const uint64_t rows = sy * sz;
  const unsigned grid =
      (unsigned)std::min<uint64_t>((rows + X_THREADS / 32 - 1) / (X_THREADS / 32), (uint64_t)ctx->sm_count * 64);
  IGN_LAUNCH(ctx, k_edt_x<T>, grid, X_THREADS, 0, lab, out, sx, rows, ax * ax, border);
  IGN_TRY((line_pass<T, false>(ctx, lab, out, sy, sx, sx, sx * sy, sx * sz, ay * ay, border)));
  if (squared) return line_pass<T, false>(ctx, lab, out, sz, sx * sy, sx, sx, sx * sy, az * az, border);
  return line_pass<T, true>(ctx, lab, out, sz, sx * sy, sx, sx, sx * sy, az * az, border);
}

int edt_check(int dtype, uint64_t sx, uint64_t sy, uint64_t sz, const float* a) {
  IGN_REQUIRE(dtype == IGN_U8 || dtype == IGN_U16 || dtype == IGN_U32 || dtype == IGN_U64, IGN_ERR_UNSUPPORTED,
              "edt: label dtype %d is not u8 / u16 / u32 / u64", dtype);
  IGN_REQUIRE(sx < (1ull << 30) && sy < (1ull << 30) && sz < (1ull << 30), IGN_ERR_OVERFLOW,
              "edt: volume %llu x %llu x %llu (each side below 2^30)", (unsigned long long)sx,
              (unsigned long long)sy, (unsigned long long)sz);
  IGN_REQUIRE(a, IGN_ERR_INVALID, "edt: null anisotropy");
  const uint64_t ext[3] = {sx, sy, sz};
  for (int i = 0; i < 3; ++i)
    IGN_REQUIRE(a[i] > 0.f && (isfinite(a[i]) || ext[i] <= 1), IGN_ERR_INVALID,
                "edt: anisotropy[%d] = %g (positive; +inf only on an axis of extent 1)", i, (double)a[i]);
  return IGN_OK;
}

}  // namespace

}  // namespace ign

using namespace ign;

extern "C" {

int ign_edt_dev(ign_ctx* ctx, const void* labels, int dtype, uint64_t sx, uint64_t sy, uint64_t sz,
                const float anisotropy[3], int black_border, int squared, float* out) {
  IGN_TRY(activate(ctx));
  IGN_TRY(edt_check(dtype, sx, sy, sz, anisotropy));
  const uint64_t n = sx * sy * sz;
  if (!n) return IGN_OK;
  IGN_REQUIRE(labels && out, IGN_ERR_INVALID, "null buffer");
  IGN_REQUIRE((uintptr_t)labels % dtype_size(dtype) == 0, IGN_ERR_INVALID,
              "edt: labels not aligned to their element size");
  IGN_REQUIRE((uintptr_t)out % 4 == 0, IGN_ERR_INVALID, "edt: out not aligned to 4 bytes");
  const int bb = black_border ? 1 : 0;
  return dispatch_label(dtype, "edt", [&](auto v) {
    return edt_run<decltype(v)>(ctx, labels, sx, sy, sz, anisotropy, bb, squared, out);
  });
}

int ign_edt(ign_ctx* ctx, const void* labels, int dtype, uint64_t sx, uint64_t sy, uint64_t sz,
            const float anisotropy[3], int black_border, int squared, float* out) {
  IGN_TRY(edt_check(dtype, sx, sy, sz, anisotropy));
  const uint64_t n = sx * sy * sz;
  return staged(ctx, {{labels, nullptr, n * dtype_size(dtype)}, {nullptr, out, n * 4}}, [&](void* const* d) {
    return ign_edt_dev(ctx, d[0], dtype, sx, sy, sz, anisotropy, black_border, squared, (float*)d[1]);
  });
}

}  // extern "C"
