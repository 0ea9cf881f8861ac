// contrast.cu -- per-voxel image kernels of the contrast-normalization, CLAHE and
// quantization tasks (igneous/tasks/image/image.py:145-432), sm_90a.
//
//   k_hist_u8 / k_hist_u16   exact luminance histograms (LuminanceLevelsTask)
//   k_stretch                per-z-slice contrast stretch + rint + clip + cast (ContrastNormalizationTask)
//   k_quantize               float32 -> uint8 (QuantizeTask)
//   k_clahe_lut, k_clahe_interp   OpenCV CLAHE::apply on every z-slice of a stack (CLAHETask)
//
// The stretch and CLAHE rules are float32 operations that must round one at a time: this
// file is compiled with -fmad=false, and the arithmetic is written with the _rn intrinsics
// as well, so no product is ever contracted into an FMA.  DESIGN.md §5b states the rules.
#include <math.h>

#include <algorithm>
#include <type_traits>

#include "common.cuh"

namespace ign {

namespace {

// ------------------------------------------------------------------ histograms
// Input is split into launches of at most HIST_CHUNK elements, so no per-CTA uint32 counter can
// overflow; each launch adds its counts into the uint64 histogram.
constexpr uint64_t HIST_CHUNK = 1ull << 31;

// uint8: one 256-bin sub-histogram per warp in shared memory (privatised, so only the lanes of
// one warp contend on a bin), summed over the warps and added to the global histogram.
__global__ void __launch_bounds__(256) k_hist_u8(const uint8_t* __restrict__ in, uint64_t n,
                                                 unsigned long long* __restrict__ hist) {
  __shared__ uint32_t sh[8][256];
  for (int i = threadIdx.x; i < 8 * 256; i += 256) (&sh[0][0])[i] = 0;
  __syncthreads();
  uint32_t* mine = sh[threadIdx.x >> 5];
  const uint64_t head = ((16 - ((uintptr_t)in & 15)) & 15) < n ? ((16 - ((uintptr_t)in & 15)) & 15) : n;
  const uint64_t nvec = (n - head) / 16;
  const uint4* v = (const uint4*)(in + head);
  for (uint64_t i = blockIdx.x * 256ull + threadIdx.x; i < nvec; i += (uint64_t)gridDim.x * 256) {
    const uint4 w = ld_stream(v + i);
    const uint32_t word[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
      for (int b = 0; b < 4; ++b) atomicAdd(&mine[(word[k] >> (8 * b)) & 255], 1u);
  }
  if (blockIdx.x == 0) {  // unaligned head and the tail after the last whole vector
    for (uint64_t i = threadIdx.x; i < head; i += 256) atomicAdd(&mine[in[i]], 1u);
    for (uint64_t i = head + nvec * 16 + threadIdx.x; i < n; i += 256) atomicAdd(&mine[in[i]], 1u);
  }
  __syncthreads();
  uint32_t s = 0;
#pragma unroll
  for (int w = 0; w < 8; ++w) s += sh[w][threadIdx.x];
  if (s) atomicAdd(&hist[threadIdx.x], (unsigned long long)s);
}

// uint16: 65,536 uint32 bins (256 KB) do not fit in a CTA's shared memory, so the bin range is
// split: a CTA with blockIdx.y = h keeps the 32,768 bins of values with top bit h (128 KB, one
// CTA per SM) and reads its share of the whole input, counting only the values of its half.
// Each input byte is read twice (the second read mostly from L2); in exchange every count is
// a shared-memory atomic, and the flush adds at most 32,768 words per CTA.
constexpr int HIST16_THREADS = 1024;
constexpr int HIST16_HALF = 32768;

__global__ void __launch_bounds__(HIST16_THREADS) k_hist_u16(const uint16_t* __restrict__ in, uint64_t n,
                                                             unsigned long long* __restrict__ hist) {
  extern __shared__ uint32_t sh16[];
  for (int i = threadIdx.x; i < HIST16_HALF; i += HIST16_THREADS) sh16[i] = 0;
  __syncthreads();
  const uint32_t half = blockIdx.y;
  const uint64_t hb = (16 - ((uintptr_t)in & 15)) & 15;
  const uint64_t head = hb / 2 < n ? hb / 2 : n;
  const uint64_t nvec = (n - head) / 8;
  const uint4* v = (const uint4*)(in + head);
  for (uint64_t i = blockIdx.x * (uint64_t)HIST16_THREADS + threadIdx.x; i < nvec;
       i += (uint64_t)gridDim.x * HIST16_THREADS) {
    const uint4 w = ld_stream(v + i);
    const uint32_t word[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        const uint32_t val = (word[k] >> (16 * b)) & 0xFFFF;
        if ((val >> 15) == half) atomicAdd(&sh16[val & (HIST16_HALF - 1)], 1u);
      }
  }
  if (blockIdx.x == 0) {  // unaligned head and the tail after the last whole vector
    for (uint64_t i = threadIdx.x; i < head; i += HIST16_THREADS)
      if ((in[i] >> 15) == half) atomicAdd(&sh16[in[i] & (HIST16_HALF - 1)], 1u);
    for (uint64_t i = head + nvec * 8 + threadIdx.x; i < n; i += HIST16_THREADS)
      if ((in[i] >> 15) == half) atomicAdd(&sh16[in[i] & (HIST16_HALF - 1)], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < HIST16_HALF; i += HIST16_THREADS)
    if (sh16[i]) atomicAdd(&hist[half * HIST16_HALF + i], (unsigned long long)sh16[i]);
}

// --------------------------------------------------------------- contrast stretch
// Streaming: each thread takes 8 consecutive voxels (one 8- or 16-byte load), no shared memory.
// Slice s of the (x, y, z, c) volume uses params[s % sz] = (f32(lower), f32(maxval_t / (upper -
// lower))); a slice that keeps its values has (0, 1), which is exact: (v - 0) * 1 == v.
template <typename T>
__device__ __forceinline__ void load8(const T* p, T* v) {
  if constexpr (sizeof(T) == 1) {
    const uint2 w = *(const uint2*)p;
    *(uint2*)v = w;
  } else if constexpr (sizeof(T) == 2) {
    *(uint4*)v = ld_stream(p);
  } else {
    *(uint4*)v = ld_stream(p);
    *(uint4*)(v + 4) = ld_stream(p + 4);
  }
}

template <typename T>
__device__ __forceinline__ void store8(T* p, const T* v) {
  if constexpr (sizeof(T) == 1) {
    st_stream(p, *(const uint2*)v);
  } else if constexpr (sizeof(T) == 2) {
    st_stream(p, *(const uint4*)v);
  } else {
    st_stream(p, *(const uint4*)v);
    st_stream(p + 4, *(const uint4*)(v + 4));
  }
}

template <typename Tout>
__device__ __forceinline__ Tout render(float r, float lo, float hi) {
  r = fminf(fmaxf(rintf(r), lo), hi);  // rint (half to even), then np.clip's max-then-min
  if constexpr (std::is_same<Tout, float>::value) return r;
  return (Tout)r;  // in range after the clip: the cast truncates toward zero like numpy's
}

template <typename Tin, typename Tout>
__global__ void __launch_bounds__(256) k_stretch(const Tin* __restrict__ in, Tout* __restrict__ out, uint64_t n,
                                                 uint64_t plane, uint64_t sz, const float2* __restrict__ params,
                                                 float lo, float hi, int vec) {
  const uint64_t g = blockIdx.x * 256ull + threadIdx.x;
  const uint64_t i0 = g * 8;
  if (i0 >= n) return;
  uint64_t q = i0 / plane, rem = i0 - q * plane;
  float2 p = params[q % sz];
  alignas(16) Tin v[8];
  alignas(16) Tout o[8];
  const bool whole = vec && i0 + 8 <= n;
  if (whole) load8(in + i0, v);
  else
    for (int k = 0; k < 8; ++k) v[k] = i0 + k < n ? in[i0 + k] : Tin(0);
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    if (rem == plane) {
      rem = 0;
      ++q;
      p = params[q % sz];
    }
    ++rem;
    const float f = __fmul_rn(__fsub_rn((float)v[k], p.x), p.y);
    o[k] = render<Tout>(f, lo, hi);
  }
  if (whole) store8(out + i0, o);
  else
    for (int k = 0; k < 8 && i0 + k < n; ++k) out[i0 + k] = o[k];
}

// -------------------------------------------------------------------- quantize
// trunc(v * 255) with saturation; NaN and products <= 0 give 0, products >= 255 give 255.
__device__ __forceinline__ uint8_t quant1(float v) {
  const float p = __fmul_rn(v, 255.0f);
  if (!(p > 0.0f)) return 0;
  if (p >= 255.0f) return 255;
  return (uint8_t)(int)p;
}

__global__ void __launch_bounds__(256) k_quantize(const float* __restrict__ in, uint8_t* __restrict__ out,
                                                  uint64_t n, int vec) {
  const uint64_t i0 = (blockIdx.x * 256ull + threadIdx.x) * 8;
  if (i0 >= n) return;
  if (vec && i0 + 8 <= n) {
    alignas(16) float v[8];
    alignas(8) uint8_t o[8];
    load8(in + i0, v);
#pragma unroll
    for (int k = 0; k < 8; ++k) o[k] = quant1(v[k]);
    store8(out + i0, o);
  } else {
    for (uint64_t i = i0; i < i0 + 8 && i < n; ++i) out[i] = quant1(in[i]);
  }
}

// ----------------------------------------------------------------------- CLAHE
// One CTA per (tile, slice) builds that tile's LUT; then k_clahe_interp streams the stack.
// Rows are the stack's x axis (contiguous in memory), columns its y axis; tiles_x tiles go
// across the columns and tiles_y across the rows (OpenCV's tileGridSize order).  When either
// extent does not divide by its tile count, OpenCV pads BOTH axes at the far end by
// tiles - extent % tiles with BORDER_REFLECT_101 (a whole tile count on an axis that did
// divide) and cuts the tiles from the padded image; the padded pixels are read through
// reflect101() here, never materialised.  The interpolation runs over the original extent.
__device__ __forceinline__ uint64_t reflect101(int64_t p, int64_t n) {
  if (n == 1) return 0;
  while (p < 0 || p >= n) p = p < 0 ? -p : 2 * (n - 1) - p;
  return (uint64_t)p;
}

// inclusive block scan of one uint32 per thread; *total = sum over the block
template <int THREADS>
__device__ __forceinline__ uint32_t block_scan(uint32_t x, uint32_t* warp_sums, uint32_t* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
    if (lane >= d) x += y;
  }
  if (lane == 31) warp_sums[warp] = x;
  __syncthreads();
  if (warp == 0) {
    uint32_t s = lane < THREADS / 32 ? warp_sums[lane] : 0;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t y = __shfl_up_sync(0xffffffffu, s, d);
      if (lane >= d) s += y;
    }
    warp_sums[lane] = s;  // inclusive prefix of the warp totals
  }
  __syncthreads();
  const uint32_t r = x + (warp ? warp_sums[warp - 1] : 0);
  *total = warp_sums[THREADS / 32 - 1];
  __syncthreads();  // warp_sums may be reused at once
  return r;
}

struct ClaheGeom {
  uint64_t rows, cols;  // extent of one slice
  uint32_t gx, gy;      // tiles across columns / rows
  uint32_t th, tw;      // tile size in the (possibly padded) image
  uint32_t lim;         // clip limit in counts, 0 = no clipping
  float lut_scale;      // f32(hist_size - 1) / f32(th * tw)
  float inv_th, inv_tw; // 1.0f / th, 1.0f / tw
};

// HS bins, of which PART are held in shared memory at once (256 for uint8; 32,768 for uint16,
// whose 65,536 uint32 bins do not fit: the tile is then counted once per half, plus once more
// for the far half when clipping needs the total clipped count before the first LUT entry).
template <typename T, int HS, int PART, int THREADS>
__global__ void __launch_bounds__(THREADS) k_clahe_lut(const T* __restrict__ in, ClaheGeom g, T* __restrict__ luts) {
  extern __shared__ uint32_t shl[];
  uint32_t* bins = shl;  // bin b lives at skew(b): thread t's PER consecutive bins fall in distinct banks
  uint32_t* wsum = shl + PART + PART / 32;
  constexpr int NPARTS = HS / PART;
  constexpr int PER = PART / THREADS;
  auto skew = [](uint32_t b) { return b + b / 32; };
  const uint32_t ntiles = g.gx * g.gy;
  const uint32_t tile = blockIdx.x % ntiles;
  const uint64_t z = blockIdx.x / ntiles;
  const uint32_t ty = tile / g.gx, tx = tile % g.gx;
  const T* slice = in + z * g.rows * g.cols;
  const uint32_t npix = g.th * g.tw;
  const int64_t r0 = (int64_t)ty * g.th, c0 = (int64_t)tx * g.tw;

  auto count = [&](int part) {
    __syncthreads();  // every thread is done reading the previous part's bins
    for (int i = threadIdx.x; i < PART + PART / 32; i += THREADS) bins[i] = 0;
    __syncthreads();
    for (uint32_t k = threadIdx.x; k < npix; k += THREADS) {
      const uint32_t cl = k / g.th, rl = k - cl * g.th;
      const uint64_t r = reflect101(r0 + rl, (int64_t)g.rows), c = reflect101(c0 + cl, (int64_t)g.cols);
      const uint32_t v = slice[r + g.rows * c];
      if (NPARTS == 1 || (int)(v / PART) == part) atomicAdd(&bins[skew(v % PART)], 1u);
    }
    __syncthreads();
  };
  auto clipped_sum = [&]() {
    uint32_t s = 0;
    for (int i = threadIdx.x; i < PART; i += THREADS) s += g.lim ? min(bins[skew(i)], g.lim) : bins[skew(i)];
    uint32_t total;
    block_scan<THREADS>(s, wsum, &total);
    return total;
  };

  uint32_t kept = 0;  // sum over all bins of min(count, lim)
  if (g.lim && NPARTS > 1)
    for (int part = 1; part < NPARTS; ++part) {
      count(part);
      kept += clipped_sum();
    }
  uint32_t carry = 0;
  uint32_t batch = 0, residual = 0, step = 1;
  T* lut = luts + (uint64_t)blockIdx.x * HS;
  for (int part = 0; part < NPARTS; ++part) {
    count(part);
    if (part == 0 && g.lim) {
      kept += clipped_sum();
      const uint32_t excess = npix - kept;  // what clipping removed, redistributed below
      batch = excess / HS;
      residual = excess - batch * HS;
      step = residual ? max((uint32_t)HS / residual, 1u) : 1u;
    }
    // clipped and redistributed count of this thread's j-th bin (read twice rather than held in
    // registers: 32 per thread would spill at 1,024 threads)
    auto clipped = [&](int j) {
      const uint32_t bin = threadIdx.x * PER + j;
      const uint32_t gbin = part * PART + bin;
      const uint32_t c = bins[skew(bin)];
      if (!g.lim) return c;
      return min(c, g.lim) + batch + ((gbin % step == 0 && gbin / step < residual) ? 1u : 0u);
    };
    uint32_t s = 0;
#pragma unroll 8
    for (int j = 0; j < PER; ++j) s += clipped(j);
    uint32_t total;
    uint32_t cum = carry + block_scan<THREADS>(s, wsum, &total) - s;
#pragma unroll 8
    for (int j = 0; j < PER; ++j) {
      cum += clipped(j);
      const float f = __fmul_rn(__uint2float_rn(cum), g.lut_scale);
      const int r = __float2int_rn(f);
      lut[part * PART + threadIdx.x * PER + j] = (T)min(max(r, 0), HS - 1);
    }
    carry += total;
  }
}

template <typename T, int HS>
__global__ void __launch_bounds__(256) k_clahe_interp(const T* in, T* out, ClaheGeom g, uint64_t n,
                                                      const T* __restrict__ luts) {
  const uint64_t i = blockIdx.x * 256ull + threadIdx.x;
  if (i >= n) return;
  const uint64_t r = i % g.rows, t = i / g.rows;
  const uint64_t c = t % g.cols, z = t / g.cols;
  const float tyf = __fsub_rn(__fmul_rn((float)r, g.inv_th), 0.5f);
  int ty1 = (int)floorf(tyf), ty2 = ty1 + 1;
  const float ya = __fsub_rn(tyf, (float)ty1), ya1 = __fsub_rn(1.0f, ya);
  ty1 = max(ty1, 0);
  ty2 = min(ty2, (int)g.gy - 1);
  const float txf = __fsub_rn(__fmul_rn((float)c, g.inv_tw), 0.5f);
  int tx1 = (int)floorf(txf), tx2 = tx1 + 1;
  const float xa = __fsub_rn(txf, (float)tx1), xa1 = __fsub_rn(1.0f, xa);
  tx1 = max(tx1, 0);
  tx2 = min(tx2, (int)g.gx - 1);
  const uint32_t v = in[i];
  const T* L = luts + z * g.gx * g.gy * (uint64_t)HS + v;
  const float l11 = L[(uint64_t)(ty1 * g.gx + tx1) * HS], l12 = L[(uint64_t)(ty1 * g.gx + tx2) * HS];
  const float l21 = L[(uint64_t)(ty2 * g.gx + tx1) * HS], l22 = L[(uint64_t)(ty2 * g.gx + tx2) * HS];
  const float top = __fadd_rn(__fmul_rn(l11, xa1), __fmul_rn(l12, xa));
  const float bot = __fadd_rn(__fmul_rn(l21, xa1), __fmul_rn(l22, xa));
  const float res = __fadd_rn(__fmul_rn(top, ya1), __fmul_rn(bot, ya));
  out[i] = (T)min(max(__float2int_rn(res), 0), HS - 1);
}

template <typename T, int HS, int PART, int THREADS>
int clahe_typed(ign_ctx* ctx, const T* in, T* out, uint64_t nz, const ClaheGeom& g) {
  ScratchFrame f(ctx);
  T* luts;
  const uint64_t items = nz * g.gx * g.gy;
  IGN_TRY(f.take(&luts, items * HS));
  const size_t smem = (PART + PART / 32 + 32) * sizeof(uint32_t);
  if (smem > 48 * 1024)
    IGN_CUDA(cudaFuncSetAttribute(k_clahe_lut<T, HS, PART, THREADS>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)smem));
  IGN_LAUNCH(ctx, (k_clahe_lut<T, HS, PART, THREADS>), (unsigned)items, THREADS, smem, in, g, luts);
  const uint64_t n = g.rows * g.cols * nz;
  IGN_LAUNCH(ctx, (k_clahe_interp<T, HS>), blocks_for(n, 256), 256, 0, in, out, g, n, (const T*)luts);
  return IGN_OK;
}

template <typename Tin, typename Tout>
int stretch_typed(ign_ctx* ctx, const void* in, void* out, uint64_t n, uint64_t plane, uint64_t sz,
                  const float2* params, float lo, float hi) {
  const int vec = ((uintptr_t)in % 16 == 0) && ((uintptr_t)out % 16 == 0);
  IGN_LAUNCH(ctx, (k_stretch<Tin, Tout>), blocks_for((n + 7) / 8, 256), 256, 0, (const Tin*)in, (Tout*)out, n,
             plane, sz, params, lo, hi, vec);
  return IGN_OK;
}

template <typename Tin>
int stretch_out(ign_ctx* ctx, int out_dtype, const void* in, void* out, uint64_t n, uint64_t plane, uint64_t sz,
                const float2* params, float lo, float hi) {
  switch (out_dtype) {
    case IGN_U8: return stretch_typed<Tin, uint8_t>(ctx, in, out, n, plane, sz, params, lo, hi);
    case IGN_U16: return stretch_typed<Tin, uint16_t>(ctx, in, out, n, plane, sz, params, lo, hi);
    case IGN_U32: return stretch_typed<Tin, uint32_t>(ctx, in, out, n, plane, sz, params, lo, hi);
    case IGN_F32: return stretch_typed<Tin, float>(ctx, in, out, n, plane, sz, params, lo, hi);
  }
  set_error("contrast_stretch: unsupported output dtype %d", out_dtype);
  return IGN_ERR_UNSUPPORTED;
}

double dtype_max(int dt) {
  switch (dt) {
    case IGN_U8: return 255.0;
    case IGN_U16: return 65535.0;
    case IGN_U32: return 4294967295.0;
    default: return 3.4028234663852886e38;  // float32
  }
}

int stretch_check(int in_dtype, int out_dtype, uint64_t sx, uint64_t sy, uint64_t sz, double minval, double maxval) {
  IGN_REQUIRE(in_dtype == IGN_U8 || in_dtype == IGN_U16, IGN_ERR_UNSUPPORTED,
              "contrast_stretch: input dtype %d is not uint8 / uint16", in_dtype);
  IGN_REQUIRE(out_dtype == IGN_U8 || out_dtype == IGN_U16 || out_dtype == IGN_U32 || out_dtype == IGN_F32,
              IGN_ERR_UNSUPPORTED, "contrast_stretch: unsupported output dtype %d", out_dtype);
  IGN_REQUIRE(sx > 0 && sy > 0 && sz > 0, IGN_ERR_INVALID, "empty volume");
  // the clip runs in float32: the bounds are checked as float32 values, so a uint32 maxval above
  // 4294967040 (which rounds to 2^32) is refused rather than cast out of range
  const double lim = dtype_max(out_dtype), low = out_dtype == IGN_F32 ? -lim : 0.0;
  const double lo32 = (double)(float)minval, hi32 = (double)(float)maxval;
  IGN_REQUIRE(lo32 >= low && hi32 <= lim && lo32 <= hi32, IGN_ERR_INVALID,
              "contrast_stretch: clip range [%.17g, %.17g] in float32 outside the output dtype's [%g, %g]", lo32,
              hi32, low, lim);
  return IGN_OK;
}

int clahe_geometry(int dtype, uint64_t rows, uint64_t cols, uint32_t gx, uint32_t gy, double clip, ClaheGeom* g) {
  IGN_REQUIRE(dtype == IGN_U8 || dtype == IGN_U16, IGN_ERR_UNSUPPORTED, "clahe: dtype %d is not uint8 / uint16", dtype);
  IGN_REQUIRE(rows > 0 && cols > 0, IGN_ERR_INVALID, "empty image");
  IGN_REQUIRE(gx > 0 && gy > 0 && gx <= 4096 && gy <= 4096, IGN_ERR_INVALID, "tile grid %u x %u", gx, gy);
  IGN_REQUIRE(clip >= 0 && clip < 1e9, IGN_ERR_INVALID, "clip limit %g", clip);
  const bool pad = rows % gy || cols % gx;
  g->rows = rows;
  g->cols = cols;
  g->gx = gx;
  g->gy = gy;
  g->th = (uint32_t)((pad ? rows + gy - rows % gy : rows) / gy);
  g->tw = (uint32_t)((pad ? cols + gx - cols % gx : cols) / gx);
  const uint64_t npix = (uint64_t)g->th * g->tw;
  IGN_REQUIRE(npix < (1ull << 31) && rows * cols < (1ull << 40), IGN_ERR_OVERFLOW, "clahe: tile too large");
  const int hs = dtype == IGN_U8 ? 256 : 65536;
  g->lim = 0;
  if (clip > 0) {
    const int64_t l = (int64_t)(clip * (double)npix / hs);
    g->lim = (uint32_t)(l < 1 ? 1 : (l > (int64_t)npix ? (int64_t)npix : l));
  }
  g->lut_scale = (float)(hs - 1) / (float)npix;
  g->inv_th = 1.0f / (float)g->th;
  g->inv_tw = 1.0f / (float)g->tw;
  return IGN_OK;
}

}  // namespace

}  // namespace ign

using namespace ign;

extern "C" {

int ign_histogram_dev(ign_ctx* ctx, const void* in, int dtype, uint64_t n, uint64_t* hist) {
  IGN_TRY(activate(ctx));
  IGN_REQUIRE(dtype == IGN_U8 || dtype == IGN_U16, IGN_ERR_UNSUPPORTED, "histogram: dtype %d is not uint8 / uint16",
              dtype);
  IGN_REQUIRE(hist && (in || !n), IGN_ERR_INVALID, "null buffer");
  IGN_REQUIRE(n < (1ull << 40), IGN_ERR_OVERFLOW, "histogram: %llu voxels (at most 2^40)", (unsigned long long)n);
  const int es = dtype_size(dtype);
  IGN_REQUIRE((uintptr_t)in % es == 0 && (uintptr_t)hist % 8 == 0, IGN_ERR_INVALID,
              "histogram: input or histogram not aligned to its element size");
  for (uint64_t at = 0; at < n; at += HIST_CHUNK) {
    const uint64_t m = n - at < HIST_CHUNK ? n - at : HIST_CHUNK;
    const char* p = (const char*)in + at * es;
    if (dtype == IGN_U8) {
      const unsigned grid = (unsigned)std::min<uint64_t>(blocks_for(m / 16 + 1, 256), (uint64_t)ctx->sm_count * 8);
      IGN_LAUNCH(ctx, k_hist_u8, grid, 256, 0, (const uint8_t*)p, m, (unsigned long long*)hist);
    } else {
      const size_t smem = HIST16_HALF * sizeof(uint32_t);
      IGN_CUDA(cudaFuncSetAttribute(k_hist_u16, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      // one 128 KB CTA per SM: half the SMs per bin half
      const unsigned gx = (unsigned)std::max<uint64_t>(
          std::min<uint64_t>(blocks_for(m / 8 + 1, HIST16_THREADS), (uint64_t)ctx->sm_count / 2), 1);
      IGN_LAUNCH(ctx, k_hist_u16, dim3(gx, 2), HIST16_THREADS, smem, (const uint16_t*)p, m, (unsigned long long*)hist);
    }
  }
  return IGN_OK;
}

int ign_histogram(ign_ctx* ctx, const void* in, int dtype, uint64_t n, uint64_t* hist) {
  const uint64_t bins = dtype == IGN_U8 ? 256 : dtype == IGN_U16 ? 65536 : 0;
  return staged(ctx, {{in, nullptr, n * dtype_size(dtype)}, {hist, hist, bins * 8}},
                [&](void* const* d) { return ign_histogram_dev(ctx, d[0], dtype, n, (uint64_t*)d[1]); });
}

int ign_contrast_stretch_dev(ign_ctx* ctx, const void* in, int in_dtype, uint64_t sx, uint64_t sy, uint64_t sz,
                             uint64_t sc, const uint32_t* lower, const uint32_t* upper, double minval, double maxval,
                             void* out, int out_dtype) {
  IGN_TRY(activate(ctx));
  IGN_REQUIRE(in && out && lower && upper, IGN_ERR_INVALID, "null buffer");
  IGN_TRY(stretch_check(in_dtype, out_dtype, sx, sy, sz, minval, maxval));
  IGN_REQUIRE((uintptr_t)in % dtype_size(in_dtype) == 0 && (uintptr_t)out % dtype_size(out_dtype) == 0,
              IGN_ERR_INVALID, "contrast_stretch: buffer not aligned to its element size");
  sc = sc ? sc : 1;
  const double maxval_t = in_dtype == IGN_U8 ? 255.0 : 65535.0;
  std::vector<float2> params(sz);
  for (uint64_t z = 0; z < sz; ++z) {
    if (lower[z] == upper[z]) {
      params[z] = make_float2(0.0f, 1.0f);
    } else {
      params[z] = make_float2((float)lower[z], (float)(maxval_t / ((double)upper[z] - (double)lower[z])));
    }
  }
  ScratchFrame f(ctx);
  float2* dp;
  IGN_TRY(f.take(&dp, sz));
  IGN_TRY(small_h2d(ctx, dp, params.data(), sz * sizeof(float2)));
  const uint64_t n = sx * sy * sz * sc;
  const float lo = (float)minval, hi = (float)maxval;
  if (in_dtype == IGN_U8) return stretch_out<uint8_t>(ctx, out_dtype, in, out, n, sx * sy, sz, dp, lo, hi);
  return stretch_out<uint16_t>(ctx, out_dtype, in, out, n, sx * sy, sz, dp, lo, hi);
}

int ign_contrast_stretch(ign_ctx* ctx, const void* in, int in_dtype, uint64_t sx, uint64_t sy, uint64_t sz,
                         uint64_t sc, const uint32_t* lower, const uint32_t* upper, double minval, double maxval,
                         void* out, int out_dtype) {
  IGN_TRY(stretch_check(in_dtype, out_dtype, sx, sy, sz, minval, maxval));
  const uint64_t n = sx * sy * sz * (sc ? sc : 1);
  return staged(ctx, {{in, nullptr, n * dtype_size(in_dtype)}, {nullptr, out, n * dtype_size(out_dtype)}},
                [&](void* const* d) {
                  return ign_contrast_stretch_dev(ctx, d[0], in_dtype, sx, sy, sz, sc, lower, upper, minval, maxval,
                                                  d[1], out_dtype);
                });
}

int ign_quantize_dev(ign_ctx* ctx, const float* in, uint64_t n, uint8_t* out) {
  IGN_TRY(activate(ctx));
  IGN_REQUIRE((in && out) || !n, IGN_ERR_INVALID, "null buffer");
  if (!n) return IGN_OK;
  IGN_REQUIRE((uintptr_t)in % 4 == 0, IGN_ERR_INVALID, "quantize: input not aligned to 4 bytes");
  const int vec = ((uintptr_t)in % 16 == 0) && ((uintptr_t)out % 8 == 0);
  IGN_LAUNCH(ctx, k_quantize, blocks_for((n + 7) / 8, 256), 256, 0, in, out, n, vec);
  return IGN_OK;
}

int ign_quantize(ign_ctx* ctx, const float* in, uint64_t n, uint8_t* out) {
  return staged(ctx, {{in, nullptr, n * 4}, {nullptr, out, n}},
                [&](void* const* d) { return ign_quantize_dev(ctx, (const float*)d[0], n, (uint8_t*)d[1]); });
}

int ign_clahe_dev(ign_ctx* ctx, const void* in, int dtype, uint64_t sx, uint64_t sy, uint64_t sz, double clip_limit,
                  uint32_t tiles_x, uint32_t tiles_y, void* out) {
  IGN_TRY(activate(ctx));
  IGN_REQUIRE(in && out, IGN_ERR_INVALID, "null buffer");
  ClaheGeom g;
  IGN_TRY(clahe_geometry(dtype, sx, sy, tiles_x, tiles_y, clip_limit, &g));
  IGN_REQUIRE((uintptr_t)in % dtype_size(dtype) == 0 && (uintptr_t)out % dtype_size(dtype) == 0, IGN_ERR_INVALID,
              "clahe: buffer not aligned to its element size");
  IGN_REQUIRE(sz > 0 && sz * tiles_x * tiles_y < (1ull << 31), IGN_ERR_INVALID, "clahe: %llu slices",
              (unsigned long long)sz);
  if (dtype == IGN_U8)
    return clahe_typed<uint8_t, 256, 256, 256>(ctx, (const uint8_t*)in, (uint8_t*)out, sz, g);
  return clahe_typed<uint16_t, 65536, HIST16_HALF, 1024>(ctx, (const uint16_t*)in, (uint16_t*)out, sz, g);
}

int ign_clahe(ign_ctx* ctx, const void* in, int dtype, uint64_t sx, uint64_t sy, uint64_t sz, double clip_limit,
              uint32_t tiles_x, uint32_t tiles_y, void* out) {
  // one staged buffer serves as in and out, so a null one of the two would not reach ign_clahe_dev
  IGN_REQUIRE(in && out, IGN_ERR_INVALID, "null buffer");
  ClaheGeom g;
  IGN_TRY(clahe_geometry(dtype, sx, sy, tiles_x, tiles_y, clip_limit, &g));
  return staged(ctx, {{in, out, sx * sy * sz * dtype_size(dtype)}}, [&](void* const* d) {
    return ign_clahe_dev(ctx, d[0], dtype, sx, sy, sz, clip_limit, tiles_x, tiles_y, d[0]);
  });
}

}  // extern "C"
