// chunks.cu -- many Precomputed chunks into / out of one device cutout in one launch
//
// The read path of a layer decodes every chunk a cutout touches into one packed buffer (chunk c an
// F-order [sx, sy, sz, nc] array at its own byte offset) and `place` copies each chunk's sub-box to
// its corner of the F-order [X, Y, Z, nc] cutout.  The write path is the reverse: `cut` copies a
// list of boxes of the cutout into one packed buffer, each box F-order contiguous -- a `raw` chunk
// file byte for byte, and what the batch encoders read -- and flags the boxes that hold only the
// background value.  `fill_box` sets one box of a cutout to one value (BlackoutTask).  All indexing is
// 64-bit: a 2048 x 2048 x 128 uint64 cutout is 4.3 GB.
#include <string.h>

#include <algorithm>

#include "common.cuh"

namespace ign {

// one row of the place table (uint64 words, IGN_PLACE_ROW of them)
struct PlaceRow {
  uint64_t sx, sy, sz, off, x0, y0, z0, bx, by, bz, dx, dy, dz;
};
// one row of the cut table (IGN_CUT_ROW words)
struct CutRow {
  uint64_t x0, y0, z0, bx, by, bz, off;
};
static_assert(sizeof(PlaceRow) == IGN_PLACE_ROW * 8, "place row layout");
static_assert(sizeof(CutRow) == IGN_CUT_ROW * 8, "cut row layout");

// blockIdx.y walks the rows, blockIdx.x / threadIdx.x the voxels of a row's box (grid-strided both ways)
template <typename T>
__global__ void __launch_bounds__(256)
    k_chunks_place(const char* __restrict__ packed, const PlaceRow* __restrict__ rows, uint64_t nrows, uint64_t nc,
                   T* __restrict__ out, uint64_t X, uint64_t Y, uint64_t Z) {
  for (uint64_t r = blockIdx.y; r < nrows; r += gridDim.y) {
    const PlaceRow w = rows[r];
    const T* src = (const T*)(packed + w.off);
    const uint64_t n = w.bx * w.by * w.bz * nc;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
      const uint64_t x = i % w.bx, y = (i / w.bx) % w.by, q = i / (w.bx * w.by), z = q % w.bz, c = q / w.bz;
      const uint64_t s = (w.x0 + x) + w.sx * ((w.y0 + y) + w.sy * ((w.z0 + z) + w.sz * c));
      const uint64_t d = (w.dx + x) + X * ((w.dy + y) + Y * ((w.dz + z) + Z * c));
      out[d] = src[s];
    }
  }
}

template <typename T>
__global__ void __launch_bounds__(256)
    k_chunks_cut(const T* __restrict__ in, uint64_t X, uint64_t Y, uint64_t Z, uint64_t nc,
                 const CutRow* __restrict__ rows, uint64_t nrows, T bg, char* __restrict__ packed,
                 uint32_t* __restrict__ all_bg) {
  for (uint64_t r = blockIdx.y; r < nrows; r += gridDim.y) {
    const CutRow w = rows[r];
    T* dst = (T*)(packed + w.off);
    const uint64_t n = w.bx * w.by * w.bz * nc;
    bool other = false;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
      const uint64_t x = i % w.bx, y = (i / w.bx) % w.by, q = i / (w.bx * w.by), z = q % w.bz, c = q / w.bz;
      const T v = in[(w.x0 + x) + X * ((w.y0 + y) + Y * ((w.z0 + z) + Z * c))];
      dst[i] = v;
      other |= v != bg;
    }
    // every writer stores the same 0: the flag starts at 1 and only ever drops
    if (__syncthreads_or(other) && threadIdx.x == 0) all_bg[r] = 0;
  }
}

// every voxel of one box of the cutout, every channel, set to v
template <typename T>
__global__ void __launch_bounds__(256)
    k_fill_box(T* __restrict__ out, uint64_t X, uint64_t Y, uint64_t Z, uint64_t x0, uint64_t y0, uint64_t z0,
               uint64_t bx, uint64_t by, uint64_t bz, uint64_t n, T v) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
    const uint64_t x = i % bx, y = (i / bx) % by, q = i / (bx * by), z = q % bz, c = q / bz;
    out[(x0 + x) + X * ((y0 + y) + Y * ((z0 + z) + Z * c))] = v;
  }
}

// the background as a T: `bits` holds the value's own bit pattern, zero-extended
template <typename T>
static T bg_value(uint64_t bits) {
  T v;
  memcpy(&v, &bits, sizeof(T));  // little endian: the low bytes
  return v;
}

// grid for `rows` rows of at most `most` elements each
static dim3 rows_grid(uint64_t rows, uint64_t most) {
  const uint64_t gx = (most + 255) / 256;
  return dim3((unsigned)(gx < 1024 ? (gx ? gx : 1) : 1024), (unsigned)(rows < 65535 ? rows : 65535));
}

}  // namespace ign

using namespace ign;

extern "C" {

int ign_chunks_place_dev(ign_ctx* ctx, const void* packed, int dtype, uint64_t nc, const uint64_t* rows,
                         uint64_t n_rows, void* cutout, uint64_t X, uint64_t Y, uint64_t Z) {
  IGN_TRY(activate(ctx));
  IGN_REQUIRE(rows || n_rows == 0, IGN_ERR_INVALID, "chunks_place: null row table");
  IGN_REQUIRE(nc >= 1 && (n_rows == 0 || (packed && cutout)), IGN_ERR_INVALID, "chunks_place: null buffer");
  const PlaceRow* hr = (const PlaceRow*)rows;
  uint64_t most = 0;
  for (uint64_t r = 0; r < n_rows; r++) {
    const PlaceRow& w = hr[r];
    IGN_REQUIRE(w.x0 + w.bx <= w.sx && w.y0 + w.by <= w.sy && w.z0 + w.bz <= w.sz, IGN_ERR_INVALID,
                "chunks_place: row %llu takes a box outside its chunk", (unsigned long long)r);
    IGN_REQUIRE(w.dx + w.bx <= X && w.dy + w.by <= Y && w.dz + w.bz <= Z, IGN_ERR_INVALID,
                "chunks_place: row %llu writes outside the cutout", (unsigned long long)r);
    const uint64_t n = w.bx * w.by * w.bz * nc;
    most = n > most ? n : most;
  }
  if (most == 0) return dispatch_chunk(dtype, "chunks_place", [](auto) { return IGN_OK; });
  ScratchFrame f(ctx);
  PlaceRow* dr;
  IGN_TRY(f.take(&dr, n_rows));
  IGN_CUDA(cudaMemcpyAsync(dr, hr, n_rows * sizeof(PlaceRow), cudaMemcpyHostToDevice, ctx->stream));
  const dim3 g = rows_grid(n_rows, most);
  return dispatch_chunk(dtype, "chunks_place", [&](auto t) -> int {
    using T = decltype(t);
    IGN_LAUNCH(ctx, k_chunks_place<T>, g, 256, 0, (const char*)packed, (const PlaceRow*)dr, n_rows, nc, (T*)cutout,
               X, Y, Z);
    return IGN_OK;
  });
}

int ign_chunks_cut_dev(ign_ctx* ctx, const void* cutout, int dtype, uint64_t X, uint64_t Y, uint64_t Z, uint64_t nc,
                       const uint64_t* rows, uint64_t n_rows, uint64_t background, void* packed, uint32_t* all_bg) {
  IGN_TRY(activate(ctx));
  IGN_REQUIRE(rows || n_rows == 0, IGN_ERR_INVALID, "chunks_cut: null row table");
  IGN_REQUIRE(nc >= 1 && (n_rows == 0 || (cutout && packed && all_bg)), IGN_ERR_INVALID, "chunks_cut: null buffer");
  const CutRow* hr = (const CutRow*)rows;
  uint64_t most = 0;
  for (uint64_t r = 0; r < n_rows; r++) {
    const CutRow& w = hr[r];
    IGN_REQUIRE(w.x0 + w.bx <= X && w.y0 + w.by <= Y && w.z0 + w.bz <= Z, IGN_ERR_INVALID,
                "chunks_cut: box %llu lies outside the cutout", (unsigned long long)r);
    const uint64_t n = w.bx * w.by * w.bz * nc;
    most = n > most ? n : most;
  }
  if (n_rows == 0) return dispatch_chunk(dtype, "chunks_cut", [](auto) { return IGN_OK; });
  ScratchFrame f(ctx);
  CutRow* dr;
  IGN_TRY(f.take(&dr, n_rows));
  IGN_CUDA(cudaMemcpyAsync(dr, hr, n_rows * sizeof(CutRow), cudaMemcpyHostToDevice, ctx->stream));
  IGN_CUDA(cudaMemsetAsync(all_bg, 1, n_rows * 4, ctx->stream));  // 0x01010101: non-zero = all background
  const dim3 g = rows_grid(n_rows, most);
  return dispatch_chunk(dtype, "chunks_cut", [&](auto t) -> int {
    using T = decltype(t);
    IGN_LAUNCH(ctx, k_chunks_cut<T>, g, 256, 0, (const T*)cutout, X, Y, Z, nc, (const CutRow*)dr, n_rows,
               bg_value<T>(background), (char*)packed, all_bg);
    return IGN_OK;
  });
}

int ign_fill_box_dev(ign_ctx* ctx, void* cutout, int dtype, uint64_t X, uint64_t Y, uint64_t Z, uint64_t nc,
                     uint64_t x0, uint64_t y0, uint64_t z0, uint64_t bx, uint64_t by, uint64_t bz, uint64_t value) {
  IGN_TRY(activate(ctx));
  IGN_REQUIRE(x0 <= X && bx <= X - x0 && y0 <= Y && by <= Y - y0 && z0 <= Z && bz <= Z - z0, IGN_ERR_INVALID,
              "fill_box: box (%llu, %llu, %llu) + (%llu, %llu, %llu) lies outside the %llu x %llu x %llu cutout",
              (unsigned long long)x0, (unsigned long long)y0, (unsigned long long)z0, (unsigned long long)bx,
              (unsigned long long)by, (unsigned long long)bz, (unsigned long long)X, (unsigned long long)Y,
              (unsigned long long)Z);
  const uint64_t n = bx * by * bz * nc;
  IGN_REQUIRE(n == 0 || cutout, IGN_ERR_INVALID, "fill_box: null cutout");
  return dispatch_chunk(dtype, "fill_box", [&](auto t) -> int {
    using T = decltype(t);
    if (n == 0) return IGN_OK;
    const unsigned grid = (unsigned)std::min<uint64_t>(blocks_for(n, 256), (uint64_t)ctx->sm_count * 32);
    IGN_LAUNCH(ctx, k_fill_box<T>, grid, 256, 0, (T*)cutout, X, Y, Z, x0, y0, z0, bx, by, bz, n, bg_value<T>(value));
    return IGN_OK;
  });
}

}  // extern "C"
