// synth.cu -- synthetic benchmark volumes generated directly in HBM
// (SURVEY.md 8(d)); bit-identical to oracle.synth_seg / oracle.synth_image.
#include "common.cuh"

namespace ign {

__device__ __forceinline__ uint64_t cell_hash(uint64_t seed, int64_t cx, int64_t cy, int64_t cz) {
  uint64_t h = mix64(seed + (uint64_t)cx * 0x100000001B3ull);
  h = mix64(h ^ ((uint64_t)cy * 0xC2B2AE3D27D4EB4Full));
  h = mix64(h ^ ((uint64_t)cz * 0x165667B19E3779F9ull));
  return h;
}

__device__ __forceinline__ int64_t floordiv(int64_t a, int64_t b) {
  int64_t q = a / b;
  if ((a % b != 0) && ((a < 0) != (b < 0))) q--;
  return q;
}

template <typename T>
__global__ void __launch_bounds__(256)
    k_synth_seg(T* __restrict__ out, uint64_t sx, uint64_t sy, uint64_t sz, int64_t ox, int64_t oy,
                int64_t oz, int pitch, uint64_t num_ids, uint64_t seed, uint64_t id_base) {
  const uint64_t total = sx * sy * sz;
  const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int64_t X = (int64_t)(t % sx) + ox;
  const int64_t Y = (int64_t)((t / sx) % sy) + oy;
  const int64_t Z = (int64_t)(t / (sx * sy)) + oz;
  const int64_t cx = floordiv(X, pitch), cy = floordiv(Y, pitch), cz = floordiv(Z, pitch);
  int64_t d1 = INT64_MAX, d2 = INT64_MAX;
  uint64_t id1 = 0;
  for (int dz = -1; dz <= 1; dz++)
    for (int dy = -1; dy <= 1; dy++)
      for (int dx = -1; dx <= 1; dx++) {
        const int64_t ccx = cx + dx, ccy = cy + dy, ccz = cz + dz;
        const uint64_t h = cell_hash(seed, ccx, ccy, ccz);
        const int64_t px = ccx * pitch + (int64_t)((h & 0xFFFF) % (uint64_t)pitch);
        const int64_t py = ccy * pitch + (int64_t)(((h >> 16) & 0xFFFF) % (uint64_t)pitch);
        const int64_t pz = ccz * pitch + (int64_t)(((h >> 32) & 0xFFFF) % (uint64_t)pitch);
        const int64_t d = (X - px) * (X - px) + (Y - py) * (Y - py) + (Z - pz) * (Z - pz);
        if (d < d1) {
          d2 = d1;
          d1 = d;
          id1 = id_base + 1 + mix64(h) % num_ids;
        } else if (d < d2) {
          d2 = d;
        }
      }
  out[t] = ((d2 - d1) < 2 * (int64_t)pitch) ? (T)0 : (T)id1;
}

__global__ void __launch_bounds__(256)
    k_synth_image(uint8_t* __restrict__ out, uint64_t sx, uint64_t sy, uint64_t sz, int64_t ox,
                  int64_t oy, int64_t oz, uint64_t seed) {
  const uint64_t total = sx * sy * sz;
  const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (t >= total) return;
  const int64_t X = (int64_t)(t % sx) + ox;
  const int64_t Y = (int64_t)((t / sx) % sy) + oy;
  const int64_t Z = (int64_t)(t / (sx * sy)) + oz;
  out[t] = (uint8_t)((cell_hash(seed, X, Y, Z) >> 11) % 255);
}

}  // namespace ign

using namespace ign;

extern "C" {

int ign_synth_seg_dev(ign_ctx* ctx, void* out, int dtype, uint64_t sx, uint64_t sy, uint64_t sz,
                      int64_t ox, int64_t oy, int64_t oz, uint32_t pitch, uint64_t num_ids,
                      uint64_t seed, uint64_t id_base) {
  IGN_TRY(activate(ctx));
  IGN_REQUIRE(out && pitch > 0 && num_ids > 0, IGN_ERR_INVALID, "bad synth_seg argument");
  const uint64_t total = sx * sy * sz;
  if (total == 0) return IGN_OK;
  IGN_REQUIRE(total / 256 < 0x7FFFFFFFull, IGN_ERR_OVERFLOW, "volume too large for one launch");
  const unsigned grid = blocks_for(total, 256);
  return dispatch_label(dtype, "synth_seg", [&](auto v) -> int {
    using T = decltype(v);
    IGN_LAUNCH(ctx, (k_synth_seg<T>), grid, 256, 0, (T*)out, sx, sy, sz, ox, oy, oz, (int)pitch, num_ids, seed, id_base);
    return IGN_OK;
  });
}

int ign_synth_image_dev(ign_ctx* ctx, uint8_t* out, uint64_t sx, uint64_t sy, uint64_t sz,
                        int64_t ox, int64_t oy, int64_t oz, uint64_t seed) {
  IGN_TRY(activate(ctx));
  IGN_REQUIRE(out, IGN_ERR_INVALID, "null buffer");
  const uint64_t total = sx * sy * sz;
  if (total == 0) return IGN_OK;
  IGN_REQUIRE(total / 256 < 0x7FFFFFFFull, IGN_ERR_OVERFLOW, "volume too large for one launch");
  IGN_LAUNCH(ctx, k_synth_image, blocks_for(total, 256), 256, 0, out, sx, sy, sz, ox, oy, oz, seed);
  return IGN_OK;
}

}  // extern "C"
