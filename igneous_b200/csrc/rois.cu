// rois.cu -- the threshold of compute_rois
//
// compute_rois (igneous/task_creation/image.py:1995-2058) thresholds each z slab of the top mip, labels it
// with cc3d (26-connected), drops dust and keeps cc3d.statistics' bounding boxes.  The threshold is here;
// the parts, dust and boxes are ign_label_parts_dev's (parts.cu).
#include <string.h>

#include <algorithm>
#include <type_traits>

#include "common.cuh"

namespace ign {

namespace {

template <typename T>
__global__ void __launch_bounds__(256) k_threshold(const T* __restrict__ in, uint64_t n, T t, uint8_t* __restrict__ out) {
  for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x)
    out[i] = in[i] > t;
}

}  // namespace

}  // namespace ign

using namespace ign;

extern "C" {

int ign_threshold_dev(ign_ctx* ctx, const void* in, int dtype, uint64_t n, uint64_t t, uint8_t* out) {
  IGN_TRY(activate(ctx));
  IGN_REQUIRE(n == 0 || (in && out), IGN_ERR_INVALID, "threshold: null buffer");
  return dispatch_chunk(dtype, "threshold", [&](auto v) -> int {
    using T = decltype(v);
    if (n == 0) return IGN_OK;
    T tt;
    if constexpr (std::is_same<T, float>::value) {
      const uint32_t bits = (uint32_t)t;
      memcpy(&tt, &bits, 4);
    } else if (t > (uint64_t)(T)~(T)0) {  // above every value of T: nothing is greater
      IGN_CUDA(cudaMemsetAsync(out, 0, n, ctx->stream));
      return IGN_OK;
    } else {
      tt = (T)t;
    }
    const unsigned grid = (unsigned)std::min<uint64_t>(blocks_for(n, 256), (uint64_t)ctx->sm_count * 32);
    IGN_LAUNCH(ctx, k_threshold<T>, grid, 256, 0, (const T*)in, n, tt, out);
    return IGN_OK;
  });
}

}  // extern "C"
