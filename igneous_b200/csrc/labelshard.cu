// labelshard.cu -- hashed label shards (neuroglancer_uint64_sharded_v1, murmurhash3_x86_128) for skeleton
// layers, sm_90a (DESIGN.md §5l).
//
// ign_shard_hash_dev hashes every label of a layer and sorts them by (shard, minishard, label) with two
// stable cub radix sorts (label, then location), then marks where each shard's run starts.  The creator
// runs it on every label of a layer; the task on its own labels, which gives their order in the file.
// ign_skeleton_restrip_dev copies each precomputed blob without its integer attribute sections: the blob
// layout is skelblob.cuh's.  ign_shard_assemble_dev writes the shard index and the minishard indices
// around payloads already in place, so a raw shard leaves the device in one copy.
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>

#include "skelblob.cuh"

namespace ign {

namespace {

__device__ __forceinline__ uint32_t rotl32(uint32_t x, int r) { return (x << r) | (x >> (32 - r)); }

__device__ __forceinline__ uint32_t fmix32(uint32_t h) {
  h ^= h >> 16;
  h *= 0x85ebca6bu;
  h ^= h >> 13;
  h *= 0xc2b2ae35u;
  h ^= h >> 16;
  return h;
}

// MurmurHash3_x86_128, seed 0, of the 8 little-endian bytes of key: no whole 16-byte block, so key is the
// tail; words 1 and 2 of the result, h1 | h2 << 32
__device__ __forceinline__ uint64_t murmur3_x86_128_lo64(uint64_t key) {
  const uint32_t c1 = 0x239b961bu, c2 = 0xab0e9789u, c3 = 0x38b34ae5u;
  uint32_t k1 = (uint32_t)key, k2 = (uint32_t)(key >> 32);
  uint32_t h1 = 0, h2 = 0, h3 = 0, h4 = 0;
  k2 *= c2;
  k2 = rotl32(k2, 16);
  k2 *= c3;
  h2 ^= k2;
  k1 *= c1;
  k1 = rotl32(k1, 15);
  k1 *= c2;
  h1 ^= k1;
  h1 ^= 8u;
  h2 ^= 8u;
  h3 ^= 8u;
  h4 ^= 8u;
  h1 += h2 + h3 + h4;
  h2 += h1;
  h3 += h1;
  h4 += h1;
  h1 = fmix32(h1);
  h2 = fmix32(h2);
  h3 = fmix32(h3);
  h4 = fmix32(h4);
  h1 += h2 + h3 + h4;
  h2 += h1;
  return (uint64_t)h1 | ((uint64_t)h2 << 32);
}

__host__ __device__ __forceinline__ uint64_t low_bits(int b) { return b >= 64 ? ~0ull : (1ull << b) - 1; }

__device__ __forceinline__ uint64_t shard_of(uint64_t loc, int mb) { return mb >= 64 ? 0 : loc >> mb; }

__global__ void __launch_bounds__(256) k_ls_locate(const uint64_t* __restrict__ labels, uint64_t n, int preshift,
                                                   uint64_t mask, uint64_t* __restrict__ loc) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) loc[i] = murmur3_x86_128_lo64(labels[i] >> preshift) & mask;
}

// head[i] = 1 where a shard's run starts; head[n] = 0
__global__ void __launch_bounds__(256) k_ls_heads(const uint64_t* __restrict__ loc, uint64_t n, int mb,
                                                  uint32_t* __restrict__ head) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  head[i] = i < n && (i == 0 || shard_of(loc[i], mb) != shard_of(loc[i - 1], mb));
}

__global__ void __launch_bounds__(256) k_ls_runs(const uint64_t* __restrict__ loc, uint64_t n, int mb,
                                                 const uint32_t* __restrict__ head, const uint32_t* __restrict__ pos,
                                                 uint64_t* __restrict__ run_start, uint64_t* __restrict__ run_shard,
                                                 uint64_t* __restrict__ n_runs) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  if (i == n) {
    run_start[pos[n]] = n;
    *n_runs = pos[n];
  } else if (head[i]) {
    run_start[pos[i]] = i;
    run_shard[pos[i]] = shard_of(loc[i], mb);
  }
}

constexpr int RS_MAX_ATTRS = 32;

struct RsAttrs {
  uint32_t bytes[RS_MAX_ATTRS];  // per vertex
  uint32_t keep[RS_MAX_ATTRS];
  int n;
  uint64_t all, kept;  // bytes per vertex of every attribute / of the kept ones
};

struct RsCtl {
  unsigned long long bad;  // lowest blob row whose length does not match its header
  unsigned long long total;
};

__device__ __forceinline__ uint32_t ld_u32_unaligned(const uint8_t* p) {
  return (uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24);
}

// size[i]: blob i's output length (0 for a bad blob); size[n] = 0 so the scan's last entry is the total
__global__ void __launch_bounds__(256) k_rs_sizes(const uint8_t* __restrict__ blobs, const uint64_t* __restrict__ off,
                                                  uint64_t n, RsAttrs a, uint64_t* __restrict__ size, RsCtl* ctl) {
  const uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i > n) return;
  if (i == n) {
    size[n] = 0;
    return;
  }
  const uint64_t s = off[i], e = off[i + 1];
  uint64_t out = 0;
  bool ok = e >= s + 8;
  if (ok) {
    const uint64_t nv = ld_u32_unaligned(blobs + s), ne = ld_u32_unaligned(blobs + s + 4);
    ok = e - s == sb_head_bytes(nv, ne) + a.all * nv;
    out = sb_head_bytes(nv, ne) + a.kept * nv;
  }
  if (!ok) {
    atomicMin(&ctl->bad, (unsigned long long)i);
    out = 0;
  }
  size[i] = out;
}

// one CTA per blob (grid-strided): the header, vertices and edges, then each kept attribute section
__global__ void __launch_bounds__(256) k_rs_copy(const uint8_t* __restrict__ blobs, const uint64_t* __restrict__ off,
                                                 uint64_t n, RsAttrs a, const uint64_t* __restrict__ out_off,
                                                 uint8_t* __restrict__ out) {
  for (uint64_t i = blockIdx.x; i < n; i += gridDim.x) {
    const uint8_t* src = blobs + off[i];
    uint8_t* dst = out + out_off[i];
    const uint64_t nv = ld_u32_unaligned(src), ne = ld_u32_unaligned(src + 4), head = sb_head_bytes(nv, ne);
    for (uint64_t b = threadIdx.x; b < head; b += blockDim.x) dst[b] = src[b];
    uint64_t s = head, d = head;
    for (int k = 0; k < a.n; ++k) {
      const uint64_t len = (uint64_t)a.bytes[k] * nv;
      if (a.keep[k]) {
        for (uint64_t b = threadIdx.x; b < len; b += blockDim.x) dst[d + b] = src[s + b];
        d += len;
      }
      s += len;
    }
  }
}

__device__ __forceinline__ uint64_t first_mini(const uint64_t* __restrict__ loc, uint64_t n, uint64_t mask,
                                               uint64_t m) {
  uint64_t lo = 0, hi = n;
  while (lo < hi) {
    const uint64_t mid = (lo + hi) >> 1;
    if ((loc[mid] & mask) < m) lo = mid + 1; else hi = mid;
  }
  return lo;
}

__device__ __forceinline__ void st_u64_unaligned(uint8_t* p, uint64_t v) {
  for (int b = 0; b < 8; ++b) p[b] = (uint8_t)(v >> (8 * b));
}

// row j's three entries of its minishard's raw index [3][k]: the label delta, the start delta (the first
// against the end of the shard index, every later one against the end of the previous payload: 0, as the
// payloads are back to back) and the size.  Minishard m's index starts 24 bytes per earlier row after the
// payloads.
__global__ void __launch_bounds__(256) k_sa_minis(const uint64_t* __restrict__ loc, const uint64_t* __restrict__ labels,
                                                  const uint64_t* __restrict__ off, uint64_t n, uint64_t mask,
                                                  uint64_t index_len, uint8_t* __restrict__ shard) {
  const uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const uint64_t m = loc[j] & mask, a = first_mini(loc, n, mask, m);
  const uint64_t b = m == mask ? n : first_mini(loc, n, mask, m + 1), k = b - a, i = j - a;
  uint8_t* w = shard + index_len + off[n] + 24 * a;
  st_u64_unaligned(w + 8 * i, labels[j] - (i ? labels[j - 1] : 0));
  st_u64_unaligned(w + 8 * (k + i), i ? 0 : off[j]);
  st_u64_unaligned(w + 8 * (2 * k + i), off[j + 1] - off[j]);
}

// shard index entry m: (start, end) of minishard m's index, relative to the end of the shard index
__global__ void __launch_bounds__(256) k_sa_index(const uint64_t* __restrict__ loc, uint64_t n, uint64_t mask,
                                                  const uint64_t* __restrict__ off, uint64_t* __restrict__ index) {
  const uint64_t m = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (m > mask) return;
  const uint64_t a = first_mini(loc, n, mask, m), b = m == mask ? n : first_mini(loc, n, mask, m + 1);
  index[2 * m] = off[n] + 24 * a;
  index[2 * m + 1] = off[n] + 24 * b;
}

}  // namespace
}  // namespace ign

using namespace ign;

extern "C" {

int ign_shard_hash_dev(ign_ctx* ctx, const uint64_t* labels, uint64_t n, int preshift_bits, int minishard_bits,
                       int shard_bits, uint64_t* labels_out, uint64_t* locations_out, uint64_t* run_start_out,
                       uint64_t* run_shard_out, uint64_t* n_runs) {
  IGN_TRY(activate(ctx));
  IGN_REQUIRE(n_runs, IGN_ERR_INVALID, "shard_hash: null n_runs");
  *n_runs = 0;
  IGN_REQUIRE(preshift_bits >= 0 && preshift_bits <= 63 && minishard_bits >= 0 && shard_bits >= 0 &&
                  minishard_bits + shard_bits <= 64, IGN_ERR_INVALID,
              "shard_hash: preshift_bits %d (0..63), minishard_bits %d + shard_bits %d (each >= 0, at most 64)",
              preshift_bits, minishard_bits, shard_bits);
  IGN_REQUIRE(n < (1ull << 31), IGN_ERR_OVERFLOW, "shard_hash: %llu labels (below 2^31)", (unsigned long long)n);
  if (n == 0) {
    if (run_start_out) IGN_CUDA(cudaMemsetAsync(run_start_out, 0, 8, ctx->stream));
    IGN_CUDA(cudaStreamSynchronize(ctx->stream));
    return IGN_OK;
  }
  IGN_REQUIRE(labels && labels_out && locations_out && run_start_out && run_shard_out, IGN_ERR_INVALID,
              "shard_hash: null buffer");
  ScratchFrame f(ctx);
  const int bits = minishard_bits + shard_bits;
  uint64_t *lab_s, *loc, *n_dev;
  uint32_t *head, *pos;
  IGN_TRY(f.take(&lab_s, n));
  IGN_TRY(f.take(&loc, n));
  IGN_TRY(f.take(&head, n + 1));
  IGN_TRY(f.take(&pos, n + 1));
  IGN_TRY(f.take(&n_dev, 1));
  size_t tb = 0, t = 0;
  IGN_CUDA(cub::DeviceRadixSort::SortKeys(nullptr, t, labels, lab_s, (int)n, 0, 64, ctx->stream));
  tb = std::max(tb, t);
  IGN_CUDA(cub::DeviceRadixSort::SortPairs(nullptr, t, loc, locations_out, lab_s, labels_out, (int)n, 0,
                                           std::max(bits, 1), ctx->stream));
  tb = std::max(tb, t);
  IGN_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, t, head, pos, (int)n + 1, ctx->stream));
  tb = std::max(tb, t);
  void* tmp;
  IGN_TRY(f.take(&tmp, tb));
  const unsigned g = blocks_for(n, 256), g1 = blocks_for(n + 1, 256);
  // LSD: labels first, then the location; both sorts are stable
  IGN_CUDA(cub::DeviceRadixSort::SortKeys(tmp, tb, labels, lab_s, (int)n, 0, 64, ctx->stream));
  IGN_LAUNCH(ctx, k_ls_locate, g, 256, 0, lab_s, n, preshift_bits, low_bits(bits), loc);
  if (bits) {
    IGN_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tb, loc, locations_out, lab_s, labels_out, (int)n, 0, bits,
                                             ctx->stream));
  } else {
    IGN_CUDA(cudaMemcpyAsync(locations_out, loc, n * 8, cudaMemcpyDeviceToDevice, ctx->stream));
    IGN_CUDA(cudaMemcpyAsync(labels_out, lab_s, n * 8, cudaMemcpyDeviceToDevice, ctx->stream));
  }
  IGN_LAUNCH(ctx, k_ls_heads, g1, 256, 0, locations_out, n, minishard_bits, head);
  IGN_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tb, head, pos, (int)n + 1, ctx->stream));
  IGN_LAUNCH(ctx, k_ls_runs, g1, 256, 0, locations_out, n, minishard_bits, head, pos, run_start_out, run_shard_out,
             n_dev);
  IGN_TRY(small_d2h(ctx, n_runs, n_dev, 8));
  IGN_TRY(small_sync(ctx));
  return IGN_OK;
}

int ign_skeleton_restrip_dev(ign_ctx* ctx, const uint8_t* blobs, const uint64_t* offsets, uint64_t n,
                             const uint32_t* attrs, int n_attrs, uint8_t* out, uint64_t capacity,
                             uint64_t* out_offsets, uint64_t* nbytes) {
  IGN_TRY(activate(ctx));
  IGN_REQUIRE(nbytes, IGN_ERR_INVALID, "skeleton_restrip: null nbytes");
  *nbytes = 0;
  IGN_REQUIRE(n_attrs >= 0 && n_attrs <= RS_MAX_ATTRS && (n_attrs == 0 || attrs), IGN_ERR_INVALID,
              "skeleton_restrip: %d vertex attributes (at most %d, with their table)", n_attrs, RS_MAX_ATTRS);
  IGN_REQUIRE(n < (1ull << 31), IGN_ERR_OVERFLOW, "skeleton_restrip: %llu blobs (below 2^31)",
              (unsigned long long)n);
  IGN_REQUIRE(offsets && out_offsets, IGN_ERR_INVALID, "skeleton_restrip: null offsets");
  RsAttrs a{};
  a.n = n_attrs;
  for (int k = 0; k < n_attrs; ++k) {
    a.bytes[k] = attrs[2 * k];
    a.keep[k] = attrs[2 * k + 1] != 0;
    a.all += a.bytes[k];
    a.kept += a.keep[k] ? a.bytes[k] : 0;
  }
  IGN_REQUIRE(n == 0 || blobs, IGN_ERR_INVALID, "skeleton_restrip: null blobs");
  ScratchFrame f(ctx);
  RsCtl* ctl;
  uint64_t* size;
  IGN_TRY(f.take(&ctl, 1));
  IGN_TRY(f.take(&size, n + 1));
  size_t tb = 0;
  IGN_CUDA(cub::DeviceScan::ExclusiveSum(nullptr, tb, size, out_offsets, (int)n + 1, ctx->stream));
  void* tmp;
  IGN_TRY(f.take(&tmp, tb));
  RsCtl init{~0ull, 0};
  IGN_TRY(small_h2d(ctx, ctl, &init, sizeof(RsCtl)));
  IGN_LAUNCH(ctx, k_rs_sizes, blocks_for(n + 1, 256), 256, 0, blobs, offsets, n, a, size, ctl);
  IGN_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tb, size, out_offsets, (int)n + 1, ctx->stream));
  RsCtl h{};
  IGN_TRY(small_d2h(ctx, &h.bad, ctl, 8));
  IGN_TRY(small_d2h(ctx, &h.total, out_offsets + n, 8));
  IGN_TRY(small_sync(ctx));
  IGN_REQUIRE(h.bad == ~0ull, IGN_ERR_INVALID,
              "skeleton_restrip: blob row %llu: its length does not match the 8 + 12 nv + 8 ne + %llu nv bytes its "
              "header and the %d vertex attributes describe", h.bad, (unsigned long long)a.all, n_attrs);
  IGN_REQUIRE(capacity >= h.total, IGN_ERR_INVALID, "skeleton_restrip: capacity %llu bytes below the %llu written",
              (unsigned long long)capacity, h.total);
  if (n) {
    IGN_REQUIRE(out, IGN_ERR_INVALID, "skeleton_restrip: null out");
    IGN_LAUNCH(ctx, k_rs_copy, (unsigned)std::min<uint64_t>(n, 1u << 20), 128, 0, blobs, offsets, n, a, out_offsets,
               out);
  }
  *nbytes = h.total;
  return IGN_OK;
}

int ign_shard_assemble_dev(ign_ctx* ctx, const uint64_t* locations, const uint64_t* labels, const uint64_t* offsets,
                           uint64_t n, int minishard_bits, uint8_t* shard, uint64_t capacity, uint64_t* nbytes) {
  IGN_TRY(activate(ctx));
  IGN_REQUIRE(nbytes, IGN_ERR_INVALID, "shard_assemble: null nbytes");
  *nbytes = 0;
  IGN_REQUIRE(minishard_bits >= 0 && minishard_bits <= 32, IGN_ERR_INVALID,
              "shard_assemble: minishard_bits %d (0..32)", minishard_bits);
  IGN_REQUIRE(n < (1ull << 40), IGN_ERR_OVERFLOW, "shard_assemble: %llu payloads", (unsigned long long)n);
  IGN_REQUIRE(offsets && shard && (n == 0 || (locations && labels)), IGN_ERR_INVALID, "shard_assemble: null buffer");
  IGN_REQUIRE(((uintptr_t)shard & 7) == 0, IGN_ERR_INVALID, "shard_assemble: the shard must be aligned to 8 bytes");
  const uint64_t mask = (1ull << minishard_bits) - 1, index_len = 16ull << minishard_bits;
  uint64_t payload = 0;
  IGN_TRY(small_d2h(ctx, &payload, offsets + n, 8));
  IGN_TRY(small_sync(ctx));
  const uint64_t total = index_len + payload + 24 * n;
  IGN_REQUIRE(capacity >= total, IGN_ERR_INVALID, "shard_assemble: capacity %llu bytes below the %llu of the file",
              (unsigned long long)capacity, (unsigned long long)total);
  if (n) IGN_LAUNCH(ctx, k_sa_minis, blocks_for(n, 256), 256, 0, locations, labels, offsets, n, mask, index_len, shard);
  IGN_LAUNCH(ctx, k_sa_index, blocks_for(mask + 1, 256), 256, 0, locations, n, mask, offsets, (uint64_t*)shard);
  *nbytes = total;
  return IGN_OK;
}

}  // extern "C"
