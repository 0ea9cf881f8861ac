// cseg.cu -- Precomputed `compressed_segmentation` chunk codec on the device
//
// SURVEY.md 8(f) row 1: the wire format either side of the hot path.  CloudVolume encodes /
// decodes it on the host around igneous/tasks/image/image.py:57-100 (every mip a
// DownsampleTask uploads) and igneous/tasks/image/ccl.py:346-356 (RelabelCCLTask's output;
// the CLI's default CCL encoding is compresso, `igneous_cli/cli.py:750`, with
// compressed_segmentation as the other segmentation codec).  Encoding where the labels
// already are shrinks the D2H of a label chunk by the compression ratio.
//
// Format (Neuroglancer): per channel [2 x u32 header per 8x8x8 block | per block: packed
// indices, then -- unless an identical table was already emitted by an earlier block of the
// channel -- the sorted lookup table]; header = (table offset : 24 | bits << 24), offset of the
// packed indices; bits in {0,1,2,4,8,16,32}; offsets in u32 words from the channel start.
// The emission order of oracle/igneous_oracle.c::orc_cseg_encode_* (block raster order, a
// table is emitted by the FIRST block that uses it) is reproduced exactly, so the streams are
// byte-identical.
//
// One encoder and one decoder serve every entry point; a single chunk is a batch of one.  N chunks
// x sc channels are S = N*sc segments, one channel stream each, and all their blocks one global
// block range (segment-major, raster order inside a segment):
//   1  k_cb_scan<T, false>  one warp per block: the distinct values are extracted in ascending
//      order (repeated warp minimum) -> n, smallest / largest value, 64-bit hash (segment included)
//   2  radix sort of (hash, block) -> the first block of every run of equal hashes is the owner
//      candidate; k_cb_verify compares each block's segment and table with its candidate's.  Equal
//      hashes do not prove equal tables: after a mismatch k_cb_resolve recomputes every owner by
//      content, so the owner is always the first block of its segment with an identical table
//   3  exclusive scan of the per-block sizes (k_cb_sizes) -> offsets; k_cb_segments places every
//      segment and checks the format's 24-bit table offsets.  Segment s = (chunk i, channel c)
//      starts at word scan[b0_s] + 2*b0_s + sc*(i + 1) of the concatenated chunk files (chunk i's
//      sc-word channel table precedes its channels)
//   4  k_cb_scan<T, true>   the same extraction again, now writing indices, tables, headers
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include <algorithm>
#include <vector>

#include "common.cuh"

namespace ign {

constexpr unsigned CS_FULL = 0xFFFFFFFFu;
constexpr int CS_MAX_BVOX = 1024;  // voxels per block (8x8x8 = 512 is the standard)

struct CsegDims {
  uint32_t sx, sy, sz, bx, by, bz, gx, gy, gz, bvox;
};

__device__ __forceinline__ uint64_t cs_shfl_xor(uint64_t v, int m) {
  return ((uint64_t)__shfl_xor_sync(CS_FULL, (uint32_t)(v >> 32), m) << 32) | __shfl_xor_sync(CS_FULL, (uint32_t)v, m);
}
__device__ __forceinline__ uint32_t cs_bits(uint32_t n) {
  if (n <= 1) return 0;
  uint32_t b = 1;
  while ((1u << b) < n) b *= 2;
  return b;
}

// lane l of the warp loads positions l, l+32, ... of block b (position p = (z*by + y)*bx + x);
// returns the mask of slots inside the volume
template <typename T, int CS_PER_LANE>
__device__ __forceinline__ uint32_t cs_load(const T* __restrict__ in, const CsegDims& d, uint64_t b, uint32_t lane,
                                            uint64_t (&val)[CS_PER_LANE]) {
  const uint32_t gxx = (uint32_t)(b % d.gx), gyy = (uint32_t)((b / d.gx) % d.gy), gzz = (uint32_t)(b / ((uint64_t)d.gx * d.gy));
  const uint32_t x0 = gxx * d.bx, y0 = gyy * d.by, z0 = gzz * d.bz;
  uint32_t have = 0;
#pragma unroll
  for (int k = 0; k < CS_PER_LANE; k++) {
    const uint32_t p = lane + 32 * k;
    val[k] = 0;
    if (p < d.bvox) {
      const uint32_t x = p % d.bx, y = (p / d.bx) % d.by, z = p / (d.bx * d.by);
      if (x0 + x < d.sx && y0 + y < d.sy && z0 + z < d.sz) {
        val[k] = (uint64_t)in[(x0 + x) + (uint64_t)d.sx * ((y0 + y) + (uint64_t)d.sy * (z0 + z))];
        have |= 1u << k;
      }
    }
  }
  return have;
}

// smallest value of the warp's slots still in `todo` (the same on every lane)
template <int CS_PER_LANE>
__device__ __forceinline__ uint64_t cs_warp_min(const uint64_t (&val)[CS_PER_LANE], uint32_t todo) {
  uint64_t m = ~0ull;
#pragma unroll
  for (int k = 0; k < CS_PER_LANE; k++)
    if ((todo >> k) & 1u) m = val[k] < m ? val[k] : m;
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) {
    const uint64_t o = cs_shfl_xor(m, s);
    m = o < m ? o : m;
  }
  return m;
}

// Do blocks a and b, both of n distinct values, hold the same values?  Called by a whole warp;
// the two sorted tables are extracted side by side and compared value by value.
template <typename T, int CS_PER_LANE>
__device__ bool cs_same_table(const T* __restrict__ in, const CsegDims& d, uint64_t a, uint64_t b, uint32_t n,
                              uint32_t lane) {
  uint64_t va[CS_PER_LANE], vb[CS_PER_LANE];
  uint32_t ta = cs_load<T, CS_PER_LANE>(in, d, a, lane, va);
  uint32_t tb = cs_load<T, CS_PER_LANE>(in, d, b, lane, vb);
  for (uint32_t i = 0; i < n; i++) {
    const uint64_t ma = cs_warp_min<CS_PER_LANE>(va, ta), mb = cs_warp_min<CS_PER_LANE>(vb, tb);
    if (ma != mb) return false;
#pragma unroll
    for (int k = 0; k < CS_PER_LANE; k++) {
      if (va[k] == ma) ta &= ~(1u << k);
      if (vb[k] == mb) tb &= ~(1u << k);
    }
  }
  return true;
}

__global__ void __launch_bounds__(256) k_iota32(uint32_t* p, uint32_t n) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = i;
}

// sorted (hash, block): the head of every run of equal hashes owns the table (the sort is stable
// and the blocks entered it in ascending order, so the head is the smallest block of the run)
__global__ void __launch_bounds__(256)
    k_cseg_heads(const unsigned long long* __restrict__ shash, uint32_t n, uint32_t* __restrict__ headpos) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) headpos[i] = (i == 0 || shash[i - 1] != shash[i]) ? i : 0u;
}
__global__ void __launch_bounds__(256)
    k_cseg_owner(const uint32_t* __restrict__ headpos, const uint32_t* __restrict__ sblock, uint32_t n,
                 uint32_t* __restrict__ owner) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) owner[sblock[i]] = sblock[headpos[i]];  // headpos: inclusive max-scan of the head positions
}

// value of voxel (x, y, z) in block b of one channel stream of nwords words; false: malformed stream
template <typename T>
__device__ __forceinline__ bool cs_decode_voxel(const uint32_t* __restrict__ in, uint64_t nwords, const CsegDims& d,
                                                uint32_t x, uint32_t y, uint32_t z, uint64_t b, uint64_t* out) {
  constexpr int WORDS = sizeof(T) / 4;
  if (2 * b + 1 >= nwords) return false;
  const uint32_t h0 = in[2 * b], h1 = in[2 * b + 1];
  const uint32_t bits = h0 >> 24;
  const uint64_t toff = h0 & 0xFFFFFFu, voff = h1;
  if (!(bits == 0 || bits == 1 || bits == 2 || bits == 4 || bits == 8 || bits == 16 || bits == 32)) return false;
  uint64_t idx = 0;
  if (bits) {
    const uint64_t bitpos = (uint64_t)(((z % d.bz) * d.by + (y % d.by)) * d.bx + (x % d.bx)) * bits;
    const uint64_t w = voff + bitpos / 32;
    if (w >= nwords) return false;
    idx = (in[w] >> (bitpos % 32)) & (bits == 32 ? 0xFFFFFFFFu : ((1u << bits) - 1u));
  }
  const uint64_t tw = toff + idx * WORDS;
  if (tw + WORDS > nwords) return false;
  uint64_t v = in[tw];
  if (WORDS == 2) v |= (uint64_t)in[tw + 1] << 32;
  *out = v;
  return true;
}

static int cseg_dims(uint64_t sx, uint64_t sy, uint64_t sz, uint32_t bx, uint32_t by, uint32_t bz, CsegDims* d) {
  IGN_REQUIRE(sx && sy && sz && bx && by && bz, IGN_ERR_INVALID, "cseg: empty chunk or block");
  IGN_REQUIRE((uint64_t)bx * by * bz <= CS_MAX_BVOX, IGN_ERR_UNSUPPORTED, "cseg: blocks of more than %d voxels are not supported", CS_MAX_BVOX);
  IGN_REQUIRE(sx < (1u << 20) && sy < (1u << 20) && sz < (1u << 20), IGN_ERR_OVERFLOW, "cseg: chunk extent too large");
  d->sx = (uint32_t)sx; d->sy = (uint32_t)sy; d->sz = (uint32_t)sz;
  d->bx = bx; d->by = by; d->bz = bz;
  d->gx = (uint32_t)((sx + bx - 1) / bx); d->gy = (uint32_t)((sy + by - 1) / by); d->gz = (uint32_t)((sz + bz - 1) / bz);
  d->bvox = bx * by * bz;
  IGN_REQUIRE((uint64_t)d->gx * d->gy * d->gz < (1u << 23), IGN_ERR_OVERFLOW,
              "cseg: %llu blocks exceed the format's 24-bit table offsets; encode Precomputed chunks, not whole volumes",
              (unsigned long long)((uint64_t)d->gx * d->gy * d->gz));
  return IGN_OK;
}

// one segment: channel c of chunk i
struct CsegSeg {
  CsegDims d;
  uint64_t in_off;    // element offset of the channel in the packed chunks
  uint64_t b0;        // first global block
  uint64_t chunk;     // i
  uint32_t chan;      // c
};

__device__ __forceinline__ uint64_t cb_find(const CsegSeg* __restrict__ segs, uint64_t nseg, uint64_t g) {
  uint64_t lo = 0, hi = nseg;  // last segment whose b0 <= g
  while (hi - lo > 1) {
    const uint64_t mid = (lo + hi) / 2;
    if (segs[mid].b0 <= g) lo = mid; else hi = mid;
  }
  return lo;
}

// One warp per block.  WRITE = false: n[g], the block's segment, hash[g] and the smallest / largest
// value lo[g], hi[g].  WRITE = true: the stream.  hash_mask keeps only some bits of the hash
// (IGN_CSEG_HASH_BITS, a test knob that forces collisions); the hash only groups candidates,
// k_cb_verify decides by content.
// k_cb_scan and k_cb_resolve hold their segment's dims in registers; under __launch_bounds__(128)
// ptxas spilled a few of them (16 / 40 bytes).  An explicit register cap lets it keep everything in
// registers.  Both launch 128 threads.
template <typename T, bool WRITE, int CS_PER_LANE>
__global__ void __maxnreg__(128)
    k_cb_scan(const T* __restrict__ in, const CsegSeg* __restrict__ segs, uint64_t nseg, uint64_t nblock, uint64_t sc,
              uint32_t* __restrict__ info_n, uint32_t* __restrict__ bseg, unsigned long long* __restrict__ hash,
              unsigned long long hash_mask, unsigned long long* __restrict__ lo, unsigned long long* __restrict__ hi,
              const unsigned long long* __restrict__ scan, const uint32_t* __restrict__ owner, uint32_t* __restrict__ out) {
  constexpr int WORDS = sizeof(T) / 4;
  const uint32_t lane = threadIdx.x & 31u;
  const uint64_t g = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5;
  if (g >= nblock) return;
  const uint64_t s = cb_find(segs, nseg, g);
  const CsegDims d = segs[s].d;
  const uint64_t b0 = segs[s].b0, chunk = segs[s].chunk;
  const uint64_t b = g - b0;
  const T* src = in + segs[s].in_off;
  uint64_t val[CS_PER_LANE];
  uint32_t idx[CS_PER_LANE] = {};
  const uint32_t have = cs_load<T, CS_PER_LANE>(src, d, b, lane, val);
  uint32_t todo = have;
  uint32_t n = 0;
  // the segment joins the hash from the start, so that it need not stay live through the extraction
  uint64_t h = WRITE ? 0 : mix64(0x9E3779B97F4A7C15ull ^ (s * 0xD6E8FEB86659FD93ull)), first = 0, m = 0;
  if (!WRITE && lane == 0) bseg[g] = (uint32_t)s;
  uint32_t* seg_out = nullptr;
  uint32_t toff = 0, eoff = 0;
  bool own = false;
  const uint32_t nb = d.gx * d.gy * d.gz;
  if (WRITE) {
    const uint64_t base0 = scan[b0];
    seg_out = out + base0 + 2 * b0 + sc * (chunk + 1);
    const uint32_t o = owner[g];
    own = o == (uint32_t)g;
    eoff = (uint32_t)(2 * nb + scan[g] - base0);
    toff = (uint32_t)(2 * nb + scan[o] - base0 + (cs_bits(info_n[o]) * d.bvox + 31) / 32);
  }
  while (__any_sync(CS_FULL, todo != 0)) {
    m = cs_warp_min<CS_PER_LANE>(val, todo);
#pragma unroll
    for (int k = 0; k < CS_PER_LANE; k++)
      if (((todo >> k) & 1u) && val[k] == m) {
        idx[k] = n;
        todo &= ~(1u << k);
      }
    if (WRITE) {
      if (own && lane == 0) {
        seg_out[toff + n * WORDS] = (uint32_t)m;
        if (WORDS == 2) seg_out[toff + n * WORDS + 1] = (uint32_t)(m >> 32);
      }
    } else {
      if (n == 0) first = m;
      h = mix64(h ^ m);
    }
    n++;
  }
  const uint32_t bits = cs_bits(n);
  if (!WRITE) {
    if (lane == 0) {
      info_n[g] = n;
      hash[g] = mix64(h + n) & hash_mask;
      lo[g] = first;
      hi[g] = m;
    }
    return;
  }
  // packed indices: word w of the block holds positions [w*32/bits, (w+1)*32/bits)
  if (bits) {
    const uint32_t per = 32 / bits;  // values per word
    const uint32_t nwords = (bits * d.bvox + 31) / 32;
    // the values of one word sit in `per` consecutive positions, i.e. in `per` consecutive lanes:
    // OR-reduce over that aligned group of lanes (per is a power of two <= 32)
#pragma unroll
    for (int k = 0; k < CS_PER_LANE; k++) {
      const uint32_t p = lane + 32 * k;
      if (32 * k >= d.bvox) break;
      const uint32_t v = ((have >> k) & 1u) ? idx[k] : 0u;
      uint32_t word = v << ((p % per) * bits);
      for (uint32_t sh = 1; sh < per; sh <<= 1) word |= __shfl_xor_sync(CS_FULL, word, sh);
      if (p < d.bvox && (p % per) == 0 && p / per < nwords) seg_out[eoff + p / per] = word;
    }
  }
  if (lane == 0) {
    seg_out[2 * b] = toff | (bits << 24);
    seg_out[2 * b + 1] = eoff;
  }
}

// owner of every block whose hash run head is in another segment or holds another table -> *collided
template <typename T, int CS_PER_LANE>
__global__ void __launch_bounds__(128)
    k_cb_verify(const T* __restrict__ in, const CsegSeg* __restrict__ segs, uint32_t nblock,
                const uint32_t* __restrict__ bseg, const uint32_t* __restrict__ n, const unsigned long long* __restrict__ lo,
                const unsigned long long* __restrict__ hi, const uint32_t* __restrict__ owner, uint32_t* __restrict__ collided) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t g = (uint32_t)((blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5);
  if (g >= nblock) return;
  const uint32_t o = owner[g];
  if (o == g) return;
  bool same = bseg[o] == bseg[g] && n[o] == n[g] && lo[o] == lo[g] && hi[o] == hi[g];
  if (same && n[g] > 2) {
    const uint32_t sg = bseg[g];
    const CsegDims d = segs[sg].d;
    const uint32_t b0 = (uint32_t)segs[sg].b0;
    same = cs_same_table<T, CS_PER_LANE>(in + segs[sg].in_off, d, o - b0, g - b0, n[g], lane);
  }
  if (!same && lane == 0) *collided = 1;
}

template <typename T, int CS_PER_LANE>
__global__ void __maxnreg__(255)
    k_cb_resolve(const T* __restrict__ in, const CsegSeg* __restrict__ segs, uint32_t nblock,
                 const uint32_t* __restrict__ bseg, const uint32_t* __restrict__ n, const unsigned long long* __restrict__ lo,
                 const unsigned long long* __restrict__ hi, const uint32_t* __restrict__ sblock,
                 const uint32_t* __restrict__ headpos, uint32_t* __restrict__ owner) {
  const uint32_t lane = threadIdx.x & 31u;
  const uint32_t i = (uint32_t)((blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5);
  if (i >= nblock) return;
  const uint32_t g = sblock[i];
  const uint32_t sg = bseg[g], ng = n[g];
  const unsigned long long log = lo[g], hig = hi[g];
  const CsegDims d = segs[sg].d;
  const T* src = in + segs[sg].in_off;
  const uint32_t b0 = (uint32_t)segs[sg].b0;
  uint32_t own = g;
  for (uint32_t base = headpos[i]; base < i && own == g; base += 32) {
    const uint32_t j = base + lane;
    const uint32_t c = j < i ? sblock[j] : 0u;
    uint32_t cand = __ballot_sync(CS_FULL, j < i && bseg[c] == sg && n[c] == ng && lo[c] == log && hi[c] == hig);
    while (cand) {
      const uint32_t cb = __shfl_sync(CS_FULL, c, __ffs(cand) - 1);
      if (ng <= 2 || cs_same_table<T, CS_PER_LANE>(src, d, cb - b0, g - b0, ng, lane)) {
        own = cb;
        break;
      }
      cand &= cand - 1;
    }
  }
  if (lane == 0) owner[g] = own;
}

template <int WORDS>
__global__ void __launch_bounds__(256)
    k_cb_sizes(const CsegSeg* __restrict__ segs, const uint32_t* __restrict__ bseg, const uint32_t* __restrict__ n,
               const uint32_t* __restrict__ owner, uint32_t nblock, unsigned long long* __restrict__ size) {
  const uint32_t g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= nblock) return;
  const uint32_t bvox = segs[bseg[g]].d.bvox;
  size[g] = (cs_bits(n[g]) * bvox + 31) / 32 + (owner[g] == g ? n[g] * WORDS : 0u);
}

// one thread per segment: its stream length (-> *too_long past the format's 24-bit offsets); with out
// set, also its entry in its chunk's channel table, (channel 0) the chunk's word offset in the output and
// (the last segment) the end of the output
__global__ void __launch_bounds__(256)
    k_cb_segments(const CsegSeg* __restrict__ segs, uint64_t nseg, uint64_t sc, const unsigned long long* __restrict__ scan,
                  uint32_t* __restrict__ too_long, uint32_t* __restrict__ out, unsigned long long* __restrict__ offsets) {
  const uint64_t s = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (s >= nseg) return;
  const CsegSeg& S = segs[s];
  const uint64_t nb = (uint64_t)S.d.gx * S.d.gy * S.d.gz;
  const uint64_t start = scan[S.b0] + 2 * S.b0 + sc * (S.chunk + 1);
  const uint64_t words = 2 * nb + scan[S.b0 + nb] - scan[S.b0];
  if (words > 0xFFFFFFull + 1024) atomicMax(too_long, 1u);
  if (!out) return;
  const uint64_t cstart = scan[segs[s - S.chan].b0] + 2 * segs[s - S.chan].b0 + sc * S.chunk;  // chunk i's first word
  out[cstart + S.chan] = (uint32_t)(start - cstart);
  if (S.chan == 0) offsets[S.chunk] = cstart;
  if (s == nseg - 1) offsets[S.chunk + 1] = start + words;
}

template <typename T>
__global__ void __launch_bounds__(256)
    k_cb_decode(const uint32_t* __restrict__ in, const unsigned long long* __restrict__ word_off,
                const CsegSeg* __restrict__ segs, uint64_t nseg, uint64_t sc, T* __restrict__ out, uint32_t* __restrict__ bad) {
  for (uint64_t s = blockIdx.y; s < nseg; s += gridDim.y) {
    const CsegSeg& S = segs[s];
    const CsegDims d = S.d;
    const uint64_t i0 = word_off[S.chunk], nw = word_off[S.chunk + 1] - i0;
    const uint32_t* chunk = in + i0;
    const uint64_t n = (uint64_t)d.sx * d.sy * d.sz;
    const uint64_t base = sc <= nw ? chunk[S.chan] : ~0ull;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
      if (base > nw) { atomicMin(bad, (uint32_t)S.chunk); break; }
      const uint32_t* ch = chunk + base;
      const uint64_t nwords = nw - base;
      const uint32_t x = (uint32_t)(i % d.sx), y = (uint32_t)((i / d.sx) % d.sy), z = (uint32_t)(i / ((uint64_t)d.sx * d.sy));
      const uint64_t b = (x / d.bx) + (uint64_t)d.gx * ((y / d.by) + (uint64_t)d.gy * (z / d.bz));
      uint64_t v;
      if (!cs_decode_voxel<T>(ch, nwords, d, x, y, z, b, &v)) { atomicMin(bad, (uint32_t)S.chunk); break; }
      out[S.in_off + i] = (T)v;
    }
  }
}

// the segment table of n chunks of shapes[i] (host n x 3) with sc channels; *nblock = blocks in all
static int cb_segments(const uint32_t* shapes, uint64_t n, uint64_t sc, uint32_t bx, uint32_t by, uint32_t bz,
                       std::vector<CsegSeg>& segs, uint64_t* nblock) {
  segs.resize(n * sc);
  uint64_t b0 = 0, off = 0;
  for (uint64_t i = 0; i < n; i++) {
    CsegDims d;
    const int st = cseg_dims(shapes[3 * i], shapes[3 * i + 1], shapes[3 * i + 2], bx, by, bz, &d);
    if (st != IGN_OK) {
      set_error("cseg batch: chunk %llu: bad shape or block size (%u x %u x %u, block %u x %u x %u)",
                (unsigned long long)i, shapes[3 * i], shapes[3 * i + 1], shapes[3 * i + 2], bx, by, bz);
      return st;
    }
    const uint64_t nb = (uint64_t)d.gx * d.gy * d.gz, vox = (uint64_t)d.sx * d.sy * d.sz;
    for (uint64_t c = 0; c < sc; c++) {
      segs[i * sc + c] = CsegSeg{d, off, b0, i, (uint32_t)c};
      off += vox;
      b0 += nb;
    }
  }
  *nblock = b0;
  return IGN_OK;
}

template <typename T>
static int cseg_encode_batch(ign_ctx* ctx, const T* in, const std::vector<CsegSeg>& hsegs, uint64_t nblock, uint64_t n,
                             uint64_t sc, uint32_t bvox, uint32_t* out, uint64_t cap_words, uint64_t* offsets,
                             uint64_t* n_words) {
  constexpr int WORDS = sizeof(T) / 4;
  const uint64_t nseg = hsegs.size();
  IGN_REQUIRE(nblock < (1ull << 31), IGN_ERR_OVERFLOW, "cseg batch: %llu blocks in one call (at most 2^31 - 1)",
              (unsigned long long)nblock);
  const uint32_t nb = (uint32_t)nblock;
  unsigned long long hash_mask = ~0ull;
  if (const char* e = getenv("IGN_CSEG_HASH_BITS")) {
    const int k = atoi(e);
    hash_mask = k >= 64 ? ~0ull : k <= 0 ? 0ull : (1ull << k) - 1;
  }
  size_t sortb = 0, scanb = 0, maxb = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, sortb, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                  (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)nb);
  cub::DeviceScan::ExclusiveSum(nullptr, scanb, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, (int)nb + 1);
  cub::DeviceScan::InclusiveScan(nullptr, maxb, (const uint32_t*)nullptr, (uint32_t*)nullptr, cub::Max(), (int)nb);
  const size_t tmpb = std::max(sortb, std::max(scanb, maxb)) + 256;
  ScratchFrame f(ctx);
  CsegSeg* segs;
  unsigned long long *hash, *shash, *lo, *hi, *scan;
  unsigned long long* size;
  uint32_t *cnt, *bseg, *blk, *sblk, *owner, *headpos, *runhead, *flags;
  void* tmp;
  IGN_TRY(f.take(&segs, nseg));
  IGN_TRY(f.take(&hash, nb));
  IGN_TRY(f.take(&shash, nb));
  IGN_TRY(f.take(&lo, nb));
  IGN_TRY(f.take(&hi, nb));
  IGN_TRY(f.take(&scan, (size_t)nb + 1));
  IGN_TRY(f.take(&cnt, (size_t)nb + 1));
  IGN_TRY(f.take(&bseg, (size_t)nb + 1));
  IGN_TRY(f.take(&blk, (size_t)nb + 1));
  IGN_TRY(f.take(&sblk, (size_t)nb + 1));
  IGN_TRY(f.take(&owner, (size_t)nb + 1));
  IGN_TRY(f.take(&size, (size_t)nb + 1));
  IGN_TRY(f.take(&headpos, (size_t)nb + 1));
  IGN_TRY(f.take(&runhead, (size_t)nb + 1));
  IGN_TRY(f.take(&flags, 2));  // [collided, too_long]
  IGN_TRY(f.take(&tmp, tmpb));
  IGN_TRY(small_h2d(ctx, segs, hsegs.data(), nseg * sizeof(CsegSeg)));
  IGN_CUDA(cudaMemsetAsync(flags, 0, 8, ctx->stream));
  const unsigned gw = blocks_for((uint64_t)nb * 32, 128);
  const bool wide = bvox > 512;
#define CB_LAUNCH_PL(kernel, ...)                                        \
  do {                                                                   \
    if (!wide) IGN_LAUNCH(ctx, (kernel<T, 16>), gw, 128, 0, __VA_ARGS__); \
    else IGN_LAUNCH(ctx, (kernel<T, 32>), gw, 128, 0, __VA_ARGS__);       \
  } while (0)
  if (!wide)
    IGN_LAUNCH(ctx, (k_cb_scan<T, false, 16>), gw, 128, 0, in, (const CsegSeg*)segs, nseg, nblock, sc, cnt, bseg, hash,
               hash_mask, lo, hi, (const unsigned long long*)nullptr, (const uint32_t*)nullptr, (uint32_t*)nullptr);
  else
    IGN_LAUNCH(ctx, (k_cb_scan<T, false, 32>), gw, 128, 0, in, (const CsegSeg*)segs, nseg, nblock, sc, cnt, bseg, hash,
               hash_mask, lo, hi, (const unsigned long long*)nullptr, (const uint32_t*)nullptr, (uint32_t*)nullptr);
  IGN_LAUNCH(ctx, k_iota32, blocks_for(nb, 256), 256, 0, blk, nb);
  {
    size_t tb = tmpb;
    IGN_CUDA(cub::DeviceRadixSort::SortPairs(tmp, tb, hash, shash, blk, sblk, (int)nb, 0, 64, ctx->stream));
    ctx->launches += 9;
  }
  IGN_LAUNCH(ctx, k_cseg_heads, blocks_for(nb, 256), 256, 0, shash, nb, headpos);
  {
    size_t tb = tmpb;
    IGN_CUDA(cub::DeviceScan::InclusiveScan(tmp, tb, headpos, runhead, cub::Max(), (int)nb, ctx->stream));
    ctx->launches += 2;
  }
  IGN_LAUNCH(ctx, k_cseg_owner, blocks_for(nb, 256), 256, 0, runhead, sblk, nb, owner);
  CB_LAUNCH_PL(k_cb_verify, in, (const CsegSeg*)segs, nb, (const uint32_t*)bseg, (const uint32_t*)cnt,
               (const unsigned long long*)lo, (const unsigned long long*)hi, (const uint32_t*)owner, flags);
  // the collision flag comes back with the total; only after a collision is there a second round trip
  uint32_t hflags[2] = {0, 0};
  unsigned long long total_data = 0;
  for (int pass = 0;; pass++) {
    IGN_LAUNCH(ctx, (k_cb_sizes<WORDS>), blocks_for(nb, 256), 256, 0, (const CsegSeg*)segs, (const uint32_t*)bseg,
               (const uint32_t*)cnt, (const uint32_t*)owner, nb, size);
    IGN_CUDA(cudaMemsetAsync(size + nb, 0, 8, ctx->stream));
    {
      size_t tb = tmpb;
      IGN_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tb, size, scan, (int)nb + 1, ctx->stream));
      ctx->launches += 2;
    }
    // the sizes pass: the 24-bit check, nothing written yet
    IGN_LAUNCH(ctx, k_cb_segments, blocks_for(nseg, 256), 256, 0, (const CsegSeg*)segs, nseg, sc,
               (const unsigned long long*)scan, flags + 1, (uint32_t*)nullptr, (unsigned long long*)nullptr);
    IGN_TRY(small_d2h(ctx, &total_data, scan + nb, 8));
    IGN_TRY(small_d2h(ctx, hflags, flags, 8));
    IGN_TRY(small_sync(ctx));
    if (pass > 0 || hflags[0] == 0) break;
    CB_LAUNCH_PL(k_cb_resolve, in, (const CsegSeg*)segs, nb, (const uint32_t*)bseg, (const uint32_t*)cnt,
                 (const unsigned long long*)lo, (const unsigned long long*)hi, (const uint32_t*)sblk,
                 (const uint32_t*)runhead, owner);
    IGN_CUDA(cudaMemsetAsync(flags + 1, 0, 4, ctx->stream));  // too_long again, from the resolved sizes
  }
#undef CB_LAUNCH_PL
  const uint64_t total = total_data + 2ull * nb + sc * n;
  *n_words = total;
  IGN_REQUIRE(hflags[1] == 0, IGN_ERR_OVERFLOW,
              "cseg: a chunk's channel stream exceeds the format's 24-bit table offsets");
  IGN_REQUIRE(total <= cap_words, IGN_ERR_OVERFLOW, "cseg: %llu words needed, the output holds %llu",
              (unsigned long long)total, (unsigned long long)cap_words);
  IGN_LAUNCH(ctx, k_cb_segments, blocks_for(nseg, 256), 256, 0, (const CsegSeg*)segs, nseg, sc,
             (const unsigned long long*)scan, flags + 1, out, (unsigned long long*)offsets);
  if (!wide)
    IGN_LAUNCH(ctx, (k_cb_scan<T, true, 16>), gw, 128, 0, in, (const CsegSeg*)segs, nseg, nblock, sc, cnt,
               (uint32_t*)nullptr, (unsigned long long*)nullptr, hash_mask, (unsigned long long*)nullptr,
               (unsigned long long*)nullptr, (const unsigned long long*)scan, (const uint32_t*)owner, out);
  else
    IGN_LAUNCH(ctx, (k_cb_scan<T, true, 32>), gw, 128, 0, in, (const CsegSeg*)segs, nseg, nblock, sc, cnt,
               (uint32_t*)nullptr, (unsigned long long*)nullptr, hash_mask, (unsigned long long*)nullptr,
               (unsigned long long*)nullptr, (const unsigned long long*)scan, (const uint32_t*)owner, out);
  return IGN_OK;
}

// n streams, stream i at streams[word_offsets[i] .. word_offsets[i+1]) (offsets on the host), of the
// chunks of shapes[i] (host n x 3) -> the packed chunks in out
static int cseg_decode_batch(ign_ctx* ctx, const uint32_t* streams, const uint64_t* word_offsets, uint64_t n_streams,
                             int dtype, const uint32_t* shapes, uint64_t sc, uint32_t bx, uint32_t by, uint32_t bz,
                             void* out) {
  for (uint64_t i = 0; i < n_streams; i++)
    IGN_REQUIRE(word_offsets[i] <= word_offsets[i + 1], IGN_ERR_INVALID, "cseg: stream %llu has a negative length",
                (unsigned long long)i);
  std::vector<CsegSeg> hsegs;
  uint64_t nblock = 0, most = 0;
  IGN_TRY(cb_segments(shapes, n_streams, sc, bx, by, bz, hsegs, &nblock));
  for (const CsegSeg& S : hsegs) most = std::max(most, (uint64_t)S.d.sx * S.d.sy * S.d.sz);
  ScratchFrame f(ctx);
  CsegSeg* segs;
  unsigned long long* woff;
  uint32_t* bad;
  IGN_TRY(f.take(&segs, hsegs.size()));
  IGN_TRY(f.take(&woff, n_streams + 1));
  IGN_TRY(f.take(&bad, 1));
  IGN_CUDA(cudaMemcpyAsync(segs, hsegs.data(), hsegs.size() * sizeof(CsegSeg), cudaMemcpyHostToDevice, ctx->stream));
  IGN_CUDA(cudaMemcpyAsync(woff, word_offsets, (n_streams + 1) * 8, cudaMemcpyHostToDevice, ctx->stream));
  IGN_CUDA(cudaMemsetAsync(bad, 0xFF, 4, ctx->stream));
  const uint64_t gx = std::min<uint64_t>(blocks_for(most, 256), 1024);
  const dim3 grid((unsigned)gx, (unsigned)std::min<uint64_t>(hsegs.size(), 65535));
  if (dtype == IGN_U32)
    IGN_LAUNCH(ctx, k_cb_decode<uint32_t>, grid, 256, 0, streams, (const unsigned long long*)woff, (const CsegSeg*)segs,
               (uint64_t)hsegs.size(), sc, (uint32_t*)out, bad);
  else
    IGN_LAUNCH(ctx, k_cb_decode<uint64_t>, grid, 256, 0, streams, (const unsigned long long*)woff, (const CsegSeg*)segs,
               (uint64_t)hsegs.size(), sc, (uint64_t*)out, bad);
  uint32_t hbad = 0;
  IGN_TRY(small_d2h(ctx, &hbad, bad, 4));
  IGN_TRY(small_sync(ctx));
  IGN_REQUIRE(hbad == 0xFFFFFFFFu, IGN_ERR_INVALID, "cseg: stream %u is malformed", hbad);
  return IGN_OK;
}

}  // namespace ign

using namespace ign;

extern "C" {

int ign_cseg_encode_dev(ign_ctx* ctx, const void* labels, int dtype, uint64_t sx, uint64_t sy, uint64_t sz,
                        uint64_t sc, uint32_t bx, uint32_t by, uint32_t bz, uint32_t* out, uint64_t cap_words,
                        uint64_t* n_words) {
  IGN_TRY(activate(ctx));
  IGN_REQUIRE(labels && out && n_words && sc >= 1, IGN_ERR_INVALID, "null argument");
  IGN_REQUIRE(dtype == IGN_U32 || dtype == IGN_U64, IGN_ERR_UNSUPPORTED, "compressed_segmentation holds uint32 / uint64 labels");
  CsegDims d;
  IGN_TRY(cseg_dims(sx, sy, sz, bx, by, bz, &d));
  const uint32_t shape[3] = {d.sx, d.sy, d.sz};
  std::vector<CsegSeg> segs;
  uint64_t nblock = 0;
  IGN_TRY(cb_segments(shape, 1, sc, bx, by, bz, segs, &nblock));
  ScratchFrame f(ctx);
  uint64_t* offsets;  // {0, *n_words}
  IGN_TRY(f.take(&offsets, 2));
  if (dtype == IGN_U32)
    IGN_TRY(cseg_encode_batch<uint32_t>(ctx, (const uint32_t*)labels, segs, nblock, 1, sc, d.bvox, out, cap_words,
                                        offsets, n_words));
  else
    IGN_TRY(cseg_encode_batch<uint64_t>(ctx, (const uint64_t*)labels, segs, nblock, 1, sc, d.bvox, out, cap_words,
                                        offsets, n_words));
  IGN_CUDA(cudaStreamSynchronize(ctx->stream));
  return IGN_OK;
}

int ign_cseg_decode_dev(ign_ctx* ctx, const uint32_t* in, uint64_t n_words, int dtype, uint64_t sx, uint64_t sy,
                        uint64_t sz, uint64_t sc, uint32_t bx, uint32_t by, uint32_t bz, void* out) {
  IGN_TRY(activate(ctx));
  IGN_REQUIRE(in && out && sc >= 1 && n_words >= sc, IGN_ERR_INVALID, "bad argument");
  IGN_REQUIRE(dtype == IGN_U32 || dtype == IGN_U64, IGN_ERR_UNSUPPORTED, "compressed_segmentation holds uint32 / uint64 labels");
  CsegDims d;
  IGN_TRY(cseg_dims(sx, sy, sz, bx, by, bz, &d));
  const uint32_t shape[3] = {d.sx, d.sy, d.sz};
  const uint64_t word_offsets[2] = {0, n_words};
  return cseg_decode_batch(ctx, in, word_offsets, 1, dtype, shape, sc, bx, by, bz, out);
}

int ign_cseg_encode_batch_dev(ign_ctx* ctx, const void* chunks, int dtype, uint64_t n_chunks, const uint32_t* shapes,
                              uint64_t sc, uint32_t bx, uint32_t by, uint32_t bz, uint32_t* out, uint64_t cap_words,
                              uint64_t* offsets, uint64_t* n_words) {
  IGN_TRY(activate(ctx));
  IGN_REQUIRE(n_words && sc >= 1 && (n_chunks == 0 || (chunks && shapes && out && offsets)), IGN_ERR_INVALID,
              "cseg batch: null argument");
  IGN_REQUIRE(dtype == IGN_U32 || dtype == IGN_U64, IGN_ERR_UNSUPPORTED, "compressed_segmentation holds uint32 / uint64 labels");
  *n_words = 0;
  if (n_chunks == 0) return IGN_OK;
  std::vector<CsegSeg> segs;
  uint64_t nblock = 0;
  IGN_TRY(cb_segments(shapes, n_chunks, sc, bx, by, bz, segs, &nblock));
  const uint32_t bvox = bx * by * bz;
  if (dtype == IGN_U32)
    return cseg_encode_batch<uint32_t>(ctx, (const uint32_t*)chunks, segs, nblock, n_chunks, sc, bvox, out, cap_words,
                                       offsets, n_words);
  return cseg_encode_batch<uint64_t>(ctx, (const uint64_t*)chunks, segs, nblock, n_chunks, sc, bvox, out, cap_words,
                                     offsets, n_words);
}

int ign_cseg_decode_batch_dev(ign_ctx* ctx, const uint32_t* streams, const uint64_t* word_offsets, uint64_t n_streams,
                              int dtype, const uint32_t* shapes, uint64_t sc, uint32_t bx, uint32_t by, uint32_t bz,
                              void* out) {
  IGN_TRY(activate(ctx));
  IGN_REQUIRE(sc >= 1 && (n_streams == 0 || (streams && word_offsets && shapes && out)), IGN_ERR_INVALID,
              "cseg batch: null argument");
  IGN_REQUIRE(dtype == IGN_U32 || dtype == IGN_U64, IGN_ERR_UNSUPPORTED, "compressed_segmentation holds uint32 / uint64 labels");
  if (n_streams == 0) return IGN_OK;
  return cseg_decode_batch(ctx, streams, word_offsets, n_streams, dtype, shapes, sc, bx, by, bz, out);
}

// host-buffer wrappers: encode needs room for the whole stream; the worst case is sc + 2*blocks +
// (label words + 1)*voxels words, and a shorter out fails with *n_words = the words needed
int ign_cseg_encode(ign_ctx* ctx, const void* labels, int dtype, uint64_t sx, uint64_t sy, uint64_t sz, uint64_t sc,
                    uint32_t bx, uint32_t by, uint32_t bz, uint32_t* out, uint64_t cap_words, uint64_t* n_words) {
  CsegDims dims;
  IGN_TRY(cseg_dims(sx, sy, sz, bx, by, bz, &dims));
  std::vector<HostBuf> bufs = {{labels, nullptr, sx * sy * sz * sc * dtype_size(dtype)}, {nullptr, out, cap_words * 4}};
  return staged(ctx, bufs, [&](void* const* d) -> int {
    IGN_TRY(ign_cseg_encode_dev(ctx, d[0], dtype, sx, sy, sz, sc, bx, by, bz, (uint32_t*)d[1], cap_words, n_words));
    bufs[1].bytes = *n_words * 4;
    return IGN_OK;
  });
}

int ign_cseg_decode(ign_ctx* ctx, const uint32_t* in, uint64_t n_words, int dtype, uint64_t sx, uint64_t sy, uint64_t sz,
                    uint64_t sc, uint32_t bx, uint32_t by, uint32_t bz, void* out) {
  CsegDims dims;
  IGN_TRY(cseg_dims(sx, sy, sz, bx, by, bz, &dims));
  return staged(ctx, {{in, nullptr, n_words * 4}, {nullptr, out, sx * sy * sz * sc * dtype_size(dtype)}},
                [&](void* const* d) {
                  return ign_cseg_decode_dev(ctx, (const uint32_t*)d[0], n_words, dtype, sx, sy, sz, sc, bx, by, bz,
                                             d[1]);
                });
}

}  // extern "C"
