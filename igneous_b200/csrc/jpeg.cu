// jpeg.cu -- Precomputed `jpeg` chunk codec on the device (grayscale, 8-bit, baseline Huffman)
//
// SURVEY.md 8(f) row 1.  EM image layers are almost always `jpeg`: the reference's CLI offers it as
// the image encoding (igneous_cli/cli.py:64), its creators record `jpeg_quality`
// (igneous/task_creation/common.py:215-236) and switch the top sharded mip of a jpeg pyramid to png
// (task_creation/image.py:708-709).  CloudVolume encodes / decodes the chunks on the host.
//
// Format: a chunk [x, y, z, 1] of uint8 is one grayscale JPEG of width sx and height sy*sz (image
// row r = y + sy*z), so the Fortran-order chunk is the raster.  The encoder writes libjpeg's default
// stream byte for byte (ITU-T T.81 baseline; oracle_jpeg/jpeg_oracle.c is the serial restatement the
// tests compare against): SOI, JFIF APP0, DQT (Annex K luminance table, IJG quality scaling, entries
// 1..255), SOF0, DHT DC + DHT AC (Annex K luminance tables), DRI when restarts are on, SOS, scan, EOI;
// the IJG accurate integer DCT ("islow", LL&M with 13-bit constants and 2 extra bits between the
// passes), quantization rounding half away from zero, partial blocks padded by repeating the last
// column and row.  The decoder reads any SOF0 / SOF1 8-bit one-component stream (any Huffman tables,
// APPn / COM segments, fill bytes, restart markers or none) and reproduces libjpeg's islow decode.
//
// Both directions take a batch of chunks per call; blocks and restart intervals are numbered over
// the whole batch.
//   encode  1 k_jpeg_fdct      8 threads per 8x8 block: edge-replicated load, level shift, FDCT,
//                              quantization, coefficients in zigzag order
//           2 k_jpeg_bits      per block: Huffman bits, the DC predicted from the previous block of
//                              its restart interval; exclusive scan -> bit offsets
//           3 k_jpeg_ibytes    per interval: bytes (padded with 1-bits); scan of its words -> every
//                              interval starts on a 32-bit word of the unstuffed buffer
//           4 k_jpeg_pack      per block: the codes at its bit offset (atomicOr on shared edge words)
//           5 k_jpeg_ffcount   per word: 0xFF bytes; scan -> k_jpeg_osize per interval: stuffed bytes
//                              + marker (+ headers); scan -> output offsets
//           6 k_jpeg_scatter   per word: the bytes, a 0x00 after every 0xFF; k_jpeg_marks writes
//                              headers, RSTn and EOI
//   decode  1 k_jpeg_scan      one CTA per stream: thread 0 parses the headers; the CTA builds the
//                              Huffman lookahead tables in shared memory, finds the scan's end and
//                              ranks its RSTn markers (block scan), then decodes one restart interval
//                              per thread, unstuffing inline, into int16 coefficients
//           2 k_jpeg_idct      8 threads per block: dequantize, islow IDCT, clamp, cropped store
// A stream without restart markers is one interval, decoded by one thread.
#include <cub/block/block_scan.cuh>
#include <cub/device/device_scan.cuh>

#include <vector>

#include "common.cuh"

namespace ign {

namespace {

constexpr int JQ_THREADS = 256;      // k_jpeg_scan CTA
constexpr uint32_t JPEG_MAX_DIM = 65535;

__constant__ uint8_t c_zigzag[64] = {  // natural index of the k-th coefficient in zigzag order
  0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
  35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
static const uint8_t ZIGZAG[64] = {
  0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
  35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
static const uint8_t LUMA_Q[64] = {  // T.81 Table K.1, natural order
  16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
  14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
  49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
// T.81 Tables K.3 / K.5: code counts per length 1..16, then the values
static const uint8_t DC_BITS[16] = {0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0};
static const uint8_t DC_VALS[12] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11};
static const uint8_t AC_BITS[16] = {0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d};
static const uint8_t AC_VALS[162] = {
  0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07, 0x22, 0x71, 0x14, 0x32,
  0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0, 0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16,
  0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28, 0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45,
  0x46, 0x47, 0x48, 0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69,
  0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89, 0x8a, 0x92, 0x93, 0x94,
  0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6,
  0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8,
  0xd9, 0xda, 0xe1, 0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8,
  0xf9, 0xfa};

// LL&M constants scaled by 2^13 (CB); PASS1 extra bits between the passes
constexpr int CB = 13, P1 = 2;
constexpr int F0298 = 2446, F0390 = 3196, F0541 = 4433, F0765 = 6270, F0899 = 7373, F1175 = 9633, F1501 = 12299,
              F1847 = 15137, F1961 = 16069, F2053 = 16819, F2562 = 20995, F3072 = 25172;
// 32-bit arithmetic: exact for 8-bit samples and for dequantized coefficients of the 8-bit range
__device__ __forceinline__ int descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }

// ------------------------------------------------------------------ encode
struct EncChunk {
  uint64_t in_off;  // first pixel in the packed input
  uint64_t b0, i0;  // first block / first restart interval of the batch
  uint32_t w, h, bw, per;  // image width, height, blocks per row, blocks per interval
  uint32_t dri;            // the DRI value (0: no restart markers)
};
struct EncParams {
  uint16_t q[64];  // quantizer, natural order
  uint16_t dc_code[12];
  uint8_t dc_len[12];
  uint16_t ac_code[256];
  uint8_t ac_len[256];
  uint8_t hdr[352];
  uint32_t hdr_len, sof_at, dri_at;
};

// index of the last entry whose `key` is <= v (entries sorted by key, entry 0 key 0)
template <typename T, typename K>
__device__ __forceinline__ uint32_t find_last(const T* a, uint32_t n, uint64_t v, K key) {
  uint32_t lo = 0, hi = n;  // answer in [lo, hi)
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if (key(a[mid]) <= v) lo = mid;
    else hi = mid;
  }
  return lo;
}

__global__ void __launch_bounds__(256)
    k_jpeg_fdct(const uint8_t* __restrict__ in, const EncChunk* __restrict__ ch, uint32_t nch, uint64_t nblk,
                const __grid_constant__ EncParams P, int16_t* __restrict__ coef) {
  __shared__ int ws[32][64];
  __shared__ uint8_t izz[64];  // zigzag position of a natural index
  if (threadIdx.x < 64) izz[c_zigzag[threadIdx.x]] = (uint8_t)threadIdx.x;
  __syncthreads();
  const uint32_t lb = threadIdx.x >> 3, t = threadIdx.x & 7;
  const uint64_t b = blockIdx.x * 32ull + lb;
  const bool ok = b < nblk;
  if (ok) {  // row t: load, level shift, 1-D DCT
    const EncChunk c = ch[find_last(ch, nch, b, [](const EncChunk& e) { return e.b0; })];
    const uint64_t l = b - c.b0;
    const uint32_t bx = (uint32_t)(l % c.bw), by = (uint32_t)(l / c.bw);
    const uint32_t y = min(by * 8 + t, c.h - 1);
    const uint8_t* row = in + c.in_off + (uint64_t)y * c.w;
    int d[8];
#pragma unroll
    for (int i = 0; i < 8; i++) d[i] = (int)row[min(bx * 8 + i, c.w - 1)] - 128;
    int t0 = d[0] + d[7], t7 = d[0] - d[7], t1 = d[1] + d[6], t6 = d[1] - d[6];
    int t2 = d[2] + d[5], t5 = d[2] - d[5], t3 = d[3] + d[4], t4 = d[3] - d[4];
    int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
    int* o = ws[lb] + 8 * t;
    o[0] = (t10 + t11) * (1 << P1);
    o[4] = (t10 - t11) * (1 << P1);
    int z1 = (t12 + t13) * F0541;
    o[2] = descale(z1 + t13 * F0765, CB - P1);
    o[6] = descale(z1 - t12 * F1847, CB - P1);
    z1 = t4 + t7;
    int z2 = t5 + t6, z3 = t4 + t6, z4 = t5 + t7, z5 = (z3 + z4) * F1175;
    t4 *= F0298; t5 *= F2053; t6 *= F3072; t7 *= F1501;
    z1 *= -F0899; z2 *= -F2562; z3 = z3 * -F1961 + z5; z4 = z4 * -F0390 + z5;
    o[7] = descale(t4 + z1 + z3, CB - P1);
    o[5] = descale(t5 + z2 + z4, CB - P1);
    o[3] = descale(t6 + z2 + z3, CB - P1);
    o[1] = descale(t7 + z1 + z4, CB - P1);
  }
  __syncwarp();
  if (!ok) return;
  // column t: 1-D DCT, quantize, store at the zigzag positions
  const int* d = ws[lb] + t;
  int t0 = d[0] + d[56], t7 = d[0] - d[56], t1 = d[8] + d[48], t6 = d[8] - d[48];
  int t2 = d[16] + d[40], t5 = d[16] - d[40], t3 = d[24] + d[32], t4 = d[24] - d[32];
  int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  int v[8];
  v[0] = descale(t10 + t11, P1);
  v[4] = descale(t10 - t11, P1);
  int z1 = (t12 + t13) * F0541;
  v[2] = descale(z1 + t13 * F0765, CB + P1);
  v[6] = descale(z1 - t12 * F1847, CB + P1);
  z1 = t4 + t7;
  int z2 = t5 + t6, z3 = t4 + t6, z4 = t5 + t7, z5 = (z3 + z4) * F1175;
  t4 *= F0298; t5 *= F2053; t6 *= F3072; t7 *= F1501;
  z1 *= -F0899; z2 *= -F2562; z3 = z3 * -F1961 + z5; z4 = z4 * -F0390 + z5;
  v[7] = descale(t4 + z1 + z3, CB + P1);
  v[5] = descale(t5 + z2 + z4, CB + P1);
  v[3] = descale(t6 + z2 + z3, CB + P1);
  v[1] = descale(t7 + z1 + z4, CB + P1);
  int16_t* out = coef + b * 64;
#pragma unroll
  for (int r = 0; r < 8; r++) {
    const int i = 8 * r + t, dv = 8 * P.q[i];  // the DCT output carries a factor 8
    const int a = v[r] < 0 ? -v[r] : v[r];
    const int qv = (a + (dv >> 1)) / dv;
    out[izz[i]] = (int16_t)(v[r] < 0 ? -qv : qv);
  }
}

struct EncTables {
  uint16_t dc_code[12];
  uint8_t dc_len[12];
  uint16_t ac_code[256];
  uint8_t ac_len[256];
};

__device__ __forceinline__ void load_tables(EncTables& s, const EncParams& P) {
  for (int i = threadIdx.x; i < 256; i += blockDim.x) {
    s.ac_code[i] = P.ac_code[i];
    s.ac_len[i] = P.ac_len[i];
    if (i < 12) { s.dc_code[i] = P.dc_code[i]; s.dc_len[i] = P.dc_len[i]; }
  }
  __syncthreads();
}

__device__ __forceinline__ int mag_bits(int v) { return v ? 32 - __clz(v < 0 ? -v : v) : 0; }

// MSB-first bits into the big-endian byte stream held in 32-bit words; words other blocks may
// share (the first and last) are written with atomicOr into the zeroed buffer
struct BitSink {
  uint32_t* raw;
  uint64_t pos;  // stream bit of the first pending bit
  uint64_t acc;
  int n;
  __device__ void put(uint32_t code, int len) {
    acc = (acc << len) | code;
    n += len;
    int room = 32 - (int)(pos & 31);
    while (n >= room) {
      const uint32_t v = (uint32_t)(acc >> (n - room)) & (room == 32 ? 0xFFFFFFFFu : ((1u << room) - 1u));
      atomicOr(raw + (pos >> 5), __byte_perm(v, 0, 0x0123));
      pos += room;
      n -= room;
      acc &= n ? ((1ull << n) - 1) : 0ull;
      room = 32;
    }
  }
  __device__ void flush() {
    if (n) {
      const int off = (int)(pos & 31);
      atomicOr(raw + (pos >> 5), __byte_perm((uint32_t)(acc << (32 - off - n)), 0, 0x0123));
    }
  }
};
struct BitCount {
  uint64_t n = 0;
  __device__ void put(uint32_t, int len) { n += len; }
};

// Huffman codes of one block (coefficients in zigzag order) given the DC prediction
template <typename Sink>
__device__ __forceinline__ void encode_block(const int16_t* __restrict__ zz, int pred, const EncTables& T, Sink& s) {
  uint64_t nz = 0;
  const uint4* z4 = reinterpret_cast<const uint4*>(zz);
#pragma unroll
  for (int j = 0; j < 8; j++) {
    const uint4 q = z4[j];
    const uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
    for (int h = 0; h < 4; h++) {
      if (w[h] & 0xFFFFu) nz |= 1ull << (8 * j + 2 * h);
      if (w[h] >> 16) nz |= 1ull << (8 * j + 2 * h + 1);
    }
  }
  const int diff = (int)zz[0] - pred;
  int n = mag_bits(diff);
  s.put(T.dc_code[n], T.dc_len[n]);
  if (n) s.put((uint32_t)(diff < 0 ? diff - 1 : diff) & ((1u << n) - 1u), n);
  nz &= ~1ull;
  int last = 0;
  while (nz) {
    const int k = __ffsll((long long)nz) - 1;
    nz &= nz - 1;
    int run = k - last - 1;
    while (run > 15) { s.put(T.ac_code[0xF0], T.ac_len[0xF0]); run -= 16; }
    const int v = zz[k];
    n = mag_bits(v);
    const int rs = (run << 4) | n;
    s.put(T.ac_code[rs], T.ac_len[rs]);
    s.put((uint32_t)(v < 0 ? v - 1 : v) & ((1u << n) - 1u), n);
    last = k;
  }
  if (last != 63) s.put(T.ac_code[0x00], T.ac_len[0x00]);
}

__device__ __forceinline__ int block_pred(const int16_t* coef, uint64_t b, const EncChunk& c) {
  return ((b - c.b0) % c.per) ? (int)coef[(b - 1) * 64] : 0;
}

__global__ void __launch_bounds__(256)
    k_jpeg_bits(const int16_t* __restrict__ coef, const EncChunk* __restrict__ ch, uint32_t nch, uint64_t nblk,
                const __grid_constant__ EncParams P, uint64_t* __restrict__ bits) {
  __shared__ EncTables T;
  load_tables(T, P);
  const uint64_t b = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (b >= nblk) return;
  const EncChunk c = ch[find_last(ch, nch, b, [](const EncChunk& e) { return e.b0; })];
  BitCount s;
  encode_block(coef + b * 64, block_pred(coef, b, c), T, s);
  bits[b] = s.n;
}

// per interval: bytes of the unstuffed data and 32-bit words it takes in the raw buffer
__global__ void __launch_bounds__(256)
    k_jpeg_ibytes(const uint64_t* __restrict__ boff, const EncChunk* __restrict__ ch, uint32_t nch, uint64_t nint,
                  uint64_t* __restrict__ ibytes, uint64_t* __restrict__ iwords) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= nint) return;
  const uint32_t ci = find_last(ch, nch, i, [](const EncChunk& e) { return e.i0; });
  const EncChunk c = ch[ci];
  const uint64_t f = c.b0 + (i - c.i0) * c.per, e = min(f + c.per, ch[ci + 1].b0);
  const uint64_t by = (boff[e] - boff[f] + 7) / 8;
  ibytes[i] = by;
  iwords[i] = (by + 3) / 4;
}

__global__ void __launch_bounds__(256)
    k_jpeg_pack(const int16_t* __restrict__ coef, const EncChunk* __restrict__ ch, uint32_t nch, uint64_t nblk,
                const __grid_constant__ EncParams P, const uint64_t* __restrict__ boff,
                const uint64_t* __restrict__ iwoff, uint32_t* __restrict__ raw) {
  __shared__ EncTables T;
  load_tables(T, P);
  const uint64_t b = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (b >= nblk) return;
  const uint32_t ci = find_last(ch, nch, b, [](const EncChunk& e) { return e.b0; });
  const EncChunk c = ch[ci];
  const uint64_t l = b - c.b0, k = l / c.per, f = c.b0 + k * c.per;
  BitSink s{raw, iwoff[c.i0 + k] * 32 + (boff[b] - boff[f]), 0, 0};
  encode_block(coef + b * 64, block_pred(coef, b, c), T, s);
  const bool last = (l + 1) % c.per == 0 || b + 1 == ch[ci + 1].b0;
  if (last) {  // pad the interval to a byte with 1-bits
    const int pad = (int)((8 - ((s.pos + s.n) & 7)) & 7);
    if (pad) s.put((1u << pad) - 1u, pad);
  }
  s.flush();
}

__global__ void __launch_bounds__(256) k_jpeg_ffcount(const uint32_t* __restrict__ raw, uint64_t nw, uint32_t* __restrict__ ff) {
  const uint64_t w = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (w >= nw) return;
  const uint32_t v = raw[w];
  ff[w] = ((v & 0xFFu) == 0xFFu) + ((v & 0xFF00u) == 0xFF00u) + ((v & 0xFF0000u) == 0xFF0000u) + ((v >> 24) == 0xFFu);
}

__global__ void __launch_bounds__(256)
    k_jpeg_osize(const uint64_t* __restrict__ ibytes, const uint64_t* __restrict__ iwoff, const uint32_t* __restrict__ ffscan,
                 const EncChunk* __restrict__ ch, uint32_t nch, uint64_t nint, uint32_t hdr_len, uint64_t* __restrict__ osize) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= nint) return;
  const EncChunk c = ch[find_last(ch, nch, i, [](const EncChunk& e) { return e.i0; })];
  osize[i] = ibytes[i] + (ffscan[iwoff[i + 1]] - ffscan[iwoff[i]]) + 2 + (i == c.i0 ? hdr_len : 0);
}

__global__ void __launch_bounds__(256)
    k_jpeg_scatter(const uint32_t* __restrict__ raw, uint64_t nw, const uint64_t* __restrict__ iwoff, uint64_t nint,
                   const uint64_t* __restrict__ ibytes, const uint32_t* __restrict__ ffscan,
                   const uint64_t* __restrict__ ooff, const EncChunk* __restrict__ ch, uint32_t nch, uint32_t hdr_len,
                   uint8_t* __restrict__ out) {
  const uint64_t w = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (w >= nw) return;
  const uint32_t i = find_last(iwoff, (uint32_t)nint, w, [](uint64_t v) { return v; });
  const EncChunk c = ch[find_last(ch, nch, i, [](const EncChunk& e) { return e.i0; })];
  const uint64_t j0 = (w - iwoff[i]) * 4;
  uint64_t o = ooff[i] + (i == c.i0 ? hdr_len : 0) + j0 + (ffscan[w] - ffscan[iwoff[i]]);
  const uint32_t v = raw[w];
  for (int k = 0; k < 4 && j0 + k < ibytes[i]; k++) {
    const uint8_t byte = (uint8_t)(v >> (8 * k));
    out[o++] = byte;
    if (byte == 0xFF) out[o++] = 0x00;
  }
}

// headers before the first interval of a chunk, RSTn / EOI after every interval, chunk offsets
__global__ void __launch_bounds__(256)
    k_jpeg_marks(const uint64_t* __restrict__ ooff, const EncChunk* __restrict__ ch, uint32_t nch, uint64_t nint,
                 const __grid_constant__ EncParams P, uint8_t* __restrict__ out, uint64_t* __restrict__ offsets) {
  const uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
  if (i >= nint) return;
  const uint32_t ci = find_last(ch, nch, i, [](const EncChunk& e) { return e.i0; });
  const EncChunk c = ch[ci];
  if (i == c.i0) {
    uint8_t* h = out + ooff[i];
    for (uint32_t k = 0; k < P.hdr_len; k++) h[k] = P.hdr[k];
    h[P.sof_at] = (uint8_t)(c.h >> 8);
    h[P.sof_at + 1] = (uint8_t)c.h;
    h[P.sof_at + 2] = (uint8_t)(c.w >> 8);
    h[P.sof_at + 3] = (uint8_t)c.w;
    if (c.dri) {
      h[P.dri_at] = (uint8_t)(c.dri >> 8);
      h[P.dri_at + 1] = (uint8_t)c.dri;
    }
    offsets[ci] = ooff[i];
  }
  const bool last = i + 1 == ch[ci + 1].i0;
  out[ooff[i + 1] - 2] = 0xFF;
  out[ooff[i + 1] - 1] = last ? 0xD9 : (uint8_t)(0xD0 + ((i - c.i0) & 7));
  if (i + 1 == nint) offsets[nch] = ooff[nint];
}

// ------------------------------------------------------------------ decode
struct DecStream {
  uint64_t off, len;  // bytes of the stream in the packed input
  uint64_t b0;        // first block of the batch
  uint64_t out_off;   // first pixel of the chunk in the output
  uint32_t w, h, bw;
};

enum { JS_OK = 0, JS_MALFORMED = 1, JS_UNSUPPORTED = 2, JS_SHAPE = 3, JS_TOO_LONG = 4 };

struct HuffDec {
  int32_t maxcode[18], mincode[17];
  int16_t valptr[17];
  uint8_t vals[256];
  uint16_t look[512];  // 9-bit lookahead: (length << 8) | value, 0 = longer code
};

struct ScanShared {
  uint8_t bits[2][4][17];
  uint8_t vals[2][4][256];
  uint8_t hdef[2][4];
  uint16_t qt[4][64];
  uint8_t qdef[4];
  HuffDec dc, ac;
  uint8_t zz[64];
  uint32_t status, scan_start, scan_end, restart, qsel, nint, nmark;
};

__device__ __forceinline__ uint32_t rd16(const uint8_t* p) { return ((uint32_t)p[0] << 8) | p[1]; }

// T.81 F.2.2.3 decoder tables from counts per length; false when the counts overflow the code space
__device__ bool huff_build(HuffDec& t, const uint8_t* bits, const uint8_t* vals) {
  int32_t code = 0;
  int k = 0;
  for (int l = 1; l <= 16; l++) {
    t.valptr[l] = (int16_t)k;
    t.mincode[l] = code;
    code += bits[l];
    k += bits[l];
    if (code > (1 << l)) return false;
    t.maxcode[l] = bits[l] ? code - 1 : -1;
    code <<= 1;
  }
  t.maxcode[17] = 0x7FFFFFFF;
  for (int i = 0; i < k; i++) t.vals[i] = vals[i];
  return true;
}

// headers of one stream, by one thread: the tables of its scan into S; the quantizer to qt_out
__device__ uint32_t parse_headers(const uint8_t* p, uint64_t n, const DecStream& st, ScanShared& S, int32_t* qt_out) {
  if (n < 4 || p[0] != 0xFF || p[1] != 0xD8) return JS_MALFORMED;
  for (int i = 0; i < 4; i++) { S.qdef[i] = 0; S.hdef[0][i] = S.hdef[1][i] = 0; }
  uint32_t fw = 0, fh = 0, restart = 0;
  int comp = -1, qsel = 0;
  bool sof = false;
  uint64_t pos = 2;
  for (;;) {
    if (pos + 2 > n || p[pos] != 0xFF) return JS_MALFORMED;
    while (pos + 1 < n && p[pos + 1] == 0xFF) pos++;  // fill bytes
    if (pos + 4 > n) return JS_MALFORMED;
    const uint32_t m = p[pos + 1];
    const uint64_t len = rd16(p + pos + 2);
    if (len < 2 || pos + 2 + len > n) return JS_MALFORMED;
    const uint8_t* s = p + pos + 4;
    const uint64_t sl = len - 2;
    pos += 2 + len;
    if (m == 0xDB) {
      for (uint64_t i = 0; i < sl;) {
        const int pq = s[i] >> 4, tq = s[i] & 15;
        if (pq > 1 || tq > 3 || i + 1 + 64 * (pq + 1) > sl) return JS_MALFORMED;
        for (int k = 0; k < 64; k++)
          S.qt[tq][c_zigzag[k]] = pq ? (uint16_t)rd16(s + i + 1 + 2 * k) : s[i + 1 + k];
        S.qdef[tq] = 1;
        i += 1 + 64 * (pq + 1);
      }
    } else if (m == 0xC4) {
      for (uint64_t i = 0; i < sl;) {
        const int tc = s[i] >> 4, th = s[i] & 15;
        if (tc > 1 || th > 3 || i + 17 > sl) return JS_MALFORMED;
        int total = 0;
        for (int l = 1; l <= 16; l++) total += (S.bits[tc][th][l] = s[i + l]);
        if (total > 256 || i + 17 + total > sl) return JS_MALFORMED;
        for (int k = 0; k < total; k++) {
          S.vals[tc][th][k] = s[i + 17 + k];
          if (tc == 0 && s[i + 17 + k] > 15) return JS_MALFORMED;
        }
        S.hdef[tc][th] = 1;
        i += 17 + total;
      }
    } else if (m == 0xDD) {
      if (sl != 2) return JS_MALFORMED;
      restart = rd16(s);
    } else if (m == 0xC0 || m == 0xC1) {
      if (sl < 6) return JS_MALFORMED;
      if (s[0] != 8 || s[5] != 1) return JS_UNSUPPORTED;  // 8-bit, one component
      if (sl != 9) return JS_MALFORMED;
      fh = rd16(s + 1);
      fw = rd16(s + 3);
      if (fh == 0) return JS_UNSUPPORTED;  // DNL
      if (fw == 0) return JS_MALFORMED;
      const int hs = s[7] >> 4, vs = s[7] & 15;
      if (hs < 1 || hs > 4 || vs < 1 || vs > 4 || s[8] > 3) return JS_MALFORMED;
      comp = s[6];
      qsel = s[8];
      sof = true;
    } else if ((m >= 0xC2 && m <= 0xCF && m != 0xC4 && m != 0xC8) || m == 0xDC) {
      return JS_UNSUPPORTED;  // progressive, lossless, hierarchical, arithmetic, DNL
    } else if (m == 0xDA) {
      if (!sof || sl < 1 || s[0] != 1) return JS_MALFORMED;
      if (sl != 6 || s[1] != comp || s[3] != 0 || s[4] != 63 || s[5] != 0) return JS_MALFORMED;
      const int td = s[2] >> 4, ta = s[2] & 15;
      if (td > 3 || ta > 3 || !S.hdef[0][td] || !S.hdef[1][ta] || !S.qdef[qsel]) return JS_MALFORMED;
      if (fw != st.w || fh != st.h) return JS_SHAPE;
      if (!huff_build(S.dc, S.bits[0][td], S.vals[0][td]) || !huff_build(S.ac, S.bits[1][ta], S.vals[1][ta]))
        return JS_MALFORMED;
      for (int k = 0; k < 64; k++) qt_out[k] = S.qt[qsel][k];
      const uint64_t nb = (uint64_t)st.bw * ((st.h + 7) / 8);
      S.restart = restart;
      S.nint = restart ? (uint32_t)((nb + restart - 1) / restart) : 1u;
      S.scan_start = (uint32_t)pos;
      return JS_OK;
    } else if (!((m >= 0xE0 && m <= 0xEF) || m == 0xFE)) {  // APPn, COM are skipped
      return JS_MALFORMED;
    }
  }
}

__device__ __forceinline__ void build_look(HuffDec& t, int p) {
  uint16_t e = 0;
  for (int l = 1; l <= 9; l++) {
    const int32_t code = p >> (9 - l);
    if (code <= t.maxcode[l]) {
      e = (uint16_t)((l << 8) | t.vals[t.valptr[l] + code - t.mincode[l]]);
      break;
    }
  }
  t.look[p] = e;
}

// MSB-first reader of one interval's entropy-coded bytes; stops at a marker or at `end`, after which
// it supplies zero bits and counts them: consuming one of them is a truncated interval
struct BitSrc {
  const uint8_t* p;
  uint64_t pos, end;
  uint64_t acc;
  int n, virt;
  bool stop, over;
  __device__ void fill() {
    while (n <= 56) {
      uint32_t b = 0;
      if (!stop) {
        if (pos < end) {
          b = p[pos];
          if (b == 0xFF) {
            if (pos + 1 < end && p[pos + 1] == 0x00) pos += 2;
            else { stop = true; b = 0; }
          } else {
            pos++;
          }
        } else {
          stop = true;
        }
      }
      if (stop) virt += 8;
      acc |= (uint64_t)b << (56 - n);
      n += 8;
    }
  }
  __device__ __forceinline__ uint32_t peek(int k) const { return (uint32_t)(acc >> (64 - k)); }
  __device__ __forceinline__ void skip(int k) {
    acc <<= k;
    n -= k;
    if (n < virt) over = true;
  }
};

__device__ __forceinline__ int huff_decode(BitSrc& r, const HuffDec& t) {
  r.fill();
  const uint32_t e = t.look[r.peek(9)];
  if (e) {
    r.skip(e >> 8);
    return e & 0xFF;
  }
  const uint32_t c16 = r.peek(16);
  for (int l = 10; l <= 16; l++) {
    const int32_t code = (int32_t)(c16 >> (16 - l));
    if (code <= t.maxcode[l]) {
      r.skip(l);
      return t.vals[t.valptr[l] + code - t.mincode[l]];
    }
  }
  return -1;
}

__device__ __forceinline__ int receive_extend(BitSrc& r, int s) {
  r.fill();
  const int v = (int)r.peek(s);
  r.skip(s);
  return v < (1 << (s - 1)) ? v - (1 << s) + 1 : v;
}

__global__ void __launch_bounds__(JQ_THREADS)
    k_jpeg_scan(const uint8_t* __restrict__ in, const DecStream* __restrict__ streams, uint32_t* __restrict__ istart,
                int32_t* __restrict__ qt, int16_t* __restrict__ coef, uint32_t* __restrict__ status) {
  using BlockScan = cub::BlockScan<uint32_t, JQ_THREADS>;
  __shared__ ScanShared S;
  __shared__ typename BlockScan::TempStorage scan_tmp;
  const uint32_t s = blockIdx.x, t = threadIdx.x;
  const DecStream st = streams[s];
  const uint8_t* p = in + st.off;
  const uint64_t n = st.len;
  if (t == 0) {
    S.status = n >= 0xFFFFFFF0ull ? (uint32_t)JS_TOO_LONG : parse_headers(p, n, st, S, qt + 64ull * s);
    S.scan_end = 0xFFFFFFFFu;
    S.nmark = 0;
  }
  if (t < 64) S.zz[t] = c_zigzag[t];
  __syncthreads();
  if (S.status != JS_OK) {
    if (t == 0) status[s] = S.status;
    return;
  }
  for (int i = t; i < 512; i += JQ_THREADS) {
    build_look(S.dc, i);
    build_look(S.ac, i);
  }
  // the scan ends at the first marker that is neither RSTn nor a fill byte
  const uint32_t ss = S.scan_start;
  for (uint64_t j = ss + t; j + 1 < n; j += JQ_THREADS) {
    const uint32_t m = p[j + 1];
    if (p[j] == 0xFF && m != 0x00 && m != 0xFF && (m & 0xF8) != 0xD0) atomicMin(&S.scan_end, (uint32_t)j);
  }
  __syncthreads();
  const uint32_t se = S.scan_end;
  if (se == 0xFFFFFFFFu || p[se + 1] != 0xD9) {
    if (t == 0) status[s] = JS_MALFORMED;
    return;
  }
  // RSTn markers before it, ranked in stream order: interval k + 1 starts after marker k
  const uint32_t nint = S.nint;
  uint32_t* ist = istart + st.b0 + s;
  uint32_t base = 0;
  bool bad = false;
  for (uint64_t tile = ss; tile < se; tile += 16ull * JQ_THREADS) {
    const uint64_t j0 = tile + 16ull * t;
    uint32_t cnt = 0;
    for (uint64_t j = j0; j < j0 + 16 && j < se; j++) cnt += p[j] == 0xFF && (p[j + 1] & 0xF8) == 0xD0;
    uint32_t rank, total;
    BlockScan(scan_tmp).ExclusiveSum(cnt, rank, total);
    rank += base;
    for (uint64_t j = j0; cnt && j < j0 + 16 && j < se; j++)
      if (p[j] == 0xFF && (p[j + 1] & 0xF8) == 0xD0) {
        if (rank + 1 < nint) ist[rank + 1] = (uint32_t)(j + 2);
        if (p[j + 1] != 0xD0 + (rank & 7)) bad = true;
        rank++;
      }
    base += total;
    __syncthreads();  // scan_tmp is reused
  }
  if (t == 0) ist[0] = ss;
  if (__syncthreads_or(bad) || base != nint - 1) {  // also publishes ist to the CTA
    if (t == 0) status[s] = JS_MALFORMED;
    return;
  }
  const uint64_t nb = (uint64_t)st.bw * ((st.h + 7) / 8);
  const uint64_t per = S.restart ? S.restart : nb;
  bool fail = false;
  for (uint32_t k = t; k < nint; k += JQ_THREADS) {
    BitSrc r{p, ist[k], se, 0, 0, 0, false, false};
    int dc = 0;
    for (uint64_t b = k * per; b < nb && b < (k + 1) * per && !fail; b++) {
      int16_t* c = coef + (st.b0 + b) * 64;
      int v = huff_decode(r, S.dc);
      if (v < 0) { fail = true; break; }
      if (v) dc += receive_extend(r, v);
      c[0] = (int16_t)dc;
      for (int i = 1; i < 64; i++) {
        const int rs = huff_decode(r, S.ac);
        if (rs < 0) { fail = true; break; }
        const int run = rs >> 4, sz = rs & 15;
        if (sz == 0) {
          if (run != 15) break;
          i += 15;
          continue;
        }
        i += run;
        if (i > 63) { fail = true; break; }
        c[S.zz[i]] = (int16_t)receive_extend(r, sz);
      }
      if (r.over) fail = true;
    }
  }
  if (fail) atomicMax(&S.status, (uint32_t)JS_MALFORMED);
  __syncthreads();
  if (t == 0) status[s] = S.status;
}

__global__ void __launch_bounds__(256)
    k_jpeg_idct(const int16_t* __restrict__ coef, const DecStream* __restrict__ streams, uint32_t ns, uint64_t nblk,
                const int32_t* __restrict__ qt, const uint32_t* __restrict__ status, uint8_t* __restrict__ out) {
  __shared__ int ws[32][64];
  const uint32_t lb = threadIdx.x >> 3, t = threadIdx.x & 7;
  const uint64_t b = blockIdx.x * 32ull + lb;
  bool ok = b < nblk;
  uint32_t si = 0;
  if (ok) {
    si = find_last(streams, ns, b, [](const DecStream& e) { return e.b0; });
    ok = status[si] == JS_OK;
  }
  if (ok) {  // column t
    const int16_t* c = coef + b * 64 + t;
    const int32_t* q = qt + 64ull * si + t;
    int d[8];
#pragma unroll
    for (int r = 0; r < 8; r++) d[r] = (int)c[8 * r] * q[8 * r];
    int z1 = (d[2] + d[6]) * F0541;
    const int t2 = z1 - d[6] * F1847, t3 = z1 + d[2] * F0765;
    const int t0 = (d[0] + d[4]) * (1 << CB), t1 = (d[0] - d[4]) * (1 << CB);
    const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
    int o0 = d[7], o1 = d[5], o2 = d[3], o3 = d[1];
    z1 = o0 + o3;
    int z2 = o1 + o2, z3 = o0 + o2, z4 = o1 + o3, z5 = (z3 + z4) * F1175;
    o0 *= F0298; o1 *= F2053; o2 *= F3072; o3 *= F1501;
    z1 *= -F0899; z2 *= -F2562; z3 = z3 * -F1961 + z5; z4 = z4 * -F0390 + z5;
    o0 += z1 + z3; o1 += z2 + z4; o2 += z2 + z3; o3 += z1 + z4;
    int* w = ws[lb] + t;
    w[0] = descale(t10 + o3, CB - P1);
    w[56] = descale(t10 - o3, CB - P1);
    w[8] = descale(t11 + o2, CB - P1);
    w[48] = descale(t11 - o2, CB - P1);
    w[16] = descale(t12 + o1, CB - P1);
    w[40] = descale(t12 - o1, CB - P1);
    w[24] = descale(t13 + o0, CB - P1);
    w[32] = descale(t13 - o0, CB - P1);
  }
  __syncwarp();
  if (!ok) return;
  const DecStream st = streams[si];
  const uint64_t l = b - st.b0;
  const uint32_t x0 = (uint32_t)(l % st.bw) * 8, y = (uint32_t)(l / st.bw) * 8 + t;
  if (y >= st.h) return;
  const int* d = ws[lb] + 8 * t;  // row t
  int z1 = (d[2] + d[6]) * F0541;
  const int t2 = z1 - d[6] * F1847, t3 = z1 + d[2] * F0765;
  const int t0 = (d[0] + d[4]) * (1 << CB), t1 = (d[0] - d[4]) * (1 << CB);
  const int t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  int o0 = d[7], o1 = d[5], o2 = d[3], o3 = d[1];
  z1 = o0 + o3;
  int z2 = o1 + o2, z3 = o0 + o2, z4 = o1 + o3, z5 = (z3 + z4) * F1175;
  o0 *= F0298; o1 *= F2053; o2 *= F3072; o3 *= F1501;
  z1 *= -F0899; z2 *= -F2562; z3 = z3 * -F1961 + z5; z4 = z4 * -F0390 + z5;
  o0 += z1 + z3; o1 += z2 + z4; o2 += z2 + z3; o3 += z1 + z4;
  const int v[8] = {t10 + o3, t11 + o2, t12 + o1, t13 + o0, t13 - o0, t12 - o1, t11 - o2, t10 - o3};
  uint8_t px[8];
#pragma unroll
  for (int x = 0; x < 8; x++) px[x] = (uint8_t)min(max(descale(v[x], CB + P1 + 3) + 128, 0), 255);
  uint8_t* dst = out + st.out_off + (uint64_t)y * st.w + x0;
  if (x0 + 8 <= st.w && ((uintptr_t)dst & 7) == 0) {
    uint2 pk;
    pk.x = px[0] | (px[1] << 8) | (px[2] << 16) | ((uint32_t)px[3] << 24);
    pk.y = px[4] | (px[5] << 8) | (px[6] << 16) | ((uint32_t)px[7] << 24);
    *reinterpret_cast<uint2*>(dst) = pk;
  } else {
#pragma unroll
    for (int x = 0; x < 8; x++)
      if (x0 + x < st.w) dst[x] = px[x];
  }
}

// ------------------------------------------------------------------ host
void huff_codes(const uint8_t bits[16], const uint8_t* vals, uint16_t* code, uint8_t* len) {
  uint32_t c = 0;
  int k = 0;
  for (int l = 1; l <= 16; l++) {
    for (int i = 0; i < bits[l - 1]; i++, k++) {
      code[vals[k]] = (uint16_t)c;
      len[vals[k]] = (uint8_t)l;
      c++;
    }
    c <<= 1;
  }
}

void enc_params(int quality, bool dri, EncParams* P) {
  memset(P, 0, sizeof(*P));
  const int s = quality < 50 ? 5000 / quality : 200 - 2 * quality;
  for (int i = 0; i < 64; i++) {
    const long v = ((long)LUMA_Q[i] * s + 50) / 100;
    P->q[i] = (uint16_t)(v < 1 ? 1 : v > 255 ? 255 : v);
  }
  huff_codes(DC_BITS, DC_VALS, P->dc_code, P->dc_len);
  huff_codes(AC_BITS, AC_VALS, P->ac_code, P->ac_len);
  std::vector<uint8_t> h;
  auto u16 = [&](unsigned v) { h.push_back((uint8_t)(v >> 8)); h.push_back((uint8_t)v); };
  u16(0xFFD8);
  u16(0xFFE0);  // JFIF 1.01, no density unit, 1:1, no thumbnail
  static const uint8_t app0[16] = {0x00, 0x10, 'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0};
  h.insert(h.end(), app0, app0 + 16);
  u16(0xFFDB); u16(67); h.push_back(0);
  for (int k = 0; k < 64; k++) h.push_back((uint8_t)P->q[ZIGZAG[k]]);
  u16(0xFFC0); u16(11); h.push_back(8);
  P->sof_at = (uint32_t)h.size();
  u16(0); u16(0);  // height, width: per chunk
  for (uint8_t b : {1, 1, 0x11, 0}) h.push_back(b);
  u16(0xFFC4); u16(3 + 16 + 12); h.push_back(0x00);
  h.insert(h.end(), DC_BITS, DC_BITS + 16);
  h.insert(h.end(), DC_VALS, DC_VALS + 12);
  u16(0xFFC4); u16(3 + 16 + 162); h.push_back(0x10);
  h.insert(h.end(), AC_BITS, AC_BITS + 16);
  h.insert(h.end(), AC_VALS, AC_VALS + 162);
  if (dri) {
    u16(0xFFDD); u16(4);
    P->dri_at = (uint32_t)h.size();
    u16(0);  // per chunk
  }
  u16(0xFFDA); u16(8);
  for (uint8_t b : {1, 1, 0x00, 0, 63, 0}) h.push_back(b);
  memcpy(P->hdr, h.data(), h.size());
  P->hdr_len = (uint32_t)h.size();
}

int check_shape(const uint32_t* shape, uint64_t c) {
  const uint64_t w = shape[3 * c], h = (uint64_t)shape[3 * c + 1] * shape[3 * c + 2];
  IGN_REQUIRE(w >= 1 && h >= 1, IGN_ERR_INVALID, "jpeg: chunk %llu is empty", (unsigned long long)c);
  IGN_REQUIRE(w <= JPEG_MAX_DIM && h <= JPEG_MAX_DIM, IGN_ERR_UNSUPPORTED,
              "jpeg: chunk %llu is %llu x %llu pixels (sx by sy*sz); JPEG holds at most 65535 per side",
              (unsigned long long)c, (unsigned long long)w, (unsigned long long)h);
  return IGN_OK;
}

size_t scan_tmp_bytes(uint64_t n) {
  size_t a = 0, b = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, a, (const uint64_t*)nullptr, (uint64_t*)nullptr, (int64_t)n);
  cub::DeviceScan::ExclusiveSum(nullptr, b, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int64_t)n);
  return (a > b ? a : b) + 256;
}

template <typename T>
int exclusive_sum(ign_ctx* ctx, void* tmp, size_t tmpb, const T* in, T* out, uint64_t n) {
  IGN_CUDA(cub::DeviceScan::ExclusiveSum(tmp, tmpb, in, out, (int64_t)n, ctx->stream));
  ctx->launches += 2;
  return IGN_OK;
}

int jpeg_encode_dev(ign_ctx* ctx, const uint8_t* in, uint64_t nch, const uint32_t* shape, int quality,
                    int64_t restart_interval, uint8_t* out, uint64_t cap, uint64_t* offsets, uint64_t* needed) {
  IGN_REQUIRE(quality >= 1 && quality <= 100, IGN_ERR_INVALID, "jpeg: quality %d outside 1..100", quality);
  IGN_REQUIRE(restart_interval <= 65535, IGN_ERR_INVALID, "jpeg: restart interval %lld exceeds 65535 blocks",
              (long long)restart_interval);
  *needed = 0;
  if (nch == 0) {
    if (offsets) offsets[0] = 0;
    return IGN_OK;
  }
  std::vector<EncChunk> ch(nch + 1);
  uint64_t px = 0, nb = 0, ni = 0;
  for (uint64_t c = 0; c < nch; c++) {
    IGN_TRY(check_shape(shape, c));
    EncChunk& e = ch[c];
    e.w = shape[3 * c];
    e.h = shape[3 * c + 1] * shape[3 * c + 2];
    e.bw = (e.w + 7) / 8;
    const uint64_t blocks = (uint64_t)e.bw * ((e.h + 7) / 8);
    e.dri = restart_interval < 0 ? e.bw : (uint32_t)restart_interval;
    e.per = e.dri ? e.dri : (uint32_t)blocks;
    e.in_off = px;
    e.b0 = nb;
    e.i0 = ni;
    px += (uint64_t)e.w * e.h;
    nb += blocks;
    ni += (blocks + e.per - 1) / e.per;
  }
  ch[nch].b0 = nb;
  ch[nch].i0 = ni;
  IGN_REQUIRE(nch < (1ull << 31) && ni < (1ull << 31), IGN_ERR_OVERFLOW, "jpeg: too many chunks in one call");
  EncParams P;
  enc_params(quality, restart_interval != 0, &P);
  const uint32_t nc = (uint32_t)nch;

  ScratchFrame f(ctx);
  EncChunk* dch;
  int16_t* coef;
  uint64_t *bits, *boff, *ibytes, *iwords, *iwoff, *osize, *ooff;
  void* tmp;
  IGN_TRY(f.take(&dch, nch + 1));
  IGN_TRY(f.take(&coef, nb * 64));
  IGN_TRY(f.take(&bits, nb + 1));
  IGN_TRY(f.take(&boff, nb + 1));
  IGN_TRY(f.take(&ibytes, ni + 1));
  IGN_TRY(f.take(&iwords, ni + 1));
  IGN_TRY(f.take(&iwoff, ni + 1));
  IGN_TRY(f.take(&osize, ni + 1));
  IGN_TRY(f.take(&ooff, ni + 1));
  size_t tmpb = scan_tmp_bytes(nb + 1);
  IGN_TRY(f.take(&tmp, tmpb));
  IGN_CUDA(cudaMemcpyAsync(dch, ch.data(), (nch + 1) * sizeof(EncChunk), cudaMemcpyHostToDevice, ctx->stream));
  IGN_LAUNCH(ctx, k_jpeg_fdct, blocks_for(nb, 32), 256, 0, in, dch, nc, nb, P, coef);
  IGN_LAUNCH(ctx, k_jpeg_bits, blocks_for(nb, 256), 256, 0, coef, dch, nc, nb, P, bits);
  IGN_CUDA(cudaMemsetAsync(bits + nb, 0, 8, ctx->stream));
  IGN_TRY(exclusive_sum(ctx, tmp, tmpb, bits, boff, nb + 1));
  IGN_LAUNCH(ctx, k_jpeg_ibytes, blocks_for(ni, 256), 256, 0, boff, dch, nc, ni, ibytes, iwords);
  IGN_CUDA(cudaMemsetAsync(iwords + ni, 0, 8, ctx->stream));
  IGN_TRY(exclusive_sum(ctx, tmp, tmpb, iwords, iwoff, ni + 1));
  uint64_t nw = 0;
  IGN_TRY(small_d2h(ctx, &nw, iwoff + ni, 8));
  IGN_TRY(small_sync(ctx));
  IGN_REQUIRE(nw < (1ull << 30), IGN_ERR_OVERFLOW, "jpeg: %llu bytes of entropy-coded data in one call exceed 4 GiB",
              (unsigned long long)nw * 4);

  ScratchFrame g(ctx);  // the data-dependent part
  uint32_t *raw, *ff, *ffscan;
  IGN_TRY(g.take(&raw, nw + 1));
  IGN_TRY(g.take(&ff, nw + 1));
  IGN_TRY(g.take(&ffscan, nw + 1));
  size_t tmpw = scan_tmp_bytes(nw + 1);
  void* tmp2 = tmp;
  if (tmpw > tmpb) IGN_TRY(g.take(&tmp2, tmpw));
  else tmpw = tmpb;
  IGN_CUDA(cudaMemsetAsync(raw, 0, (nw + 1) * 4, ctx->stream));
  IGN_LAUNCH(ctx, k_jpeg_pack, blocks_for(nb, 256), 256, 0, coef, dch, nc, nb, P, boff, iwoff, raw);
  IGN_LAUNCH(ctx, k_jpeg_ffcount, blocks_for(nw, 256), 256, 0, raw, nw, ff);
  IGN_CUDA(cudaMemsetAsync(ff + nw, 0, 4, ctx->stream));
  IGN_TRY(exclusive_sum(ctx, tmp2, tmpw, ff, ffscan, nw + 1));
  IGN_LAUNCH(ctx, k_jpeg_osize, blocks_for(ni, 256), 256, 0, ibytes, iwoff, ffscan, dch, nc, ni, P.hdr_len, osize);
  IGN_CUDA(cudaMemsetAsync(osize + ni, 0, 8, ctx->stream));
  IGN_TRY(exclusive_sum(ctx, tmp, tmpb, osize, ooff, ni + 1));
  uint64_t total = 0;
  IGN_TRY(small_d2h(ctx, &total, ooff + ni, 8));
  IGN_TRY(small_sync(ctx));
  *needed = total;
  if (out == nullptr || total > cap) return IGN_OK;
  uint64_t* doff;
  IGN_TRY(g.take(&doff, nch + 1));
  IGN_LAUNCH(ctx, k_jpeg_scatter, blocks_for(nw, 256), 256, 0, raw, nw, iwoff, ni, ibytes, ffscan, ooff, dch, nc,
             P.hdr_len, out);
  IGN_LAUNCH(ctx, k_jpeg_marks, blocks_for(ni, 256), 256, 0, ooff, dch, nc, ni, P, out, doff);
  IGN_CUDA(cudaMemcpyAsync(offsets, doff, (nch + 1) * 8, cudaMemcpyDeviceToHost, ctx->stream));
  IGN_CUDA(cudaStreamSynchronize(ctx->stream));
  return IGN_OK;
}

const char* js_reason(uint32_t st) {
  switch (st) {
    case JS_UNSUPPORTED: return "not a baseline / extended sequential 8-bit one-component Huffman stream "
                                "(progressive, arithmetic, lossless, 12-bit, multi-component and DNL streams are not supported)";
    case JS_SHAPE: return "its dimensions do not match the chunk shape";
    case JS_TOO_LONG: return "longer than 4 GiB";
    default: return "malformed or truncated";
  }
}

int jpeg_decode_dev(ign_ctx* ctx, const uint8_t* in, const uint64_t* offsets, uint64_t ns, const uint32_t* shape,
                    uint8_t* out) {
  if (ns == 0) return IGN_OK;
  IGN_REQUIRE(ns < (1u << 31), IGN_ERR_OVERFLOW, "jpeg: too many streams in one call");
  std::vector<DecStream> st(ns + 1);
  uint64_t nb = 0, px = 0;
  for (uint64_t s = 0; s < ns; s++) {
    IGN_TRY(check_shape(shape, s));
    IGN_REQUIRE(offsets[s + 1] >= offsets[s], IGN_ERR_INVALID, "jpeg: stream offsets decrease at %llu", (unsigned long long)s);
    DecStream& d = st[s];
    d.off = offsets[s];
    d.len = offsets[s + 1] - offsets[s];
    d.w = shape[3 * s];
    d.h = shape[3 * s + 1] * shape[3 * s + 2];
    d.bw = (d.w + 7) / 8;
    d.b0 = nb;
    d.out_off = px;
    nb += (uint64_t)d.bw * ((d.h + 7) / 8);
    px += (uint64_t)d.w * d.h;
  }
  st[ns].b0 = nb;
  ScratchFrame f(ctx);
  DecStream* dst;
  int16_t* coef;
  uint32_t *istart, *status;
  int32_t* qt;
  IGN_TRY(f.take(&dst, ns + 1));
  IGN_TRY(f.take(&coef, nb * 64));
  IGN_TRY(f.take(&istart, nb + ns));
  IGN_TRY(f.take(&qt, ns * 64));
  IGN_TRY(f.take(&status, ns));
  IGN_CUDA(cudaMemcpyAsync(dst, st.data(), (ns + 1) * sizeof(DecStream), cudaMemcpyHostToDevice, ctx->stream));
  IGN_CUDA(cudaMemsetAsync(coef, 0, nb * 128, ctx->stream));
  IGN_LAUNCH(ctx, k_jpeg_scan, (unsigned)ns, JQ_THREADS, 0, in, dst, istart, qt, coef, status);
  IGN_LAUNCH(ctx, k_jpeg_idct, blocks_for(nb, 32), 256, 0, coef, dst, (uint32_t)ns, nb, qt, status, out);
  std::vector<uint32_t> hs(ns);
  IGN_CUDA(cudaMemcpyAsync(hs.data(), status, ns * 4, cudaMemcpyDeviceToHost, ctx->stream));
  IGN_CUDA(cudaStreamSynchronize(ctx->stream));
  for (uint64_t s = 0; s < ns; s++)
    if (hs[s] != JS_OK) {
      set_error("jpeg: stream %llu is %s", (unsigned long long)s, js_reason(hs[s]));
      return hs[s] == JS_UNSUPPORTED ? IGN_ERR_UNSUPPORTED : IGN_ERR_INVALID;
    }
  return IGN_OK;
}

}  // namespace

}  // namespace ign

using namespace ign;

extern "C" {

int ign_jpeg_encode_dev(ign_ctx* ctx, const uint8_t* chunks, uint64_t n_chunks, const uint32_t* shapes, int quality,
                        int64_t restart_interval, uint8_t* out, uint64_t cap, uint64_t* offsets, uint64_t* n_bytes) {
  IGN_TRY(activate(ctx));
  IGN_REQUIRE(shapes && offsets && n_bytes && (chunks || n_chunks == 0), IGN_ERR_INVALID, "null argument");
  return jpeg_encode_dev(ctx, chunks, n_chunks, shapes, quality, restart_interval, out, cap, offsets, n_bytes);
}

int ign_jpeg_encode(ign_ctx* ctx, const uint8_t* chunks, uint64_t n_chunks, const uint32_t* shapes, int quality,
                    int64_t restart_interval, uint8_t* out, uint64_t cap, uint64_t* offsets, uint64_t* n_bytes) {
  IGN_REQUIRE(shapes && offsets && n_bytes && (chunks || n_chunks == 0), IGN_ERR_INVALID, "null argument");
  uint64_t px = 0;
  for (uint64_t c = 0; c < n_chunks; c++) px += (uint64_t)shapes[3 * c] * shapes[3 * c + 1] * shapes[3 * c + 2];
  std::vector<HostBuf> bufs = {{chunks, nullptr, px}, {nullptr, out, out ? cap : 0}};
  return staged(ctx, bufs, [&](void* const* d) -> int {
    IGN_TRY(jpeg_encode_dev(ctx, (const uint8_t*)d[0], n_chunks, shapes, quality, restart_interval, (uint8_t*)d[1],
                            cap, offsets, n_bytes));
    bufs[1].bytes = *n_bytes <= cap ? *n_bytes : 0;
    return IGN_OK;
  });
}

int ign_jpeg_decode_dev(ign_ctx* ctx, const uint8_t* streams, const uint64_t* offsets, uint64_t n_streams,
                        const uint32_t* shapes, uint8_t* out) {
  IGN_TRY(activate(ctx));
  IGN_REQUIRE(offsets && shapes && ((streams && out) || n_streams == 0), IGN_ERR_INVALID, "null argument");
  return jpeg_decode_dev(ctx, streams, offsets, n_streams, shapes, out);
}

int ign_jpeg_decode(ign_ctx* ctx, const uint8_t* streams, const uint64_t* offsets, uint64_t n_streams,
                    const uint32_t* shapes, uint8_t* out) {
  IGN_REQUIRE(offsets && shapes && ((streams && out) || n_streams == 0), IGN_ERR_INVALID, "null argument");
  uint64_t px = 0;
  for (uint64_t c = 0; c < n_streams; c++) px += (uint64_t)shapes[3 * c] * shapes[3 * c + 1] * shapes[3 * c + 2];
  IGN_REQUIRE(offsets[n_streams] >= offsets[0], IGN_ERR_INVALID, "jpeg: stream offsets decrease");
  return staged(ctx, {{streams, nullptr, offsets[n_streams]}, {nullptr, out, px}}, [&](void* const* d) {
    return jpeg_decode_dev(ctx, (const uint8_t*)d[0], offsets, n_streams, shapes, (uint8_t*)d[1]);
  });
}

}  // extern "C"
