/*
 * igneous_oracle.c -- CPU restatement of the igneous per-chunk hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is product code: only
 * tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl
 * reference legs may load this library, and only as the checker.
 *
 * The reference (seung-lab/igneous @ 3b6e5b6) holds no arithmetic of its own
 * for this path; it calls un-vendored third-party wheels that are absent from
 * the reference checkout and from this image:
 *   tinybrain >= 1.5.0               (requirements.txt:22)
 *   connected-components-3d >= 3.10.1 (requirements.txt:5)
 *   zmesh >= 1.13.1,<2.0             (requirements.txt:26)
 * This file restates their published algorithms, anchored on the reference's
 * call sites:
 *   igneous/tasks/image/image.py:46-55,91   (pooling)
 *   igneous/tasks/image/ccl.py:169-175      (CCL + dust)
 *   igneous/tasks/mesh/mesh.py:151,245,371-383 (mesher)
 *
 * PARITY STATUS (see DESIGN.md "Oracle"):
 *   - CCL: pinned structurally by the reference's own tests
 *     (test/test_ccl_tasks.py:188-208, 213-249) + cross-checked against
 *     scipy.ndimage.label in tests/test_oracle.py.
 *   - mode pooling: rule documented (COUNTLESS 2D); tie-break KATs in
 *     SURVEY.md 8(c).  Odd-edge handling: parity unpinned.
 *   - averaging: rounding rule (floor) and 4-mip renormalisation recalled
 *     from upstream tinybrain; parity unpinned (kept as a runtime enum).
 *   - marching cubes: classic Lorensen/Bourke table; corner convention,
 *     winding and vertex order: parity unpinned (compared after
 *     canonicalisation).
 *
 * All arrays are Fortran order: index = x + sx*(y + sy*z).
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORC_OK 0
#define ORC_EINVAL -1
#define ORC_ENOMEM -2

/* ------------------------------------------------------------------ */
/* Mode pooling 2x2x1 (tinybrain.downsample_segmentation, one mip).    */
/* Rule per 2x2 block a=(x,y) b=(x+1,y) c=(x,y+1) d=(x+1,y+1):         */
/*   out = a if (a==b || a==c) else (b if b==c else d)                 */
/* Odd extents: the lone column/row has only (a,c) / (a,b) -> a        */
/* (two samples: mode is a whenever they agree; tie -> first).         */
/* sparse: zeros are not counted (mode over the non-zero samples, ties  */
/* resolved in a,b,c,d order; all zero -> 0).                          */
/* ------------------------------------------------------------------ */
#define DEF_MODE_POOL(T, NAME)                                              \
  int NAME(const T* in, uint64_t sx, uint64_t sy, uint64_t sz, T* out,      \
           int sparse) {                                                    \
    const uint64_t ox = (sx + 1) / 2, oy = (sy + 1) / 2;                    \
    for (uint64_t z = 0; z < sz; z++) {                                     \
      for (uint64_t y = 0; y < oy; y++) {                                   \
        for (uint64_t x = 0; x < ox; x++) {                                 \
          const uint64_t x0 = 2 * x, y0 = 2 * y;                            \
          const int hx = (x0 + 1 < sx), hy = (y0 + 1 < sy);                 \
          const T a = in[x0 + sx * (y0 + sy * z)];                          \
          T r;                                                              \
          if (!sparse) {                                                    \
            if (hx && hy) {                                                 \
              const T b = in[x0 + 1 + sx * (y0 + sy * z)];                  \
              const T c = in[x0 + sx * (y0 + 1 + sy * z)];                  \
              const T d = in[x0 + 1 + sx * (y0 + 1 + sy * z)];              \
              r = (a == b || a == c) ? a : ((b == c) ? b : d);              \
            } else {                                                        \
              r = a;                                                        \
            }                                                               \
          } else {                                                          \
            T v[4];                                                         \
            int n = 0;                                                      \
            if (a) v[n++] = a;                                              \
            if (hx) {                                                       \
              T b = in[x0 + 1 + sx * (y0 + sy * z)];                        \
              if (b) v[n++] = b;                                            \
            }                                                               \
            if (hy) {                                                       \
              T c = in[x0 + sx * (y0 + 1 + sy * z)];                        \
              if (c) v[n++] = c;                                            \
            }                                                               \
            if (hx && hy) {                                                 \
              T d = in[x0 + 1 + sx * (y0 + 1 + sy * z)];                    \
              if (d) v[n++] = d;                                            \
            }                                                               \
            if (n == 0) r = 0;                                              \
            else if (n <= 2) r = v[0];                                      \
            else if (n == 3)                                                \
              r = (v[0] == v[1] || v[0] == v[2]) ? v[0]                     \
                  : ((v[1] == v[2]) ? v[1] : v[0]);                         \
            else                                                            \
              r = (v[0] == v[1] || v[0] == v[2]) ? v[0]                     \
                  : ((v[1] == v[2]) ? v[1] : v[3]);                         \
          }                                                                 \
          out[x + ox * (y + oy * z)] = r;                                   \
        }                                                                   \
      }                                                                     \
    }                                                                       \
    return ORC_OK;                                                          \
  }

DEF_MODE_POOL(uint8_t, orc_mode_pool_2x2x1_u8)
DEF_MODE_POOL(uint16_t, orc_mode_pool_2x2x1_u16)
DEF_MODE_POOL(uint32_t, orc_mode_pool_2x2x1_u32)
DEF_MODE_POOL(uint64_t, orc_mode_pool_2x2x1_u64)

/* ------------------------------------------------------------------ */
/* Average pooling 2x2x1 (tinybrain.downsample_with_averaging).        */
/* Upstream keeps un-normalised 2x2 sums in a wider integer: level k   */
/* of a group of four is rendered as accum >> 2k (floor), after the    */
/* fourth level the accumulator is renormalised (accum >>= 8) and the  */
/* next group starts from those truncated values.  Odd extents mirror  */
/* the lone row/column (counted twice) so the divisor stays 4.         */
/* rounding: 0 floor (upstream, recalled), 1 half-up, 2 half-even.     */
/* ------------------------------------------------------------------ */
static uint64_t orc_render(uint64_t acc, unsigned shift, int rounding) {
  if (rounding == 0 || shift == 0) return acc >> shift;
  const uint64_t half = 1ull << (shift - 1);
  if (rounding == 1) return (acc + half) >> shift;
  /* half-even */
  uint64_t q = acc >> shift, rem = acc & ((1ull << shift) - 1);
  if (rem > half || (rem == half && (q & 1))) q++;
  return q;
}

/* accumulate one 2x2x1 level of 64-bit sums (mirror odd edges) */
static uint64_t* orc_accum_2x2(const uint64_t* in, uint64_t sx, uint64_t sy,
                               uint64_t sz) {
  const uint64_t ox = (sx + 1) / 2, oy = (sy + 1) / 2;
  uint64_t* acc = (uint64_t*)malloc(sizeof(uint64_t) * ox * oy * sz);
  if (!acc) return NULL;
  for (uint64_t z = 0; z < sz; z++)
    for (uint64_t y = 0; y < oy; y++)
      for (uint64_t x = 0; x < ox; x++) {
        const uint64_t x0 = 2 * x, y0 = 2 * y;
        const uint64_t x1 = (x0 + 1 < sx) ? x0 + 1 : x0;
        const uint64_t y1 = (y0 + 1 < sy) ? y0 + 1 : y0;
        acc[x + ox * (y + oy * z)] =
            in[x0 + sx * (y0 + sy * z)] + in[x1 + sx * (y0 + sy * z)] +
            in[x0 + sx * (y1 + sy * z)] + in[x1 + sx * (y1 + sy * z)];
      }
  return acc;
}

#define DEF_AVG_POOL(T, NAME)                                                 \
  int NAME(const T* in, uint64_t sx, uint64_t sy, uint64_t sz, int num_mips,  \
           T** outs, int rounding) {                                          \
    if (num_mips < 1) return ORC_EINVAL;                                      \
    uint64_t n = sx * sy * sz;                                                \
    uint64_t* cur = (uint64_t*)malloc(sizeof(uint64_t) * (n ? n : 1));        \
    if (!cur) return ORC_ENOMEM;                                              \
    for (uint64_t i = 0; i < n; i++) cur[i] = in[i];                          \
    for (int mip = 0; mip < num_mips; mip++) {                                \
      uint64_t* acc = orc_accum_2x2(cur, sx, sy, sz);                         \
      free(cur);                                                              \
      if (!acc) return ORC_ENOMEM;                                            \
      sx = (sx + 1) / 2;                                                      \
      sy = (sy + 1) / 2;                                                      \
      n = sx * sy * sz;                                                       \
      const unsigned shift = 2 * ((mip % 4) + 1);                             \
      for (uint64_t i = 0; i < n; i++)                                        \
        outs[mip][i] = (T)orc_render(acc[i], shift, rounding);                \
      if (shift == 8)                                                         \
        for (uint64_t i = 0; i < n; i++)                                      \
          acc[i] = orc_render(acc[i], shift, rounding);                       \
      cur = acc;                                                              \
    }                                                                         \
    free(cur);                                                                \
    return ORC_OK;                                                            \
  }

DEF_AVG_POOL(uint8_t, orc_avg_pool_2x2x1_u8)
DEF_AVG_POOL(uint16_t, orc_avg_pool_2x2x1_u16)
DEF_AVG_POOL(uint32_t, orc_avg_pool_2x2x1_u32)

/* float32: plain mean of the four (mirrored) samples at every level,   */
/* op order ((a+b)+(c+d))*0.25f.  Parity unpinned.                     */
int orc_avg_pool_2x2x1_f32(const float* in, uint64_t sx, uint64_t sy,
                           uint64_t sz, int num_mips, float** outs,
                           int rounding) {
  (void)rounding;
  const float* cur = in;
  for (int mip = 0; mip < num_mips; mip++) {
    const uint64_t ox = (sx + 1) / 2, oy = (sy + 1) / 2;
    float* o = outs[mip];
    for (uint64_t z = 0; z < sz; z++)
      for (uint64_t y = 0; y < oy; y++)
        for (uint64_t x = 0; x < ox; x++) {
          const uint64_t x0 = 2 * x, y0 = 2 * y;
          const uint64_t x1 = (x0 + 1 < sx) ? x0 + 1 : x0;
          const uint64_t y1 = (y0 + 1 < sy) ? y0 + 1 : y0;
          const float a = cur[x0 + sx * (y0 + sy * z)];
          const float b = cur[x1 + sx * (y0 + sy * z)];
          const float c = cur[x0 + sx * (y1 + sy * z)];
          const float d = cur[x1 + sx * (y1 + sy * z)];
          o[x + ox * (y + oy * z)] = ((a + b) + (c + d)) * 0.25f;
        }
    cur = o;
    sx = ox;
    sy = oy;
  }
  return ORC_OK;
}

/* ------------------------------------------------------------------ */
/* Block pooling with factors 1 or 2 per axis (the other                */
/* tinybrain.downsample_* factors igneous can request: (2,2,2) for      */
/* --volumetric, igneous_cli/cli.py; DownsampleMethods, types.py:6-12). */
/* One level.  Samples of a block are visited x fastest, then y, then z.*/
/*  mode  (sparse = zeros ignored; all zero -> 0):                      */
/*    planar factor (fx*fy*fz == 4) and exactly four samples left:      */
/*      the COUNTLESS 2-D pick of the 2x2x1 kernel, so that (2,2,1)     */
/*      through this path equals orc_mode_pool_2x2x1;                   */
/*    otherwise: the value with the highest count, ties -> the earliest */
/*      sample (what replicate-the-edge + first-maximum gives).         */
/*  average: sum over the block with the lone row/column/slice of an    */
/*    odd extent counted twice (divisor stays fx*fy*fz), rendered with  */
/*    the rounding enum of the 2x2x1 kernel.  Recursive per mip.        */
/*    sparse: mean of the non-zero samples (replicated edge samples     */
/*    included), 0 when there are none.                                 */
/* PARITY UNPINNED: tie-break and edge rules are recalled, not pinned.  */
/* ------------------------------------------------------------------ */
#define DEF_BLOCK_MODE(T, NAME)                                              \
  int NAME(const T* in, uint64_t sx, uint64_t sy, uint64_t sz, uint32_t fx,  \
           uint32_t fy, uint32_t fz, int sparse, T* out) {                   \
    if (fx < 1 || fx > 2 || fy < 1 || fy > 2 || fz < 1 || fz > 2)           \
      return ORC_EINVAL;                                                     \
    const uint64_t ox = (sx + fx - 1) / fx, oy = (sy + fy - 1) / fy,         \
                   oz = (sz + fz - 1) / fz;                                  \
    const int planar = (fx * fy * fz == 4);                                  \
    for (uint64_t z = 0; z < oz; z++)                                        \
      for (uint64_t y = 0; y < oy; y++)                                      \
        for (uint64_t x = 0; x < ox; x++) {                                  \
          T v[8];                                                            \
          int n = 0;                                                         \
          for (uint32_t dz = 0; dz < fz && z * fz + dz < sz; dz++)           \
            for (uint32_t dy = 0; dy < fy && y * fy + dy < sy; dy++)         \
              for (uint32_t dx = 0; dx < fx && x * fx + dx < sx; dx++) {     \
                const T s = in[(x * fx + dx) +                               \
                               sx * ((y * fy + dy) + sy * (z * fz + dz))];   \
                if (!sparse || s != 0) v[n++] = s;                           \
              }                                                              \
          T r = 0;                                                           \
          if (planar && n == 4) {                                            \
            r = (v[0] == v[1] || v[0] == v[2]) ? v[0]                        \
                : ((v[1] == v[2]) ? v[1] : v[3]);                            \
          } else {                                                           \
            int best = 0;                                                    \
            for (int t = 0; t < n; t++) {                                    \
              int ct = 0;                                                    \
              for (int q = 0; q < n; q++) ct += (v[q] == v[t]);              \
              if (ct > best) {                                               \
                best = ct;                                                   \
                r = v[t];                                                    \
              }                                                              \
            }                                                                \
          }                                                                  \
          out[x + ox * (y + oy * z)] = r;                                    \
        }                                                                    \
    return ORC_OK;                                                           \
  }

DEF_BLOCK_MODE(uint8_t, orc_block_mode_u8)
DEF_BLOCK_MODE(uint16_t, orc_block_mode_u16)
DEF_BLOCK_MODE(uint32_t, orc_block_mode_u32)
DEF_BLOCK_MODE(uint64_t, orc_block_mode_u64)

static uint64_t orc_render_div(uint64_t acc, uint64_t n, int rounding) {
  if (n == 0) return 0;
  uint64_t q = acc / n;
  const uint64_t rem2 = 2 * (acc - q * n);
  if (rounding == 1) q += (rem2 >= n);
  else if (rounding == 2) q += (rem2 > n || (rem2 == n && (q & 1)));
  return q;
}

#define DEF_BLOCK_AVG(T, NAME)                                               \
  int NAME(const T* in, uint64_t sx, uint64_t sy, uint64_t sz, uint32_t fx,  \
           uint32_t fy, uint32_t fz, int flag, T* out) {                     \
    if (fx < 1 || fx > 2 || fy < 1 || fy > 2 || fz < 1 || fz > 2)           \
      return ORC_EINVAL;                                                     \
    const int rounding = flag % 3, sparse = flag >= 3;                       \
    const uint64_t ox = (sx + fx - 1) / fx, oy = (sy + fy - 1) / fy,         \
                   oz = (sz + fz - 1) / fz;                                  \
    const unsigned shift = (fx == 2) + (fy == 2) + (fz == 2);                \
    for (uint64_t z = 0; z < oz; z++)                                        \
      for (uint64_t y = 0; y < oy; y++)                                      \
        for (uint64_t x = 0; x < ox; x++) {                                  \
          uint64_t acc = 0, nonzero = 0;                                     \
          for (uint32_t dz = 0; dz < fz; dz++)                               \
            for (uint32_t dy = 0; dy < fy; dy++)                             \
              for (uint32_t dx = 0; dx < fx; dx++) {                         \
                uint64_t xx = x * fx + dx, yy = y * fy + dy, zz = z * fz + dz; \
                if (xx >= sx) xx = sx - 1;                                   \
                if (yy >= sy) yy = sy - 1;                                   \
                if (zz >= sz) zz = sz - 1;                                   \
                acc += in[xx + sx * (yy + sy * zz)];                         \
                nonzero += (in[xx + sx * (yy + sy * zz)] != 0);              \
              }                                                              \
          out[x + ox * (y + oy * z)] =                                       \
              sparse ? (T)orc_render_div(acc, nonzero, rounding)             \
                     : (T)orc_render(acc, shift, rounding);                  \
        }                                                                    \
    return ORC_OK;                                                           \
  }

DEF_BLOCK_AVG(uint8_t, orc_block_avg_u8)
DEF_BLOCK_AVG(uint16_t, orc_block_avg_u16)
DEF_BLOCK_AVG(uint32_t, orc_block_avg_u32)

/* float32: pairwise sums in x, then y, then z (each a float add), times   */
/* the exact reciprocal of the block size                                  */
int orc_block_avg_f32(const float* in, uint64_t sx, uint64_t sy, uint64_t sz,
                      uint32_t fx, uint32_t fy, uint32_t fz, int flag,
                      float* out) {
  const int sparse = flag >= 3;
  if (fx < 1 || fx > 2 || fy < 1 || fy > 2 || fz < 1 || fz > 2) return ORC_EINVAL;
  const uint64_t ox = (sx + fx - 1) / fx, oy = (sy + fy - 1) / fy,
                 oz = (sz + fz - 1) / fz;
  const float scale = 1.0f / (float)(fx * fy * fz);
  for (uint64_t z = 0; z < oz; z++)
    for (uint64_t y = 0; y < oy; y++)
      for (uint64_t x = 0; x < ox; x++) {
        float zs[2] = {0.0f, 0.0f};
        int nonzero = 0;
        for (uint32_t dz = 0; dz < fz; dz++) {
          float ys[2] = {0.0f, 0.0f};
          for (uint32_t dy = 0; dy < fy; dy++) {
            float xs[2] = {0.0f, 0.0f};
            for (uint32_t dx = 0; dx < fx; dx++) {
              uint64_t xx = x * fx + dx, yy = y * fy + dy, zz = z * fz + dz;
              if (xx >= sx) xx = sx - 1;
              if (yy >= sy) yy = sy - 1;
              if (zz >= sz) zz = sz - 1;
              xs[dx] = in[xx + sx * (yy + sy * zz)];
              nonzero += (xs[dx] != 0.0f);
            }
            ys[dy] = (fx == 2) ? (float)(xs[0] + xs[1]) : xs[0];
          }
          zs[dz] = (fy == 2) ? (float)(ys[0] + ys[1]) : ys[0];
        }
        const float sum = (fz == 2) ? (float)(zs[0] + zs[1]) : zs[0];
        if (sparse) out[x + ox * (y + oy * z)] = nonzero ? sum / (float)nonzero : 0.0f;
        else out[x + ox * (y + oy * z)] = sum * scale;
      }
  return ORC_OK;
}

/* ------------------------------------------------------------------ */
/* 6-connected multi-label CCL (cc3d.connected_components,             */
/* connectivity=6; called at igneous/tasks/image/ccl.py:173,235,339).  */
/* Two voxels are connected iff they are face adjacent and hold the    */
/* same non-zero value.  Output ids 1..N are assigned in order of the  */
/* first voxel of each component in Fortran raster order (== rank of   */
/* the component's minimum linear index); background stays 0.          */
/* ------------------------------------------------------------------ */
static uint64_t uf_find(uint64_t* p, uint64_t i) {
  while (p[i] != i) {
    p[i] = p[p[i]];
    i = p[i];
  }
  return i;
}
static void uf_union(uint64_t* p, uint64_t a, uint64_t b) {
  a = uf_find(p, a);
  b = uf_find(p, b);
  if (a < b) p[b] = a;
  else if (b < a) p[a] = b;
}

#define DEF_CCL6(T, NAME)                                                    \
  int NAME(const T* in, uint64_t sx, uint64_t sy, uint64_t sz,               \
           uint64_t* out, uint64_t* n_out) {                                 \
    const uint64_t n = sx * sy * sz;                                         \
    uint64_t* p = (uint64_t*)malloc(sizeof(uint64_t) * (n ? n : 1));         \
    if (!p) return ORC_ENOMEM;                                               \
    for (uint64_t i = 0; i < n; i++) p[i] = i;                               \
    for (uint64_t z = 0; z < sz; z++)                                        \
      for (uint64_t y = 0; y < sy; y++)                                      \
        for (uint64_t x = 0; x < sx; x++) {                                  \
          const uint64_t i = x + sx * (y + sy * z);                          \
          const T v = in[i];                                                 \
          if (!v) continue;                                                  \
          if (x && in[i - 1] == v) uf_union(p, i, i - 1);                    \
          if (y && in[i - sx] == v) uf_union(p, i, i - sx);                  \
          if (z && in[i - sx * sy] == v) uf_union(p, i, i - sx * sy);        \
        }                                                                    \
    uint64_t next = 0;                                                       \
    /* roots are minimum indices: a raster scan meets the root first */      \
    for (uint64_t i = 0; i < n; i++) {                                       \
      if (!in[i]) { out[i] = 0; continue; }                                  \
      const uint64_t r = uf_find(p, i);                                      \
      if (r == i) out[i] = ++next;                                           \
      else out[i] = out[r];                                                  \
    }                                                                        \
    free(p);                                                                 \
    if (n_out) *n_out = next;                                                \
    return ORC_OK;                                                           \
  }

DEF_CCL6(uint8_t, orc_ccl6_u8)
DEF_CCL6(uint16_t, orc_ccl6_u16)
DEF_CCL6(uint32_t, orc_ccl6_u32)
DEF_CCL6(uint64_t, orc_ccl6_u64)

/* ------------------------------------------------------------------ */
/* Multi-label marching cubes (zmesh.Mesher.mesh, mesh.py:245).        */
/* For every 2x2x2 cube and every distinct non-zero corner label L the */
/* classic 256-case table is evaluated with bit i set iff corner i==L. */
/* Vertices sit on edge midpoints; coordinates are emitted in integer  */
/* half-voxel units (2*x + dx).  Triangles are emitted per label in    */
/* cube raster order (x fastest), table order inside a cube.           */
/*                                                                     */
/* Corner numbering (Bourke): 0:(0,0,0) 1:(1,0,0) 2:(1,1,0) 3:(0,1,0)   */
/*                            4:(0,0,1) 5:(1,0,1) 6:(1,1,1) 7:(0,1,1)   */
/* Edge numbering: 0:0-1 1:1-2 2:2-3 3:3-0 4:4-5 5:5-6 6:6-7 7:7-4     */
/*                 8:0-4 9:1-5 10:2-6 11:3-7                           */
/* ------------------------------------------------------------------ */
#include "mc_table.h"

/* edge midpoint offsets in half-voxel units relative to 2*(x,y,z) */
static const int8_t orc_edge_mid[12][3] = {
    {1, 0, 0}, {2, 1, 0}, {1, 2, 0}, {0, 1, 0}, {1, 0, 2}, {2, 1, 2},
    {1, 2, 2}, {0, 1, 2}, {0, 0, 1}, {2, 0, 1}, {2, 2, 1}, {0, 2, 1}};
static const int8_t orc_corner[8][3] = {{0, 0, 0}, {1, 0, 0}, {1, 1, 0},
                                        {0, 1, 0}, {0, 0, 1}, {1, 0, 1},
                                        {1, 1, 1}, {0, 1, 1}};

/*
 * Two-call protocol: with tri_label == NULL only counts triangles.
 * tri_label[t]  : label of triangle t
 * tri_verts[9t..]: three vertices (x,y,z) in half-voxel integer units,
 * ordered: all cubes in raster order, labels inside a cube in ascending
 * corner order of first appearance, triangles in table order.
 * flip != 0 reverses the winding of every triangle.
 */
#define DEF_MC(T, NAME)                                                       \
  int NAME(const T* in, uint64_t sx, uint64_t sy, uint64_t sz,                \
           uint64_t* n_tri, uint64_t* tri_label, uint32_t* tri_verts,         \
           int flip) {                                                        \
    uint64_t nt = 0;                                                          \
    if (sx < 2 || sy < 2 || sz < 2) { *n_tri = 0; return ORC_OK; }            \
    for (uint64_t z = 0; z + 1 < sz; z++)                                     \
      for (uint64_t y = 0; y + 1 < sy; y++)                                   \
        for (uint64_t x = 0; x + 1 < sx; x++) {                               \
          T c[8];                                                             \
          int any = 0;                                                        \
          for (int k = 0; k < 8; k++) {                                       \
            c[k] = in[(x + orc_corner[k][0]) +                                \
                      sx * ((y + orc_corner[k][1]) +                          \
                            sy * (z + orc_corner[k][2]))];                    \
            any |= (c[k] != 0);                                               \
          }                                                                   \
          if (!any) continue;                                                 \
          for (int k = 0; k < 8; k++) {                                       \
            const T L = c[k];                                                 \
            if (!L) continue;                                                 \
            int seen = 0;                                                     \
            for (int j = 0; j < k; j++) seen |= (c[j] == L);                  \
            if (seen) continue;                                               \
            int idx = 0;                                                      \
            for (int j = 0; j < 8; j++) idx |= (c[j] == L) << j;              \
            const int8_t* tt = mc_tri_table[idx];                             \
            for (int e = 0; tt[e] >= 0; e += 3) {                             \
              if (tri_label) {                                                \
                tri_label[nt] = (uint64_t)L;                                  \
                for (int v = 0; v < 3; v++) {                                 \
                  const int ed = tt[e + (flip ? 2 - v : v)];                  \
                  tri_verts[9 * nt + 3 * v + 0] =                             \
                      (uint32_t)(2 * x + orc_edge_mid[ed][0]);                \
                  tri_verts[9 * nt + 3 * v + 1] =                             \
                      (uint32_t)(2 * y + orc_edge_mid[ed][1]);                \
                  tri_verts[9 * nt + 3 * v + 2] =                             \
                      (uint32_t)(2 * z + orc_edge_mid[ed][2]);                \
                }                                                             \
              }                                                               \
              nt++;                                                           \
            }                                                                 \
          }                                                                   \
        }                                                                     \
    *n_tri = nt;                                                              \
    return ORC_OK;                                                            \
  }

DEF_MC(uint8_t, orc_marching_cubes_u8)
DEF_MC(uint16_t, orc_marching_cubes_u16)
DEF_MC(uint32_t, orc_marching_cubes_u32)
DEF_MC(uint64_t, orc_marching_cubes_u64)

/* table accessors so tests can validate the table itself */
const int8_t* orc_mc_tri_table(void) { return &mc_tri_table[0][0]; }

/* ------------------------------------------------------------------ */
/* Weld (Mesher.get without simplification, mesh.py:376-381): per      */
/* label, unique vertices ordered by packed (z,y,x) key; faces keep    */
/* cube raster order.  Outputs are grouped by ascending label.         */
/*   tri_order[T]   : input triangle index of output triangle t        */
/*   uniq_label[U], uniq_xyz[3U] : unique vertices (label major)       */
/*   faces[3T]      : index into the unique vertex list (GLOBAL index; */
/*                    subtract the label's first vertex for local ids) */
/* ------------------------------------------------------------------ */
typedef struct { uint64_t label, key; uint64_t corner; } orc_vrec;
typedef struct { uint64_t label, idx; } orc_trec;

static int orc_cmp_v(const void* a, const void* b) {
  const orc_vrec *x = (const orc_vrec*)a, *y = (const orc_vrec*)b;
  if (x->label != y->label) return x->label < y->label ? -1 : 1;
  if (x->key != y->key) return x->key < y->key ? -1 : 1;
  return 0;
}
static int orc_cmp_t(const void* a, const void* b) {
  const orc_trec *x = (const orc_trec*)a, *y = (const orc_trec*)b;
  if (x->label != y->label) return x->label < y->label ? -1 : 1;
  return x->idx < y->idx ? -1 : (x->idx > y->idx ? 1 : 0);
}

int orc_weld(const uint64_t* tri_label, const uint32_t* tri_verts, uint64_t T,
             uint64_t* tri_order, uint64_t* uniq_label, uint32_t* uniq_xyz,
             uint32_t* faces, uint64_t* n_uniq) {
  *n_uniq = 0;
  if (T == 0) return ORC_OK;
  orc_trec* tr = (orc_trec*)malloc(sizeof(orc_trec) * T);
  orc_vrec* vr = (orc_vrec*)malloc(sizeof(orc_vrec) * 3 * T);
  uint64_t* newpos = (uint64_t*)malloc(sizeof(uint64_t) * T);
  if (!tr || !vr || !newpos) { free(tr); free(vr); free(newpos); return ORC_ENOMEM; }
  for (uint64_t t = 0; t < T; t++) { tr[t].label = tri_label[t]; tr[t].idx = t; }
  qsort(tr, T, sizeof(orc_trec), orc_cmp_t);
  for (uint64_t t = 0; t < T; t++) { tri_order[t] = tr[t].idx; newpos[tr[t].idx] = t; }
  for (uint64_t t = 0; t < T; t++)
    for (int v = 0; v < 3; v++) {
      const uint32_t* p = tri_verts + 9 * t + 3 * v;
      vr[3 * t + v].label = tri_label[t];
      vr[3 * t + v].key = ((uint64_t)p[2] << 42) | ((uint64_t)p[1] << 21) | p[0];
      vr[3 * t + v].corner = 3 * newpos[t] + v;
    }
  qsort(vr, 3 * T, sizeof(orc_vrec), orc_cmp_v);
  uint64_t u = 0;
  for (uint64_t i = 0; i < 3 * T; i++) {
    if (i == 0 || vr[i].label != vr[i - 1].label || vr[i].key != vr[i - 1].key) {
      uniq_label[u] = vr[i].label;
      uniq_xyz[3 * u + 0] = (uint32_t)(vr[i].key & 0x1FFFFF);
      uniq_xyz[3 * u + 1] = (uint32_t)((vr[i].key >> 21) & 0x1FFFFF);
      uniq_xyz[3 * u + 2] = (uint32_t)(vr[i].key >> 42);
      u++;
    }
    faces[vr[i].corner] = (uint32_t)(u - 1);
  }
  *n_uniq = u;
  free(tr); free(vr); free(newpos);
  return ORC_OK;
}

/* ------------------------------------------------------------------ */
/* Synthetic jittered-Voronoi segmentation (SURVEY.md 8(d)); same      */
/* integer hash as igneous_b200/csrc/synth.cu and oracle.synth_seg_np. */
/* ------------------------------------------------------------------ */
static uint64_t orc_mix64(uint64_t z) {
  z += 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}
static uint64_t orc_cell_hash(uint64_t seed, int64_t cx, int64_t cy, int64_t cz) {
  uint64_t h = orc_mix64(seed + (uint64_t)cx * 0x100000001B3ull);
  h = orc_mix64(h ^ ((uint64_t)cy * 0xC2B2AE3D27D4EB4Full));
  h = orc_mix64(h ^ ((uint64_t)cz * 0x165667B19E3779F9ull));
  return h;
}
static int64_t orc_floordiv(int64_t a, int64_t b) {
  int64_t q = a / b;
  if ((a % b != 0) && ((a < 0) != (b < 0))) q--;
  return q;
}

int orc_synth_seg_u64(uint64_t* out, uint64_t sx, uint64_t sy, uint64_t sz,
                      int64_t ox, int64_t oy, int64_t oz, int pitch,
                      uint64_t num_ids, uint64_t seed, uint64_t id_base) {
  for (uint64_t z = 0; z < sz; z++)
    for (uint64_t y = 0; y < sy; y++)
      for (uint64_t x = 0; x < sx; x++) {
        const int64_t X = (int64_t)x + ox, Y = (int64_t)y + oy, Z = (int64_t)z + oz;
        const int64_t cx = orc_floordiv(X, pitch), cy = orc_floordiv(Y, pitch),
                      cz = orc_floordiv(Z, pitch);
        int64_t d1 = INT64_MAX, d2 = INT64_MAX;
        uint64_t id1 = 0;
        for (int dz = -1; dz <= 1; dz++)
          for (int dy = -1; dy <= 1; dy++)
            for (int dx = -1; dx <= 1; dx++) {
              const int64_t ccx = cx + dx, ccy = cy + dy, ccz = cz + dz;
              const uint64_t h = orc_cell_hash(seed, ccx, ccy, ccz);
              const int64_t px = ccx * pitch + (int64_t)((h & 0xFFFF) % (uint64_t)pitch);
              const int64_t py = ccy * pitch + (int64_t)(((h >> 16) & 0xFFFF) % (uint64_t)pitch);
              const int64_t pz = ccz * pitch + (int64_t)(((h >> 32) & 0xFFFF) % (uint64_t)pitch);
              const int64_t d = (X - px) * (X - px) + (Y - py) * (Y - py) + (Z - pz) * (Z - pz);
              if (d < d1) { d2 = d1; d1 = d; id1 = id_base + 1 + orc_mix64(h) % num_ids; }
              else if (d < d2) { d2 = d; }
            }
        out[x + sx * (y + sy * z)] = ((d2 - d1) < 2 * (int64_t)pitch) ? 0 : id1;
      }
  return ORC_OK;
}

/* ------------------------------------------------------------------ */
/* Quadric edge-collapse simplification (Mesher.get(reduction_factor,   */
/* max_error), igneous/tasks/mesh/mesh.py:376-381).                    */
/*                                                                     */
/* PARITY UNPINNED: zmesh's simplifier (zi_lib, sequential heap order) */
/* is absent; this restates the product's own deterministic algorithm  */
/* so the GPU implementation can be checked bit for bit:               */
/*   - per-vertex Garland-Heckbert plane quadrics (unit normals);      */
/*   - boundary vertices are locked (chunk borders must still stitch); */
/*   - rounds: every interior edge gets cost = min over {u, v, mid} of */
/*     p^T (Qu+Qv) p, valid iff cost <= max_err^2, the link condition  */
/*     holds and no incident face flips; each vertex takes the minimum */
/*     (float32 cost, half-edge id) key over its edges (key1), then    */
/*     the minimum over its neighbours (key2); an edge collapses iff   */
/*     its key equals key2 of both endpoints -> collapses of one round */
/*     are independent.  Stop rules are per label (see orc_simplify).  */
/* All arithmetic in double without FMA contraction.                   */
/* ------------------------------------------------------------------ */
#include <math.h>
#include <stdio.h>
#define SIMP_NONE 0xFFFFFFFFu
#define SIMP_MAXV 32
#define SIMP_KEYMAX 0xFFFFFFFFFFFFFFFFull

typedef struct {
  uint64_t U, T;
  double* pos;       /* 3U */
  double* Q;         /* 10U */
  uint32_t* face;    /* 3T */
  const uint32_t* flabel;
  uint8_t* falive;
  uint8_t* valive;
  uint8_t* vbound;
  uint32_t *next, *head, *tail;
  uint64_t *key1, *key2;
} simp_t;

static void simp_plane_quadric(const double* a, const double* b, const double* c, double* K, int* ok) {
  const double ux = b[0] - a[0], uy = b[1] - a[1], uz = b[2] - a[2];
  const double vx = c[0] - a[0], vy = c[1] - a[1], vz = c[2] - a[2];
  double nx = uy * vz - uz * vy, ny = uz * vx - ux * vz, nz = ux * vy - uy * vx;
  const double len = sqrt(nx * nx + ny * ny + nz * nz);
  if (!(len > 0.0)) { *ok = 0; return; }
  nx = nx / len; ny = ny / len; nz = nz / len;
  const double d = -(nx * a[0] + ny * a[1] + nz * a[2]);
  K[0] = nx * nx; K[1] = nx * ny; K[2] = nx * nz; K[3] = nx * d;
  K[4] = ny * ny; K[5] = ny * nz; K[6] = ny * d;
  K[7] = nz * nz; K[8] = nz * d; K[9] = d * d;
  *ok = 1;
}

static double simp_qeval(const double* q, const double* p) {
  const double x = p[0], y = p[1], z = p[2];
  return q[0] * x * x + 2.0 * q[1] * x * y + 2.0 * q[2] * x * z + 2.0 * q[3] * x +
         q[4] * y * y + 2.0 * q[5] * y * z + 2.0 * q[6] * y + q[7] * z * z + 2.0 * q[8] * z + q[9];
}

/* twin of half-edge (u->v) of face f: another alive face containing u and v.
   returns count of such faces, *twin = node id (3g+c) of g's corner holding u */
static int simp_twins(const simp_t* s, uint32_t f, uint32_t u, uint32_t v, uint32_t* twin) {
  int cnt = 0;
  for (uint32_t h = s->head[u]; h != SIMP_NONE; h = s->next[h]) {
    const uint32_t g = h / 3;
    if (g == f || !s->falive[g]) continue;
    const uint32_t* fv = s->face + 3 * g;
    if (fv[0] == v || fv[1] == v || fv[2] == v) {
      if (cnt == 0) *twin = h;
      cnt++;
    }
  }
  return cnt;
}

typedef struct { int valid; double cost; uint32_t keep, remove; double p[3]; } simp_eval_t;

static int simp_ring(const simp_t* s, uint32_t w, uint32_t* faces, uint32_t* nbr, int* nf, int* nn) {
  *nf = 0; *nn = 0;
  for (uint32_t h = s->head[w]; h != SIMP_NONE; h = s->next[h]) {
    const uint32_t g = h / 3;
    if (!s->falive[g]) continue;
    if (*nf >= SIMP_MAXV) return 0;
    faces[(*nf)++] = g;
    const uint32_t* fv = s->face + 3 * g;
    for (int k = 0; k < 3; k++) {
      const uint32_t x = fv[k];
      if (x == w) continue;
      int seen = 0;
      for (int j = 0; j < *nn; j++) seen |= (nbr[j] == x);
      if (!seen) {
        if (*nn >= SIMP_MAXV) return 0;
        nbr[(*nn)++] = x;
      }
    }
  }
  return 1;
}

/* cheap part: placement and quadric cost (no ring walks) */
static void simp_cost(const simp_t* s, uint32_t u, uint32_t v, double max_err2, simp_eval_t* e) {
  e->valid = 0;
  if (s->vbound[u] && s->vbound[v]) return;
  double q[10];
  for (int i = 0; i < 10; i++) q[i] = s->Q[10 * (uint64_t)u + i] + s->Q[10 * (uint64_t)v + i];
  const double* pu = s->pos + 3 * (uint64_t)u;
  const double* pv = s->pos + 3 * (uint64_t)v;
  double best[3], cost;
  if (s->vbound[u]) {
    e->keep = u; e->remove = v;
    best[0] = pu[0]; best[1] = pu[1]; best[2] = pu[2];
    cost = simp_qeval(q, best);
  } else if (s->vbound[v]) {
    e->keep = v; e->remove = u;
    best[0] = pv[0]; best[1] = pv[1]; best[2] = pv[2];
    cost = simp_qeval(q, best);
  } else {
    e->keep = u < v ? u : v;
    e->remove = u < v ? v : u;
    const double* pk = s->pos + 3 * (uint64_t)e->keep;
    const double* pr = s->pos + 3 * (uint64_t)e->remove;
    double mid[3] = {(pk[0] + pr[0]) * 0.5, (pk[1] + pr[1]) * 0.5, (pk[2] + pr[2]) * 0.5};
    const double ck = simp_qeval(q, pk), cr = simp_qeval(q, pr), cm = simp_qeval(q, mid);
    cost = ck; best[0] = pk[0]; best[1] = pk[1]; best[2] = pk[2];
    if (cr < cost) { cost = cr; best[0] = pr[0]; best[1] = pr[1]; best[2] = pr[2]; }
    if (cm < cost) { cost = cm; best[0] = mid[0]; best[1] = mid[1]; best[2] = mid[2]; }
  }
  if (cost < 0.0) cost = 0.0;
  if (!(cost <= max_err2)) return;
  e->valid = 1;
  e->cost = cost;
  e->p[0] = best[0]; e->p[1] = best[1]; e->p[2] = best[2];
}

/* full validation of a round winner: link condition + no face flips */
static void simp_evaluate(const simp_t* s, uint32_t u, uint32_t v, double max_err2, simp_eval_t* e) {
  simp_cost(s, u, v, max_err2, e);
  if (!e->valid) return;
  e->valid = 0;
  const double* best = e->p;
  uint32_t fu[SIMP_MAXV], fv[SIMP_MAXV], nu[SIMP_MAXV], nv[SIMP_MAXV];
  int nfu, nfv, nnu, nnv;
  if (!simp_ring(s, u, fu, nu, &nfu, &nnu)) return;
  if (!simp_ring(s, v, fv, nv, &nfv, &nnv)) return;
  int common = 0;
  for (int i = 0; i < nnu; i++)
    for (int j = 0; j < nnv; j++) common += (nu[i] == nv[j]);
  int shared = 0;
  for (int i = 0; i < nfu; i++)
    for (int j = 0; j < nfv; j++) shared += (fu[i] == fv[j]);
  if (shared != 2 || common != 2) return; /* link condition for an interior edge */
  /* ... except on a tetrahedron: a surviving face {u, a, b} next to a face {v, a, b} (a, b the
     wings) would become a second face on {k, a, b}, a zero-volume pair of opposite windings */
  for (int i = 0; i < nfu; i++) {
    const uint32_t* fx = s->face + 3 * (uint64_t)fu[i];
    if (fx[0] == v || fx[1] == v || fx[2] == v) continue; /* dies */
    for (int j = 0; j < nfv; j++) {
      const uint32_t* fy = s->face + 3 * (uint64_t)fv[j];
      int same = 0; /* both of a, b in fy: fy is {v, a, b} */
      for (int k = 0; k < 3; k++)
        if (fx[k] != u) same += (fy[0] == fx[k]) | (fy[1] == fx[k]) | (fy[2] == fx[k]);
      if (same == 2) return;
    }
  }
  for (int pass = 0; pass < 2; pass++) {
    const uint32_t* fl = pass ? fv : fu;
    const int n = pass ? nfv : nfu;
    const uint32_t w = pass ? v : u, other = pass ? u : v;
    for (int i = 0; i < n; i++) {
      const uint32_t* fx = s->face + 3 * (uint64_t)fl[i];
      if (fx[0] == other || fx[1] == other || fx[2] == other) continue; /* dies */
      const double* P[3];
      const double* N[3];
      for (int k = 0; k < 3; k++) {
        P[k] = s->pos + 3 * (uint64_t)fx[k];
        N[k] = (fx[k] == w) ? best : P[k];
      }
      const double ax = P[1][0] - P[0][0], ay = P[1][1] - P[0][1], az = P[1][2] - P[0][2];
      const double bx = P[2][0] - P[0][0], by = P[2][1] - P[0][1], bz = P[2][2] - P[0][2];
      const double n0x = ay * bz - az * by, n0y = az * bx - ax * bz, n0z = ax * by - ay * bx;
      const double cx = N[1][0] - N[0][0], cy = N[1][1] - N[0][1], cz = N[1][2] - N[0][2];
      const double dx = N[2][0] - N[0][0], dy = N[2][1] - N[0][1], dz = N[2][2] - N[0][2];
      const double n1x = cy * dz - cz * dy, n1y = cz * dx - cx * dz, n1z = cx * dy - cy * dx;
      const double dot = n0x * n1x + n0y * n1y + n0z * n1z;
      if (!(dot > 0.0)) return;
    }
  }
  e->valid = 1;
}

/* invertible 32-bit mixer (lowbias32) and its inverse: equal-cost edges get a
   pseudo-random, per-round priority instead of raster order (which would leave
   one local minimum per flat region and stall the rounds) */
static uint32_t simp_mix(uint32_t x) {
  x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16;
  return x;
}
static uint32_t simp_unmix(uint32_t x) {
  x ^= x >> 16; x *= 0x43021123U; x ^= x >> 15 ^ x >> 30; x *= 0x1d69e2a5U; x ^= x >> 16;
  return x;
}
/* 16-bit variant (odd multipliers and xor-shifts are bijections of [0, 65536)) */
static uint32_t simp_mix16(uint32_t x) {
  x &= 0xFFFFu;
  x = (x * 0x2F35u) & 0xFFFFu; x ^= x >> 7;
  x = (x * 0x4A6Bu) & 0xFFFFu; x ^= x >> 9;
  x = (x * 0x9E37u) & 0xFFFFu; x ^= x >> 8;
  return x;
}
static uint32_t simp_unmix16(uint32_t x) {
  x &= 0xFFFFu;
  x ^= x >> 8; x = (x * 0x7787u) & 0xFFFFu;
  x ^= x >> 9; x = (x * 0x1243u) & 0xFFFFu;
  x ^= x >> 7; x ^= x >> 14; x = (x * 0xEB1Du) & 0xFFFFu;
  return x;
}
/* Priority key of an edge: (cost, per-round pseudo-random tie-break that also names the
   half-edge).  Labels whose half-edge ids fit 16 bits (3 * faces <= 65536: every label the
   product keeps in shared memory) use a 32-bit key -- the float cost truncated to its upper
   16 magnitude bits (8 exponent + 8 mantissa bits), then a 16-bit permutation of the id --
   so that the product can post keys with native 32-bit shared-memory atomics; larger labels
   keep the full float cost and a 32-bit permutation in a 64-bit key. */
static uint64_t simp_key(double cost, uint32_t h, uint32_t salt, int fmt16) {
  const float c = (float)cost;
  uint32_t bits;
  memcpy(&bits, &c, 4);
  if (fmt16) return (uint64_t)((((bits >> 15) & 0xFFFFu) << 16) | simp_mix16((h ^ salt) & 0xFFFFu));
  return ((uint64_t)bits << 32) | simp_mix(h ^ salt);
}
static uint32_t simp_key_edge(uint64_t key, uint32_t salt, int fmt16) {
  if (fmt16) return simp_unmix16((uint32_t)(key & 0xFFFFu)) ^ (salt & 0xFFFFu);
  return simp_unmix((uint32_t)(key & 0xFFFFFFFFu)) ^ salt;
}
uint32_t orc_simp_mix(uint32_t x) { return simp_mix(x); }
uint32_t orc_simp_unmix(uint32_t x) { return simp_unmix(x); }
uint32_t orc_simp_mix16(uint32_t x) { return simp_mix16(x); }
uint32_t orc_simp_unmix16(uint32_t x) { return simp_unmix16(x); }

/*
 * pos: 3U doubles (in/out), face: 3T global vertex ids (in/out), flabel: T dense labels 1..K,
 * target[K+1]: stop when a label's alive faces <= target.  tri_off[K+1]: first face of
 * each label (priorities use label-local half-edge ids so that the result does not depend
 * on the order labels are stored in).  valive/falive are outputs.
 * Returns the number of rounds executed in *rounds.  rep[U] (optional, NULL to skip): the surviving
 * vertex each input vertex was collapsed into (itself when it survives).
 */
int orc_simplify(uint64_t U, uint64_t T, double* pos, uint32_t* face, const uint32_t* flabel,
                 uint32_t K, const uint32_t* target, const uint32_t* tri_off, double max_err2, int max_rounds,
                 uint8_t* valive, uint8_t* falive, int* rounds, uint32_t* rep) {
  simp_t s;
  s.U = U; s.T = T; s.pos = pos; s.face = face; s.flabel = flabel; s.falive = falive; s.valive = valive;
  s.Q = (double*)calloc(10 * (U ? U : 1), sizeof(double));
  s.vbound = (uint8_t*)calloc(U ? U : 1, 1);
  s.next = (uint32_t*)malloc(sizeof(uint32_t) * (3 * T + 1));
  s.head = (uint32_t*)malloc(sizeof(uint32_t) * (U + 1));
  s.tail = (uint32_t*)malloc(sizeof(uint32_t) * (U + 1));
  s.key1 = (uint64_t*)malloc(sizeof(uint64_t) * (U + 1));
  s.key2 = (uint64_t*)malloc(sizeof(uint64_t) * (U + 1));
  uint32_t* alive_faces = (uint32_t*)calloc(K + 2, sizeof(uint32_t));
  uint8_t* label_active = (uint8_t*)calloc(K + 2, 1);
  uint8_t* estate = (uint8_t*)calloc(3 * T + 1, 1);
  uint8_t* vdirty = (uint8_t*)calloc(U + 1, 1);
  if (!estate || !vdirty) return ORC_ENOMEM;
  if (!s.Q || !s.vbound || !s.next || !s.head || !s.tail || !s.key1 || !s.key2 || !alive_faces || !label_active)
    return ORC_ENOMEM;
  for (uint64_t v = 0; v < U; v++) { s.head[v] = s.tail[v] = SIMP_NONE; valive[v] = 1; }
  if (rep) for (uint64_t v = 0; v < U; v++) rep[v] = (uint32_t)v;
  /* incident lists in ascending node order */
  for (uint64_t h = 0; h < 3 * T; h++) {
    const uint32_t v = face[h];
    s.next[h] = SIMP_NONE;
    if (s.head[v] == SIMP_NONE) s.head[v] = (uint32_t)h;
    else s.next[s.tail[v]] = (uint32_t)h;
    s.tail[v] = (uint32_t)h;
  }
  for (uint64_t f = 0; f < T; f++) { falive[f] = 1; alive_faces[flabel[f]]++; }
  uint8_t* fmt16 = (uint8_t*)calloc(K + 2, 1); /* key format of each label (see simp_key) */
  if (!fmt16) return ORC_ENOMEM;
  for (uint32_t l = 1; l <= K; l++) fmt16[l] = 3ull * alive_faces[l] <= 65536ull;
  /* quadrics: per vertex, faces in list order */
  for (uint64_t v = 0; v < U; v++)
    for (uint32_t h = s.head[v]; h != SIMP_NONE; h = s.next[h]) {
      const uint32_t* fv = face + 3 * (uint64_t)(h / 3);
      double Kq[10];
      int ok;
      simp_plane_quadric(pos + 3 * (uint64_t)fv[0], pos + 3 * (uint64_t)fv[1], pos + 3 * (uint64_t)fv[2], Kq, &ok);
      if (ok) for (int i = 0; i < 10; i++) s.Q[10 * v + i] += Kq[i];
    }
  /* boundary vertices: an edge without exactly one twin */
  for (uint64_t h = 0; h < 3 * T; h++) {
    const uint32_t f = (uint32_t)(h / 3), c = (uint32_t)(h % 3);
    const uint32_t u = face[3 * (uint64_t)f + c], v = face[3 * (uint64_t)f + (c + 1) % 3];
    uint32_t tw;
    if (simp_twins(&s, f, u, v, &tw) != 1) { s.vbound[u] = 1; s.vbound[v] = 1; }
  }
  /* stop rules are per label (labels are independent: the product runs each label to
     completion inside one CTA): a label is finished when its faces <= target at the
     start of a round, when a round produced no winner for it (nothing collapsed or
     parked: fixed point), or after four consecutive rounds that each removed fewer than
     0.2% of its remaining faces. */
  uint8_t* stopped = (uint8_t*)calloc(K + 2, 1);
  uint32_t* slow = (uint32_t*)calloc(K + 2, sizeof(uint32_t));
  uint32_t* nsel = (uint32_t*)calloc(K + 2, sizeof(uint32_t));
  uint32_t* ncol = (uint32_t*)calloc(K + 2, sizeof(uint32_t));
  if (!stopped || !slow || !nsel || !ncol) return ORC_ENOMEM;
  int r = 0;
  for (; r < max_rounds; r++) {
    int any_label = 0;
    for (uint32_t l = 1; l <= K; l++) {
      label_active[l] = !stopped[l] && alive_faces[l] > target[l];
      any_label |= label_active[l];
      nsel[l] = ncol[l] = 0;
    }
    if (!any_label) break;
    const uint32_t salt = (uint32_t)r * 0x9E3779B9u; /* fresh tie-break priorities every round: with a fixed salt the same validation failures win again and again (8738 instead of 454 faces on the reference's box volume) */
    for (uint64_t v = 0; v < U; v++) s.key1[v] = SIMP_KEYMAX;
    /* E: one key per edge (the half-edge with u < v), from the cheap cost only */
    for (uint64_t h = 0; h < 3 * T; h++) {
      const uint32_t f = (uint32_t)(h / 3), c = (uint32_t)(h % 3);
      if (!falive[f] || !label_active[flabel[f]]) continue;
      const uint32_t u = face[3 * (uint64_t)f + c], v = face[3 * (uint64_t)f + (c + 1) % 3];
      if (!(u < v)) continue;
      if (estate[h] == 1) {
        if (vdirty[u] || vdirty[v]) estate[h] = 0; /* neighbourhood changed: try again */
        else continue;
      }
      simp_eval_t e;
      simp_cost(&s, u, v, max_err2, &e);
      if (!e.valid) continue;
      const uint64_t key = simp_key(e.cost, (uint32_t)h - 3 * tri_off[flabel[f]], salt, fmt16[flabel[f]]); /* label-local id */
      if (key < s.key1[u]) s.key1[u] = key;
      if (key < s.key1[v]) s.key1[v] = key;
    }
    for (uint64_t w = 0; w < U; w++) {
      if (!valive[w]) { s.key2[w] = SIMP_KEYMAX; continue; }
      uint64_t m = s.key1[w];
      for (uint32_t h = s.head[w]; h != SIMP_NONE; h = s.next[h]) {
        const uint32_t g = h / 3;
        if (!falive[g]) continue;
        for (int k = 0; k < 3; k++) {
          const uint64_t kk = s.key1[face[3 * (uint64_t)g + k]];
          if (kk < m) m = kk;
        }
      }
      s.key2[w] = m;
    }
    /* dirty flags of inactive labels are irrelevant from now on (a label never becomes
       active again), those of active labels were consumed by the edge pass */
    memset(vdirty, 0, U ? U : 1);
    /* select on the pre-round state, then apply (selected collapses are independent);
       winners that fail the full validation are parked until their neighbourhood changes */
    for (uint64_t a = 0; a < U; a++) {
      const uint64_t key = s.key1[a];
      if (!valive[a] || key == SIMP_KEYMAX) continue;
      const uint32_t lab = flabel[s.head[a] / 3];
      const uint32_t h = simp_key_edge(key, salt, fmt16[lab]) + 3 * tri_off[lab];
      const uint32_t f = h / 3, c = h % 3;
      const uint32_t u = face[3 * (uint64_t)f + c], v = face[3 * (uint64_t)f + (c + 1) % 3];
      if (a != u) continue;
      if (s.key2[u] != key || s.key2[v] != key) continue;
      simp_eval_t e;
      simp_evaluate(&s, u, v, max_err2, &e);
      nsel[lab]++;
      if (!e.valid) { estate[h] = 1; continue; }
      const uint32_t k = e.keep, rm = e.remove;
      pos[3 * (uint64_t)k + 0] = e.p[0]; pos[3 * (uint64_t)k + 1] = e.p[1]; pos[3 * (uint64_t)k + 2] = e.p[2];
      for (int i = 0; i < 10; i++) s.Q[10 * (uint64_t)k + i] = s.Q[10 * (uint64_t)k + i] + s.Q[10 * (uint64_t)rm + i];
      for (uint32_t hh = s.head[rm]; hh != SIMP_NONE; hh = s.next[hh]) {
        const uint32_t g = hh / 3;
        if (!falive[g]) continue;
        uint32_t* fv = face + 3 * (uint64_t)g;
        if (fv[0] == k || fv[1] == k || fv[2] == k) { falive[g] = 0; alive_faces[flabel[g]]--; }
        else fv[hh % 3] = k;
      }
      s.next[s.tail[k]] = s.head[rm];
      s.tail[k] = s.tail[rm];
      valive[rm] = 0;
      if (rep) rep[rm] = k;
      ncol[lab]++;
      vdirty[k] = 1;
      for (uint32_t hh = s.head[k]; hh != SIMP_NONE; hh = s.next[hh]) {
        const uint32_t g = hh / 3;
        if (!falive[g]) continue;
        vdirty[face[3 * (uint64_t)g]] = 1; vdirty[face[3 * (uint64_t)g + 1]] = 1; vdirty[face[3 * (uint64_t)g + 2]] = 1;
      }
    }
    for (uint32_t l = 1; l <= K; l++) {
      if (!label_active[l]) continue;
      if (getenv("ORC_SIMP_TRACE")) fprintf(stderr, "round %d label %u winners %u collapses %u alive %u\n", r, l, nsel[l], ncol[l], alive_faces[l]);
      if (nsel[l] == 0) { stopped[l] = 1; continue; }
      if ((uint64_t)ncol[l] * 1000 < (uint64_t)alive_faces[l]) slow[l]++; else slow[l] = 0;
      if (slow[l] >= 4) stopped[l] = 1;
    }
  }
  free(stopped); free(slow); free(nsel); free(ncol);
  *rounds = r;
  if (rep) for (uint64_t v = 0; v < U; v++) while (!valive[rep[v]]) rep[v] = rep[rep[v]];
  free(s.Q); free(s.vbound); free(s.next); free(s.head); free(s.tail); free(s.key1); free(s.key2);
  free(alive_faces); free(label_active); free(estate); free(vdirty); free(fmt16);
  return ORC_OK;
}

/* ------------------------------------------------------------------ */
/* compressed_segmentation chunk codec (Precomputed `encoding:          */
/* compressed_segmentation`, the wire format either side of the path:   */
/* SURVEY.md 8(f) row 1; CloudVolume decodes / encodes it on the host   */
/* around igneous/tasks/image/image.py:57-100 and ccl.py:346-356).      */
/* Restated from the published Neuroglancer format description and the  */
/* reference encoder's emission order (recalled; the library is absent  */
/* offline) -- PARITY UNPINNED for the encoder's byte layout; the       */
/* decoder accepts any conforming stream.                               */
/*   file    = [channel offsets u32 x C] channel_0 ... channel_{C-1}    */
/*   channel = block headers (2 x u32 per block, x fastest) followed by */
/*             per block: packed indices, then (if not seen before in   */
/*             this channel) the sorted lookup table                    */
/*   header  = word0: table offset (24 bits) | bits << 24               */
/*             word1: offset of the packed indices                      */
/*             (offsets in u32 units from the start of the channel)     */
/*   bits    = 0, 1, 2, 4, 8, 16 or 32 per voxel; voxel (x,y,z) of a    */
/*             block sits at bit ((z*by + y)*bx + x) * bits, LSB first; */
/*             positions outside the volume stay 0                     */
/* Arrays are Fortran order [x, y, z, c].  Encoders return the number   */
/* of u32 words written (or needed, when out == NULL / cap too small).  */
/* ------------------------------------------------------------------ */
typedef struct {
  uint64_t hash;
  uint32_t offset, n;
  uint32_t first_word; /* index into the output of the table itself */
} cseg_table_t;

static uint64_t cseg_hash(const uint64_t* v, uint32_t n) {
  uint64_t h = 0x9E3779B97F4A7C15ull ^ n;
  for (uint32_t i = 0; i < n; i++) {
    h ^= v[i] + 0x9E3779B97F4A7C15ull + (h << 6) + (h >> 2);
  }
  return h;
}

static int cseg_cmp_u64(const void* a, const void* b) {
  const uint64_t x = *(const uint64_t*)a, y = *(const uint64_t*)b;
  return (x > y) - (x < y);
}

#define DEF_CSEG_ENCODE(T, NAME, WORDS)                                        \
  int64_t NAME(const T* in, uint64_t sx, uint64_t sy, uint64_t sz,             \
               uint64_t sc, uint32_t bx, uint32_t by, uint32_t bz,             \
               uint32_t* out, uint64_t cap) {                                  \
    if (!in || !bx || !by || !bz || !sx || !sy || !sz || !sc) return ORC_EINVAL; \
    const uint64_t gx = (sx + bx - 1) / bx, gy = (sy + by - 1) / by,           \
                   gz = (sz + bz - 1) / bz;                                    \
    const uint64_t nblock = gx * gy * gz, bvox = (uint64_t)bx * by * bz;       \
    uint64_t size = sc; /* words used so far (channel offset table first) */   \
    uint64_t* vals = (uint64_t*)malloc(sizeof(uint64_t) * bvox);               \
    uint64_t* uniq = (uint64_t*)malloc(sizeof(uint64_t) * bvox);               \
    cseg_table_t* cache = (cseg_table_t*)malloc(sizeof(cseg_table_t) * nblock); \
    uint64_t* tables = NULL; /* copies of cached tables for comparison */      \
    uint64_t tables_cap = 0, tables_n = 0;                                     \
    if (!vals || !uniq || !cache) { free(vals); free(uniq); free(cache); return ORC_ENOMEM; } \
    int64_t rc = 0;                                                            \
    for (uint64_t c = 0; c < sc && rc == 0; c++) {                             \
      const T* chan = in + c * sx * sy * sz;                                   \
      const uint64_t base = size;                                              \
      if (out && c < cap) out[c] = (uint32_t)base;                             \
      uint64_t ncache = 0;                                                     \
      tables_n = 0;                                                            \
      for (uint64_t i = 0; i < 2 * nblock; i++)                                \
        if (out && size + i < cap) out[size + i] = 0;                          \
      size += 2 * nblock;                                                      \
      for (uint64_t gzz = 0; gzz < gz && rc == 0; gzz++)                       \
        for (uint64_t gyy = 0; gyy < gy && rc == 0; gyy++)                     \
          for (uint64_t gxx = 0; gxx < gx && rc == 0; gxx++) {                 \
            const uint64_t bi = gxx + gx * (gyy + gy * gzz);                   \
            const uint64_t x0 = gxx * bx, y0 = gyy * by, z0 = gzz * bz;        \
            const uint64_t ax = (sx - x0 < bx) ? sx - x0 : bx,                 \
                           ay = (sy - y0 < by) ? sy - y0 : by,                 \
                           az = (sz - z0 < bz) ? sz - z0 : bz;                 \
            uint64_t nv = 0;                                                   \
            for (uint64_t z = 0; z < az; z++)                                  \
              for (uint64_t y = 0; y < ay; y++)                                \
                for (uint64_t x = 0; x < ax; x++)                              \
                  vals[nv++] = (uint64_t)chan[(x0 + x) + sx * ((y0 + y) + sy * (z0 + z))]; \
            memcpy(uniq, vals, sizeof(uint64_t) * nv);                         \
            qsort(uniq, nv, sizeof(uint64_t), cseg_cmp_u64);                   \
            uint64_t nu = 0;                                                   \
            for (uint64_t i = 0; i < nv; i++)                                  \
              if (i == 0 || uniq[i] != uniq[i - 1]) uniq[nu++] = uniq[i];      \
            uint32_t bits = 0;                                                 \
            if (nu > 1) { bits = 1; while ((1ull << bits) < nu) bits *= 2; }   \
            const uint64_t enc_words = (bits * bvox + 31) / 32;                \
            const uint64_t enc_off = size - base;                              \
            for (uint64_t i = 0; i < enc_words; i++)                           \
              if (out && size + i < cap) out[size + i] = 0;                    \
            if (bits) {                                                        \
              uint64_t k = 0;                                                  \
              for (uint64_t z = 0; z < az; z++)                                \
                for (uint64_t y = 0; y < ay; y++)                              \
                  for (uint64_t x = 0; x < ax; x++) {                          \
                    const uint64_t v = vals[k++];                              \
                    uint64_t lo = 0, hi = nu; /* index of v in uniq */         \
                    while (lo + 1 < hi) {                                      \
                      const uint64_t mid = (lo + hi) / 2;                      \
                      if (uniq[mid] <= v) lo = mid; else hi = mid;             \
                    }                                                          \
                    const uint64_t bitpos = ((z * by + y) * bx + x) * bits;    \
                    const uint64_t w = size + bitpos / 32;                     \
                    if (out && w < cap) out[w] |= (uint32_t)(lo << (bitpos % 32)); \
                  }                                                            \
            }                                                                  \
            size += enc_words;                                                 \
            /* lookup table: reuse an identical one of this channel */         \
            const uint64_t hsh = cseg_hash(uniq, (uint32_t)nu);                \
            uint64_t toff = ~0ull;                                             \
            for (uint64_t i = 0; i < ncache; i++)                              \
              if (cache[i].hash == hsh && cache[i].n == nu &&                  \
                  memcmp(tables + cache[i].first_word, uniq, sizeof(uint64_t) * nu) == 0) { \
                toff = cache[i].offset;                                        \
                break;                                                         \
              }                                                                \
            if (toff == ~0ull) {                                               \
              toff = size - base;                                              \
              if (tables_n + nu > tables_cap) {                                \
                tables_cap = (tables_n + nu) * 2 + 64;                         \
                uint64_t* nt = (uint64_t*)realloc(tables, sizeof(uint64_t) * tables_cap); \
                if (!nt) { rc = ORC_ENOMEM; break; }                           \
                tables = nt;                                                   \
              }                                                                \
              memcpy(tables + tables_n, uniq, sizeof(uint64_t) * nu);          \
              cache[ncache].hash = hsh;                                        \
              cache[ncache].n = (uint32_t)nu;                                  \
              cache[ncache].offset = (uint32_t)toff;                           \
              cache[ncache].first_word = (uint32_t)tables_n;                   \
              ncache++;                                                        \
              tables_n += nu;                                                  \
              for (uint64_t i = 0; i < nu; i++) {                              \
                if (out && size < cap) out[size] = (uint32_t)(uniq[i] & 0xFFFFFFFFull); \
                size++;                                                        \
                if (WORDS == 2) {                                              \
                  if (out && size < cap) out[size] = (uint32_t)(uniq[i] >> 32); \
                  size++;                                                      \
                }                                                              \
              }                                                                \
            }                                                                  \
            if (toff > 0xFFFFFFull) { rc = ORC_EINVAL; break; }                \
            const uint64_t hw = base + 2 * bi;                                 \
            if (out && hw + 1 < cap) {                                         \
              out[hw] = (uint32_t)toff | (bits << 24);                         \
              out[hw + 1] = (uint32_t)enc_off;                                 \
            }                                                                  \
          }                                                                    \
    }                                                                          \
    free(vals); free(uniq); free(cache); free(tables);                         \
    return rc ? rc : (int64_t)size;                                            \
  }

DEF_CSEG_ENCODE(uint32_t, orc_cseg_encode_u32, 1)
DEF_CSEG_ENCODE(uint64_t, orc_cseg_encode_u64, 2)

#define DEF_CSEG_DECODE(T, NAME, WORDS)                                        \
  int NAME(const uint32_t* in, uint64_t nwords, uint64_t sx, uint64_t sy,      \
           uint64_t sz, uint64_t sc, uint32_t bx, uint32_t by, uint32_t bz,    \
           T* out) {                                                           \
    if (!in || !out || !bx || !by || !bz || nwords < sc) return ORC_EINVAL;    \
    const uint64_t gx = (sx + bx - 1) / bx, gy = (sy + by - 1) / by,           \
                   gz = (sz + bz - 1) / bz;                                    \
    for (uint64_t c = 0; c < sc; c++) {                                        \
      const uint64_t base = in[c];                                             \
      T* chan = out + c * sx * sy * sz;                                        \
      if (base + 2 * gx * gy * gz > nwords) return ORC_EINVAL;                 \
      for (uint64_t gzz = 0; gzz < gz; gzz++)                                  \
        for (uint64_t gyy = 0; gyy < gy; gyy++)                                \
          for (uint64_t gxx = 0; gxx < gx; gxx++) {                            \
            const uint64_t bi = gxx + gx * (gyy + gy * gzz);                   \
            const uint32_t h0 = in[base + 2 * bi], h1 = in[base + 2 * bi + 1]; \
            const uint32_t bits = h0 >> 24;                                    \
            const uint64_t toff = base + (h0 & 0xFFFFFFu), voff = base + h1;   \
            if (!(bits == 0 || bits == 1 || bits == 2 || bits == 4 ||          \
                  bits == 8 || bits == 16 || bits == 32)) return ORC_EINVAL;   \
            const uint64_t x0 = gxx * bx, y0 = gyy * by, z0 = gzz * bz;        \
            for (uint64_t z = 0; z < bz && z0 + z < sz; z++)                   \
              for (uint64_t y = 0; y < by && y0 + y < sy; y++)                 \
                for (uint64_t x = 0; x < bx && x0 + x < sx; x++) {             \
                  uint64_t idx = 0;                                            \
                  if (bits) {                                                  \
                    const uint64_t bitpos = ((z * by + y) * bx + x) * bits;    \
                    const uint64_t w = voff + bitpos / 32;                     \
                    if (w >= nwords) return ORC_EINVAL;                        \
                    idx = (in[w] >> (bitpos % 32)) &                           \
                          (bits == 32 ? 0xFFFFFFFFu : ((1u << bits) - 1u));    \
                  }                                                            \
                  const uint64_t tw = toff + idx * WORDS;                      \
                  if (tw + WORDS > nwords) return ORC_EINVAL;                  \
                  uint64_t v = in[tw];                                         \
                  if (WORDS == 2) v |= (uint64_t)in[tw + 1] << 32;             \
                  chan[(x0 + x) + sx * ((y0 + y) + sy * (z0 + z))] = (T)v;     \
                }                                                              \
          }                                                                    \
    }                                                                          \
    return ORC_OK;                                                             \
  }

DEF_CSEG_DECODE(uint32_t, orc_cseg_decode_u32, 1)
DEF_CSEG_DECODE(uint64_t, orc_cseg_decode_u64, 2)
