/* jpeg_oracle.c -- serial restatement of the grayscale JPEG chunk codec (TEST INFRASTRUCTURE ONLY)
 *
 * Written from ITU-T T.81 (baseline sequential DCT, Huffman coding, Annex K tables) and the
 * IJG's published integer DCT (Loeffler-Ligtenberg-Moschytz, 13-bit constants, 2 extra bits
 * between the passes).  The encoder writes what libjpeg writes with its defaults for one
 * 8-bit component: SOI, JFIF APP0, one DQT (Annex K luminance table scaled by the IJG quality
 * rule), SOF0, DHT DC, DHT AC (Annex K luminance tables), DRI when the restart interval is not 0,
 * SOS, the scan, EOI.  The decoder reads any baseline / extended sequential (SOF0 / SOF1) 8-bit
 * grayscale stream and reproduces libjpeg's accurate integer (islow) decode.
 *
 * An image is `w` columns by `h` rows, row-major: a Precomputed chunk [x, y, z] in Fortran order
 * is the image of width sx and height sy*sz.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

enum { ORC_JPEG_OK = 0, ORC_JPEG_MALFORMED = -2, ORC_JPEG_UNSUPPORTED = -3, ORC_JPEG_SHAPE = -4 };

static const uint8_t ZIGZAG[64] = {  /* natural index of the k-th coefficient in zigzag order */
  0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28,
  35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

static const uint8_t LUMA_Q[64] = {  /* T.81 Table K.1, natural order */
  16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
  14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
  49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};

/* T.81 Tables K.3 and K.5: code counts per length 1..16, then the values */
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

/* LL&M constants, scaled by 2^13 */
#define CB 13
#define P1 2
#define F0298 2446
#define F0390 3196
#define F0541 4433
#define F0765 6270
#define F0899 7373
#define F1175 9633
#define F1501 12299
#define F1847 15137
#define F1961 16069
#define F2053 16819
#define F2562 20995
#define F3072 25172
#define DESCALE(x, n) (((x) + ((int64_t)1 << ((n)-1))) >> (n))

/* IJG quality rule: 1..100 -> percentage scale of the Annex K table, entries clamped to 1..255 */
static void quant_table(int quality, uint16_t q[64]) {
  if (quality < 1) quality = 1;
  if (quality > 100) quality = 100;
  const int s = quality < 50 ? 5000 / quality : 200 - 2 * quality;
  for (int i = 0; i < 64; i++) {
    long v = ((long)LUMA_Q[i] * s + 50) / 100;
    q[i] = (uint16_t)(v < 1 ? 1 : v > 255 ? 255 : v);
  }
}

/* ------------------------------------------------------------------ encoder */
typedef struct {
  uint8_t* out;
  size_t cap, n;
  uint32_t acc;  /* pending bits, MSB first */
  int nacc;
} Writer;

static void put_byte(Writer* w, uint8_t b) {
  if (w->n < w->cap) w->out[w->n] = b;
  w->n++;
}
static void put_u16(Writer* w, unsigned v) {
  put_byte(w, (uint8_t)(v >> 8));
  put_byte(w, (uint8_t)v);
}
static void put_bits(Writer* w, uint32_t code, int len) {
  for (int i = len - 1; i >= 0; i--) {
    w->acc = (w->acc << 1) | ((code >> i) & 1u);
    if (++w->nacc == 8) {
      put_byte(w, (uint8_t)w->acc);
      if ((uint8_t)w->acc == 0xFF) put_byte(w, 0x00);
      w->acc = 0;
      w->nacc = 0;
    }
  }
}
static void flush_bits(Writer* w) {  /* pad the last byte with 1-bits */
  if (w->nacc) put_bits(w, 0x7F, 8 - w->nacc);
}

/* T.81 Annex C: code of every value of a table given by its counts per length */
static void huff_codes(const uint8_t bits[16], const uint8_t* vals, uint16_t code[256], uint8_t len[256]) {
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

static int nbits(int v) {
  if (v < 0) v = -v;
  int n = 0;
  while (v) { n++; v >>= 1; }
  return n;
}

/* islow FDCT of level-shifted samples; out = 8x the orthonormal DCT */
static void fdct(const int in[64], int out[64]) {
  int64_t ws[64];
  for (int r = 0; r < 8; r++) {
    const int* d = in + 8 * r;
    int64_t t0 = d[0] + d[7], t7 = d[0] - d[7], t1 = d[1] + d[6], t6 = d[1] - d[6];
    int64_t t2 = d[2] + d[5], t5 = d[2] - d[5], t3 = d[3] + d[4], t4 = d[3] - d[4];
    int64_t t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
    int64_t* o = ws + 8 * r;
    o[0] = (t10 + t11) * (1 << P1);
    o[4] = (t10 - t11) * (1 << P1);
    int64_t z1 = (t12 + t13) * F0541;
    o[2] = DESCALE(z1 + t13 * F0765, CB - P1);
    o[6] = DESCALE(z1 - t12 * F1847, CB - P1);
    z1 = t4 + t7;
    int64_t z2 = t5 + t6, z3 = t4 + t6, z4 = t5 + t7, z5 = (z3 + z4) * F1175;
    t4 *= F0298; t5 *= F2053; t6 *= F3072; t7 *= F1501;
    z1 *= -F0899; z2 *= -F2562; z3 = z3 * -F1961 + z5; z4 = z4 * -F0390 + z5;
    o[7] = DESCALE(t4 + z1 + z3, CB - P1);
    o[5] = DESCALE(t5 + z2 + z4, CB - P1);
    o[3] = DESCALE(t6 + z2 + z3, CB - P1);
    o[1] = DESCALE(t7 + z1 + z4, CB - P1);
  }
  for (int c = 0; c < 8; c++) {
    const int64_t* d = ws + c;
    int64_t t0 = d[0] + d[56], t7 = d[0] - d[56], t1 = d[8] + d[48], t6 = d[8] - d[48];
    int64_t t2 = d[16] + d[40], t5 = d[16] - d[40], t3 = d[24] + d[32], t4 = d[24] - d[32];
    int64_t t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
    int* o = out + c;
    o[0] = (int)DESCALE(t10 + t11, P1);
    o[32] = (int)DESCALE(t10 - t11, P1);
    int64_t z1 = (t12 + t13) * F0541;
    o[16] = (int)DESCALE(z1 + t13 * F0765, CB + P1);
    o[48] = (int)DESCALE(z1 - t12 * F1847, CB + P1);
    z1 = t4 + t7;
    int64_t z2 = t5 + t6, z3 = t4 + t6, z4 = t5 + t7, z5 = (z3 + z4) * F1175;
    t4 *= F0298; t5 *= F2053; t6 *= F3072; t7 *= F1501;
    z1 *= -F0899; z2 *= -F2562; z3 = z3 * -F1961 + z5; z4 = z4 * -F0390 + z5;
    o[56] = (int)DESCALE(t4 + z1 + z3, CB + P1);
    o[40] = (int)DESCALE(t5 + z2 + z4, CB + P1);
    o[24] = (int)DESCALE(t6 + z2 + z3, CB + P1);
    o[8] = (int)DESCALE(t7 + z1 + z4, CB + P1);
  }
}

/* Encode a w x h image at `quality` with a restart marker every `restart` blocks (0: none).
 * Returns the stream's size; the stream is written only when it fits in `cap`. */
size_t orc_jpeg_encode(const uint8_t* img, uint32_t w, uint32_t h, int quality, uint32_t restart, uint8_t* out,
                       size_t cap) {
  Writer wr = {out, cap, 0, 0, 0};
  uint16_t q[64];
  quant_table(quality, q);
  put_u16(&wr, 0xFFD8);
  static const uint8_t app0[16] = {0x00, 0x10, 'J', 'F', 'I', 'F', 0, 1, 1, 0, 0, 1, 0, 1, 0, 0};
  put_u16(&wr, 0xFFE0);
  for (int i = 0; i < 16; i++) put_byte(&wr, app0[i]);
  put_u16(&wr, 0xFFDB); put_u16(&wr, 67); put_byte(&wr, 0);
  for (int k = 0; k < 64; k++) put_byte(&wr, (uint8_t)q[ZIGZAG[k]]);
  put_u16(&wr, 0xFFC0); put_u16(&wr, 11); put_byte(&wr, 8); put_u16(&wr, h); put_u16(&wr, w);
  put_byte(&wr, 1); put_byte(&wr, 1); put_byte(&wr, 0x11); put_byte(&wr, 0);
  put_u16(&wr, 0xFFC4); put_u16(&wr, 3 + 16 + 12); put_byte(&wr, 0x00);
  for (int i = 0; i < 16; i++) put_byte(&wr, DC_BITS[i]);
  for (int i = 0; i < 12; i++) put_byte(&wr, DC_VALS[i]);
  put_u16(&wr, 0xFFC4); put_u16(&wr, 3 + 16 + 162); put_byte(&wr, 0x10);
  for (int i = 0; i < 16; i++) put_byte(&wr, AC_BITS[i]);
  for (int i = 0; i < 162; i++) put_byte(&wr, AC_VALS[i]);
  if (restart) { put_u16(&wr, 0xFFDD); put_u16(&wr, 4); put_u16(&wr, restart); }
  put_u16(&wr, 0xFFDA); put_u16(&wr, 8); put_byte(&wr, 1); put_byte(&wr, 1); put_byte(&wr, 0x00);
  put_byte(&wr, 0); put_byte(&wr, 63); put_byte(&wr, 0);

  uint16_t dcc[256], acc[256];
  uint8_t dcl[256], acl[256];
  huff_codes(DC_BITS, DC_VALS, dcc, dcl);
  huff_codes(AC_BITS, AC_VALS, acc, acl);
  const uint32_t bw = (w + 7) / 8, bh = (h + 7) / 8;
  const uint64_t nb = (uint64_t)bw * bh;
  int last_dc = 0;
  unsigned rst = 0;
  for (uint64_t b = 0; b < nb; b++) {
    if (restart && b && b % restart == 0) {
      flush_bits(&wr);
      put_u16(&wr, 0xFFD0 + (rst++ & 7));
      last_dc = 0;
    }
    const uint32_t bx = (uint32_t)(b % bw), by = (uint32_t)(b / bw);
    int s[64], c[64];
    for (int r = 0; r < 8; r++)
      for (int x = 0; x < 8; x++) {
        uint32_t yy = by * 8 + r, xx = bx * 8 + x;  /* edge blocks repeat the last row / column */
        if (yy >= h) yy = h - 1;
        if (xx >= w) xx = w - 1;
        s[8 * r + x] = (int)img[(uint64_t)yy * w + xx] - 128;
      }
    fdct(s, c);
    int zz[64];
    for (int k = 0; k < 64; k++) {  /* round half away from zero; the DCT carries a factor 8 */
      const int i = ZIGZAG[k], d = 8 * q[i];
      int v = c[i];
      zz[k] = v < 0 ? -((-v + d / 2) / d) : (v + d / 2) / d;
    }
    int diff = zz[0] - last_dc;
    last_dc = zz[0];
    int n = nbits(diff);
    put_bits(&wr, dcc[n], dcl[n]);
    if (n) put_bits(&wr, (uint32_t)(diff < 0 ? diff - 1 : diff) & ((1u << n) - 1), n);
    int run = 0;
    for (int k = 1; k < 64; k++) {
      const int v = zz[k];
      if (v == 0) { run++; continue; }
      while (run > 15) { put_bits(&wr, acc[0xF0], acl[0xF0]); run -= 16; }
      n = nbits(v);
      const int rs = (run << 4) | n;
      put_bits(&wr, acc[rs], acl[rs]);
      put_bits(&wr, (uint32_t)(v < 0 ? v - 1 : v) & ((1u << n) - 1), n);
      run = 0;
    }
    if (run) put_bits(&wr, acc[0x00], acl[0x00]);
  }
  flush_bits(&wr);
  put_u16(&wr, 0xFFD9);
  return wr.n;
}

/* ------------------------------------------------------------------ decoder */
typedef struct {
  int defined;
  uint8_t bits[17];
  uint8_t vals[256];
  int32_t maxcode[18], valptr[17], mincode[17];
} Huff;

static int huff_build(Huff* t) {  /* T.81 F.2.2.3 decoder tables; 0 if the counts overflow the code space */
  int32_t code = 0;
  int k = 0;
  for (int l = 1; l <= 16; l++) {
    t->valptr[l] = k;
    t->mincode[l] = code;
    code += t->bits[l];
    k += t->bits[l];
    if (code > (1 << l)) return 0;
    t->maxcode[l] = t->bits[l] ? code - 1 : -1;
    code <<= 1;
  }
  t->maxcode[17] = 0x7FFFFFFF;
  return 1;
}

typedef struct {
  const uint8_t* p;
  size_t pos, end;  /* entropy-coded bytes of one restart interval: [pos, end) */
  uint32_t acc;
  int nacc;
  int over;  /* bits requested past the interval's end */
} Reader;

static int get_bit(Reader* r) {
  if (r->nacc == 0) {
    if (r->pos >= r->end) { r->over = 1; return 0; }
    uint8_t b = r->p[r->pos++];
    if (b == 0xFF) {  /* a stuffed zero follows every data 0xFF inside the interval */
      if (r->pos >= r->end || r->p[r->pos] != 0x00) { r->over = 1; return 0; }
      r->pos++;
    }
    r->acc = b;
    r->nacc = 8;
  }
  r->nacc--;
  return (r->acc >> r->nacc) & 1;
}
static int get_bits(Reader* r, int n) {
  int v = 0;
  for (int i = 0; i < n; i++) v = (v << 1) | get_bit(r);
  return v;
}
static int decode_huff(Reader* r, const Huff* t) {
  int32_t code = get_bit(r);
  int l = 1;
  while (code > t->maxcode[l]) {
    if (++l > 16) return -1;
    code = (code << 1) | get_bit(r);
  }
  return t->vals[t->valptr[l] + code - t->mincode[l]];
}
static int extend(int v, int n) { return v < (1 << (n - 1)) ? v - (1 << n) + 1 : v; }

static void idct_put(const int16_t coef[64], const uint16_t q[64], uint8_t* out, uint32_t w, uint32_t h, uint32_t x0,
                     uint32_t y0) {
  int ws[64];
  for (int c = 0; c < 8; c++) {
    int64_t d[8];
    for (int r = 0; r < 8; r++) d[r] = (int64_t)coef[8 * r + c] * q[8 * r + c];
    int64_t z1 = (d[2] + d[6]) * F0541;
    int64_t t2 = z1 - d[6] * F1847, t3 = z1 + d[2] * F0765;
    int64_t t0 = (d[0] + d[4]) * (1 << CB), t1 = (d[0] - d[4]) * (1 << CB);
    int64_t t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
    int64_t o0 = d[7], o1 = d[5], o2 = d[3], o3 = d[1];
    z1 = o0 + o3;
    int64_t z2 = o1 + o2, z3 = o0 + o2, z4 = o1 + o3, z5 = (z3 + z4) * F1175;
    o0 *= F0298; o1 *= F2053; o2 *= F3072; o3 *= F1501;
    z1 *= -F0899; z2 *= -F2562; z3 = z3 * -F1961 + z5; z4 = z4 * -F0390 + z5;
    o0 += z1 + z3; o1 += z2 + z4; o2 += z2 + z3; o3 += z1 + z4;
    ws[c] = (int)DESCALE(t10 + o3, CB - P1);
    ws[56 + c] = (int)DESCALE(t10 - o3, CB - P1);
    ws[8 + c] = (int)DESCALE(t11 + o2, CB - P1);
    ws[48 + c] = (int)DESCALE(t11 - o2, CB - P1);
    ws[16 + c] = (int)DESCALE(t12 + o1, CB - P1);
    ws[40 + c] = (int)DESCALE(t12 - o1, CB - P1);
    ws[24 + c] = (int)DESCALE(t13 + o0, CB - P1);
    ws[32 + c] = (int)DESCALE(t13 - o0, CB - P1);
  }
  for (int r = 0; r < 8; r++) {
    const int* d = ws + 8 * r;
    int64_t z1 = (int64_t)(d[2] + d[6]) * F0541;
    int64_t t2 = z1 - (int64_t)d[6] * F1847, t3 = z1 + (int64_t)d[2] * F0765;
    int64_t t0 = (int64_t)(d[0] + d[4]) * (1 << CB), t1 = (int64_t)(d[0] - d[4]) * (1 << CB);
    int64_t t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
    int64_t o0 = d[7], o1 = d[5], o2 = d[3], o3 = d[1];
    z1 = o0 + o3;
    int64_t z2 = o1 + o2, z3 = o0 + o2, z4 = o1 + o3, z5 = (z3 + z4) * F1175;
    o0 *= F0298; o1 *= F2053; o2 *= F3072; o3 *= F1501;
    z1 *= -F0899; z2 *= -F2562; z3 = z3 * -F1961 + z5; z4 = z4 * -F0390 + z5;
    o0 += z1 + z3; o1 += z2 + z4; o2 += z2 + z3; o3 += z1 + z4;
    const int64_t v[8] = {t10 + o3, t11 + o2, t12 + o1, t13 + o0, t13 - o0, t12 - o1, t11 - o2, t10 - o3};
    if (y0 + r >= h) break;
    for (int x = 0; x < 8 && x0 + x < w; x++) {
      int64_t p = DESCALE(v[x], CB + P1 + 3) + 128;
      out[(uint64_t)(y0 + r) * w + x0 + x] = (uint8_t)(p < 0 ? 0 : p > 255 ? 255 : p);
    }
  }
}

static unsigned rd16(const uint8_t* p) { return ((unsigned)p[0] << 8) | p[1]; }

/* Decode a stream that must hold a w x h 8-bit grayscale image. */
int orc_jpeg_decode(const uint8_t* data, size_t n, uint32_t w, uint32_t h, uint8_t* out) {
  uint16_t qt[4][64];
  int qdef[4] = {0, 0, 0, 0};
  Huff ht[2][4];
  memset(ht, 0, sizeof(ht));
  uint32_t restart = 0, fw = 0, fh = 0;
  int have_sof = 0, comp_id = -1, qsel = 0;
  size_t pos = 2;
  if (n < 4 || data[0] != 0xFF || data[1] != 0xD8) return ORC_JPEG_MALFORMED;
  for (;;) {  /* header segments up to SOS */
    if (pos + 2 > n || data[pos] != 0xFF) return ORC_JPEG_MALFORMED;
    while (pos + 1 < n && data[pos + 1] == 0xFF) pos++;  /* fill bytes */
    if (pos + 4 > n) return ORC_JPEG_MALFORMED;
    const uint8_t m = data[pos + 1];
    const size_t len = rd16(data + pos + 2);
    if (len < 2 || pos + 2 + len > n) return ORC_JPEG_MALFORMED;
    const uint8_t* s = data + pos + 4;
    const size_t sl = len - 2;
    pos += 2 + len;
    if (m == 0xDB) {
      size_t i = 0;
      while (i < sl) {
        const int pq = s[i] >> 4, tq = s[i] & 15;
        if (pq > 1 || tq > 3 || i + 1 + 64 * (pq + 1) > sl) return ORC_JPEG_MALFORMED;
        for (int k = 0; k < 64; k++)
          qt[tq][ZIGZAG[k]] = pq ? (uint16_t)rd16(s + i + 1 + 2 * k) : s[i + 1 + k];
        qdef[tq] = 1;
        i += 1 + 64 * (pq + 1);
      }
    } else if (m == 0xC4) {
      size_t i = 0;
      while (i < sl) {
        const int tc = s[i] >> 4, th = s[i] & 15;
        if (tc > 1 || th > 3 || i + 17 > sl) return ORC_JPEG_MALFORMED;
        Huff* t = &ht[tc][th];
        int total = 0;
        for (int l = 1; l <= 16; l++) total += (t->bits[l] = s[i + l]);
        if (total > 256 || i + 17 + total > sl) return ORC_JPEG_MALFORMED;
        memcpy(t->vals, s + i + 17, total);
        if (!huff_build(t)) return ORC_JPEG_MALFORMED;
        if (tc == 0)
          for (int k = 0; k < total; k++)
            if (t->vals[k] > 15) return ORC_JPEG_MALFORMED;
        t->defined = 1;
        i += 17 + total;
      }
    } else if (m == 0xDD) {
      if (sl != 2) return ORC_JPEG_MALFORMED;
      restart = rd16(s);
    } else if (m == 0xC0 || m == 0xC1) {
      if (sl < 6) return ORC_JPEG_MALFORMED;
      if (s[0] != 8 || s[5] != 1) return ORC_JPEG_UNSUPPORTED;  /* 8-bit, one component */
      if (sl != 9) return ORC_JPEG_MALFORMED;
      fh = rd16(s + 1);
      fw = rd16(s + 3);
      if (fh == 0) return ORC_JPEG_UNSUPPORTED;  /* height given by a DNL marker */
      if (fw == 0) return ORC_JPEG_MALFORMED;
      comp_id = s[6];
      if ((s[7] >> 4) < 1 || (s[7] >> 4) > 4 || (s[7] & 15) < 1 || (s[7] & 15) > 4 || s[8] > 3) return ORC_JPEG_MALFORMED;
      qsel = s[8];
      have_sof = 1;
    } else if ((m >= 0xC2 && m <= 0xCF && m != 0xC4 && m != 0xC8) || m == 0xDC) {
      return ORC_JPEG_UNSUPPORTED;  /* progressive, lossless, hierarchical, arithmetic, DNL */
    } else if (m == 0xDA) {
      if (!have_sof) return ORC_JPEG_MALFORMED;
      if (sl < 1 || s[0] != 1) return ORC_JPEG_MALFORMED;
      if (sl != 6 || s[1] != comp_id || s[3] != 0 || s[4] != 63 || s[5] != 0) return ORC_JPEG_MALFORMED;
      const int td = s[2] >> 4, ta = s[2] & 15;
      if (td > 3 || ta > 3 || !ht[0][td].defined || !ht[1][ta].defined || !qdef[qsel]) return ORC_JPEG_MALFORMED;
      if (fw != w || fh != h) return ORC_JPEG_SHAPE;
      const Huff *dc = &ht[0][td], *ac = &ht[1][ta];
      const uint32_t bw = (w + 7) / 8, bh = (h + 7) / 8;
      const uint64_t nb = (uint64_t)bw * bh;
      const uint64_t per = restart ? restart : nb;
      for (uint64_t b0 = 0, k = 0; b0 < nb; b0 += per, k++) {
        size_t e = pos;  /* the interval's data runs to the next marker */
        while (e + 1 < n && !(data[e] == 0xFF && data[e + 1] != 0x00 && data[e + 1] != 0xFF)) e++;
        if (e + 1 >= n) return ORC_JPEG_MALFORMED;
        Reader r = {data, pos, e, 0, 0, 0};
        int last_dc = 0;
        for (uint64_t b = b0; b < nb && b < b0 + per; b++) {
          int16_t coef[64];
          memset(coef, 0, sizeof(coef));
          int t = decode_huff(&r, dc);
          if (t < 0) return ORC_JPEG_MALFORMED;
          if (t) last_dc += extend(get_bits(&r, t), t);
          coef[0] = (int16_t)last_dc;
          for (int i = 1; i < 64; i++) {
            const int rs = decode_huff(&r, ac);
            if (rs < 0) return ORC_JPEG_MALFORMED;
            const int run = rs >> 4, sz = rs & 15;
            if (sz == 0) {
              if (run != 15) break;
              i += 15;
              continue;
            }
            i += run;
            if (i > 63) return ORC_JPEG_MALFORMED;
            coef[ZIGZAG[i]] = (int16_t)extend(get_bits(&r, sz), sz);
          }
          if (r.over) return ORC_JPEG_MALFORMED;
          idct_put(coef, qt[qsel], out, w, h, (uint32_t)(b % bw) * 8, (uint32_t)(b / bw) * 8);
        }
        /* data[e] is 0xFF; fill bytes may precede the marker code */
        while (e + 1 < n && data[e + 1] == 0xFF) e++;
        const uint8_t mk = data[e + 1];
        if (b0 + per < nb) {
          if (mk != 0xD0 + (k & 7)) return ORC_JPEG_MALFORMED;
          pos = e + 2;
        } else {
          if (mk != 0xD9) return ORC_JPEG_MALFORMED;
          return ORC_JPEG_OK;
        }
      }
      return ORC_JPEG_MALFORMED;
    } else if ((m >= 0xE0 && m <= 0xEF) || m == 0xFE) {
      /* APPn, COM: skipped */
    } else {
      return ORC_JPEG_MALFORMED;
    }
  }
}
