/* merge_oracle.c -- serial C checker of the skeleton merge and postprocess rule of DESIGN.md §5h, over the
 * packed layout of ign_skeleton_merge_dev (test infrastructure only; shares no code with the kernels or with
 * tests/skelmergeref.py).
 *
 * Per label: crop and concatenate its fragments, consolidate, and unless the cable length exceeds
 * max_cable_length: dust, loops, connect pieces, ticks, consolidate.  Every operation on float32 values is
 * rounded on its own (build with -ffp-contract=off).
 *
 * Returns 0, 1 (allocation failed), 2 (an edge index outside its fragment), 3 (a non-finite vertex),
 * 4 (capacity too small). */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct { uint32_t a, b; int alive; } Edge;

static float v_len(const float* v, uint32_t a, uint32_t b) {
  float dx = v[3 * b] - v[3 * a], dy = v[3 * b + 1] - v[3 * a + 1], dz = v[3 * b + 2] - v[3 * a + 2];
  float xx = dx * dx, yy = dy * dy, zz = dz * dz;
  float s = xx + yy;
  s = s + zz;
  return sqrtf(s);
}

static double v_dist(const float* v, uint32_t a, uint32_t b) {
  double dx = (double)v[3 * a] - (double)v[3 * b], dy = (double)v[3 * a + 1] - (double)v[3 * b + 1];
  double dz = (double)v[3 * a + 2] - (double)v[3 * b + 2];
  double s = dx * dx + dy * dy;
  s = s + dz * dz;
  return sqrt(s);
}

static uint32_t uf_find(uint32_t* p, uint32_t x) {
  while (p[x] != x) {
    p[x] = p[p[x]];
    x = p[x];
  }
  return x;
}

static int uf_union(uint32_t* p, uint32_t a, uint32_t b) {
  a = uf_find(p, a);
  b = uf_find(p, b);
  if (a == b) return 0;
  if (a < b) p[b] = a; else p[a] = b;
  return 1;
}

/* ---------------------------------------------------------------- consolidate */
static const float* g_keys;  /* qsort context */

static int cmp_vert(const void* pa, const void* pb) {
  uint32_t i = *(const uint32_t*)pa, j = *(const uint32_t*)pb;
  for (int d = 0; d < 3; ++d) {
    float x = g_keys[3 * i + d], y = g_keys[3 * j + d];
    if (x < y) return -1;
    if (x > y) return 1;
  }
  return i < j ? -1 : (i > j);
}

static int cmp_u64(const void* pa, const void* pb) {
  uint64_t a = *(const uint64_t*)pa, b = *(const uint64_t*)pb;
  return a < b ? -1 : (a > b);
}

typedef struct {
  uint32_t nv, ne;
  float* v;
  float* r;
  uint8_t* t;
  uint64_t* e; /* (lo << 32) | hi, sorted */
} Skel;

static void skel_free(Skel* s) {
  free(s->v);
  free(s->r);
  free(s->t);
  free(s->e);
  memset(s, 0, sizeof(*s));
}

/* vertices v (n), edges ek (m pairs of indices into v) -> out, consolidated */
static int consolidate(uint32_t n, const float* v, const float* r, const uint8_t* t, uint64_t m,
                       const uint32_t* ea, const uint32_t* eb, Skel* out) {
  memset(out, 0, sizeof(*out));
  uint32_t* ord = malloc(sizeof(uint32_t) * (n + 1));
  uint32_t* uid = malloc(sizeof(uint32_t) * (n + 1));
  uint32_t* first = malloc(sizeof(uint32_t) * (n + 1));
  float* k = malloc(sizeof(float) * 3 * (n + 1));
  uint64_t* ek = malloc(sizeof(uint64_t) * (m + 1));
  uint32_t* used = malloc(sizeof(uint32_t) * (n + 1));
  if (!ord || !uid || !first || !k || !ek || !used) goto oom;
  for (uint32_t i = 0; i < n; ++i) {
    ord[i] = i;
    for (int d = 0; d < 3; ++d) k[3 * i + d] = v[3 * i + d] + 0.0f;
  }
  g_keys = k;
  qsort(ord, n, sizeof(uint32_t), cmp_vert);
  uint32_t u = 0;
  for (uint32_t p = 0; p < n; ++p) {
    uint32_t i = ord[p];
    if (p == 0 || memcmp(&k[3 * i], &k[3 * ord[p - 1]], 12) != 0) {
      /* equal floats other than +-0 have equal bits, and -0 is gone */
      first[u++] = i;
    }
    uid[i] = u - 1;
  }
  uint64_t ne = 0;
  for (uint64_t e = 0; e < m; ++e) {
    uint32_t a = uid[ea[e]], b = uid[eb[e]];
    if (a == b) continue;
    if (a > b) { uint32_t x = a; a = b; b = x; }
    ek[ne++] = ((uint64_t)a << 32) | b;
  }
  qsort(ek, ne, sizeof(uint64_t), cmp_u64);
  uint64_t w = 0;
  for (uint64_t e = 0; e < ne; ++e)
    if (e == 0 || ek[e] != ek[e - 1]) ek[w++] = ek[e];
  ne = w;
  for (uint32_t i = 0; i < u; ++i) used[i] = 0;
  for (uint64_t e = 0; e < ne; ++e) used[ek[e] >> 32] = used[(uint32_t)ek[e]] = 1;
  uint32_t nv = 0;
  for (uint32_t i = 0; i < u; ++i) used[i] = used[i] ? nv++ : 0xFFFFFFFFu;
  out->nv = nv;
  out->ne = (uint32_t)ne;
  out->v = malloc(sizeof(float) * 3 * (nv + 1));
  out->r = malloc(sizeof(float) * (nv + 1));
  out->t = malloc(nv + 1);
  out->e = malloc(sizeof(uint64_t) * (ne + 1));
  if (!out->v || !out->r || !out->t || !out->e) goto oom;
  for (uint32_t i = 0; i < u; ++i) {
    if (used[i] == 0xFFFFFFFFu) continue;
    memcpy(&out->v[3 * used[i]], &v[3 * first[i]], 12);
    out->r[used[i]] = r[first[i]];
    out->t[used[i]] = t[first[i]];
  }
  for (uint64_t e = 0; e < ne; ++e) out->e[e] = ((uint64_t)used[ek[e] >> 32] << 32) | used[(uint32_t)ek[e]];
  free(ord); free(uid); free(first); free(k); free(ek); free(used);
  return 0;
oom:
  free(ord); free(uid); free(first); free(k); free(ek); free(used);
  skel_free(out);
  return 1;
}

/* ---------------------------------------------------------------- postprocess on a fixed vertex set */
typedef struct {
  uint32_t n;
  const float* v;
  const float* r;
  Edge* e;
  uint64_t m, cap;
  uint32_t* deg;
} Graph;

static void g_degrees(Graph* g) {
  memset(g->deg, 0, sizeof(uint32_t) * g->n);
  for (uint64_t i = 0; i < g->m; ++i)
    if (g->e[i].alive) g->deg[g->e[i].a]++, g->deg[g->e[i].b]++;
}

static int cmp_edge(const void* pa, const void* pb) {
  const Edge *x = pa, *y = pb;
  if (x->a != y->a) return x->a < y->a ? -1 : 1;
  return x->b < y->b ? -1 : (x->b > y->b);
}

/* drop dead edges and sort by (lo, hi) */
static void g_tidy(Graph* g) {
  uint64_t w = 0;
  for (uint64_t i = 0; i < g->m; ++i)
    if (g->e[i].alive) g->e[w++] = g->e[i];
  g->m = w;
  qsort(g->e, g->m, sizeof(Edge), cmp_edge);
}

static void g_add(Graph* g, uint32_t a, uint32_t b) {
  if (a > b) { uint32_t x = a; a = b; b = x; }
  for (uint64_t i = 0; i < g->m; ++i)
    if (g->e[i].alive && g->e[i].a == a && g->e[i].b == b) return;
  g->e[g->m].a = a;
  g->e[g->m].b = b;
  g->e[g->m].alive = 1;
  g->m++;
}

static int dust(Graph* g, double thr, uint32_t* p, double* cable) {
  for (uint32_t i = 0; i < g->n; ++i) p[i] = i, cable[i] = 0.0;
  for (uint64_t i = 0; i < g->m; ++i) uf_union(p, g->e[i].a, g->e[i].b);
  for (uint64_t i = 0; i < g->m; ++i) cable[uf_find(p, g->e[i].a)] += (double)v_len(g->v, g->e[i].a, g->e[i].b);
  for (uint64_t i = 0; i < g->m; ++i)
    if (cable[uf_find(p, g->e[i].a)] < thr) g->e[i].alive = 0;
  g_tidy(g);
  return 0;
}

/* one cycle per call; 1 when a cycle was handled */
static int one_loop(Graph* g, uint32_t* p, uint32_t* off, uint32_t* adj, uint32_t* prev, uint32_t* path) {
  uint32_t n = g->n;
  g_tidy(g);
  for (uint32_t i = 0; i < n; ++i) p[i] = i;
  uint64_t c = g->m;
  for (uint64_t i = 0; i < g->m; ++i)
    if (!uf_union(p, g->e[i].a, g->e[i].b)) { c = i; break; }
  if (c == g->m) return 0;
  /* tree edges 0..c-1: adjacency, then the tree path from a to b */
  memset(off, 0, sizeof(uint32_t) * (n + 1));
  for (uint64_t i = 0; i < c; ++i) off[g->e[i].a + 1]++, off[g->e[i].b + 1]++;
  for (uint32_t i = 0; i < n; ++i) off[i + 1] += off[i];
  for (uint32_t i = 0; i < n; ++i) prev[i] = off[i];  /* fill cursors */
  for (uint64_t i = 0; i < c; ++i) {
    adj[prev[g->e[i].a]++] = g->e[i].b;
    adj[prev[g->e[i].b]++] = g->e[i].a;
  }
  uint32_t a = g->e[c].a, b = g->e[c].b;
  for (uint32_t i = 0; i < n; ++i) prev[i] = 0xFFFFFFFFu;
  prev[a] = a;
  uint32_t* stack = p;  /* union-find is done with */
  uint32_t top = 0;
  stack[top++] = a;
  while (top) {
    uint32_t x = stack[--top];
    for (uint32_t j = off[x]; j < off[x + 1]; ++j)
      if (prev[adj[j]] == 0xFFFFFFFFu) prev[adj[j]] = x, stack[top++] = adj[j];
  }
  uint32_t k = 0;
  for (uint32_t x = b;; x = prev[x]) {
    path[k++] = x;
    if (x == a) break;
  }
  for (uint32_t i = 0; i < k / 2; ++i) { uint32_t x = path[i]; path[i] = path[k - 1 - i]; path[k - 1 - i] = x; }
  /* ring edge i joins path[i] and path[(i + 1) % k] */
  g_degrees(g);
  uint32_t br[3], nb = 0;
  for (uint32_t i = 0; i < k; ++i)
    if (g->deg[path[i]] >= 3) { if (nb < 3) br[nb] = i; nb++; }
#define RING_DROP(i)                                                             \
  do {                                                                           \
    uint32_t x_ = path[(i)], y_ = path[((i) + 1) % k];                           \
    if (x_ > y_) { uint32_t s_ = x_; x_ = y_; y_ = s_; }                         \
    for (uint64_t q_ = 0; q_ < g->m; ++q_)                                       \
      if (g->e[q_].alive && g->e[q_].a == x_ && g->e[q_].b == y_) g->e[q_].alive = 0; \
  } while (0)
  if (nb == 0) {
    for (uint32_t i = 0; i < k; ++i) RING_DROP(i);
  } else if (nb == 1) {
    uint32_t bv = path[br[0]], f = bv;
    double best = -1.0;
    for (uint32_t i = 0; i < k; ++i) {
      double d = v_dist(g->v, bv, path[i]);
      if (d > best || (d == best && path[i] < f)) best = d, f = path[i];
    }
    for (uint32_t i = 0; i < k; ++i) RING_DROP(i);
    g_add(g, bv, f);
  } else if (nb == 2) {
    uint32_t i = br[0], j = br[1];
    uint32_t len1 = j - i, len2 = k - len1;
    uint32_t m1 = 0xFFFFFFFFu, m2 = 0xFFFFFFFFu;
    for (uint32_t q = i + 1; q < j; ++q) if (path[q] < m1) m1 = path[q];
    for (uint32_t q = j + 1; q < k + i; ++q) if (path[q % k] < m2) m2 = path[q % k];
    int keep1 = len1 != len2 ? len1 < len2 : m1 < m2;
    if (keep1) { for (uint32_t q = j; q < k + i; ++q) RING_DROP(q % k); }
    else { for (uint32_t q = i; q < j; ++q) RING_DROP(q); }
  } else {
    uint32_t bi = 0, ba = 0, bb = 0;
    float bl = -1.0f;
    for (uint32_t i = 0; i < k; ++i) {
      uint32_t x = path[i], y = path[(i + 1) % k];
      if (x > y) { uint32_t s = x; x = y; y = s; }
      float l = v_len(g->v, x, y);
      if (l > bl || (l == bl && (x < ba || (x == ba && y < bb)))) bl = l, ba = x, bb = y, bi = i;
    }
    RING_DROP(bi);
  }
#undef RING_DROP
  return 1;
}

typedef struct { double d; uint32_t a, b; } Cand;

static int cmp_cand(const void* pa, const void* pb) {
  const Cand *x = pa, *y = pb;
  if (x->d != y->d) return x->d < y->d ? -1 : 1;
  if (x->a != y->a) return x->a < y->a ? -1 : 1;
  return x->b < y->b ? -1 : (x->b > y->b);
}

/* Kruskal over the candidates */
static int connect(Graph* g, uint32_t* p) {
  uint32_t n = g->n;
  g_degrees(g);
  for (uint32_t i = 0; i < n; ++i) p[i] = i;
  for (uint64_t i = 0; i < g->m; ++i) uf_union(p, g->e[i].a, g->e[i].b);
  uint32_t roots = 0;
  for (uint32_t i = 0; i < n; ++i) roots += g->deg[i] && uf_find(p, i) == i;
  if (roots < 2) return 0;
  uint64_t nc = 0, cap = 1024;
  Cand* c = malloc(sizeof(Cand) * cap);
  if (!c) return 1;
  for (uint32_t a = 0; a < n; ++a) {
    if (!g->deg[a]) continue;
    uint32_t ra = uf_find(p, a);
    for (uint32_t b = a + 1; b < n; ++b) {
      if (!g->deg[b] || uf_find(p, b) == ra) continue;
      double d = v_dist(g->v, a, b);
      if (!(d < (double)g->r[a] + (double)g->r[b])) continue;
      if (nc == cap) {
        Cand* q = realloc(c, sizeof(Cand) * (cap *= 2));
        if (!q) { free(c); return 1; }
        c = q;
      }
      c[nc].d = d, c[nc].a = a, c[nc].b = b, nc++;
    }
  }
  qsort(c, nc, sizeof(Cand), cmp_cand);
  for (uint64_t i = 0; i < nc; ++i)
    if (uf_union(p, c[i].a, c[i].b)) {
      g->e[g->m].a = c[i].a, g->e[g->m].b = c[i].b, g->e[g->m].alive = 1;
      g->m++;
    }
  free(c);
  g_tidy(g);
  return 0;
}

static int ticks(Graph* g, double thr, uint32_t* p, uint32_t* off, uint32_t* adj, uint32_t* eid) {
  uint32_t n = g->n;
  g_tidy(g);
  g_degrees(g);
  for (uint32_t i = 0; i < n; ++i) p[i] = i;
  for (uint64_t i = 0; i < g->m; ++i) uf_union(p, g->e[i].a, g->e[i].b);
  memset(off, 0, sizeof(uint32_t) * (n + 1));
  for (uint64_t i = 0; i < g->m; ++i) off[g->e[i].a + 1]++, off[g->e[i].b + 1]++;
  for (uint32_t i = 0; i < n; ++i) off[i + 1] += off[i];
  uint32_t* cur = malloc(sizeof(uint32_t) * (n + 1));
  uint8_t* done = calloc(n + 1, 1);
  if (!cur || !done) { free(cur); free(done); return 1; }
  memcpy(cur, off, sizeof(uint32_t) * n);
  for (uint64_t i = 0; i < g->m; ++i) {
    adj[cur[g->e[i].a]] = g->e[i].b, eid[cur[g->e[i].a]++] = (uint32_t)i;
    adj[cur[g->e[i].b]] = g->e[i].a, eid[cur[g->e[i].b]++] = (uint32_t)i;
  }
  for (uint32_t i = 0; i < n; ++i) p[i] = uf_find(p, i);
  for (;;) {
    /* the shortest tick over every component that still has a branch vertex and is not done */
    uint32_t* nbr = cur;  /* reused: branch count per root */
    memset(nbr, 0, sizeof(uint32_t) * n);
    for (uint32_t i = 0; i < n; ++i) if (g->deg[i] >= 3) nbr[p[i]]++;
    int any = 0;
    for (uint32_t c = 0; c < n; ++c) {
      if (!nbr[c] || done[c]) continue;
      double bl = INFINITY;
      uint32_t bleaf = 0xFFFFFFFFu;
      for (uint32_t leaf = 0; leaf < n; ++leaf) {
        if (p[leaf] != c || g->deg[leaf] != 1) continue;
        uint32_t prv = 0xFFFFFFFFu, x = leaf;
        double len = 0.0;
        do {
          uint32_t y = 0xFFFFFFFFu;
          for (uint32_t j = off[x]; j < off[x + 1]; ++j)
            if (g->e[eid[j]].alive && adj[j] != prv) { y = adj[j]; break; }
          len += (double)v_len(g->v, x < y ? x : y, x < y ? y : x);
          prv = x, x = y;
        } while (g->deg[x] < 3);
        if (len < bl) bl = len, bleaf = leaf;
      }
      if (!(bl < thr)) { done[c] = 1; continue; }
      any = 1;
      uint32_t prv = 0xFFFFFFFFu, x = bleaf;
      do {
        uint32_t y = 0xFFFFFFFFu, q = 0;
        for (uint32_t j = off[x]; j < off[x + 1]; ++j)
          if (g->e[eid[j]].alive && adj[j] != prv) { y = adj[j]; q = eid[j]; break; }
        g->e[q].alive = 0;
        g->deg[x]--, g->deg[y]--;
        prv = x, x = y;
      } while (g->deg[x] + 1 < 3);
      break;  /* degrees changed: count branch vertices again */
    }
    if (!any) break;
  }
  free(cur);
  free(done);
  g_tidy(g);
  return 0;
}

static int postprocess(Skel* s, double dust_thr, double tick_thr, Skel* out) {
  uint32_t n = s->nv;
  Graph g = {n, s->v, s->r, NULL, s->ne, 2 * (uint64_t)s->ne + n + 1, NULL};
  g.e = malloc(sizeof(Edge) * g.cap);
  g.deg = malloc(sizeof(uint32_t) * (n + 1));
  uint32_t* p = malloc(sizeof(uint32_t) * (n + 1));
  uint32_t* off = malloc(sizeof(uint32_t) * (n + 2));
  uint32_t* adj = malloc(sizeof(uint32_t) * (2 * g.cap + 1));
  uint32_t* eid = malloc(sizeof(uint32_t) * (2 * g.cap + 1));
  uint32_t* prev = malloc(sizeof(uint32_t) * (n + 1));
  uint32_t* path = malloc(sizeof(uint32_t) * (n + 1));
  double* cable = malloc(sizeof(double) * (n + 1));
  uint32_t *ea = NULL, *eb = NULL;
  int rc = 1;
  if (!g.e || !g.deg || !p || !off || !adj || !eid || !prev || !path || !cable) goto done;
  for (uint32_t i = 0; i < s->ne; ++i)
    g.e[i].a = (uint32_t)(s->e[i] >> 32), g.e[i].b = (uint32_t)s->e[i], g.e[i].alive = 1;
  if (dust_thr > 0 && dust(&g, dust_thr, p, cable)) goto done;
  while (one_loop(&g, p, off, adj, prev, path)) {}
  if (connect(&g, p)) goto done;
  if (tick_thr > 0 && ticks(&g, tick_thr, p, off, adj, eid)) goto done;
  g_tidy(&g);
  ea = malloc(sizeof(uint32_t) * (g.m + 1));
  eb = malloc(sizeof(uint32_t) * (g.m + 1));
  if (!ea || !eb) goto done;
  for (uint64_t i = 0; i < g.m; ++i) ea[i] = g.e[i].a, eb[i] = g.e[i].b;
  rc = consolidate(n, s->v, s->r, s->t, g.m, ea, eb, out);
done:
  free(g.e); free(g.deg); free(p); free(off); free(adj); free(eid); free(prev); free(path); free(cable);
  free(ea); free(eb);
  return rc;
}

static double cable_length(const Skel* s) {
  double c = 0.0;
  for (uint32_t i = 0; i < s->ne; ++i) c += (double)v_len(s->v, (uint32_t)(s->e[i] >> 32), (uint32_t)s->e[i]);
  return c;
}

static uint64_t blob_bytes(uint64_t nv, uint64_t ne, int vt) { return 8 + 16 * nv + 8 * ne + (vt ? nv : 0); }

uint64_t orc_skeleton_merge_capacity(uint64_t n_labels, uint64_t n_vertices, uint64_t n_edges) {
  return 16 * n_labels + 25 * n_vertices + 8 * n_edges;
}

int orc_skeleton_merge(uint64_t n_labels, const uint64_t* label_frag, const uint64_t* frag_vert,
                       const uint64_t* frag_edge, const double* frag_box, const float* vertices, const float* radius,
                       const uint8_t* vtypes, const uint32_t* edges, double dust_thr, double tick_thr,
                       double max_cable, int vertex_types, uint8_t* blobs, uint64_t capacity, uint64_t* table,
                       uint64_t* nbytes) {
  uint64_t nf = label_frag[n_labels], nvert = frag_vert[nf], nedge = frag_edge[nf];
  for (uint64_t i = 0; i < 3 * nvert; ++i)
    if (!isfinite(vertices[i])) return 3;
  for (uint64_t f = 0; f < nf; ++f)
    for (uint64_t e = frag_edge[f]; e < frag_edge[f + 1]; ++e)
      if (edges[2 * e] >= frag_vert[f + 1] - frag_vert[f] || edges[2 * e + 1] >= frag_vert[f + 1] - frag_vert[f])
        return 2;
  if (capacity < orc_skeleton_merge_capacity(n_labels, nvert, nedge)) return 4;
  uint64_t at = 0;
  for (uint64_t l = 0; l < n_labels; ++l) {
    uint64_t v0 = frag_vert[label_frag[l]], v1 = frag_vert[label_frag[l + 1]];
    uint64_t e0 = frag_edge[label_frag[l]], e1 = frag_edge[label_frag[l + 1]];
    uint32_t n = (uint32_t)(v1 - v0);
    uint32_t* map = malloc(sizeof(uint32_t) * (n + 1));
    uint32_t* ea = malloc(sizeof(uint32_t) * (e1 - e0 + 1));
    uint32_t* eb = malloc(sizeof(uint32_t) * (e1 - e0 + 1));
    float* v = malloc(sizeof(float) * 3 * (n + 1));
    float* r = malloc(sizeof(float) * (n + 1));
    uint8_t* t = malloc(n + 1);
    if (!map || !ea || !eb || !v || !r || !t) return 1;
    uint32_t kept = 0;
    uint64_t m = 0;
    for (uint64_t f = label_frag[l]; f < label_frag[l + 1]; ++f) {
      const double* box = frag_box + 6 * f;
      for (uint64_t i = frag_vert[f]; i < frag_vert[f + 1]; ++i) {
        int in = 1;
        for (int d = 0; d < 3; ++d) {
          double c = (double)vertices[3 * i + d];
          in &= box[d] <= c && c <= box[3 + d];
        }
        map[i - v0] = in ? kept : 0xFFFFFFFFu;
        if (in) {
          memcpy(&v[3 * kept], &vertices[3 * i], 12);
          r[kept] = radius[i];
          t[kept] = vtypes[i];
          kept++;
        }
      }
      for (uint64_t e = frag_edge[f]; e < frag_edge[f + 1]; ++e) {
        uint32_t a = map[frag_vert[f] - v0 + edges[2 * e]], b = map[frag_vert[f] - v0 + edges[2 * e + 1]];
        if (a == 0xFFFFFFFFu || b == 0xFFFFFFFFu) continue;
        ea[m] = a, eb[m] = b, m++;
      }
    }
    Skel fused, post;
    int rc = consolidate(kept, v, r, t, m, ea, eb, &fused);
    free(map); free(ea); free(eb); free(v); free(r); free(t);
    if (rc) return rc;
    Skel* s = &fused;
    if (!(cable_length(&fused) > max_cable)) {
      rc = postprocess(&fused, dust_thr, tick_thr, &post);
      if (rc) { skel_free(&fused); return rc; }
      s = &post;
    }
    table[4 * l] = l;
    table[4 * l + 1] = at;
    table[4 * l + 2] = s->nv;
    table[4 * l + 3] = s->ne;
    uint8_t* o = blobs + at;
    uint32_t h[2] = {s->nv, s->ne};
    memcpy(o, h, 8);
    memcpy(o + 8, s->v, 12 * (size_t)s->nv);
    uint32_t* oe = (uint32_t*)(o + 8 + 12 * (size_t)s->nv);
    for (uint32_t i = 0; i < s->ne; ++i) oe[2 * i] = (uint32_t)(s->e[i] >> 32), oe[2 * i + 1] = (uint32_t)s->e[i];
    memcpy(o + 8 + 12 * (size_t)s->nv + 8 * (size_t)s->ne, s->r, 4 * (size_t)s->nv);
    if (vertex_types) memcpy(o + 8 + 16 * (size_t)s->nv + 8 * (size_t)s->ne, s->t, s->nv);
    uint64_t end = at + blob_bytes(s->nv, s->ne, vertex_types);
    for (uint64_t b = end; b & 7; ++b) blobs[b] = 0;
    at = (end + 7) & ~7ull;
    *nbytes = end;
    if (s == &post) skel_free(&post);
    skel_free(&fused);
  }
  if (n_labels == 0) *nbytes = 0;
  return 0;
}
