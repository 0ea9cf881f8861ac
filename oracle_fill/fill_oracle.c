/*
 * fill_oracle.c -- serial C restatement of the hole-filling rule (DESIGN.md §5a), the checker of
 * ign_fill_holes / ign_dilate_multilabel.  Test infrastructure only; never linked into the product.
 *
 * Written from the rule's text, not from csrc/fill.cu: components by a voxel union-find, contacts
 * by a sort of pair keys, merge rounds that rebuild the region graph from the component contacts
 * every round, enclosure by an iterative DFS with low-links.  Volumes are uint64, Fortran order.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct {
  uint64_t key, w;
} orc_kw;

static int cmp_u64(const void* a, const void* b) {
  const uint64_t x = *(const uint64_t*)a, y = *(const uint64_t*)b;
  return x < y ? -1 : (x > y);
}
static int cmp_kw(const void* a, const void* b) { return cmp_u64(a, b); }

static uint32_t uf_find(uint32_t* p, uint32_t i) {
  while (p[i] != i) {
    p[i] = p[p[i]];
    i = p[i];
  }
  return i;
}
static void uf_unite(uint32_t* p, uint32_t a, uint32_t b) {
  a = uf_find(p, a);
  b = uf_find(p, b);
  if (a < b) p[b] = a;
  else if (b < a) p[a] = b;
}

/* one multilabel dilation step of the background (mesh.py:211-218) */
void orc_dilate_multilabel(const uint64_t* X, uint64_t sx, uint64_t sy, uint64_t sz, uint64_t* out) {
  for (uint64_t z = 0; z < sz; z++)
    for (uint64_t y = 0; y < sy; y++)
      for (uint64_t x = 0; x < sx; x++) {
        const uint64_t i = (z * sy + y) * sx + x;
        out[i] = X[i];
        if (X[i] != 0) continue;
        uint64_t v[26];
        int m = 0;
        for (int dz = -1; dz <= 1; dz++)
          for (int dy = -1; dy <= 1; dy++)
            for (int dx = -1; dx <= 1; dx++) {
              const int64_t gx = (int64_t)x + dx, gy = (int64_t)y + dy, gz = (int64_t)z + dz;
              if ((dx | dy | dz) == 0 || gx < 0 || gy < 0 || gz < 0 || gx >= (int64_t)sx || gy >= (int64_t)sy ||
                  gz >= (int64_t)sz)
                continue;
              const uint64_t u = X[((uint64_t)gz * sy + (uint64_t)gy) * sx + (uint64_t)gx];
              if (u) v[m++] = u;
            }
        if (m == 0) continue;
        qsort(v, (size_t)m, sizeof(uint64_t), cmp_u64);
        uint64_t best = 0;
        int bestc = 0;
        for (int a = 0; a < m;) {  /* ascending runs: a later run wins only with a strictly larger count */
          int b = a;
          while (b < m && v[b] == v[a]) b++;
          if (b - a > bestc) {
            bestc = b - a;
            best = v[a];
          }
          a = b;
        }
        out[i] = best;
      }
}

/* steps 2-5 on one volume: filled.  axes: bit mask of the axes whose box faces are the outside */
static int fill_pass(const uint64_t* X, uint64_t sx, uint64_t sy, uint64_t sz, unsigned axes, int p, uint64_t* filled) {
  const uint64_t n = sx * sy * sz;
  uint32_t* par = malloc(n * 4);
  uint32_t* comp = malloc(n * 4);
  if (!par || !comp) return -1;
  for (uint64_t i = 0; i < n; i++) par[i] = (uint32_t)i;
  for (uint64_t z = 0; z < sz; z++)
    for (uint64_t y = 0; y < sy; y++)
      for (uint64_t x = 0; x < sx; x++) {
        const uint64_t i = (z * sy + y) * sx + x;
        if (x && X[i - 1] == X[i]) uf_unite(par, (uint32_t)i, (uint32_t)(i - 1));
        if (y && X[i - sx] == X[i]) uf_unite(par, (uint32_t)i, (uint32_t)(i - sx));
        if (z && X[i - sx * sy] == X[i]) uf_unite(par, (uint32_t)i, (uint32_t)(i - sx * sy));
      }
  uint32_t N = 0;
  for (uint64_t i = 0; i < n; i++) {  /* roots are the first voxels: numbered before their members */
    const uint32_t r = uf_find(par, (uint32_t)i);
    comp[i] = r == i ? ++N : comp[r];
  }
  free(par);
  uint64_t* value = calloc(N + 1, 8);
  uint64_t* wo = calloc(N + 1, 8);
  /* contacts: (min, max) keys of differing face neighbours, sorted and counted */
  uint64_t m = 0;
  for (int pass = 0; pass < 2; pass++) {
    uint64_t* keys = pass ? malloc((m ? m : 1) * 8) : NULL;
    uint64_t k = 0;
    for (uint64_t z = 0; z < sz; z++)
      for (uint64_t y = 0; y < sy; y++)
        for (uint64_t x = 0; x < sx; x++) {
          const uint64_t i = (z * sy + y) * sx + x;
          const uint32_t c = comp[i];
          const uint64_t nb[3] = {x + 1 < sx ? i + 1 : i, y + 1 < sy ? i + sx : i, z + 1 < sz ? i + sx * sy : i};
          for (int a = 0; a < 3; a++) {
            const uint32_t d = comp[nb[a]];
            if (d == c) continue;
            if (pass) keys[k] = c < d ? ((uint64_t)c << 32 | d) : ((uint64_t)d << 32 | c);
            k++;
          }
          if (pass) continue;
          value[c] = X[i];
          const uint64_t co[3] = {x, y, z}, ext[3] = {sx, sy, sz};
          for (int a = 0; a < 3; a++)
            if (axes >> a & 1u) wo[c] += (co[a] == 0) + (co[a] + 1 == ext[a]);
        }
    if (!pass) {
      m = k;
      continue;
    }
    qsort(keys, (size_t)m, 8, cmp_u64);
    /* component edges, run-length encoded in place: ea / eb / ew */
    uint64_t E = 0;
    uint32_t *ea = malloc((m ? m : 1) * 4), *eb = malloc((m ? m : 1) * 4);
    uint64_t* ew = malloc((m ? m : 1) * 8);
    for (uint64_t a = 0; a < m;) {
      uint64_t b = a;
      while (b < m && keys[b] == keys[a]) b++;
      ea[E] = (uint32_t)(keys[a] >> 32);
      eb[E] = (uint32_t)keys[a];
      ew[E] = b - a;
      E++;
      a = b;
    }
    free(keys);
    /* ---- merge rounds (p > 0); rt[c] = region of c (chains of absorptions) */
    uint32_t* rt = malloc((N + 1) * 4);
    for (uint32_t c = 0; c <= N; c++) rt[c] = c;
    orc_kw* re = malloc((E ? E : 1) * sizeof(orc_kw));
    uint64_t* rwo = calloc(N + 1, 8);
    uint64_t* area = calloc(N + 1, 8);
    uint64_t* bw = calloc(N + 1, 8);
    uint32_t* bt = calloc(N + 1, 4);
    uint32_t* tgt = calloc(N + 1, 4);
    uint32_t* abs_r = malloc((N + 1) * 4);
    uint32_t* abs_t = malloc((N + 1) * 4);
    uint64_t R = 0;  /* region edges of the current round */
    for (;;) {
      /* region graph from the component contacts */
      R = 0;
      for (uint64_t e = 0; e < E; e++) {
        const uint32_t a = uf_find(rt, ea[e]), b = uf_find(rt, eb[e]);
        if (a == b) continue;
        re[R].key = a < b ? ((uint64_t)a << 32 | b) : ((uint64_t)b << 32 | a);
        re[R].w = ew[e];
        R++;
      }
      qsort(re, (size_t)R, sizeof(orc_kw), cmp_kw);
      uint64_t u = 0;
      for (uint64_t a = 0; a < R;) {
        uint64_t b = a, w = 0;
        while (b < R && re[b].key == re[a].key) w += re[b++].w;
        re[u].key = re[a].key;
        re[u].w = w;
        u++;
        a = b;
      }
      R = u;
      if (p <= 0) break;
      memset(rwo, 0, (N + 1) * 8);
      memset(area, 0, (N + 1) * 8);
      memset(bw, 0, (N + 1) * 8);
      memset(bt, 0, (N + 1) * 4);
      memset(tgt, 0, (N + 1) * 4);
      for (uint32_t c = 1; c <= N; c++) rwo[uf_find(rt, c)] += wo[c];
      for (uint32_t r = 1; r <= N; r++) area[r] = rwo[r];
      for (uint64_t e = 0; e < R; e++) {
        const uint32_t a = (uint32_t)(re[e].key >> 32), b = (uint32_t)re[e].key;
        const uint64_t w = re[e].w;
        area[a] += w;
        area[b] += w;
        if (w > bw[a] || (w == bw[a] && b < bt[a])) { bw[a] = w; bt[a] = b; }
        if (w > bw[b] || (w == bw[b] && a < bt[b])) { bw[b] = w; bt[b] = a; }
      }
      int any = 0;
      for (uint32_t r = 1; r <= N; r++)
        if (rt[r] == r && rwo[r] == 0 && bw[r] > 0 && 100 * bw[r] >= (uint64_t)(100 - p) * area[r]) {
          tgt[r] = bt[r];
          any = 1;
        }
      if (!any) break;
      uint32_t na = 0;
      for (uint32_t r = 1; r <= N; r++) {
        if (!tgt[r]) continue;
        const uint32_t t = tgt[r];
        if (!tgt[t] || (tgt[t] == r && (area[r] < area[t] || (area[r] == area[t] && r > t)))) {
          abs_r[na] = r;
          abs_t[na++] = t;
        }
      }
      if (!na) {  /* a longer cycle: the candidate of smallest area, ties to the larger root */
        uint32_t pick = 0;
        for (uint32_t r = 1; r <= N; r++)
          if (tgt[r] && (!pick || area[r] < area[pick] || (area[r] == area[pick] && r > pick))) pick = r;
        abs_r[na] = pick;
        abs_t[na++] = tgt[pick];
      }
      for (uint32_t k2 = 0; k2 < na; k2++) rt[abs_r[k2]] = abs_t[k2];
    }
    if (p <= 0) memset(rwo, 0, (N + 1) * 8);
    if (p <= 0)
      for (uint32_t c = 1; c <= N; c++) rwo[c] = wo[c];
    /* ---- enclosure: CSR of the region graph plus the outside (node 0) */
    uint64_t* deg = calloc(N + 2, 8);
    for (uint64_t e = 0; e < R; e++) {
      deg[(uint32_t)(re[e].key >> 32) + 1]++;
      deg[(uint32_t)re[e].key + 1]++;
    }
    for (uint32_t r = 1; r <= N; r++)
      if (rt[r] == r && rwo[r]) {
        deg[1]++;
        deg[r + 1]++;
      }
    for (uint32_t i2 = 1; i2 <= N + 1; i2++) deg[i2] += deg[i2 - 1];
    uint32_t* adj = malloc((deg[N + 1] ? deg[N + 1] : 1) * 4);
    uint64_t* fill_at = malloc((N + 1) * 8);
    memcpy(fill_at, deg, (N + 1) * 8);
    for (uint64_t e = 0; e < R; e++) {
      const uint32_t a = (uint32_t)(re[e].key >> 32), b = (uint32_t)re[e].key;
      adj[fill_at[a]++] = b;
      adj[fill_at[b]++] = a;
    }
    for (uint32_t r = 1; r <= N; r++)
      if (rt[r] == r && rwo[r]) {
        adj[fill_at[0]++] = r;
        adj[fill_at[r]++] = 0;
      }
    const uint32_t NONE = 0xFFFFFFFFu;
    uint32_t* disc = malloc((N + 1) * 4);
    uint32_t* low = malloc((N + 1) * 4);
    uint32_t* up = malloc((N + 1) * 4);
    uint64_t* it = malloc((N + 1) * 8);
    uint32_t* stack = malloc((N + 1) * 4);
    uint32_t* order = malloc((N + 1) * 4);
    uint32_t* filler = calloc(N + 1, 4);
    for (uint32_t r = 0; r <= N; r++) disc[r] = NONE;
    uint32_t t = 0, sp = 0, no = 0;
    disc[0] = low[0] = t++;
    up[0] = NONE;
    it[0] = deg[0];
    stack[sp++] = 0;
    while (sp) {
      const uint32_t v = stack[sp - 1];
      if (it[v] < deg[v + 1]) {
        const uint32_t w = adj[it[v]++];
        if (disc[w] == NONE) {
          up[w] = v;
          disc[w] = low[w] = t++;
          it[w] = deg[w];
          order[no++] = w;
          stack[sp++] = w;
        } else if (w != up[v] && disc[w] < low[v]) {
          low[v] = disc[w];
        }
      } else {
        sp--;
        if (v && low[v] < low[up[v]]) low[up[v]] = low[v];
      }
    }
    for (uint32_t k2 = 0; k2 < no; k2++) {
      const uint32_t c = order[k2], v = up[c];
      if (v == 0) continue;
      filler[c] = filler[v] ? filler[v] : ((low[c] >= disc[v] && value[v] != 0) ? v : 0);
    }
    uint64_t* table = malloc((N + 1) * 8);
    for (uint32_t c = 1; c <= N; c++) {
      const uint32_t r = uf_find(rt, c);
      table[c] = filler[r] ? value[filler[r]] : (value[r] ? value[r] : value[c]);
    }
    for (uint64_t i = 0; i < n; i++) filled[i] = table[comp[i]];
    free(table); free(filler); free(order); free(stack); free(it); free(up); free(low); free(disc);
    free(fill_at); free(adj); free(deg); free(abs_t); free(abs_r); free(tgt); free(bt); free(bw); free(area);
    free(rwo); free(re); free(rt); free(ew); free(eb); free(ea);
  }
  free(wo);
  free(value);
  free(comp);
  return 0;
}

/* fastmorph.fill_holes_v2(X0, fix_borders, merge_threshold = 1 - p/100) (mesh.py:220-228) */
int orc_fill_holes(const uint64_t* X0, uint64_t sx, uint64_t sy, uint64_t sz, int fix_borders, int p,
                   uint64_t* filled, uint64_t* holes) {
  const uint64_t n = sx * sy * sz;
  uint64_t* cur = malloc(n * 8);
  if (!cur) return -1;
  memcpy(cur, X0, n * 8);
  if (fix_borders) {
    const uint64_t ext[3] = {sx, sy, sz};
    for (int axis = 0; axis < 3; axis++)
      for (int side = 0; side < 2; side++) {
        const uint64_t idx = side ? ext[axis] - 1 : 0;
        if (side && idx == 0) continue;
        const uint64_t na = axis == 0 ? sy : sx, nb = axis == 2 ? sy : sz;
        uint64_t* pl = malloc(na * nb * 8);
        uint64_t* pf = malloc(na * nb * 8);
        for (uint64_t b = 0; b < nb; b++)
          for (uint64_t a = 0; a < na; a++) {
            const uint64_t x = axis == 0 ? idx : a, y = axis == 1 ? idx : (axis == 0 ? a : b), z = axis == 2 ? idx : b;
            pl[b * na + a] = cur[(z * sy + y) * sx + x];
          }
        if (fill_pass(pl, na, nb, 1, 3u, p, pf)) return -1;
        for (uint64_t b = 0; b < nb; b++)
          for (uint64_t a = 0; a < na; a++) {
            const uint64_t x = axis == 0 ? idx : a, y = axis == 1 ? idx : (axis == 0 ? a : b), z = axis == 2 ? idx : b;
            cur[(z * sy + y) * sx + x] = pf[b * na + a];
          }
        free(pl);
        free(pf);
      }
  }
  const int rc = fill_pass(cur, sx, sy, sz, 7u, p, filled);
  free(cur);
  for (uint64_t i = 0; i < n; i++) holes[i] = (filled[i] != X0[i] && X0[i] != 0) ? X0[i] : 0;
  return rc;
}
