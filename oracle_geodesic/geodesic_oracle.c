/* Serial checker of the geodesic rule (DESIGN.md 5e): a binary-heap Dijkstra over the voxel lattice
 * with explicit float additions, and the parent rule applied to its converged distances.
 * TEST INFRASTRUCTURE ONLY.  Labels are u64, volumes F-order. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct { float d; uint64_t v; } item;

static void push(item* h, uint64_t* n, item it) {
  uint64_t i = (*n)++;
  while (i > 0 && h[(i - 1) / 2].d > it.d) {
    h[i] = h[(i - 1) / 2];
    i = (i - 1) / 2;
  }
  h[i] = it;
}

static item pop(item* h, uint64_t* n) {
  item top = h[0], last = h[--*n];
  uint64_t i = 0;
  for (;;) {
    uint64_t c = 2 * i + 1;
    if (c >= *n) break;
    if (c + 1 < *n && h[c + 1].d < h[c].d) c++;
    if (h[c].d >= last.d) break;
    h[i] = h[c];
    i = c;
  }
  h[i] = last;
  return top;
}

/* neighbours in (dz, dy, dx) raster order, dx fastest; returns how many */
static int neighbours(int connectivity, const float* a, int off[26][3], float w[26]) {
  int maxdiag = connectivity == 6 ? 1 : connectivity == 18 ? 2 : 3, n = 0;
  for (int dz = -1; dz <= 1; dz++)
    for (int dy = -1; dy <= 1; dy++)
      for (int dx = -1; dx <= 1; dx++) {
        int m = abs(dx) + abs(dy) + abs(dz);
        if (m == 0 || m > maxdiag) continue;
        off[n][0] = dx, off[n][1] = dy, off[n][2] = dz;
        if (a) {
          double x = (double)a[0] * dx, y = (double)a[1] * dy, z = (double)a[2] * dz;
          w[n] = (float)sqrt(x * x + y * y + z * z);
        }
        n++;
      }
  return n;
}

/* 0 ok; 1 allocation failed; 2 a reached voxel without a parent under the rule (dist is still complete);
 * 3 a source outside the volume or on label 0 */
int orc_geodesic(const uint64_t* lab, uint64_t sx, uint64_t sy, uint64_t sz, int connectivity, const float* aniso,
                 const float* weights, const uint64_t* sources, uint64_t ns, float* dist, uint32_t* parents) {
  const uint64_t n = sx * sy * sz;
  int off[26][3];
  float w[26];
  const int nn = neighbours(connectivity, weights ? NULL : aniso, off, w);
  /* every lowering pushes once, and a voxel is lowered at most once per edge into it */
  item* heap = (item*)malloc(sizeof(item) * (n * (uint64_t)nn + ns + 1));
  uint8_t* is_source = (uint8_t*)calloc(n ? n : 1, 1);
  if (!heap || !is_source) {
    free(heap);
    free(is_source);
    return 1;
  }
  uint64_t hn = 0;
  for (uint64_t i = 0; i < n; i++) dist[i] = INFINITY;
  for (uint64_t i = 0; i < ns; i++) {
    if (sources[i] >= n || lab[sources[i]] == 0) {
      free(heap);
      free(is_source);
      return 3;
    }
    dist[sources[i]] = 0.0f;
    is_source[sources[i]] = 1;
    push(heap, &hn, (item){0.0f, sources[i]});
  }
  while (hn) {
    const item it = pop(heap, &hn);
    if (it.d > dist[it.v]) continue;
    const int64_t x = it.v % sx, y = (it.v / sx) % sy, z = it.v / (sx * sy);
    for (int k = 0; k < nn; k++) {
      const int64_t qx = x + off[k][0], qy = y + off[k][1], qz = z + off[k][2];
      if (qx < 0 || qy < 0 || qz < 0 || qx >= (int64_t)sx || qy >= (int64_t)sy || qz >= (int64_t)sz) continue;
      const uint64_t q = (uint64_t)qx + sx * ((uint64_t)qy + sy * (uint64_t)qz);
      if (lab[q] != lab[it.v]) continue;
      const float cand = it.d + (weights ? weights[q] : w[k]);
      if (cand < dist[q]) {
        dist[q] = cand;
        push(heap, &hn, (item){cand, q});
      }
    }
  }
  free(heap);
  int rc = 0;
  if (parents) {
    for (uint64_t q = 0; q < n; q++) {
      parents[q] = 0;
      if (lab[q] == 0 || is_source[q] || isinf(dist[q])) continue;
      const int64_t x = q % sx, y = (q / sx) % sy, z = q / (sx * sy);
      for (int k = 0; k < nn && !parents[q]; k++) {
        const int64_t px = x + off[k][0], py = y + off[k][1], pz = z + off[k][2];
        if (px < 0 || py < 0 || pz < 0 || px >= (int64_t)sx || py >= (int64_t)sy || pz >= (int64_t)sz) continue;
        const uint64_t p = (uint64_t)px + sx * ((uint64_t)py + sy * (uint64_t)pz);
        if (lab[p] != lab[q]) continue;
        const float cand = dist[p] + (weights ? weights[q] : w[k]);
        if (cand == dist[q] && (dist[p] < dist[q] || (dist[p] == dist[q] && p < q))) parents[q] = (uint32_t)p + 1;
      }
      if (!parents[q]) rc = 2;
    }
  }
  free(is_source);
  return rc;
}
