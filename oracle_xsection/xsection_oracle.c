/* Serial C checker of the cross-sectional area rule of DESIGN.md §5i -- TEST INFRASTRUCTURE ONLY.
 *
 * orc_xs_normals follows the rule literally: per component, the root r is the vertex farthest in hops from the
 * component's lowest vertex, every other vertex's parent its lowest neighbour one hop nearer r; the leaves are
 * taken shallowest first (ties to the lowest index) and each walks its whole path to r; a vertex takes its
 * normal on the first path that reaches it, from the window of the path's voxel steps around its position.
 * orc_xs_sections walks each point's section breadth first with a per-point stamp over the whole volume and
 * adds up each cut voxel's area by inclusion-exclusion over the corners of its box.  Built with
 * -ffp-contract=off so that every float64 operation rounds on its own. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

static int64_t sym(int64_t j, int64_t len) {
  int64_t m = j % (2 * len);
  if (m < 0) m += 2 * len;
  return m < len ? m : 2 * len - 1 - m;
}

/* 0 ok, 1 allocation failed, 2 an edge index out of range */
int orc_xs_normals(uint64_t nv, const int64_t* vox, uint64_t ne, const uint32_t* edges, const double* a,
                   uint64_t window, double* out) {
  int rc = 1;
  uint64_t *start = calloc(nv + 1, 8), *pos = NULL;
  uint32_t *nbr = NULL, *queue = NULL, *parent = NULL, *leaves = NULL, *path = NULL;
  int64_t *hop = NULL, *dep = NULL;
  unsigned char* done = NULL;
  if (!start) return 1;
  for (uint64_t e = 0; e < ne; e++) {
    if (edges[2 * e] >= nv || edges[2 * e + 1] >= nv) { free(start); return 2; }
    if (edges[2 * e] == edges[2 * e + 1]) continue;
    start[edges[2 * e] + 1]++;
    start[edges[2 * e + 1] + 1]++;
  }
  for (uint64_t v = 0; v < nv; v++) start[v + 1] += start[v];
  pos = malloc((nv + 1) * 8);
  nbr = malloc((start[nv] + 1) * 4);
  queue = malloc((nv + 1) * 4);
  parent = malloc((nv + 1) * 4);
  leaves = malloc((nv + 1) * 4);
  path = malloc((nv + 1) * 4);
  hop = malloc((nv + 1) * 8);
  dep = malloc((nv + 1) * 8);
  done = calloc(nv + 1, 1);
  if (!pos || !nbr || !queue || !parent || !leaves || !path || !hop || !dep || !done) goto out;
  memcpy(pos, start, nv * 8);
  for (uint64_t e = 0; e < ne; e++) {
    uint32_t u = edges[2 * e], w = edges[2 * e + 1];
    if (u == w) continue;
    nbr[pos[u]++] = w;
    nbr[pos[w]++] = u;
  }
  for (uint64_t v = 0; v < nv; v++) hop[v] = dep[v] = -1;
  for (uint64_t s = 0; s < nv; s++) {
    if (hop[s] >= 0) continue;
    uint64_t qn = 0;
    queue[qn++] = (uint32_t)s;
    hop[s] = 0;
    for (uint64_t h = 0; h < qn; h++)
      for (uint64_t e = start[queue[h]]; e < start[queue[h] + 1]; e++)
        if (hop[nbr[e]] < 0) { hop[nbr[e]] = hop[queue[h]] + 1; queue[qn++] = nbr[e]; }
    if (qn == 1) { out[3 * s] = out[3 * s + 1] = out[3 * s + 2] = 0.0; done[s] = 1; continue; }
    uint32_t r = (uint32_t)s;
    for (uint64_t h = 0; h < qn; h++) {
      uint32_t u = queue[h];
      if (hop[u] > hop[r] || (hop[u] == hop[r] && u < r)) r = u;
    }
    qn = 0;
    queue[qn++] = r;
    dep[r] = 0;
    for (uint64_t h = 0; h < qn; h++)
      for (uint64_t e = start[queue[h]]; e < start[queue[h] + 1]; e++)
        if (dep[nbr[e]] < 0) { dep[nbr[e]] = dep[queue[h]] + 1; queue[qn++] = nbr[e]; }
    /* parents, then the leaves: vertices nobody names as parent */
    for (uint64_t h = 0; h < qn; h++) {
      uint32_t u = queue[h], p = UINT32_MAX;
      for (uint64_t e = start[u]; e < start[u + 1]; e++)
        if (dep[nbr[e]] == dep[u] - 1 && nbr[e] < p) p = nbr[e];
      parent[u] = p;
    }
    uint64_t nl = 0;
    for (uint64_t h = 0; h < qn; h++) {
      uint32_t u = queue[h];
      int leaf = u != r;
      for (uint64_t e = start[u]; e < start[u + 1] && leaf; e++)
        if (parent[nbr[e]] == u) leaf = 0;
      if (leaf) leaves[nl++] = u;
    }
    /* shallowest first, ties to the lowest index (insertion sort: small lists) */
    for (uint64_t i = 1; i < nl; i++) {
      uint32_t x = leaves[i];
      uint64_t j = i;
      while (j > 0 && (dep[leaves[j - 1]] > dep[x] || (dep[leaves[j - 1]] == dep[x] && leaves[j - 1] > x))) {
        leaves[j] = leaves[j - 1];
        j--;
      }
      leaves[j] = x;
    }
    for (uint64_t l = 0; l < nl; l++) {
      int64_t len = 0;
      for (uint32_t u = leaves[l];; u = parent[u]) {
        path[len++] = u;
        if (u == r) break;
      }
      for (int64_t i = 0; i < len; i++) {
        uint32_t v = path[i];
        if (done[v]) continue;
        done[v] = 1;
        int64_t sum[3] = {0, 0, 0};
        int64_t lo = i - (int64_t)(window / 2);
        for (int64_t j = lo; j < lo + (int64_t)window; j++) {
          int64_t p = sym(j, len);
          if (p == len - 1) p = len - 2;
          for (int k = 0; k < 3; k++) sum[k] += vox[3 * (uint64_t)path[p] + k] - vox[3 * (uint64_t)path[p + 1] + k];
        }
        if (!sum[0] && !sum[1] && !sum[2]) {
          int64_t p = i == len - 1 ? len - 2 : i;
          for (int k = 0; k < 3; k++) sum[k] = vox[3 * (uint64_t)path[p] + k] - vox[3 * (uint64_t)path[p + 1] + k];
        }
        for (int k = 0; k < 3; k++) out[3 * (uint64_t)v + k] = (double)sum[k] * a[k];
      }
    }
  }
  rc = 0;
out:
  free(start); free(pos); free(nbr); free(queue); free(parent); free(leaves); free(path); free(hop); free(dep);
  free(done);
  return rc;
}

/* area of {y in [-a/2, a/2]^3 : n.y = -s}: |n| d/dt of the volume below the plane, corner by corner */
static double box_area(const double* n, const double* a, double s) {
  double e[3], nz = 1.0, zero = 1.0;
  int idx[3], m = 0;
  for (int i = 0; i < 3; i++) {
    if (n[i] != 0.0) { idx[m++] = i; nz *= fabs(n[i]); } else zero *= a[i];
    e[i] = fabs(n[i]) * a[i] * 0.5;
  }
  if (m == 1) return zero;
  double norm = sqrt((n[0] * n[0] + n[1] * n[1]) + n[2] * n[2]);
  double f = 0.0;
  for (int c = 0; c < (1 << m); c++) {
    double corner = 0.0;
    int odd = 0;
    for (int i = 0; i < m; i++) {
      int up = (c >> i) & 1;
      corner += up ? e[idx[i]] : -e[idx[i]];
      odd ^= up;
    }
    double w = -s - corner;
    if (w <= 0.0) continue;
    double term = m == 3 ? w * w : w;
    f += odd ? -term : term;
  }
  return m == 3 ? zero * f * norm / (2.0 * nz) : zero * f * norm / nz;
}

/* labels uint64 F-order; 0 ok, 1 allocation failed, 3 a point outside the volume */
int orc_xs_sections(const uint64_t* labels, uint64_t sx, uint64_t sy, uint64_t sz, uint64_t np,
                    const uint64_t* voxel, const uint64_t* label, const double* normal, const double* a,
                    float* area, uint8_t* contacts, uint64_t* visited) {
  uint64_t n = sx * sy * sz;
  uint64_t* stamp = calloc(n ? n : 1, 8);
  uint64_t* queue = malloc((n ? n : 1) * 8);
  if (!stamp || !queue) { free(stamp); free(queue); return 1; }
  *visited = 0;
  for (uint64_t p = 0; p < np; p++) {
    const double* nn = normal + 3 * p;
    area[p] = 0.f;
    contacts[p] = 0;
    if (voxel[p] >= n) { free(stamp); free(queue); return 3; }
    if ((nn[0] == 0.0 && nn[1] == 0.0 && nn[2] == 0.0) || labels[voxel[p]] != label[p]) continue;
    int64_t c[3] = {(int64_t)(voxel[p] % sx), (int64_t)(voxel[p] / sx % sy), (int64_t)(voxel[p] / sx / sy)};
    double h = 0.5 * ((fabs(nn[0]) * a[0] + fabs(nn[1]) * a[1]) + fabs(nn[2]) * a[2]);
    uint64_t qn = 0;
    queue[qn++] = voxel[p];
    stamp[voxel[p]] = p + 1;
    double sum = 0.0;
    uint8_t faces = 0;
    for (uint64_t k = 0; k < qn; k++) {
      int64_t x = (int64_t)(queue[k] % sx), y = (int64_t)(queue[k] / sx % sy), z = (int64_t)(queue[k] / sx / sy);
      double d0 = (double)(x - c[0]) * a[0], d1 = (double)(y - c[1]) * a[1], d2 = (double)(z - c[2]) * a[2];
      sum += box_area(nn, a, (nn[0] * d0 + nn[1] * d1) + nn[2] * d2);
      faces |= (x == 0) | (x == (int64_t)sx - 1) << 1 | (y == 0) << 2 | (y == (int64_t)sy - 1) << 3 |
               (z == 0) << 4 | (z == (int64_t)sz - 1) << 5;
      for (int dz = -1; dz <= 1; dz++)
        for (int dy = -1; dy <= 1; dy++)
          for (int dx = -1; dx <= 1; dx++) {
            int64_t X = x + dx, Y = y + dy, Z = z + dz;
            if (X < 0 || Y < 0 || Z < 0 || X >= (int64_t)sx || Y >= (int64_t)sy || Z >= (int64_t)sz) continue;
            uint64_t v = (uint64_t)X + sx * ((uint64_t)Y + sy * (uint64_t)Z);
            if (stamp[v] == p + 1 || labels[v] != label[p]) continue;
            double e0 = (double)(X - c[0]) * a[0], e1 = (double)(Y - c[1]) * a[1], e2 = (double)(Z - c[2]) * a[2];
            double s = (nn[0] * e0 + nn[1] * e1) + nn[2] * e2;
            if (!(fabs(s) < h)) continue;
            stamp[v] = p + 1;
            queue[qn++] = v;
          }
    }
    *visited += qn;
    area[p] = (float)sum;
    contacts[p] = faces;
  }
  free(stamp);
  free(queue);
  return 0;
}
