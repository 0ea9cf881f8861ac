/* Serial checker of the TEASAR path loop (DESIGN.md 5f), one object at a time: for every path a fresh
 * binary-heap Dijkstra from the skeleton set S over the object's voxels (fix_branching) or the given
 * parents, the trace rule, and the invalidation boxes.  TEST INFRASTRUCTURE ONLY.  Objects are u32
 * ids 1..k of an F-order volume; the fields come from the caller. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define NONE 0xFFFFFFFFu

typedef struct { float d; uint32_t v; } hitem;

static void hpush(hitem* h, uint64_t* n, hitem it) {
  uint64_t i = (*n)++;
  while (i > 0 && h[(i - 1) / 2].d > it.d) {
    h[i] = h[(i - 1) / 2];
    i = (i - 1) / 2;
  }
  h[i] = it;
}

static hitem hpop(hitem* h, uint64_t* n) {
  hitem top = h[0], last = h[--*n];
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

typedef struct {
  const uint32_t* obj;
  uint64_t sx, sy, sz;
  const float *aniso, *dbf, *daf, *pdrf;
  const uint32_t* parents;
  float scale, cnst;
  uint32_t* nxt;    /* NONE outside S */
  uint8_t* valid;
  float* D;
  hitem* heap;
  int64_t lo[3], hi[3];  /* the object's bounding box, inclusive */
  uint64_t bad;     /* 1 + the voxel without a next voxel */
} loop;

/* neighbour k (raster order, dx fastest) of q, or -1 off the volume or off q's object */
static int64_t nbr(const loop* L, uint64_t q, int k) {
  int kk = k < 13 ? k : k + 1;
  int64_t dx = kk % 3 - 1, dy = (kk / 3) % 3 - 1, dz = kk / 9 - 1;
  int64_t x = q % L->sx + dx, y = (q / L->sx) % L->sy + dy, z = q / (L->sx * L->sy) + dz;
  if (x < 0 || y < 0 || z < 0 || x >= (int64_t)L->sx || y >= (int64_t)L->sy || z >= (int64_t)L->sz) return -1;
  uint64_t p = (uint64_t)x + L->sx * ((uint64_t)y + L->sy * (uint64_t)z);
  return L->obj[p] == L->obj[q] ? (int64_t)p : -1;
}

/* D = least cost from S over the object's voxels vox[0..nv), entering p costs pdrf[p] */
static void solve(loop* L, const uint32_t* vox, uint64_t nv) {
  uint64_t hn = 0;
  for (uint64_t i = 0; i < nv; i++) {
    L->D[vox[i]] = INFINITY;
    if (L->nxt[vox[i]] != NONE) {
      L->D[vox[i]] = 0.0f;
      hpush(L->heap, &hn, (hitem){0.0f, vox[i]});
    }
  }
  while (hn) {
    hitem it = hpop(L->heap, &hn);
    if (it.d > L->D[it.v]) continue;
    for (int k = 0; k < 26; k++) {
      int64_t q = nbr(L, it.v, k);
      if (q < 0) continue;
      float cand = it.d + L->pdrf[q];
      if (cand < L->D[q]) {
        L->D[q] = cand;
        hpush(L->heap, &hn, (hitem){cand, (uint32_t)q});
      }
    }
  }
}

/* 0 ok, 2 a path voxel without a next voxel */
static int trace(loop* L, const uint32_t* vox, uint64_t nv, uint64_t t) {
  if (!L->parents) solve(L, vox, nv);
  uint64_t q = t;
  for (;;) {
    /* invalidate the box of q */
    float r = L->scale * L->dbf[q] + L->cnst;
    const int64_t c[3] = {(int64_t)(q % L->sx), (int64_t)((q / L->sx) % L->sy), (int64_t)(q / (L->sx * L->sy))};
    int64_t b0[3], b1[3];
    for (int i = 0; i < 3; i++) {
      /* the half extent floor(r / a), clamped before the cast: the box is clipped to the object anyway */
      float hf = floorf(r / L->aniso[i]);
      int64_t h = hf > (float)(L->hi[i] - L->lo[i] + 1) ? L->hi[i] - L->lo[i] + 1 : (int64_t)hf;
      b0[i] = c[i] - h > L->lo[i] ? c[i] - h : L->lo[i];
      b1[i] = c[i] + h < L->hi[i] ? c[i] + h : L->hi[i];
    }
    for (int64_t pz = b0[2]; pz <= b1[2]; pz++) {
      for (int64_t py = b0[1]; py <= b1[1]; py++) {
        for (int64_t px = b0[0]; px <= b1[0]; px++) {
          uint64_t p = (uint64_t)px + L->sx * ((uint64_t)py + L->sy * (uint64_t)pz);
          if (L->obj[p] == L->obj[q]) L->valid[p] = 0;
        }
      }
    }
    if (L->nxt[q] != NONE) return 0;
    int64_t p = -1;
    if (L->parents) {
      if (L->parents[q]) p = (int64_t)L->parents[q] - 1;
    } else {
      for (int k = 0; k < 26 && p < 0; k++) {
        int64_t c = nbr(L, q, k);
        if (c < 0) continue;
        float dp = L->D[c], dq = L->D[q];
        if (dp + L->pdrf[q] == dq && (dp < dq || (dp == dq && (uint64_t)c < q))) p = c;
      }
    }
    if (p < 0) {
      L->bad = q + 1;
      return 2;
    }
    L->nxt[q] = (uint32_t)p;
    q = (uint64_t)p;
  }
}

/* 0 ok; 1 allocation failed; 2 a path voxel without a next voxel (*bad = its index + 1); 3 a root off its
 * object.  parents == NULL: fix_branching.  nxt_out: n entries, NONE outside the skeleton, the voxel
 * itself at a root. */
int orc_teasar(const uint32_t* obj, uint64_t sx, uint64_t sy, uint64_t sz, uint64_t k, const float* aniso,
               const float* dbf, const float* daf, const float* pdrf, const uint32_t* parents, const uint64_t* roots,
               const uint64_t* before, uint64_t nb, const uint64_t* after, uint64_t na, float scale, float cnst,
               uint64_t max_paths, uint32_t* nxt_out, uint64_t* bad) {
  const uint64_t n = sx * sy * sz;
  loop L = {obj, sx, sy, sz, aniso, dbf, daf, pdrf, parents, scale, cnst, nxt_out, NULL, NULL, NULL, {0}, {0}, 0};
  uint64_t* start = (uint64_t*)calloc(k + 2, sizeof(uint64_t));
  uint32_t* vox = (uint32_t*)malloc(sizeof(uint32_t) * (n ? n : 1));
  L.valid = (uint8_t*)calloc(n ? n : 1, 1);
  L.D = (float*)malloc(sizeof(float) * (n ? n : 1));
  int rc = 0;
  if (!start || !vox || !L.valid || !L.D) {
    rc = 1;
    goto done;
  }
  for (uint64_t i = 0; i < n; i++) nxt_out[i] = NONE;
  /* each object's voxels in ascending index: vox[start[o] .. start[o + 1]) */
  for (uint64_t i = 0; i < n; i++) start[obj[i] + 1]++;
  for (uint64_t o = 1; o <= k + 1; o++) start[o] += start[o - 1];
  {
    /* a solve pushes the sources and at most once per edge into a voxel */
    uint64_t most = 0;
    for (uint64_t o = 1; o <= k; o++)
      if (start[o + 1] - start[o] > most) most = start[o + 1] - start[o];
    L.heap = (hitem*)malloc(sizeof(hitem) * (27 * most + 1));
    if (!L.heap) {
      rc = 1;
      goto done;
    }
  }
  {
    uint64_t* fill = (uint64_t*)malloc(sizeof(uint64_t) * (k + 1));
    if (!fill) {
      rc = 1;
      goto done;
    }
    memcpy(fill, start, sizeof(uint64_t) * (k + 1));
    for (uint64_t i = 0; i < n; i++) vox[fill[obj[i]]++] = (uint32_t)i;
    free(fill);
  }
  for (uint64_t o = 1; o <= k && !rc; o++) {
    const uint32_t* ov = vox + start[o];
    const uint64_t nv = start[o + 1] - start[o];
    const uint64_t r = roots[o];
    if (r >= n || obj[r] != o) {
      rc = 3;
      break;
    }
    for (int i = 0; i < 3; i++) L.lo[i] = INT64_MAX, L.hi[i] = -1;
    for (uint64_t i = 0; i < nv; i++) {
      const int64_t c[3] = {(int64_t)(ov[i] % sx), (int64_t)((ov[i] / sx) % sy), (int64_t)(ov[i] / (sx * sy))};
      for (int j = 0; j < 3; j++) {
        if (c[j] < L.lo[j]) L.lo[j] = c[j];
        if (c[j] > L.hi[j]) L.hi[j] = c[j];
      }
      L.valid[ov[i]] = 1;
    }
    nxt_out[r] = (uint32_t)r;
    int64_t last = -1;
    for (uint64_t i = 0; i < nb; i++)
      if (before[i] < n && obj[before[i]] == o) last = (int64_t)i;
    for (int64_t i = 0; i < last && !rc; i++)
      if (before[i] < n && obj[before[i]] == o) rc = trace(&L, ov, nv, before[i]);
    for (uint64_t paths = 0; paths < max_paths && !rc; paths++) {
      int64_t best = -1;
      for (uint64_t i = 0; i < nv; i++)
        if (L.valid[ov[i]] && (best < 0 || daf[ov[i]] > daf[best])) best = ov[i];
      if (best < 0) break;
      rc = trace(&L, ov, nv, (uint64_t)best);
    }
    for (uint64_t i = 0; i < na && !rc; i++)
      if (after[i] < n && obj[after[i]] == o) rc = trace(&L, ov, nv, after[i]);
  }
done:
  if (bad) *bad = L.bad;
  free(start);
  free(vox);
  free(L.valid);
  free(L.D);
  free(L.heap);
  return rc;
}
