/* TEST INFRASTRUCTURE ONLY — CPU restatement ("port") of the reference LIO hot path.
 *
 * Nothing in the product (lidar-slam-detection_b200/, liblsdreg.so) may include, link or call this
 * file.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs
 * use it, as the checker.  All citations are relative to /root/reference.
 *
 * Pinning status (DESIGN.md "Oracle"):
 *   - iVox k-NN, ikd-Tree k-NN, esti_plane: pinned against the compiled reference (oracle/_ref,
 *     tests/test_oracle_vs_ref.py) and the golden vectors it generated (tests/golden/).
 *   - PCL VoxelGrid: PCL 1.9.1 is not vendored in the reference tree -> restated from the
 *     published algorithm (pcl/filters/impl/voxel_grid.hpp, PCL 1.9.1); PARITY UNPINNED.
 *
 * Build: oracle/Makefile (gcc -O3 -ffp-contract=off, no -march=native: fp32 distance arithmetic
 * is evaluated left-to-right without FMA exactly like the reference x86-64 build).
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <omp.h>

/* ===================================================================================== */
/* a1  pcl::VoxelGrid<PointXYZINormal>::filter — call site laserMapping.cpp:1206-1207,   */
/*     leaf 0.5 (laserMapping.cpp:1027,1073).  Semantics (PCL 1.9.1 voxel_grid.hpp):     */
/*     bbox -> min_b = floor(min*inv_leaf); idx = (ijk-min_b).(1,dx,dx*dy); sort by idx;  */
/*     per-run centroid of all fields (fp32 sums in input order); output ascending idx.   */
/* ===================================================================================== */
typedef struct { int idx; int pi; } OrcVoxKey;

static int cmp_voxkey(const void* a, const void* b) {
  const OrcVoxKey* x = (const OrcVoxKey*)a; const OrcVoxKey* y = (const OrcVoxKey*)b;
  if (x->idx != y->idx) return x->idx < y->idx ? -1 : 1;
  return x->pi < y->pi ? -1 : (x->pi > y->pi);  /* stable: input order inside a voxel */
}

/* in/out: [n,4] = x,y,z,intensity.  Returns the number of output points, or -1 when the grid
 * would overflow int32 (PCL then warns and returns the input unchanged: out = in, caller uses n). */
int orc_voxelgrid(const float* in, int n, float leaf, float* out, int* out_vidx) {
  if (n <= 0) return 0;
  float inv = 1.0f / leaf;
  float mn[3] = {in[0], in[1], in[2]}, mx[3] = {in[0], in[1], in[2]};
  for (int i = 1; i < n; i++)
    for (int d = 0; d < 3; d++) {
      float v = in[4 * i + d];
      if (v < mn[d]) mn[d] = v;
      if (v > mx[d]) mx[d] = v;
    }
  int64_t dx = (int64_t)((mx[0] - mn[0]) * inv) + 1;
  int64_t dy = (int64_t)((mx[1] - mn[1]) * inv) + 1;
  int64_t dz = (int64_t)((mx[2] - mn[2]) * inv) + 1;
  if (dx * dy * dz > (int64_t)INT32_MAX) {
    memcpy(out, in, sizeof(float) * 4 * (size_t)n);
    return -1;
  }
  int minb[3], maxb[3], divb[3];
  for (int d = 0; d < 3; d++) {
    minb[d] = (int)floorf(mn[d] * inv);
    maxb[d] = (int)floorf(mx[d] * inv);
    divb[d] = maxb[d] - minb[d] + 1;
  }
  int mul[3] = {1, divb[0], divb[0] * divb[1]};
  OrcVoxKey* keys = (OrcVoxKey*)malloc(sizeof(OrcVoxKey) * (size_t)n);
  for (int i = 0; i < n; i++) {
    int i0 = (int)(floorf(in[4 * i + 0] * inv) - (float)minb[0]);
    int i1 = (int)(floorf(in[4 * i + 1] * inv) - (float)minb[1]);
    int i2 = (int)(floorf(in[4 * i + 2] * inv) - (float)minb[2]);
    keys[i].idx = i0 * mul[0] + i1 * mul[1] + i2 * mul[2];
    keys[i].pi = i;
  }
  qsort(keys, (size_t)n, sizeof(OrcVoxKey), cmp_voxkey);
  int m = 0;
  for (int s = 0; s < n;) {
    int e = s;
    float acc[4] = {0, 0, 0, 0};
    while (e < n && keys[e].idx == keys[s].idx) {
      const float* p = in + 4 * (size_t)keys[e].pi;
      acc[0] += p[0]; acc[1] += p[1]; acc[2] += p[2]; acc[3] += p[3];
      e++;
    }
    float cnt = (float)(e - s);
    for (int d = 0; d < 4; d++) out[4 * (size_t)m + d] = acc[d] / cnt;
    if (out_vidx) out_vidx[m] = keys[s].idx;
    m++;
    s = e;
  }
  free(keys);
  return m;
}

/* ===================================================================================== */
/* a2/a3  faster_lio::IVox  (include/ivox3d/ivox3d.h:31-261, ivox3d_node.hpp:38-127)      */
/* ===================================================================================== */
typedef struct { float x, y, z; int id; } OrcPt;
typedef struct { int kx, ky, kz; int used; int n, cap; OrcPt* pts; } OrcCell;
typedef struct {
  float res, inv_res;
  int nearby_n; int nearby[125][3];
  size_t tab_size, n_cells, n_points; OrcCell* tab;
} OrcIvox;

static uint64_t cell_hash(int x, int y, int z) {
  uint64_t h = (uint64_t)(uint32_t)x * 0x9E3779B97F4A7C15ull;
  h ^= ((uint64_t)(uint32_t)y + 0x7F4A7C15ull) * 0xC2B2AE3D27D4EB4Full;
  h ^= ((uint64_t)(uint32_t)z + 0x165667B1ull) * 0xD6E8FEB86659FD93ull;
  h ^= h >> 29; h *= 0xBF58476D1CE4E5B9ull; h ^= h >> 32;
  return h;
}

/* GenerateNearbyGrids, ivox3d.h:178-215 */
static void set_nearby(OrcIvox* m, int nearby) {
  static const int n18[19][3] = {{0,0,0},{-1,0,0},{1,0,0},{0,1,0},{0,-1,0},{0,0,-1},{0,0,1},{1,1,0},{-1,1,0},
    {1,-1,0},{-1,-1,0},{1,0,1},{-1,0,1},{1,0,-1},{-1,0,-1},{0,1,1},{0,-1,1},{0,1,-1},{0,-1,-1}};
  m->nearby_n = 0;
  if (nearby == 0) { m->nearby_n = 1; memset(m->nearby[0], 0, sizeof(int) * 3); }
  else if (nearby == 6 || nearby == 18) {
    int c = nearby == 6 ? 7 : 19;
    for (int i = 0; i < c; i++) memcpy(m->nearby[i], n18[i], sizeof(int) * 3);
    m->nearby_n = c;
  } else if (nearby == 26) { /* ivox3d.h:191-198: the NEARBY18 list (in its order), then the eight corners in this order */
    static const int corners[8][3] = {{1, 1, 1}, {-1, 1, 1}, {1, -1, 1}, {1, 1, -1}, {-1, -1, 1}, {-1, 1, -1}, {1, -1, -1}, {-1, -1, -1}};
    for (int i = 0; i < 19; i++) memcpy(m->nearby[i], n18[i], sizeof(int) * 3);
    for (int i = 0; i < 8; i++) memcpy(m->nearby[19 + i], corners[i], sizeof(int) * 3);
    m->nearby_n = 27;
  } else { /* NEARBY74: 5x5x3, ivox3d.h:205-211 */
    for (int i = -2; i <= 2; i++) for (int j = -2; j <= 2; j++) for (int k = -1; k <= 1; k++) {
      int* d = m->nearby[m->nearby_n++]; d[0] = i; d[1] = j; d[2] = k; }
  }
}

OrcIvox* orc_ivox_create(float res, int nearby, size_t expected_cells) {
  OrcIvox* m = (OrcIvox*)calloc(1, sizeof(OrcIvox));
  m->res = res;
  m->inv_res = (float)(1.0 / (double)res); /* ivox3d.h:58 */
  set_nearby(m, nearby);
  size_t t = 1024;
  while (t < expected_cells * 2) t <<= 1;
  m->tab_size = t;
  m->tab = (OrcCell*)calloc(t, sizeof(OrcCell));
  return m;
}
void orc_ivox_set_nearby(OrcIvox* m, int nearby) { set_nearby(m, nearby); }
void orc_ivox_destroy(OrcIvox* m) {
  if (!m) return;
  for (size_t i = 0; i < m->tab_size; i++) free(m->tab[i].pts);
  free(m->tab); free(m);
}
size_t orc_ivox_num_cells(const OrcIvox* m) { return m->n_cells; }
size_t orc_ivox_num_points(const OrcIvox* m) { return m->n_points; }

static OrcCell* find_cell(const OrcIvox* m, int x, int y, int z) {
  size_t mask = m->tab_size - 1, s = cell_hash(x, y, z) & mask;
  for (;;) {
    OrcCell* c = &m->tab[s];
    if (!c->used) return NULL;
    if (c->kx == x && c->ky == y && c->kz == z) return c;
    s = (s + 1) & mask;
  }
}
static void grow(OrcIvox* m);
static OrcCell* find_or_add_cell(OrcIvox* m, int x, int y, int z) {
  if ((m->n_cells + 1) * 2 > m->tab_size) grow(m);
  size_t mask = m->tab_size - 1, s = cell_hash(x, y, z) & mask;
  for (;;) {
    OrcCell* c = &m->tab[s];
    if (!c->used) { c->used = 1; c->kx = x; c->ky = y; c->kz = z; m->n_cells++; return c; }
    if (c->kx == x && c->ky == y && c->kz == z) return c;
    s = (s + 1) & mask;
  }
}
static void grow(OrcIvox* m) {
  OrcCell* old = m->tab; size_t on = m->tab_size;
  m->tab_size = on * 2; m->tab = (OrcCell*)calloc(m->tab_size, sizeof(OrcCell));
  size_t mask = m->tab_size - 1;
  for (size_t i = 0; i < on; i++) if (old[i].used) {
    size_t s = cell_hash(old[i].kx, old[i].ky, old[i].kz) & mask;
    while (m->tab[s].used) s = (s + 1) & mask;
    m->tab[s] = old[i];
  }
  free(old);
}

/* Pos2Grid, ivox3d.h:258-261: round(pt * inv_res) with round-half-away-from-zero */
static inline void pos2grid(const OrcIvox* m, const float* p, int* k) {
  k[0] = (int)roundf(p[0] * m->inv_res);
  k[1] = (int)roundf(p[1] * m->inv_res);
  k[2] = (int)roundf(p[2] * m->inv_res);
}

/* AddPoints, ivox3d.h:231-256 (LRU eviction not restated: capacity is raised above the map size,
 * BASELINE.md §3 config 2).  Point i gets id ids ? ids[i] : id0 + i. */
void orc_ivox_add(OrcIvox* m, const float* xyz, int stride, int n, int id0, const int* ids) {
  for (int i = 0; i < n; i++) {
    const float* p = xyz + (size_t)stride * i;
    int k[3]; pos2grid(m, p, k);
    OrcCell* c = find_or_add_cell(m, k[0], k[1], k[2]);
    if (c->n == c->cap) { c->cap = c->cap ? c->cap * 2 : 4; c->pts = (OrcPt*)realloc(c->pts, sizeof(OrcPt) * (size_t)c->cap); }
    OrcPt* q = &c->pts[c->n++];
    q->x = p[0]; q->y = p[1]; q->z = p[2]; q->id = ids ? ids[i] : id0 + i;
    m->n_points++;
  }
}

typedef struct { float d2; int id; float x, y, z; } OrcCand;
/* canonical order used everywhere in this repo: ascending (d2, id) */
/* KD_TREE::Delete_Point_Boxes (ikd_Tree.cpp:536-556, Delete_by_range :648-672): a point is deleted iff
 * min <= p < max on every axis, for any of the boxes.  boxes: [n_boxes, 6] = (min xyz, max xyz).  Returns #deleted. */
size_t orc_ivox_delete_boxes(OrcIvox* m, const float* boxes, int n_boxes) {
  size_t del = 0;
  for (size_t s = 0; s < m->tab_size; s++) {
    OrcCell* c = &m->tab[s];
    if (!c->used) continue;
    int w = 0;
    for (int j = 0; j < c->n; j++) {
      const OrcPt* p = &c->pts[j];
      int inside = 0;
      for (int b = 0; b < n_boxes && !inside; b++) {
        const float* B = boxes + 6 * b;
        inside = B[0] <= p->x && B[3] > p->x && B[1] <= p->y && B[4] > p->y && B[2] <= p->z && B[5] > p->z;
      }
      if (inside) del++; else c->pts[w++] = *p;
    }
    c->n = w;
  }
  m->n_points -= del;
  return del;
}

static inline int cand_less(const OrcCand* a, const OrcCand* b) {
  return a->d2 < b->d2 || (a->d2 == b->d2 && a->id < b->id);
}
static inline void topk_insert(OrcCand* best, int* nb, int k, const OrcCand* c) {
  if (*nb == k && !cand_less(c, &best[k - 1])) return;
  int j = *nb < k ? (*nb)++ : k - 1;
  while (j > 0 && cand_less(c, &best[j - 1])) { best[j] = best[j - 1]; j--; }
  best[j] = *c;
}
/* distance2, ivox3d_node.hpp:11-14: (dx*dx + dy*dy) + dz*dz in fp32 */
static inline float dist2f(const float* a, const OrcPt* b) {
  float dx = b->x - a[0], dy = b->y - a[1], dz = b->z - a[2];
  return dx * dx + dy * dy + dz * dz;
}

/* GetClosestPoint(pt, out, k, max_sq), ivox3d.h:139-171 + KNNPointByCondition,
 * ivox3d_node.hpp:107-127.  The reference keeps per-cell top-k then the global top-k; the union of
 * per-cell top-k contains the global top-k, so this is the k smallest with d2 < max_sq in the
 * stencil.  Returned in canonical (d2,id) order; the reference's order is "nearest first, rest
 * unspecified (nth_element)". */
static int ivox_knn_one(const OrcIvox* m, const float* q, int k, double max_sq, OrcCand* best) {
  int key[3]; pos2grid(m, q, key);
  int nb = 0;
  for (int c = 0; c < m->nearby_n; c++) {
    const OrcCell* cell = find_cell(m, key[0] + m->nearby[c][0], key[1] + m->nearby[c][1], key[2] + m->nearby[c][2]);
    if (!cell) continue;
    for (int j = 0; j < cell->n; j++) {
      float d = dist2f(q, &cell->pts[j]);
      if ((double)d < max_sq) {
        OrcCand cd = {d, cell->pts[j].id, cell->pts[j].x, cell->pts[j].y, cell->pts[j].z};
        topk_insert(best, &nb, k, &cd);
      }
    }
  }
  return nb;
}

/* ---- the reference's neighbour ORDER -------------------------------------------------------------------------------
 * GetClosestPoint hands its candidates to std::nth_element twice (ivox3d.h:159-164) and KNNPointByCondition once per voxel
 * with more than K points in range (ivox3d_node.hpp:118-123); the five neighbours reach esti_plane in the order libstdc++'s
 * introselect leaves them in (bits/stl_algo.h: __introselect, __unguarded_partition_pivot, __move_median_to_first,
 * __unguarded_partition, __insertion_sort, __heap_select), and esti_plane's fp32 solve depends on the row order.  What
 * follows restates that algorithm (comparison: DistPoint::operator<, the distance alone) on the candidate sequence the
 * reference builds: nearby_grids_ order, then the voxel's points_ order (= insertion order). */
static inline int ref_less(const OrcCand* a, const OrcCand* b) { return a->d2 < b->d2; }
static inline void ref_swap(OrcCand* a, OrcCand* b) { OrcCand t = *a; *a = *b; *b = t; }
static void ref_adjust_heap(OrcCand* first, long hole, long len, OrcCand value) {   /* std::__adjust_heap + __push_heap */
  const long top = hole;
  long child = hole;
  while (child < (len - 1) / 2) {
    child = 2 * (child + 1);
    if (ref_less(first + child, first + (child - 1))) child--;
    first[hole] = first[child];
    hole = child;
  }
  if ((len & 1) == 0 && child == (len - 2) / 2) {
    child = 2 * (child + 1);
    first[hole] = first[child - 1];
    hole = child - 1;
  }
  long parent = (hole - 1) / 2;
  while (hole > top && ref_less(first + parent, &value)) {
    first[hole] = first[parent];
    hole = parent;
    parent = (hole - 1) / 2;
  }
  first[hole] = value;
}
static long orc_heap_select_calls = 0;   /* how often introselect's depth limit was hit (tests make sure it is) */
long orc_heap_select_count(void) { return orc_heap_select_calls; }
static void ref_heap_select(OrcCand* first, OrcCand* middle, OrcCand* last) {       /* std::__heap_select */
  orc_heap_select_calls++;
  const long len = middle - first;
  if (len >= 2)
    for (long parent = (len - 2) / 2;; parent--) {                                  /* std::__make_heap */
      OrcCand v = first[parent];
      ref_adjust_heap(first, parent, len, v);
      if (parent == 0) break;
    }
  for (OrcCand* i = middle; i < last; i++)
    if (ref_less(i, first)) {                                                        /* std::__pop_heap(first, middle, i) */
      OrcCand v = *i;
      *i = *first;
      ref_adjust_heap(first, 0, len, v);
    }
}
static void ref_nth_element(OrcCand* first, OrcCand* nth, OrcCand* last) {          /* std::nth_element */
  if (first == last || nth == last) return;
  long depth = 0;
  for (long n = last - first; n > 1; n >>= 1) depth++;                              /* std::__lg */
  depth *= 2;
  while (last - first > 3) {
    if (depth == 0) {
      ref_heap_select(first, nth + 1, last);
      ref_swap(first, nth);
      return;
    }
    depth--;
    OrcCand* mid = first + (last - first) / 2;
    OrcCand *a = first + 1, *b = mid, *c = last - 1;                                /* __move_median_to_first(first, a, b, c) */
    if (ref_less(a, b)) {
      if (ref_less(b, c)) ref_swap(first, b);
      else if (ref_less(a, c)) ref_swap(first, c);
      else ref_swap(first, a);
    } else if (ref_less(a, c)) ref_swap(first, a);
    else if (ref_less(b, c)) ref_swap(first, c);
    else ref_swap(first, b);
    OrcCand *lo = first + 1, *hi = last;                                             /* __unguarded_partition(first + 1, last, first) */
    for (;;) {
      while (ref_less(lo, first)) lo++;
      hi--;
      while (ref_less(first, hi)) hi--;
      if (!(lo < hi)) break;
      ref_swap(lo, hi);
      lo++;
    }
    if (lo <= nth) first = lo; else last = lo;
  }
  for (OrcCand* i = first + 1; i < last; i++) {                                      /* __insertion_sort */
    OrcCand v = *i;
    if (ref_less(&v, first)) {
      for (OrcCand* j = i; j > first; j--) *j = *(j - 1);
      *first = v;
    } else {
      OrcCand* j = i;
      while (ref_less(&v, j - 1)) { *j = *(j - 1); j--; }
      *j = v;
    }
  }
}
/* the restated nth_element on its own (tests pin it against std::nth_element on the reference's DistPoint, oracle/ref_lio.cpp) */
void orc_nth_element(const float* dist, int* idx_inout, int n, int first, int nth, int last) {
  OrcCand* c = (OrcCand*)malloc(sizeof(OrcCand) * (size_t)(n > 0 ? n : 1));
  for (int i = 0; i < n; i++) { c[i].d2 = dist[idx_inout[i]]; c[i].id = idx_inout[i]; c[i].x = c[i].y = c[i].z = 0.f; }
  ref_nth_element(c + first, c + nth, c + last);
  for (int i = 0; i < n; i++) idx_inout[i] = c[i].id;
  free(c);
}
#define ORC_REF_CAND_MAX 4096
/* GetClosestPoint exactly as the reference runs it, order included; `best` receives min(n, k) candidates in the reference's order */
static int ivox_knn_one_ref(const OrcIvox* m, const float* q, int k, double max_sq, OrcCand* best) {
  int key[3]; pos2grid(m, q, key);
  OrcCand stack_c[256];
  OrcCand* cand = stack_c;
  int cap = 256, n = 0;
  for (int c = 0; c < m->nearby_n; c++) {
    const OrcCell* cell = find_cell(m, key[0] + m->nearby[c][0], key[1] + m->nearby[c][1], key[2] + m->nearby[c][2]);
    if (!cell) continue;
    const int old = n;
    if (n + cell->n > cap) {
      const int ncap = 2 * (n + cell->n);
      OrcCand* nc = (OrcCand*)malloc(sizeof(OrcCand) * (size_t)ncap);
      memcpy(nc, cand, sizeof(OrcCand) * (size_t)n);
      if (cand != stack_c) free(cand);
      cand = nc; cap = ncap;
    }
    for (int j = 0; j < cell->n; j++) {
      const float d = dist2f(q, &cell->pts[j]);
      if ((double)d < max_sq) { OrcCand cd = {d, cell->pts[j].id, cell->pts[j].x, cell->pts[j].y, cell->pts[j].z}; cand[n++] = cd; }
    }
    if (n - old > k) { ref_nth_element(cand + old, cand + old + k - 1, cand + n); n = old + k; }
  }
  if (n > k) { ref_nth_element(cand, cand + k - 1, cand + n); n = k; }
  if (n > 0) ref_nth_element(cand, cand, cand + n);
  for (int j = 0; j < n; j++) best[j] = cand[j];
  if (cand != stack_c) free(cand);
  return n;
}

/* Exact k-NN within radius (d2 <= max_sq) by shell expansion over the same grid: equals the
 * ikd-Tree result Nearest_Search (ikd_Tree.cpp:367-397, :869-1013) whenever the reference accepts
 * it (5 found and d2[4] <= 5, laserMapping.cpp:846-847). */
static int exact_knn_one(const OrcIvox* m, const float* q, int k, double max_sq, OrcCand* best) {
  int key[3]; pos2grid(m, q, key);
  int nb = 0;
  int rmax = (int)ceil(sqrt(max_sq) / (double)m->res) + 1;
  for (int r = 0; r <= rmax; r++) {
    if (r >= 1 && nb == k) {
      double lo = (double)(r - 1) * (double)m->res * (1.0 - 1e-5); /* unseen points are farther than this */
      if ((double)best[k - 1].d2 < lo * lo) break;
    }
    for (int i = -r; i <= r; i++) for (int j = -r; j <= r; j++) for (int l = -r; l <= r; l++) {
      int a = abs(i) > abs(j) ? abs(i) : abs(j); if (abs(l) > a) a = abs(l);
      if (a != r) continue;
      const OrcCell* cell = find_cell(m, key[0] + i, key[1] + j, key[2] + l);
      if (!cell) continue;
      for (int p = 0; p < cell->n; p++) {
        float d = dist2f(q, &cell->pts[p]);
        if ((double)d <= max_sq) {
          OrcCand cd = {d, cell->pts[p].id, cell->pts[p].x, cell->pts[p].y, cell->pts[p].z};
          topk_insert(best, &nb, k, &cd);
        }
      }
    }
  }
  return nb;
}

/* mode 0: iVox stencil (d2 < max_sq), canonical (d2, id) order; mode 2: the same neighbours in the reference's own order;
 * mode 1: exact within radius (d2 <= max_sq).
 * q stride in floats; outputs [nq,k] (-1 / 0 padded), out_xyz [nq,k,3] optional. */
void orc_knn(const OrcIvox* m, int mode, const float* q, int stride, int nq, int k, double max_sq,
             int* out_ids, float* out_d2, float* out_xyz, int* out_cnt, int nthreads) {
  omp_set_num_threads(nthreads > 0 ? nthreads : 1);
#pragma omp parallel for schedule(dynamic, 256)
  for (int i = 0; i < nq; i++) {
    OrcCand best[64];
    int kk = k > 64 ? 64 : k;
    int nb = mode == 0 ? ivox_knn_one(m, q + (size_t)stride * i, kk, max_sq, best)
             : mode == 2 ? ivox_knn_one_ref(m, q + (size_t)stride * i, kk, max_sq, best)     /* the reference's order */
                         : exact_knn_one(m, q + (size_t)stride * i, kk, max_sq, best);
    out_cnt[i] = nb;
    for (int j = 0; j < k; j++) {
      out_ids[(size_t)i * k + j] = j < nb ? best[j].id : -1;
      out_d2[(size_t)i * k + j] = j < nb ? best[j].d2 : -1.f;
      if (out_xyz) {
        float* o = out_xyz + ((size_t)i * k + j) * 3;
        o[0] = j < nb ? best[j].x : 0; o[1] = j < nb ? best[j].y : 0; o[2] = j < nb ? best[j].z : 0;
      }
    }
  }
}

/* ===================================================================================== */
/* a5  esti_plane<float>  (include/common_lib.h:236-268): 5x3 A n = -1 solved with Eigen's */
/*     ColPivHouseholderQR in fp32 (Eigen/src/QR/ColPivHouseholderQR.h:480-570,            */
/*     Householder/Householder.h:65-130), normalise, reject if any point is > thr off.     */
/* ===================================================================================== */
#define FEPS 1.1920929e-07f
/* Eigen's reductions as the reference's x86-64 (SSE2, 4-float packets, no FMA) build orders them — the reference's plane
 * coefficients are defined by that order (DESIGN.md section 4):
 *   fixed size 5 (a whole column; Core/Redux.h, LinearVectorizedTraversal + CompleteUnrolling): one packet of the first four
 *     terms reduced as (t0 + t2) + (t1 + t3) (arch/SSE/PacketMath.h predux), then + t4;
 *   run-time size n (Redux.h:243-270, expression without direct access => no alignment peeling): n >= 4: first four terms as one
 *     packet, the rest added one by one; n < 4: left to right;
 *   fixed size 3 without packets (DefaultTraversal + CompleteUnrolling, redux_novec_unroller): t0 + (t1 + t2). */
static float red_dyn(const float* t, int n) {
  if (n >= 4) {
    float s = (t[0] + t[2]) + (t[1] + t[3]);
    for (int i = 4; i < n; i++) s += t[i];
    return s;
  }
  float s = t[0];
  for (int i = 1; i < n; i++) s += t[i];
  return s;
}
static float red_fix5(const float* t) { return ((t[0] + t[2]) + (t[1] + t[3])) + t[4]; }
/* A is column-major 5x3 (A[c][r]) like Eigen's m_qr */
static float sqn_tail(float A[3][5], int c, int r0) {   /* squared norm of A[r0..4][c] (run-time size) */
  float t[5]; int n = 0;
  for (int r = r0; r < 5; r++) t[n++] = A[c][r] * A[c][r];
  return n ? red_dyn(t, n) : 0.f;
}
static float dot_tail(float A[3][5], int ce, const float* v, int r0) {   /* sum_{r>=r0} A[r][ce] * v[r] (run-time size) */
  float t[5]; int n = 0;
  for (int r = r0; r < 5; r++) t[n++] = A[ce][r] * v[r];
  return n ? red_dyn(t, n) : 0.f;
}
/* the factorisation + solve of A n = b; returns nonzero pivots.  qr/hc/perm as Eigen's matrixQR() / hCoeffs() / colsPermutation() */
static int esti_qr(const float* pts, float A[3][5], float hc[3], int perm[3], float x[3]) {
  float b[5];
  for (int r = 0; r < 5; r++) { A[0][r] = pts[3 * r]; A[1][r] = pts[3 * r + 1]; A[2][r] = pts[3 * r + 2]; b[r] = -1.0f; }
  const int rows = 5, cols = 3, size = 3;
  float nu[3], nd[3];
  int trans[3];
  for (int k = 0; k < cols; k++) {
    float t[5];
    for (int r = 0; r < 5; r++) t[r] = A[k][r] * A[k][r];
    nu[k] = nd[k] = sqrtf(red_fix5(t));
  }
  float mxn = nu[0]; if (nu[1] > mxn) mxn = nu[1]; if (nu[2] > mxn) mxn = nu[2];
  const float th_helper = (mxn * FEPS) * (mxn * FEPS) / (float)rows;
  const float downdate = sqrtf(FEPS);
  int nonzero = size;
  for (int k = 0; k < size; k++) {
    int big = k; float bn = nu[k];
    for (int j = k + 1; j < cols; j++) if (nu[j] > bn) { bn = nu[j]; big = j; }
    if (nonzero == size && bn * bn < th_helper * (float)(rows - k)) nonzero = k;
    trans[k] = big;
    if (big != k) {
      for (int r = 0; r < rows; r++) { float t = A[k][r]; A[k][r] = A[big][r]; A[big][r] = t; }
      float t = nu[k]; nu[k] = nu[big]; nu[big] = t;
      t = nd[k]; nd[k] = nd[big]; nd[big] = t;
    }
    /* makeHouseholderInPlace on A[k..4][k] (Householder.h:65-100) */
    const float tail = sqn_tail(A, k, k + 1);
    const float c0 = A[k][k];
    float beta, tau;
    if (tail <= 1.17549435e-38f) { tau = 0.f; beta = c0; for (int r = k + 1; r < rows; r++) A[k][r] = 0.f; }
    else {
      beta = sqrtf(c0 * c0 + tail);
      if (c0 >= 0.f) beta = -beta;
      const float den = c0 - beta;
      for (int r = k + 1; r < rows; r++) A[k][r] = A[k][r] / den;
      tau = (beta - c0) / beta;
    }
    hc[k] = tau; A[k][k] = beta;
    /* applyHouseholderOnTheLeft to the trailing columns (Householder.h:110-135): tmp = essential^T bottom; tmp += row0;
     * row0 -= tau tmp; bottom -= (tau essential) tmp */
    if (tau != 0.f && k + 1 < rows) {
      float te[5];
      for (int r = k + 1; r < rows; r++) te[r] = tau * A[k][r];
      for (int j = k + 1; j < cols; j++) {
        float tmp = dot_tail(A, k, A[j], k + 1);
        tmp += A[j][k];
        A[j][k] -= tau * tmp;
        for (int r = k + 1; r < rows; r++) A[j][r] -= te[r] * tmp;
      }
    }
    for (int j = k + 1; j < cols; j++) {
      if (nu[j] != 0.f) {
        float t = fabsf(A[j][k]) / nu[j];
        t = (1.f + t) * (1.f - t);
        if (t < 0.f) t = 0.f;
        const float rr = nu[j] / nd[j];
        const float t2 = t * (rr * rr);
        if (t2 <= downdate) { nd[j] = sqrtf(sqn_tail(A, j, k + 1)); nu[j] = nd[j]; }
        else nu[j] *= sqrtf(t);
      }
    }
  }
  perm[0] = 0; perm[1] = 1; perm[2] = 2;   /* applyTranspositionOnTheRight(k, trans[k]) for k = 0.. */
  for (int k = 0; k < size; k++) { const int t = perm[k]; perm[k] = perm[trans[k]]; perm[trans[k]] = t; }
  /* solve (ColPivHouseholderQR.h _solve_impl): c = H_{nz-1} .. H_0 b, upper-triangular solve column by column, un-permute */
  x[0] = x[1] = x[2] = 0.f;
  if (nonzero > 0) {
    for (int k = 0; k < nonzero; k++) {
      if (hc[k] == 0.f) continue;
      float tmp = dot_tail(A, k, b, k + 1);
      tmp += b[k];
      b[k] -= hc[k] * tmp;
      for (int r = k + 1; r < rows; r++) b[r] -= (hc[k] * A[k][r]) * tmp;
    }
    /* triangular_solve_vector<.., OnTheLeft, Upper, false, ColMajor>: from the last column up, axpy into the rows above */
    for (int i = nonzero - 1; i >= 0; i--) {
      if (b[i] != 0.f) {
        b[i] /= A[i][i];
        for (int r = 0; r < i; r++) b[r] -= b[i] * A[i][r];
      }
    }
    for (int i = 0; i < nonzero; i++) x[perm[i]] = b[i];
  }
  return nonzero;
}
void orc_esti_plane_qr(const float* pts5, int n, float* qr15, float* hc3, int* perm3, int* nzp, float* x3) {
  for (int i = 0; i < n; i++) {
    float A[3][5];
    nzp[i] = esti_qr(pts5 + 15 * (size_t)i, A, hc3 + 3 * (size_t)i, perm3 + 3 * (size_t)i, x3 + 3 * (size_t)i);
    for (int c = 0; c < 3; c++) for (int r = 0; r < 5; r++) qr15[15 * (size_t)i + 5 * c + r] = A[c][r];
  }
}
int orc_esti_plane(const float* pts, float thr, float* pabcd) {
  float A[3][5], hc[3], x[3]; int perm[3];
  esti_qr(pts, A, hc, perm, x);
  const float n = sqrtf(x[0] * x[0] + (x[1] * x[1] + x[2] * x[2]));   /* fixed size 3: t0 + (t1 + t2) */
  pabcd[0] = x[0] / n; pabcd[1] = x[1] / n; pabcd[2] = x[2] / n; pabcd[3] = (float)(1.0 / (double)n);
  for (int j = 0; j < 5; j++) {
    float v = pabcd[0] * pts[3 * j] + pabcd[1] * pts[3 * j + 1] + pabcd[2] * pts[3 * j + 2] + pabcd[3];
    if (fabs((double)v) > (double)thr) return 0;
  }
  return 1;
}
void orc_esti_plane_batch(const float* pts5, int n, float thr, float* pabcd, int* ok) {
  for (int i = 0; i < n; i++) ok[i] = orc_esti_plane(pts5 + 15 * (size_t)i, thr, pabcd + 4 * (size_t)i);
}

/* ===================================================================================== */
/* a3+a5+a6+a7+a8  h_share_model_geometric  (src/laserMapping.cpp:813-982) and the         */
/*     HTH / H^T h products the ESKF forms from it (esekfom.hpp:1782-1809).                */
/* ===================================================================================== */
static void mat3_vec(const double* R, const double* v, double* o) {
  for (int i = 0; i < 3; i++) o[i] = R[3 * i] * v[0] + R[3 * i + 1] * v[1] + R[3 * i + 2] * v[2];
}
static void mat3T_vec(const double* R, const double* v, double* o) {
  for (int i = 0; i < 3; i++) o[i] = R[i] * v[0] + R[3 + i] * v[1] + R[6 + i] * v[2];
}
/* cyclic Jacobi for a symmetric 3x3 (stands in for Eigen::SelfAdjointEigenSolver,
 * laserMapping.cpp:941-943; only |v.n| and V diag(mask) V^T are used, both sign/order free) */
static void eig3_sym(const double* Ain, double* w, double* V) {
  double A[9]; memcpy(A, Ain, sizeof(A));
  for (int i = 0; i < 9; i++) V[i] = (i % 4 == 0) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 60; sweep++) {
    double off = fabs(A[1]) + fabs(A[2]) + fabs(A[5]);
    if (off < 1e-300) break;
    for (int p = 0; p < 2; p++) for (int q = p + 1; q < 3; q++) {
      double apq = A[3 * p + q];
      if (fabs(apq) < 1e-300) continue;
      double th = (A[3 * q + q] - A[3 * p + p]) / (2.0 * apq);
      double t = (th >= 0 ? 1.0 : -1.0) / (fabs(th) + sqrt(th * th + 1.0));
      double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
      for (int k = 0; k < 3; k++) { double akp = A[3 * k + p], akq = A[3 * k + q]; A[3 * k + p] = c * akp - s * akq; A[3 * k + q] = s * akp + c * akq; }
      for (int k = 0; k < 3; k++) { double apk = A[3 * p + k], aqk = A[3 * q + k]; A[3 * p + k] = c * apk - s * aqk; A[3 * q + k] = s * apk + c * aqk; }
      for (int k = 0; k < 3; k++) { double vkp = V[3 * k + p], vkq = V[3 * k + q]; V[3 * k + p] = c * vkp - s * vkq; V[3 * k + q] = s * vkp + c * vkq; }
    }
  }
  w[0] = A[0]; w[1] = A[4]; w[2] = A[8];
}

/* One call of the measurement model.
 *   body      [n,4] downsampled scan in the lidar frame (feats_down_body)
 *   R,t       state rot (row-major 3x3), pos;  R_LI,t_LI extrinsics (offset_R_L_I, offset_T_L_I)
 *   search    ekfom_data.converge: redo the k-NN (laserMapping.cpp:842)
 *   knn_mode  0 = iVox NEARBY stencil (live path), 1 = exact (ikd-Tree path, accept d2[4] <= 5)
 * Per-scan persistent arrays (Nearest_Points, point_selected_surf): near_xyz [n,5,3],
 * near_ids [n,5], near_cnt [n], selected [n].  Outputs: world [n,4], plane [n,4] = (normal, pd2),
 * HTH [36] (the non-zero 6x6 block of the 15x15), HTh [6], res_sum, n_eff, degenerate.
 * hx_out [n,6] / h_out [n] (optional) receive the compacted Jacobian rows and -pd2.
 * Returns n_eff (0 -> ekfom_data.valid = false, "No Effective Points"). */
int orc_lio_hmodel(const OrcIvox* map, const float* body, int n, const double* R, const double* t,
                   const double* R_LI, const double* t_LI, int search, int knn_mode,
                   float* near_xyz, int* near_ids, int* near_cnt, unsigned char* selected,
                   float* world, float* plane, double* HTH, double* HTh, double* res_sum,
                   int* degenerate, int degenerate_detect_en, double* hx_out, double* h_out,
                   int nthreads) {
  omp_set_num_threads(nthreads > 0 ? nthreads : 1);
#pragma omp parallel for schedule(dynamic, 256)
  for (int i = 0; i < n; i++) {
    const float* pb = body + 4 * (size_t)i;
    double p_body[3] = {pb[0], pb[1], pb[2]}, pl[3], pw[3];
    mat3_vec(R_LI, p_body, pl);
    for (int d = 0; d < 3; d++) pl[d] += t_LI[d];
    mat3_vec(R, pl, pw);
    float* w = world + 4 * (size_t)i;
    for (int d = 0; d < 3; d++) w[d] = (float)(pw[d] + t[d]);
    w[3] = pb[3];
    if (search) {
      OrcCand best[5];
      /* knn_mode & 4: neighbours in the order the reference's GetClosestPoint leaves them in (std::nth_element) */
      int nb = (knn_mode & 1) ? exact_knn_one(map, w, 5, 5.0, best)
               : (knn_mode & 4) ? ivox_knn_one_ref(map, w, 5, 5.0, best) : ivox_knn_one(map, w, 5, 5.0, best);
      /* knn_mode & 2: the reference's stale list.  IVox::GetClosestPoint returns before clearing its output when no
       * candidate is in range (ivox3d.h:155-157), and Nearest_Points[i] is a file-scope vector that outlives the scan
       * (laserMapping.cpp:1273): such a point keeps the neighbours row i had the last time it found any. */
      if ((knn_mode & 2) && nb == 0) { selected[i] = near_cnt[i] >= 5; goto searched; }
      near_cnt[i] = nb;
      for (int j = 0; j < 5; j++) {
        near_ids[5 * (size_t)i + j] = j < nb ? best[j].id : -1;
        float* o = near_xyz + (5 * (size_t)i + j) * 3;
        o[0] = j < nb ? best[j].x : 0; o[1] = j < nb ? best[j].y : 0; o[2] = j < nb ? best[j].z : 0;
      }
      selected[i] = nb >= 5; /* laserMapping.cpp:847,850 */
    }
  searched:
    if (!selected[i]) continue;
    selected[i] = 0;
    float pabcd[4];
    if (orc_esti_plane(near_xyz + 15 * (size_t)i, 0.1f, pabcd)) {
      float pd2 = pabcd[0] * w[0] + pabcd[1] * w[1] + pabcd[2] * w[2] + pabcd[3];
      double nb2 = sqrt(p_body[0] * p_body[0] + p_body[1] * p_body[1] + p_body[2] * p_body[2]);
      float s = (float)(1 - 0.9 * fabs((double)pd2) / sqrt(nb2)); /* laserMapping.cpp:861 */
      if (s > 0.9) {
        selected[i] = 1;
        float* pl4 = plane + 4 * (size_t)i;
        pl4[0] = pabcd[0]; pl4[1] = pabcd[1]; pl4[2] = pabcd[2]; pl4[3] = pd2;
      }
    }
  }
  /* compaction + H rows (laserMapping.cpp:875-932), extrinsic_est_en = false */
  double* hx = (double*)malloc(sizeof(double) * 6 * (size_t)(n > 0 ? n : 1));
  double* hh = (double*)malloc(sizeof(double) * (size_t)(n > 0 ? n : 1));
  int ne = 0; double total = 0.0;
  for (int i = 0; i < n; i++) {
    if (!selected[i]) continue;
    const float* pb = body + 4 * (size_t)i; const float* pl4 = plane + 4 * (size_t)i;
    total += (double)fabsf(pl4[3]); /* res_last[i] = abs(pd2) */
    double pbe[3] = {pb[0], pb[1], pb[2]}, pt[3];
    mat3_vec(R_LI, pbe, pt);
    for (int d = 0; d < 3; d++) pt[d] += t_LI[d];
    double nv[3] = {pl4[0], pl4[1], pl4[2]}, C[3];
    mat3T_vec(R, nv, C); /* s.rot.conjugate() * norm_vec */
    double Ax = pt[1] * C[2] - pt[2] * C[1], Ay = pt[2] * C[0] - pt[0] * C[2], Az = pt[0] * C[1] - pt[1] * C[0];
    double* row = hx + 6 * (size_t)ne;
    row[0] = nv[0]; row[1] = nv[1]; row[2] = nv[2]; row[3] = Ax; row[4] = Ay; row[5] = Az;
    hh[ne] = -(double)pl4[3];
    ne++;
  }
  *res_sum = total; *degenerate = 0;
  memset(HTH, 0, sizeof(double) * 36); memset(HTh, 0, sizeof(double) * 6);
  if (ne < 1) { free(hx); free(hh); return 0; }
  if (degenerate_detect_en) { /* laserMapping.cpp:934-980 */
    double H3[9] = {0};
    for (int j = 0; j < ne; j++) for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) H3[3 * a + b] += hx[6 * (size_t)j + a] * hx[6 * (size_t)j + b];
    double ew[3], V[9]; eig3_sym(H3, ew, V);
    int mask[3] = {1, 1, 1}, deg = 0;
    for (int i = 0; i < 3; i++) {
      float contri = 0, strong = 0;
      for (int j = 0; j < ne; j++) {
        double r0 = hx[6 * (size_t)j], r1 = hx[6 * (size_t)j + 1], r2 = hx[6 * (size_t)j + 2];
        double nn = sqrt(r0 * r0 + r1 * r1 + r2 * r2);
        float dotp = (float)fabs((r0 / nn) * V[i] + (r1 / nn) * V[3 + i] + (r2 / nn) * V[6 + i]);
        if (dotp > 0.1736) contri += dotp;
        if (dotp > 0.7070) strong += dotp;
      }
      if (contri < 250.0 && strong < 50.0) { mask[i] = 0; deg = 1; }
    }
    if (deg) { /* mat_p = (V^T)^-1 V2 = V diag(mask) V^T ; rows n -> mat_p n */
      double P[9] = {0};
      for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) for (int i = 0; i < 3; i++) if (mask[i]) P[3 * a + b] += V[3 * a + i] * V[3 * b + i];
      for (int j = 0; j < ne; j++) {
        double* row = hx + 6 * (size_t)j; double o[3];
        mat3_vec(P, row, o); row[0] = o[0]; row[1] = o[1]; row[2] = o[2];
      }
      *degenerate = 1;
    }
  }
  for (int j = 0; j < ne; j++) {
    const double* row = hx + 6 * (size_t)j;
    for (int a = 0; a < 6; a++) { for (int b = 0; b < 6; b++) HTH[6 * a + b] += row[a] * row[b]; HTh[a] += row[a] * hh[j]; }
  }
  if (hx_out) memcpy(hx_out, hx, sizeof(double) * 6 * (size_t)ne);
  if (h_out) memcpy(h_out, hh, sizeof(double) * (size_t)ne);
  free(hx); free(hh);
  return ne;
}

/* ===================================================================================== */
/* a10  map_incremental  (src/laserMapping.cpp:523-576).  flag[i]: 0 skip, 1 PointToAdd,   */
/*      2 PointNoNeedDownsample.  Points are then added with id = id0 + i.                 */
/* ===================================================================================== */
static inline float calc_dist3(const float* a, const float* b) {
  return (a[0] - b[0]) * (a[0] - b[0]) + (a[1] - b[1]) * (a[1] - b[1]) + (a[2] - b[2]) * (a[2] - b[2]);
}
int orc_map_incremental(OrcIvox* map, const float* body, int n, const double* R, const double* t,
                        const double* R_LI, const double* t_LI, const float* near_xyz, const int* near_cnt,
                        int ekf_inited, double fsize, float* world, unsigned char* flag, int id0, int id_t2) {
  int added = 0;
  for (int i = 0; i < n; i++) {
    const float* pb = body + 4 * (size_t)i;
    double p_body[3] = {pb[0], pb[1], pb[2]}, pl[3], pw[3];
    mat3_vec(R_LI, p_body, pl);
    for (int d = 0; d < 3; d++) pl[d] += t_LI[d];
    mat3_vec(R, pl, pw);
    float* w = world + 4 * (size_t)i;
    for (int d = 0; d < 3; d++) w[d] = (float)(pw[d] + t[d]);
    w[3] = pb[3];
    int f = 1;
    if (near_cnt[i] > 0 && ekf_inited) {
      const float* nr = near_xyz + 15 * (size_t)i;
      float mid[3];
      for (int d = 0; d < 3; d++) mid[d] = (float)(floor((double)w[d] / fsize) * fsize + 0.5 * fsize);
      float dist = calc_dist3(w, mid);
      /* float subtraction, std::fabs(float), then compared against a double (laserMapping.cpp:545) */
      if ((double)fabsf(nr[0] - mid[0]) > 0.5 * fsize && (double)fabsf(nr[1] - mid[1]) > 0.5 * fsize &&
          (double)fabsf(nr[2] - mid[2]) > 0.5 * fsize) {
        f = 2;
      } else {
        for (int r = 0; r < 5; r++) {
          if (near_cnt[i] < 5) break;
          if (calc_dist3(nr + 3 * r, mid) < dist) { f = 0; break; }
        }
      }
    }
    flag[i] = (unsigned char)f;
  }
  for (int pass = 1; pass <= 2; pass++) /* PointToAdd first, then PointNoNeedDownsample */
    for (int i = 0; i < n; i++) if (flag[i] == pass) { int id = id0 + i + (pass == 2 ? id_t2 : 0); /* id_t2 = n: ids grow in insertion order */ orc_ivox_add(map, world + 4 * (size_t)i, 4, 1, 0, &id); added++; }
  return added;
}

/* ===================================================================================== */
/* a15  NDT (P2D, DIRECT1/7/27) — restated from the reference's CUDA functors, which are   */
/*      __host__ __device__ arithmetic over a hash of Gaussian voxels:                     */
/*        slam/thirdparty/fast_gicp/src/fast_gicp/cuda/gaussian_voxelmap.cu:76-202         */
/*        .../covariance_regularization.cu:15-52,105-116 (PLANE: V diag(1e-3,1,1) V^-1)    */
/*        .../find_voxel_correspondences.cu:16-111, ndt_compute_derivatives.cu:15-102      */
/*        include/fast_gicp/cuda/vector3_hash.cuh:35-38 (coord = floor(x/res - 0.5))       */
/*      Pin status: the reference NDT exists only as CUDA (thrust) code; it recompiles for  */
/*      sm_90a (oracle/ref_cuda.cu) and pins this restatement on the GPU box               */
/*      (tests/test_gpu_ref_cuda.py), within the bounds its lossy voxel table allows.       */
/*      fp32 per-element arithmetic as the reference; sums are carried in double (the      */
/*      reference reduces fp32 tuples in thrust's unspecified tree order).                 */
/*      PLANE-regularised covariance: V diag(1e-3,1,1) V^T  =>  C^-1 = I + 999 n n^T with  */
/*      n the eigenvector of the smallest eigenvalue; used in that closed form.            */
/* ===================================================================================== */
typedef struct { int kx, ky, kz, used, n; double sum[3], sxx[9]; float mean[3], nrm[3]; } OrcNdtVox;
typedef struct { float res; size_t tab_size, n_vox; OrcNdtVox* tab; } OrcNdt;

static inline void ndt_coord(const float* p, float res, int* c) {
  c[0] = (int)floorf(p[0] / res - 0.5f); c[1] = (int)floorf(p[1] / res - 0.5f); c[2] = (int)floorf(p[2] / res - 0.5f);
}
static OrcNdtVox* ndt_find(const OrcNdt* m, int x, int y, int z) {
  size_t mask = m->tab_size - 1, s = cell_hash(x, y, z) & mask;
  for (;;) {
    OrcNdtVox* v = &m->tab[s];
    if (!v->used) return NULL;
    if (v->kx == x && v->ky == y && v->kz == z) return v;
    s = (s + 1) & mask;
  }
}
OrcNdt* orc_ndt_build(const float* pts, int stride, int n, float res) {
  OrcNdt* m = (OrcNdt*)calloc(1, sizeof(OrcNdt));
  m->res = res;
  size_t t = 1024; while (t < (size_t)n * 2) t <<= 1;
  m->tab_size = t; m->tab = (OrcNdtVox*)calloc(t, sizeof(OrcNdtVox));
  size_t mask = t - 1;
  for (int i = 0; i < n; i++) {
    const float* p = pts + (size_t)stride * i;
    int c[3]; ndt_coord(p, res, c);
    size_t s = cell_hash(c[0], c[1], c[2]) & mask;
    OrcNdtVox* v;
    for (;;) { v = &m->tab[s]; if (!v->used) { v->used = 1; v->kx = c[0]; v->ky = c[1]; v->kz = c[2]; m->n_vox++; break; }
               if (v->kx == c[0] && v->ky == c[1] && v->kz == c[2]) break; s = (s + 1) & mask; }
    v->n++;
    for (int a = 0; a < 3; a++) { v->sum[a] += (double)p[a]; for (int b = 0; b < 3; b++) v->sxx[3 * a + b] += (double)p[a] * (double)p[b]; }
  }
  for (size_t s = 0; s < t; s++) {
    OrcNdtVox* v = &m->tab[s];
    if (!v->used) continue;
    /* The reference accumulates these moments in fp32 with atomicAdd in arbitrary thread order
     * (gaussian_voxelmap.cu:138-147): its own result scatters run to run by the fp32 cancellation
     * error of sum(xx^T) - mean sum^T.  Both restatements (this one and the CUDA path) carry the
     * moments in double, the value that scatter is centred on. */
    double cov[9], mean[3];
    for (int a = 0; a < 3; a++) { mean[a] = v->sum[a] / (double)v->n; v->mean[a] = (float)mean[a]; }
    for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) cov[3 * a + b] = (v->sxx[3 * a + b] - mean[a] * v->sum[b]) / (double)v->n;
    double A[9], w[3], V[9];
    for (int k = 0; k < 9; k++) A[k] = cov[k];
    for (int a = 0; a < 3; a++) for (int b = a + 1; b < 3; b++) A[3 * a + b] = A[3 * b + a] = 0.5 * (A[3 * a + b] + A[3 * b + a]);
    eig3_sym(A, w, V);
    int k0 = 0; if (w[1] < w[k0]) k0 = 1; if (w[2] < w[k0]) k0 = 2;
    for (int a = 0; a < 3; a++) v->nrm[a] = (float)V[3 * a + k0];
  }
  return m;
}
void orc_ndt_destroy(OrcNdt* m) { if (m) { free(m->tab); free(m); } }
size_t orc_ndt_num_voxels(const OrcNdt* m) { return m->n_vox; }

static const int ndt_off7[7][3] = {{0,0,0},{1,0,0},{-1,0,0},{0,1,0},{0,-1,0},{0,0,1},{0,0,-1}};
/* linearize at T_lin (row-major 4x4 double), evaluate at T_eval.  H36/b6 may be NULL.  n_off in {1,7,27}. */
double orc_ndt_cost(const OrcNdt* m, const float* src, int stride, int n, const double* T_lin, const double* T_eval,
                    int n_off, double* H36, double* b6, int* n_corr) {
  float Rl[9], tl[3], R[9], t[3];
  for (int a = 0; a < 3; a++) { for (int b = 0; b < 3; b++) { Rl[3 * a + b] = (float)T_lin[4 * a + b]; R[3 * a + b] = (float)T_eval[4 * a + b]; } tl[a] = (float)T_lin[4 * a + 3]; t[a] = (float)T_eval[4 * a + 3]; }
  double H[36] = {0}, b[6] = {0}, err = 0; int nc = 0;
  const float k_sq = m->res * m->res;
  for (int i = 0; i < n; i++) {
    const float* a = src + (size_t)stride * i;
    float pl[3], tA[3];
    for (int r = 0; r < 3; r++) { pl[r] = Rl[3 * r] * a[0] + Rl[3 * r + 1] * a[1] + Rl[3 * r + 2] * a[2] + tl[r];
                                  tA[r] = R[3 * r] * a[0] + R[3 * r + 1] * a[1] + R[3 * r + 2] * a[2] + t[r]; }
    int c[3]; ndt_coord(pl, m->res, c);
    for (int o = 0; o < n_off; o++) {
      int ox, oy, oz;
      if (n_off == 27) { ox = o / 9 - 1; oy = (o / 3) % 3 - 1; oz = o % 3 - 1; }
      else { ox = ndt_off7[o][0]; oy = ndt_off7[o][1]; oz = ndt_off7[o][2]; }
      const OrcNdtVox* v = ndt_find(m, c[0] + ox, c[1] + oy, c[2] + oz);
      if (!v) continue;
      nc++;
      if (v->n <= 6) continue; /* ndt_compute_derivatives.cu:62-64 */
      float e[3], Ce[3];
      for (int r = 0; r < 3; r++) e[r] = v->mean[r] - tA[r];
      float ne = v->nrm[0] * e[0] + v->nrm[1] * e[1] + v->nrm[2] * e[2];
      for (int r = 0; r < 3; r++) Ce[r] = e[r] + 999.0f * v->nrm[r] * ne;
      float x = sqrtf(e[0] * e[0] + e[1] * e[1] + e[2] * e[2]);
      float w = k_sq / (k_sq + x * x); /* cauchy, :15-18 */
      err += (double)(w * (e[0] * Ce[0] + e[1] * Ce[1] + e[2] * Ce[2]));
      if (!H36) continue;
      /* J = [skew(tA) | -I] (3x6) */
      float J[3][6] = {{0, -tA[2], tA[1], -1, 0, 0}, {tA[2], 0, -tA[0], 0, -1, 0}, {-tA[1], tA[0], 0, 0, 0, -1}};
      float M[3][6]; /* C^-1 J */
      for (int cc = 0; cc < 6; cc++) {
        float nj = v->nrm[0] * J[0][cc] + v->nrm[1] * J[1][cc] + v->nrm[2] * J[2][cc];
        for (int r = 0; r < 3; r++) M[r][cc] = J[r][cc] + 999.0f * v->nrm[r] * nj;
      }
      for (int p = 0; p < 6; p++) {
        for (int q = 0; q < 6; q++) H[6 * p + q] += (double)(w * (J[0][p] * M[0][q] + J[1][p] * M[1][q] + J[2][p] * M[2][q]));
        b[p] += (double)(w * (J[0][p] * Ce[0] + J[1][p] * Ce[1] + J[2][p] * Ce[2]));
      }
    }
  }
  if (H36) { memcpy(H36, H, sizeof(H)); memcpy(b6, b, sizeof(b)); }
  if (n_corr) *n_corr = nc;
  return err;
}

/* ===================================================================================== */
/* a12/a13  FastGICP (fast_gicp_impl.hpp:119-303): k-NN covariances with PLANE             */
/*      regularisation (U diag(1,1,1e-3) V^T  =  I - 0.999 n n^T), 1-NN correspondences    */
/*      within max_corr, D2D cost, all double.  Neighbour search is exact (the reference   */
/*      uses pcl::search::KdTree/FLANN: exact k-NN, method-independent up to ties).         */
/*      Pinned against the compiled reference FastGICP / FastVGICP (oracle/ref_reg.cpp,      */
/*      PCL shimmed): tests/test_oracle_reg.py.                                              */
/* ===================================================================================== */
/* normals[n,3] (double) = smallest-eigenvalue direction of the k-NN covariance; cnt[n] = #neighbours used */
void orc_gicp_normals(const OrcIvox* map, const float* pts, int stride, int n, int k, double max_sq, double* normals, int* cnt,
                      int nthreads) {
  omp_set_num_threads(nthreads > 0 ? nthreads : 1);
#pragma omp parallel for schedule(dynamic, 256)
  for (int i = 0; i < n; i++) {
    OrcCand best[64];
    int kk = k > 64 ? 64 : k;
    int nb = exact_knn_one(map, pts + (size_t)stride * i, kk, max_sq, best);
    if (nb < kk && n > nb) {
      /* The reference takes the k nearest neighbours wherever they are (pcl::search::KdTree::nearestKSearch,
       * fast_gicp_impl.hpp:259): max_sq only bounds the fast grid search.  A point with fewer than k neighbours inside
       * the radius (sparse rings of a scan at long range) gets the true k-NN by an exact scan of the cloud. */
      nb = 0;
      for (int j = 0; j < n; j++) {
        const float* b = pts + (size_t)stride * j;
        OrcPt pj = {b[0], b[1], b[2], j};
        OrcCand cd = {dist2f(pts + (size_t)stride * i, &pj), j, b[0], b[1], b[2]};
        topk_insert(best, &nb, kk, &cd);
      }
    }
    cnt[i] = nb;
    double mean[3] = {0, 0, 0}, C[9] = {0};
    for (int j = 0; j < nb; j++) { mean[0] += best[j].x; mean[1] += best[j].y; mean[2] += best[j].z; }
    for (int a = 0; a < 3; a++) mean[a] /= (double)k; /* rowwise().mean() over k columns (zero-padded if fewer) */
    for (int j = 0; j < k; j++) {
      double d[3] = {(j < nb ? best[j].x : 0.0) - mean[0], (j < nb ? best[j].y : 0.0) - mean[1], (j < nb ? best[j].z : 0.0) - mean[2]};
      for (int a = 0; a < 3; a++) for (int b = 0; b < 3; b++) C[3 * a + b] += d[a] * d[b];
    }
    for (int a = 0; a < 9; a++) C[a] /= (double)k;
    double w[3], V[9]; eig3_sym(C, w, V);
    int k0 = 0; if (w[1] < w[k0]) k0 = 1; if (w[2] < w[k0]) k0 = 2;
    for (int a = 0; a < 3; a++) normals[3 * (size_t)i + a] = V[3 * a + k0];
  }
}
static void inv3(const double* A, double* I) {
  double c00 = A[4] * A[8] - A[5] * A[7], c01 = A[5] * A[6] - A[3] * A[8], c02 = A[3] * A[7] - A[4] * A[6];
  double det = A[0] * c00 + A[1] * c01 + A[2] * c02, id = 1.0 / det;
  I[0] = c00 * id; I[1] = (A[2] * A[7] - A[1] * A[8]) * id; I[2] = (A[1] * A[5] - A[2] * A[4]) * id;
  I[3] = c01 * id; I[4] = (A[0] * A[8] - A[2] * A[6]) * id; I[5] = (A[2] * A[3] - A[0] * A[5]) * id;
  I[6] = c02 * id; I[7] = (A[1] * A[6] - A[0] * A[7]) * id; I[8] = (A[0] * A[4] - A[1] * A[3]) * id;
}
/* corr[n] in/out: when update != 0 correspondences (1-NN ids within max_corr, else -1) and Mahalanobis
 * matrices maha[n,9] are recomputed at T (update_correspondences); otherwise reused (compute_error). */
double orc_gicp_cost(const OrcIvox* tgt_map, const float* tgt, int tstride, const double* tgt_nrm, const float* src, int sstride,
                     const double* src_nrm, int n, const double* T, double max_corr, int update, int* corr, double* maha,
                     double* H36, double* b6, int nthreads) {
  double R[9], t[3];
  for (int a = 0; a < 3; a++) { for (int b = 0; b < 3; b++) R[3 * a + b] = T[4 * a + b]; t[a] = T[4 * a + 3]; }
  if (update) {
    float Rf[9], tf[3];
    for (int a = 0; a < 9; a++) Rf[a] = (float)R[a];
    for (int a = 0; a < 3; a++) tf[a] = (float)t[a];
    omp_set_num_threads(nthreads > 0 ? nthreads : 1);
#pragma omp parallel for schedule(dynamic, 256)
    for (int i = 0; i < n; i++) {
      const float* a = src + (size_t)sstride * i;
      float q[3];
      for (int r = 0; r < 3; r++) q[r] = Rf[3 * r] * a[0] + Rf[3 * r + 1] * a[1] + Rf[3 * r + 2] * a[2] + tf[r];
      OrcCand best[1];
      int nb = exact_knn_one(tgt_map, q, 1, max_corr * max_corr, best);
      corr[i] = (nb > 0 && (double)best[0].d2 < max_corr * max_corr) ? best[0].id : -1;
      if (corr[i] < 0) continue;
      const double* nb_ = tgt_nrm + 3 * (size_t)corr[i]; const double* na = src_nrm + 3 * (size_t)i;
      double Rn[3]; mat3_vec(R, na, Rn);
      double RCR[9];
      for (int p = 0; p < 3; p++) for (int c = 0; c < 3; c++) RCR[3 * p + c] = (p == c ? 2.0 : 0.0) - 0.999 * (nb_[p] * nb_[c] + Rn[p] * Rn[c]);
      inv3(RCR, maha + 9 * (size_t)i);
    }
  }
  double H[36] = {0}, b[6] = {0}, err = 0;
  for (int i = 0; i < n; i++) {
    if (corr[i] < 0) continue;
    const float* a = src + (size_t)sstride * i; const float* bb = tgt + (size_t)tstride * corr[i];
    double A[3] = {a[0], a[1], a[2]}, tA[3], e[3], Me[3];
    mat3_vec(R, A, tA);
    for (int r = 0; r < 3; r++) { tA[r] += t[r]; e[r] = (double)bb[r] - tA[r]; }
    const double* M = maha + 9 * (size_t)i;
    mat3_vec(M, e, Me);
    err += e[0] * Me[0] + e[1] * Me[1] + e[2] * Me[2];
    if (!H36) continue;
    double J[3][6] = {{0, -tA[2], tA[1], -1, 0, 0}, {tA[2], 0, -tA[0], 0, -1, 0}, {-tA[1], tA[0], 0, 0, 0, -1}};
    double MJ[3][6];
    for (int c = 0; c < 6; c++) for (int r = 0; r < 3; r++) MJ[r][c] = M[3 * r] * J[0][c] + M[3 * r + 1] * J[1][c] + M[3 * r + 2] * J[2][c];
    for (int p = 0; p < 6; p++) {
      for (int q = 0; q < 6; q++) H[6 * p + q] += J[0][p] * MJ[0][q] + J[1][p] * MJ[1][q] + J[2][p] * MJ[2][q];
      b[p] += J[0][p] * Me[0] + J[1][p] * Me[1] + J[2][p] * Me[2];
    }
  }
  if (H36) { memcpy(H36, H, sizeof(H)); memcpy(b6, b, sizeof(b)); }
  return err;
}

/* ===================================================================================== */
/* a14  FastVGICP (fast_vgicp_impl.hpp:72-207) + GaussianVoxelMap, ADDITIVE voxels          */
/*      (fast_vgicp_voxel.hpp:108-182): target voxel = mean of the points and MEAN of their */
/*      PLANE-regularised covariances (I - 0.999 n n^T); coord = floor(x/res - 0.5) in      */
/*      double; correspondences = voxels at coord + offsets (DIRECT1/7/27) of the           */
/*      transformed source point; weight sqrt(num_points).  Pinned against the compiled     */
/*      reference (oracle/_ref/libref_reg.so) in tests/test_oracle_reg.py.                  */
/* ===================================================================================== */
typedef struct { int kx, ky, kz, used, n; double mean[3], cov[9]; } OrcVgVox;
typedef struct { double res; size_t tab_size, n_vox; OrcVgVox* tab; } OrcVg;

static OrcVgVox* vg_find(const OrcVg* m, int x, int y, int z) {
  size_t mask = m->tab_size - 1, s = cell_hash(x, y, z) & mask;
  for (;;) {
    OrcVgVox* v = &m->tab[s];
    if (!v->used) return NULL;
    if (v->kx == x && v->ky == y && v->kz == z) return v;
    s = (s + 1) & mask;
  }
}
static inline void vg_coord(const double* p, double res, int* c) {
  for (int a = 0; a < 3; a++) c[a] = (int)floor(p[a] / res - 0.5);
}
/* normals[n,3]: the targets' covariance directions from orc_gicp_normals */
OrcVg* orc_vgicp_build(const float* pts, int stride, int n, const double* normals, double res) {
  OrcVg* m = (OrcVg*)calloc(1, sizeof(OrcVg));
  m->res = res;
  size_t t = 1024; while (t < (size_t)n * 2) t <<= 1;
  m->tab_size = t; m->tab = (OrcVgVox*)calloc(t, sizeof(OrcVgVox));
  size_t mask = t - 1;
  for (int i = 0; i < n; i++) {
    const float* pf = pts + (size_t)stride * i;
    double p[3] = {pf[0], pf[1], pf[2]};
    int c[3]; vg_coord(p, res, c);
    size_t s = cell_hash(c[0], c[1], c[2]) & mask;
    OrcVgVox* v;
    for (;;) { v = &m->tab[s]; if (!v->used) { v->used = 1; v->kx = c[0]; v->ky = c[1]; v->kz = c[2]; m->n_vox++; break; }
               if (v->kx == c[0] && v->ky == c[1] && v->kz == c[2]) break; s = (s + 1) & mask; }
    v->n++;
    const double* nr = normals + 3 * (size_t)i;
    for (int a = 0; a < 3; a++) { v->mean[a] += p[a]; for (int b = 0; b < 3; b++) v->cov[3 * a + b] += (a == b ? 1.0 : 0.0) - 0.999 * nr[a] * nr[b]; }
  }
  for (size_t s = 0; s < t; s++) {
    OrcVgVox* v = &m->tab[s];
    if (!v->used) continue;
    for (int a = 0; a < 3; a++) v->mean[a] /= (double)v->n;
    for (int a = 0; a < 9; a++) v->cov[a] /= (double)v->n;
  }
  return m;
}
void orc_vgicp_destroy(OrcVg* m) { if (m) { free(m->tab); free(m); } }
size_t orc_vgicp_num_voxels(const OrcVg* m) { return m->n_vox; }
int orc_vgicp_voxel(const OrcVg* m, int x, int y, int z, double* mean, double* cov) {
  const OrcVgVox* v = vg_find(m, x, y, z);
  if (!v) return 0;
  memcpy(mean, v->mean, sizeof(v->mean)); memcpy(cov, v->cov, sizeof(v->cov));
  return v->n;
}
/* update != 0: correspondences (voxel table slots, corr[n_off*n], -1 = none) and Mahalanobis matrices
 * maha[n_off*n, 9] are recomputed at T; otherwise reused.  Returns the weighted error. */
double orc_vgicp_cost(const OrcVg* m, const float* src, int stride, const double* src_nrm, int n, const double* T, int n_off,
                      int update, long long* corr, double* maha, double* H36, double* b6, int* n_corr) {
  double R[9], t[3];
  for (int a = 0; a < 3; a++) { for (int b = 0; b < 3; b++) R[3 * a + b] = T[4 * a + b]; t[a] = T[4 * a + 3]; }
  if (update) {
    for (int i = 0; i < n; i++) {
      const float* a = src + (size_t)stride * i;
      double A[3] = {a[0], a[1], a[2]}, tA[3];
      mat3_vec(R, A, tA);
      for (int r = 0; r < 3; r++) tA[r] += t[r];
      int c[3]; vg_coord(tA, m->res, c);
      double Rn[3]; mat3_vec(R, src_nrm + 3 * (size_t)i, Rn);
      for (int o = 0; o < n_off; o++) {
        int ox, oy, oz;
        if (n_off == 27) { ox = o / 9 - 1; oy = (o / 3) % 3 - 1; oz = o % 3 - 1; }
        else { ox = ndt_off7[o][0]; oy = ndt_off7[o][1]; oz = ndt_off7[o][2]; }
        const OrcVgVox* v = vg_find(m, c[0] + ox, c[1] + oy, c[2] + oz);
        const size_t q = (size_t)o * n + i;
        corr[q] = v ? (long long)(v - m->tab) : -1;
        if (!v) continue;
        double RCR[9];
        for (int p = 0; p < 3; p++) for (int cc = 0; cc < 3; cc++) RCR[3 * p + cc] = v->cov[3 * p + cc] + (p == cc ? 1.0 : 0.0) - 0.999 * Rn[p] * Rn[cc];
        inv3(RCR, maha + 9 * q);
      }
    }
  }
  double H[36] = {0}, b[6] = {0}, err = 0; int nc = 0;
  for (int o = 0; o < n_off; o++) for (int i = 0; i < n; i++) {
    const size_t q = (size_t)o * n + i;
    if (corr[q] < 0) continue;
    nc++;
    const OrcVgVox* v = m->tab + corr[q];
    const float* a = src + (size_t)stride * i;
    double A[3] = {a[0], a[1], a[2]}, tA[3], e[3], Me[3];
    mat3_vec(R, A, tA);
    for (int r = 0; r < 3; r++) { tA[r] += t[r]; e[r] = v->mean[r] - tA[r]; }
    const double* M = maha + 9 * q;
    mat3_vec(M, e, Me);
    const double w = sqrt((double)v->n);
    err += w * (e[0] * Me[0] + e[1] * Me[1] + e[2] * Me[2]);
    if (!H36) continue;
    double J[3][6] = {{0, -tA[2], tA[1], -1, 0, 0}, {tA[2], 0, -tA[0], 0, -1, 0}, {-tA[1], tA[0], 0, 0, 0, -1}};
    double MJ[3][6];
    for (int c = 0; c < 6; c++) for (int r = 0; r < 3; r++) MJ[r][c] = M[3 * r] * J[0][c] + M[3 * r + 1] * J[1][c] + M[3 * r + 2] * J[2][c];
    for (int p = 0; p < 6; p++) {
      for (int q2 = 0; q2 < 6; q2++) H[6 * p + q2] += w * (J[0][p] * MJ[0][q2] + J[1][p] * MJ[1][q2] + J[2][p] * MJ[2][q2]);
      b[p] += w * (J[0][p] * Me[0] + J[1][p] * Me[1] + J[2][p] * Me[2]);
    }
  }
  if (H36) { memcpy(H36, H, sizeof(H)); memcpy(b6, b, sizeof(b)); }
  if (n_corr) *n_corr = nc;
  return err;
}

/* a16  pcl::Registration::getFitnessScore(max_range) (PCL 1.9.1 registration.hpp): mean of the squared
 * 1-NN distances d2 <= max_range (the reference compares the SQUARED distance with max_range). */
double orc_fitness(const OrcIvox* tgt_map, const float* src, int stride, int n, const double* T, double max_range, double search_sq) {
  float R[9], t[3];
  for (int a = 0; a < 3; a++) { for (int b = 0; b < 3; b++) R[3 * a + b] = (float)T[4 * a + b]; t[a] = (float)T[4 * a + 3]; }
  double sum = 0; int nr = 0;
  for (int i = 0; i < n; i++) {
    const float* a = src + (size_t)stride * i; float q[3];
    for (int r = 0; r < 3; r++) q[r] = R[3 * r] * a[0] + R[3 * r + 1] * a[1] + R[3 * r + 2] * a[2] + t[r];
    OrcCand best[1];
    int nb = exact_knn_one(tgt_map, q, 1, search_sq, best);
    if (nb > 0 && (double)best[0].d2 <= max_range) { sum += (double)best[0].d2; nr++; }
  }
  return nr > 0 ? sum / nr : 1.7976931348623157e308;
}
