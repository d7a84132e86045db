/* The CPU minimum spanning forest the device msf is checked against: Kruskal's
 * algorithm with a union-find, under the same key and canonical edge list as
 * algorithm::msf.  Test infrastructure written for this project.
 *
 * Graph: the edge {i, j}, i != j, for every stored entry A(i,j) or A(j,i); its weight is
 * the smaller of the stored values, -0.0 read as +0.0; self-loops are dropped.  Edges
 * are ranked by (w, min(i,j), max(i,j)).  Values come in as doubles, which hold every
 * FP32 and INT32 value exactly. */
#include <stdlib.h>

typedef struct {
  int u, v;
  double w;
} Edge;

/* (u, v, w): groups the entries of one edge together, the lightest first */
static int byEnds(const void* a, const void* b) {
  const Edge* x = (const Edge*)a;
  const Edge* y = (const Edge*)b;
  if (x->u != y->u) return x->u < y->u ? -1 : 1;
  if (x->v != y->v) return x->v < y->v ? -1 : 1;
  return x->w < y->w ? -1 : (x->w > y->w ? 1 : 0);
}

/* the key (w, u, v) */
static int byKey(const void* a, const void* b) {
  const Edge* x = (const Edge*)a;
  const Edge* y = (const Edge*)b;
  if (x->w != y->w) return x->w < y->w ? -1 : 1;
  if (x->u != y->u) return x->u < y->u ? -1 : 1;
  return x->v < y->v ? -1 : (x->v > y->v ? 1 : 0);
}

static int findRoot(int* parent, int x) {
  while (parent[x] != x) {
    parent[x] = parent[parent[x]];
    x = parent[x];
  }
  return x;
}

/* The minimum spanning forest of the n x n CSR (rp, ci, val).  out_rp [n + 1], out_ci
 * and out_val [2 (n - 1) at least] receive F: both directions of every forest edge, rows
 * sorted by column.  *weight = the sum of the forest's weights in (min, max) order.
 * Returns the number of forest edges, -1 on a NaN off the diagonal, -2 when out of
 * memory. */
long long orc_msf(int n, const int* rp, const int* ci, const double* val, int* out_rp,
                  int* out_ci, double* out_val, double* weight) {
  const long long nnz = n > 0 ? rp[n] : 0;
  Edge* e = (Edge*)malloc((size_t)(nnz > 0 ? nnz : 1)*sizeof(Edge));
  int* parent = (int*)malloc((size_t)(n > 0 ? n : 1)*sizeof(int));
  unsigned char* kept = (unsigned char*)calloc((size_t)(nnz > 0 ? nnz : 1), 1);
  if (e == NULL || parent == NULL || kept == NULL) {
    free(e); free(parent); free(kept);
    return -2;
  }
  long long m = 0;
  for (int i = 0; i < n; ++i)
    for (int k = rp[i]; k < rp[i + 1]; ++k) {
      const int j = ci[k];
      if (j == i) continue;
      const double w = val[k];
      if (w != w) {
        free(e); free(parent); free(kept);
        return -1;
      }
      e[m].u = i < j ? i : j;
      e[m].v = i < j ? j : i;
      e[m].w = w == 0.0 ? 0.0 : w;
      ++m;
    }
  /* one edge per (u, v), with the smaller weight */
  qsort(e, (size_t)m, sizeof(Edge), byEnds);
  long long me = 0;
  for (long long k = 0; k < m; ++k)
    if (me == 0 || e[me - 1].u != e[k].u || e[me - 1].v != e[k].v) e[me++] = e[k];
  /* Kruskal */
  qsort(e, (size_t)me, sizeof(Edge), byKey);
  for (int i = 0; i < n; ++i) parent[i] = i;
  long long nf = 0;
  for (long long k = 0; k < me; ++k) {
    const int a = findRoot(parent, e[k].u);
    const int b = findRoot(parent, e[k].v);
    if (a == b) continue;
    parent[a < b ? b : a] = a < b ? a : b;
    kept[k] = 1;
    ++nf;
  }
  long long f = 0;
  for (long long k = 0; k < me; ++k)
    if (kept[k]) e[f++] = e[k];
  qsort(e, (size_t)nf, sizeof(Edge), byEnds);
  /* F: row u holds v and row v holds u; each row's columns come out sorted because
   * the lower neighbours (edges (v', u), v' < u, in v' order) are placed before the
   * upper ones (edges (u, v'), in v' order) */
  double sum = 0.0;
  for (int i = 0; i <= n; ++i) out_rp[i] = 0;
  for (long long k = 0; k < nf; ++k) {
    ++out_rp[e[k].u + 1];
    ++out_rp[e[k].v + 1];
    sum += e[k].w;
  }
  for (int i = 0; i < n; ++i) out_rp[i + 1] += out_rp[i];
  int* fill = parent;                    /* the union-find is no longer needed */
  for (int i = 0; i < n; ++i) fill[i] = out_rp[i];
  for (long long k = 0; k < nf; ++k) {   /* lower neighbours: rows v, in u order */
    const int at = fill[e[k].v]++;
    out_ci[at] = e[k].u;
    out_val[at] = e[k].w;
  }
  for (long long k = 0; k < nf; ++k) {   /* upper neighbours: rows u, in v order */
    const int at = fill[e[k].u]++;
    out_ci[at] = e[k].v;
    out_val[at] = e[k].w;
  }
  *weight = sum;
  free(e); free(parent); free(kept);
  return nf;
}
