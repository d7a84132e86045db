/* oracle/gb_oracle.c — CPU restatement of the reference's algorithms for the
 * direction-optimised mxv/vxm + masked-mxm path (see gb_oracle.h for the scope
 * and the TEST-INFRASTRUCTURE-ONLY rule).  Each function cites the reference
 * file:line it follows.  Plain C, single thread.
 */
#include "gb_oracle.h"

#include <float.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

/* ------------------------------------------------------------------------- */
/* Semiring table: reference graphblas/stddef.hpp:14-138 (binary ops),       */
/* :160-173 (monoid identities), :194-213 (semirings).                       */
/* ------------------------------------------------------------------------- */
enum { OP_OR, OP_AND, OP_PLUS, OP_MINUS, OP_MUL, OP_DIV, OP_MIN, OP_MAX,
       OP_GT, OP_LT, OP_NE, OP_SECOND };

static float apply_op(int op, float a, float b) {
  switch (op) {
    case OP_OR:     return (a != 0.f || b != 0.f) ? 1.f : 0.f;
    case OP_AND:    return (a != 0.f && b != 0.f) ? 1.f : 0.f;
    case OP_PLUS:   return a + b;
    case OP_MINUS:  return a - b;
    case OP_MUL:    return a * b;
    case OP_DIV:    return a / b;
    case OP_MIN:    return fminf(a, b);      /* CUDA min(a,b): a NaN operand is ignored */
    case OP_MAX:    return fmaxf(a, b);
    case OP_GT:     return a > b ? 1.f : 0.f;
    case OP_LT:     return a < b ? 1.f : 0.f;
    case OP_NE:     return a != b ? 1.f : 0.f;
    case OP_SECOND: return b;
  }
  return 0.f;
}

typedef struct { int add; int mul; float identity; } semiring_t;

static semiring_t semiring(int id) {
  semiring_t s = { OP_PLUS, OP_MUL, 0.f };
  switch (id) {
    case ORC_LOGICAL_OR_AND:        s.add = OP_OR;   s.mul = OP_AND;    s.identity = 0.f; break;
    case ORC_PLUS_MULTIPLIES:       s.add = OP_PLUS; s.mul = OP_MUL;    s.identity = 0.f; break;
    case ORC_MINIMUM_PLUS:          s.add = OP_MIN;  s.mul = OP_PLUS;   s.identity = FLT_MAX; break;
    case ORC_MAXIMUM_MULTIPLIES:    s.add = OP_MAX;  s.mul = OP_MUL;    s.identity = 0.f; break;
    case ORC_PLUS_DIVIDES:          s.add = OP_PLUS; s.mul = OP_DIV;    s.identity = 0.f; break;
    case ORC_PLUS_GREATER:          s.add = OP_PLUS; s.mul = OP_GT;     s.identity = 0.f; break;
    case ORC_GREATER_PLUS:          s.add = OP_GT;   s.mul = OP_PLUS;   s.identity = FLT_MIN; break;
    case ORC_PLUS_MINUS:            s.add = OP_PLUS; s.mul = OP_MINUS;  s.identity = 0.f; break;
    case ORC_PLUS_LESS:             s.add = OP_PLUS; s.mul = OP_LT;     s.identity = 0.f; break;
    case ORC_CUSTOM_LESS_PLUS:      s.add = OP_LT;   s.mul = OP_PLUS;   s.identity = FLT_MAX; break;
    case ORC_MINIMUM_MULTIPLIES:    s.add = OP_MIN;  s.mul = OP_MUL;    s.identity = FLT_MAX; break;
    case ORC_MULTIPLIES_MULTIPLIES: s.add = OP_MUL;  s.mul = OP_MUL;    s.identity = 1.f; break;
    case ORC_NOT_EQUAL_TO_PLUS:     s.add = OP_NE;   s.mul = OP_PLUS;   s.identity = FLT_MAX; break;
    case ORC_MINIMUM_SELECT_SECOND: s.add = OP_MIN;  s.mul = OP_SECOND; s.identity = FLT_MAX; break;
    case ORC_PLUS_NOT_EQUAL_TO:     s.add = OP_PLUS; s.mul = OP_NE;     s.identity = 0.f; break;
    case ORC_CUSTOM_LESS_LESS:      s.add = OP_LT;   s.mul = OP_LT;     s.identity = FLT_MAX; break;
    case ORC_MINIMUM_NOT_EQUAL_TO:  s.add = OP_MIN;  s.mul = OP_NE;     s.identity = FLT_MAX; break;
    default: break;
  }
  return s;
}

float orc_identity(int id) { return semiring(id).identity; }
float orc_add(int id, float a, float b) { return apply_op(semiring(id).add, a, b); }
float orc_mul(int id, float a, float b) { return apply_op(semiring(id).mul, a, b); }

/* ------------------------------------------------------------------------- */
/* BFS: reference graphblas/algorithm/test_bfs.hpp:11-61.  FIFO queue of      */
/* discovered vertices, level of a neighbour = level of the dequeued vertex   */
/* + 1, source level 1, undiscovered 0; stops expanding past `stop`.          */
/* ------------------------------------------------------------------------- */
int orc_bfs(int nrows, const int* rowptr, const int* colind, int* levels,
            int src, int stop) {
  int i, depth = 1;
  int* queue = (int*)malloc((size_t)(nrows > 0 ? nrows : 1) * sizeof(int));
  long long head = 0, tail = 0;
  for (i = 0; i < nrows; ++i) levels[i] = 0;
  levels[src] = 1;
  queue[tail++] = src;
  while (head < tail) {
    int node = queue[head++];
    int next = levels[node] + 1;
    int e;
    if (next > stop) break;
    for (e = rowptr[node]; e < rowptr[node + 1]; ++e) {
      int nb = colind[e];
      if (levels[nb] == 0) {
        levels[nb] = next;
        if (depth < next) depth = next;
        queue[tail++] = nb;
      }
    }
  }
  free(queue);
  return depth;
}

/* ------------------------------------------------------------------------- */
/* SSSP: reference graphblas/algorithm/test_sssp.hpp:15-79.  Lazy Dijkstra:   */
/* a (distance, vertex) min-heap with duplicate entries, a popped vertex is   */
/* marked processed, relaxations skip processed vertices and edges of weight  */
/* FLT_MAX.  "depth" counts rounds that each drain the heap as it stood at    */
/* the start of the round (test_sssp.hpp:44-45,74).                           */
/* ------------------------------------------------------------------------- */
typedef struct { float d; int v; } heap_item;

static int heap_less(heap_item a, heap_item b) {
  /* std::pair<float,int> ordering used by std::greater in the reference */
  return (a.d < b.d) || (a.d == b.d && a.v < b.v);
}

static void heap_push(heap_item** h, long long* n, long long* cap, heap_item x) {
  long long i;
  if (*n == *cap) {
    *cap = *cap ? *cap * 2 : 1024;
    *h = (heap_item*)realloc(*h, (size_t)(*cap) * sizeof(heap_item));
  }
  i = (*n)++;
  while (i > 0) {
    long long p = (i - 1) / 2;
    if (!heap_less(x, (*h)[p])) break;
    (*h)[i] = (*h)[p];
    i = p;
  }
  (*h)[i] = x;
}

static heap_item heap_pop(heap_item* h, long long* n) {
  heap_item top = h[0];
  heap_item x = h[--(*n)];
  long long i = 0;
  while (1) {
    long long l = 2 * i + 1, r = l + 1, m = l;
    if (l >= *n) break;
    if (r < *n && heap_less(h[r], h[l])) m = r;
    if (!heap_less(h[m], x)) break;
    h[i] = h[m];
    i = m;
  }
  if (*n > 0) h[i] = x;
  return top;
}

int orc_sssp(int nrows, const int* rowptr, const int* colind, const float* val,
             float* dist, int src) {
  unsigned char* processed = (unsigned char*)calloc((size_t)(nrows > 0 ? nrows : 1), 1);
  heap_item* heap = NULL;
  long long hn = 0, hcap = 0;
  int i, depth = 0;
  heap_item first;
  for (i = 0; i < nrows; ++i) dist[i] = FLT_MAX;
  dist[src] = 0.f;
  first.d = 0.f; first.v = src;
  heap_push(&heap, &hn, &hcap, first);
  while (hn > 0) {
    long long round = hn, k;
    for (k = 0; k < round; ++k) {
      heap_item it = heap_pop(heap, &hn);
      int e;
      processed[it.v] = 1;
      for (e = rowptr[it.v]; e < rowptr[it.v + 1]; ++e) {
        int nb = colind[e];
        float w = val[e];
        if (!processed[nb] && w != FLT_MAX) {
          float nd = it.d + w;
          if (nd < dist[nb]) {
            heap_item x;
            dist[nb] = nd;
            x.d = nd; x.v = nb;
            heap_push(&heap, &hn, &hcap, x);
          }
        }
      }
    }
    depth++;
  }
  free(heap);
  free(processed);
  return depth;
}

/* ------------------------------------------------------------------------- */
/* PageRank: reference graphblas/algorithm/test_pr.hpp:15-80.  All arithmetic */
/* in float, in the reference's order: pagerank[v] starts at (1-alpha)/n,     */
/* every node pushes alpha*(p[node]/outdeg[node]) along its row, then         */
/* resultant = sum (p_old - p_new)^2; stop when fabs(resultant) < eps.        */
/* ------------------------------------------------------------------------- */
int orc_pr(int nrows, const int* rowptr, const int* colind, float* pr,
           float alpha, float eps, int max_niter) {
  float* next = (float*)malloc((size_t)(nrows > 0 ? nrows : 1) * sizeof(float));
  float* outdeg = (float*)malloc((size_t)(nrows > 0 ? nrows : 1) * sizeof(float));
  int it, node, depth = 0;
  for (node = 0; node < nrows; ++node) pr[node] = 1.f / nrows;
  for (node = 0; node < nrows; ++node)
    outdeg[node] = (float)(rowptr[node + 1] - rowptr[node]);
  for (it = 0; it < max_niter; ++it) {
    float resultant = 0.f;
    for (node = 0; node < nrows; ++node) next[node] = (1.f - alpha) / nrows;
    for (node = 0; node < nrows; ++node) {
      float contrib = pr[node] / outdeg[node];
      int e;
      for (e = rowptr[node]; e < rowptr[node + 1]; ++e)
        next[colind[e]] += alpha * contrib;
    }
    for (node = 0; node < nrows; ++node) {
      float diff = pr[node] - next[node];
      resultant += diff * diff;
      pr[node] = next[node];
    }
    if (fabsf(resultant) < eps) break;
    depth++;
  }
  free(next);
  free(outdeg);
  return depth;
}

/* ------------------------------------------------------------------------- */
/* Triangle count: reference graphblas/algorithm/test_tc.hpp:15-85.  For      */
/* every stored entry (node, neighbour) the two sorted adjacency lists are    */
/* intersected by a two-pointer merge; every match counts one.                */
/* ------------------------------------------------------------------------- */
long long orc_tc(int nrows, const int* rowptr, const int* colind) {
  long long count = 0;
  int node;
  for (node = 0; node < nrows; ++node) {
    int e;
    for (e = rowptr[node]; e < rowptr[node + 1]; ++e) {
      int nb = colind[e];
      int p = rowptr[node], pe = rowptr[node + 1];
      int q = rowptr[nb], qe = rowptr[nb + 1];
      while (p < pe && q < qe) {
        int x = colind[p], y = colind[q];
        if (x < y) ++p;
        else if (x > y) ++q;
        else { ++count; ++p; ++q; }
      }
    }
  }
  return count;
}

/* ------------------------------------------------------------------------- */
/* Masked mxm, int plus-times: the definition C(i,j) = sum_k A(i,k)*B(k,j)    */
/* for (i,j) in the mask (reference backend/cuda/spgemm.hpp:22-110 computes  */
/* the same dot products on the device).  The shorter list is walked and each */
/* key binary-searched in the longer one, so hub entries of R-MAT graphs cost */
/* min*log(max) instead of a merge over both lists.                            */
/* ------------------------------------------------------------------------- */
static int lower_bound_i32(const int* a, int lo, int hi, int key) {
  while (lo < hi) {
    int mid = lo + (hi - lo) / 2;
    if (a[mid] < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

void orc_mxm_masked(int nrows, const int* a_rowptr, const int* a_colind,
                    const int* a_val, const int* b_colptr, const int* b_rowind,
                    const int* b_val, const int* m_rowptr, const int* m_colind,
                    const int* m_val, long long* out) {
  int i;
  for (i = 0; i < nrows; ++i) {
    int e;
    const int pb = a_rowptr[i], pe = a_rowptr[i + 1];
    for (e = m_rowptr[i]; e < m_rowptr[i + 1]; ++e) {
      const int j = m_colind[e];
      const int qb = b_colptr[j], qe = b_colptr[j + 1];
      long long acc = 0;
      if (m_val[e] != 0) {
        if (pe - pb <= qe - qb) {
          int p, q = qb;
          for (p = pb; p < pe && q < qe; ++p) {
            q = lower_bound_i32(b_rowind, q, qe, a_colind[p]);
            if (q < qe && b_rowind[q] == a_colind[p])
              acc += (long long)a_val[p] * b_val[q];
          }
        } else {
          int q, p = pb;
          for (q = qb; q < qe && p < pe; ++q) {
            p = lower_bound_i32(a_colind, p, pe, b_rowind[q]);
            if (p < pe && a_colind[p] == b_rowind[q])
              acc += (long long)a_val[p] * b_val[q];
          }
        }
      }
      out[e] = acc;
    }
  }
}

/* ------------------------------------------------------------------------- */
/* vxm over a semiring, push formulation: reference test/gvxm.cu:41-55        */
/* (dense u), :103-119 (sparse u), :169-192 (sparse u + mask), generalised    */
/* from (+,*) to the semiring functors.  w starts "absent"; the first product */
/* landing on a column initialises it with add(identity, product).            */
/* ------------------------------------------------------------------------- */
void orc_vxm(int id, int nrows, int ncols, const int* rowptr, const int* colind,
             const float* val, const float* u, const unsigned char* u_present,
             const float* mask, int scmp, float* w, unsigned char* w_present) {
  semiring_t s = semiring(id);
  int row, col;
  for (col = 0; col < ncols; ++col) {
    w[col] = s.identity;
    if (w_present) w_present[col] = 0;
  }
  for (row = 0; row < nrows; ++row) {
    int e;
    if (u_present && !u_present[row]) continue;
    for (e = rowptr[row]; e < rowptr[row + 1]; ++e) {
      float prod = apply_op(s.mul, val[e], u[row]);
      col = colind[e];
      w[col] = apply_op(s.add, w[col], prod);
      if (w_present) w_present[col] = 1;
    }
  }
  if (mask) {
    for (col = 0; col < ncols; ++col) {
      int drop = scmp ? (mask[col] != 0.f) : (mask[col] == 0.f);
      if (drop) {
        w[col] = 0.f;
        if (w_present) w_present[col] = 0;
      }
    }
  }
}

/* reference test/greduce.cu:63-75 (row sums) */
void orc_reduce_rows(int nrows, const int* rowptr, const float* val, float* w) {
  int row;
  for (row = 0; row < nrows; ++row) {
    float acc = 0.f;
    int e;
    for (e = rowptr[row]; e < rowptr[row + 1]; ++e) acc += val[e];
    w[row] = acc;
  }
}

/* ------------------------------------------------------------------------- */
/* Loader semantics.  reference graphblas/util.hpp:264-329: when undirected,  */
/* every non-loop edge (r,c) also contributes (c,r); tuples are sorted by     */
/* (row, col); self-loops and repeated (row,col) pairs are dropped; then      */
/* coo2csr (:502-556) counts rows and prefix-sums.                            */
/* ------------------------------------------------------------------------- */
static int cmp_u64(const void* a, const void* b) {
  unsigned long long x = *(const unsigned long long*)a;
  unsigned long long y = *(const unsigned long long*)b;
  return (x > y) - (x < y);
}

long long orc_build_csr(int nrows, long long nedges, const int* src,
                        const int* dst, int undirected, int* rowptr,
                        int* colind) {
  long long cap = undirected ? 2 * nedges : nedges;
  unsigned long long* keys =
      (unsigned long long*)malloc((size_t)(cap > 0 ? cap : 1) * sizeof(unsigned long long));
  long long n = 0, i, kept = 0;
  int r;
  for (i = 0; i < nedges; ++i) {
    unsigned long long a = (unsigned int)src[i], b = (unsigned int)dst[i];
    keys[n++] = (a << 32) | b;
    if (undirected && a != b) keys[n++] = (b << 32) | a;
  }
  qsort(keys, (size_t)n, sizeof(unsigned long long), cmp_u64);
  for (r = 0; r <= nrows; ++r) rowptr[r] = 0;
  for (i = 0; i < n; ++i) {
    int a = (int)(keys[i] >> 32), b = (int)(keys[i] & 0xffffffffu);
    if (a == b) continue;                              /* self-loop */
    if (i > 0 && keys[i] == keys[i - 1]) continue;     /* duplicate */
    colind[kept++] = b;
    rowptr[a + 1]++;
  }
  for (r = 0; r < nrows; ++r) rowptr[r + 1] += rowptr[r];
  free(keys);
  return kept;
}

/* reference graphblas/backend/cuda/tri.hpp:21-48 */
long long orc_tril(int nrows, int* rowptr, int* colind) {
  long long kept = 0, read = 0;
  int row;
  for (row = 0; row < nrows; ++row) {
    long long end = rowptr[row + 1];
    rowptr[row] = (int)kept;
    for (; read < end; ++read)
      if (colind[read] <= row) colind[kept++] = colind[read];
  }
  rowptr[nrows] = (int)kept;
  return kept;
}

/* ------------------------------------------------------------------------- */
/* R-MAT generator (ours; the reference ships none).  One SplitMix64 draw per */
/* (edge, level); the top 32 bits pick the quadrant against integer           */
/* thresholds floor(0.57*2^32), +floor(0.19*2^32), +floor(0.19*2^32).         */
/* ------------------------------------------------------------------------- */
static unsigned long long splitmix64(unsigned long long x) {
  unsigned long long z = x + 0x9E3779B97F4A7C15ull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

void orc_rmat_edges(int scale, long long nedges, unsigned long long seed,
                    long long first_edge, int* src, int* dst) {
  const unsigned int T1 = 2448131358u, T2 = 3264175144u, T3 = 4080218930u;
  long long e;
  for (e = 0; e < nedges; ++e) {
    unsigned long long ge = (unsigned long long)(first_edge + e);
    unsigned int s = 0, d = 0;
    int l;
    for (l = 0; l < scale; ++l) {
      unsigned long long key = (seed << 48) ^ (ge << 6) ^ (unsigned long long)l;
      unsigned int r = (unsigned int)(splitmix64(key) >> 32);
      unsigned int sb = (r >= T2) ? 1u : 0u;
      unsigned int db = ((r >= T1 && r < T2) || r >= T3) ? 1u : 0u;
      s = (s << 1) | sb;
      d = (d << 1) | db;
    }
    src[e] = (int)s;
    dst[e] = (int)d;
  }
}
