/* CPU k-truss and truss decomposition: the checker of the device ktruss and trussness
 * (tests/truss_reference.py binds it).
 *
 * Input: a CSR (n, rowptr, colind) with sorted, duplicate-free rows and a symmetric
 * pattern; entries with colind == row (self-loops) are skipped.  Each undirected edge
 * {u, v} is counted once, from its (min, max) entry.
 *
 * orc_trussness: the sequential bucket peel of Wang & Cheng (VLDB 2012).  Edges sit in
 * buckets by current support, as in the Batagelj-Zaversnik core decomposition; the
 * edge of least support s is removed with tau = s + 2, and each triangle it still
 * closes lowers the support of its other two edges when theirs is above s.
 * orc_ktruss: a queue peel for one k: every edge with support below k - 2 is queued,
 * and removing one lowers the support of the other two edges of each triangle it still
 * closes, queueing any that falls below k - 2.
 * Both return per entry, in both directions, tau or the k-truss support (-1 for a
 * removed edge or a self-loop). */
#include <stdlib.h>

typedef struct {
  int n;
  const int* ptr;
  const int* ind;
  long long nnz;
  int* eid;          /* [nnz] the canonical entry of each entry's edge, -1 for a loop */
  int* row;          /* [nnz] the row of each entry */
} Graph;

static int lower_bound(const int* a, int lo, int hi, int key) {
  while (lo < hi) {
    int mid = lo + (hi - lo)/2;
    if (a[mid] < key) lo = mid + 1; else hi = mid;
  }
  return lo;
}

static int graph_init(Graph* g, int n, const int* ptr, const int* ind) {
  g->n = n;
  g->ptr = ptr;
  g->ind = ind;
  g->nnz = n > 0 ? ptr[n] : 0;
  g->eid = (int*)malloc((size_t)(g->nnz > 0 ? g->nnz : 1)*sizeof(int));
  g->row = (int*)malloc((size_t)(g->nnz > 0 ? g->nnz : 1)*sizeof(int));
  if (!g->eid || !g->row) return -1;
  for (int u = 0; u < n; ++u)
    for (int p = ptr[u]; p < ptr[u + 1]; ++p) {
      int v = ind[p];
      g->row[p] = u;
      if (u < v) g->eid[p] = p;
      else if (u > v) g->eid[p] = lower_bound(ind, ptr[v], ptr[v + 1], u);
      else g->eid[p] = -1;
    }
  return 0;
}

static void graph_free(Graph* g) {
  free(g->eid);
  free(g->row);
}

/* Calls visit(ctx, f, g) for each w in N(u) ∩ N(v), w not u or v, with f and g the
 * canonical entries of {u, w} and {v, w}. */
typedef void (*Visit)(void* ctx, int f, int g);

static void triangles(const Graph* G, int e, Visit visit, void* ctx) {
  int u = G->row[e], v = G->ind[e];
  int p = G->ptr[u], pe = G->ptr[u + 1], q = G->ptr[v], qe = G->ptr[v + 1];
  int swap = pe - p > qe - q;    /* p walks the shorter list */
  if (swap) {
    int t = p; p = q; q = t;
    t = pe; pe = qe; qe = t;
  }
  int search = qe - q > 16*(pe - p);   /* much longer: search it, else merge */
  while (p < pe && q < qe) {
    int a = G->ind[p];
    if (search) q = lower_bound(G->ind, q, qe, a);
    if (q >= qe) break;
    int b = G->ind[q];
    if (a < b) ++p;
    else if (b < a) ++q;
    else {
      if (a != u && a != v)
        visit(ctx, swap ? G->eid[q] : G->eid[p], swap ? G->eid[p] : G->eid[q]);
      ++p;
      ++q;
    }
  }
}

/* sup[e] = the triangles of G on each canonical entry e, each triangle found once:
 * edges are oriented from lower to higher (degree, id), and for each u the out-lists of
 * its out-neighbours are matched against a mark of its own out-list (Chiba-Nishizeki
 * order, so a hub's long list is never walked once per neighbour). */
static int supports(const Graph* G, int* sup) {
  int n = G->n;
  long long nnz = G->nnz;
  int* optr = (int*)calloc((size_t)n + 1, sizeof(int));
  int* oind = (int*)malloc((size_t)(nnz > 0 ? nnz : 1)*sizeof(int));
  int* oeid = (int*)malloc((size_t)(nnz > 0 ? nnz : 1)*sizeof(int));
  int* owner = (int*)malloc((size_t)(n > 0 ? n : 1)*sizeof(int));
  int* mark = (int*)malloc((size_t)(n > 0 ? n : 1)*sizeof(int));
  if (!optr || !oind || !oeid || !owner || !mark) return -1;
#define DEG(x) (G->ptr[(x) + 1] - G->ptr[(x)])
#define BEFORE(x, y) (DEG(x) < DEG(y) || (DEG(x) == DEG(y) && (x) < (y)))
  for (int u = 0; u < n; ++u) {
    owner[u] = -1;
    optr[u + 1] = optr[u];
    for (int p = G->ptr[u]; p < G->ptr[u + 1]; ++p) {
      int w = G->ind[p];
      if (w != u && BEFORE(u, w)) {
        oind[optr[u + 1]] = w;
        oeid[optr[u + 1]] = G->eid[p];
        ++optr[u + 1];
      }
    }
  }
  for (long long e = 0; e < nnz; ++e) sup[e] = 0;
  for (int u = 0; u < n; ++u) {
    for (int p = optr[u]; p < optr[u + 1]; ++p) {
      owner[oind[p]] = u;
      mark[oind[p]] = oeid[p];
    }
    for (int p = optr[u]; p < optr[u + 1]; ++p) {
      int v = oind[p];
      for (int q = optr[v]; q < optr[v + 1]; ++q) {
        int w = oind[q];
        if (owner[w] == u) {
          ++sup[oeid[p]];
          ++sup[oeid[q]];
          ++sup[mark[w]];
        }
      }
    }
  }
#undef BEFORE
#undef DEG
  free(optr); free(oind); free(oeid); free(owner); free(mark);
  return 0;
}

/* ---- truss decomposition -------------------------------------------------------------- */

typedef struct {
  int* sup;
  int* pos;          /* an edge's place in order */
  int* order;        /* edges by support */
  int* bin;          /* first place of each support */
  char* gone;
  int s;             /* the support of the edge being removed */
} Buckets;

static void lower(Buckets* b, int f) {
  if (b->sup[f] <= b->s) return;
  int sf = b->sup[f];
  int first = b->bin[sf];
  int other = b->order[first];
  if (other != f) {               /* f to the front of its bucket */
    int pf = b->pos[f];
    b->order[first] = f;
    b->pos[f] = first;
    b->order[pf] = other;
    b->pos[other] = pf;
  }
  b->bin[sf] += 1;
  b->sup[f] -= 1;
}

static void peel_visit(void* ctx, int f, int g) {
  Buckets* b = (Buckets*)ctx;
  if (b->gone[f] || b->gone[g]) return;
  lower(b, f);
  lower(b, g);
}

int orc_trussness(int n, const int* ptr, const int* ind, int* tau) {
  Graph G;
  if (graph_init(&G, n, ptr, ind)) return -1;
  long long nnz = G.nnz;
  size_t cap = (size_t)(nnz > 0 ? nnz : 1);
  Buckets b;
  b.sup = (int*)malloc(cap*sizeof(int));
  b.pos = (int*)malloc(cap*sizeof(int));
  b.order = (int*)malloc(cap*sizeof(int));
  b.bin = (int*)calloc((size_t)n + 2, sizeof(int));
  b.gone = (char*)calloc(cap, 1);
  if (supports(&G, b.sup)) return -1;
  int m = 0, maxs = 0;
  for (long long e = 0; e < nnz; ++e)
    if (G.eid[e] == e) {
      ++m;
      if (b.sup[e] > maxs) maxs = b.sup[e];
      b.bin[b.sup[e]] += 1;
    }
  int start = 0;
  for (int s = 0; s <= maxs; ++s) {   /* bin[s] = first place of support s */
    int c = b.bin[s];
    b.bin[s] = start;
    start += c;
  }
  for (long long e = 0; e < nnz; ++e)
    if (G.eid[e] == e) {
      b.pos[e] = b.bin[b.sup[e]]++;
      b.order[b.pos[e]] = (int)e;
    }
  for (int s = maxs; s > 0; --s) b.bin[s] = b.bin[s - 1];
  b.bin[0] = 0;
  int kmax = 0;
  for (int i = 0; i < m; ++i) {
    int e = b.order[i];
    b.s = b.sup[e];
    tau[e] = b.s + 2;
    if (tau[e] > kmax) kmax = tau[e];
    b.gone[e] = 1;
    triangles(&G, e, peel_visit, &b);
  }
  for (long long p = 0; p < nnz; ++p) tau[p] = G.eid[p] >= 0 ? tau[G.eid[p]] : -1;
  free(b.sup); free(b.pos); free(b.order); free(b.bin); free(b.gone);
  graph_free(&G);
  return kmax;
}

/* ---- one k-truss ---------------------------------------------------------------------- */

typedef struct {
  int* sup;
  char* gone;        /* removed or queued */
  int* queue;
  long long tail;
  int k;
} Queue;

static void drop(Queue* q, int f) {
  q->sup[f] -= 1;
  if (!q->gone[f] && q->sup[f] < q->k - 2) {
    q->gone[f] = 1;
    q->queue[q->tail++] = f;
  }
}

static char* g_dead;   /* edges whose triangles are already charged */

static void ktruss_visit(void* ctx, int f, int g) {
  Queue* q = (Queue*)ctx;
  if (g_dead[f] || g_dead[g]) return;
  drop(q, f);
  drop(q, g);
}

long long orc_ktruss(int n, const int* ptr, const int* ind, int k, int* sup) {
  Graph G;
  if (graph_init(&G, n, ptr, ind)) return -1;
  long long nnz = G.nnz;
  size_t cap = (size_t)(nnz > 0 ? nnz : 1);
  Queue q;
  q.sup = sup;
  q.gone = (char*)calloc(cap, 1);
  q.queue = (int*)malloc(cap*sizeof(int));
  q.tail = 0;
  q.k = k;
  g_dead = (char*)calloc(cap, 1);
  if (supports(&G, sup)) return -1;
  for (long long e = 0; e < nnz; ++e)
    if (G.eid[e] == e && sup[e] < k - 2) {
      q.gone[e] = 1;
      q.queue[q.tail++] = (int)e;
    }
  for (long long h = 0; h < q.tail; ++h) {
    int e = q.queue[h];
    g_dead[e] = 1;
    triangles(&G, e, ktruss_visit, &q);
  }
  long long kept = 0;
  for (long long e = 0; e < nnz; ++e)
    if (G.eid[e] == e && !q.gone[e]) ++kept;
  for (long long p = nnz - 1; p >= 0; --p) {
    int e = G.eid[p];
    sup[p] = (e >= 0 && !q.gone[e]) ? sup[e] : -1;
  }
  free(q.gone); free(q.queue); free(g_dead);
  g_dead = NULL;
  graph_free(&G);
  return kept;
}
