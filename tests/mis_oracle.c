/* tests/mis_oracle.c — CPU greedy maximal independent set, the checker of the device
 * MIS (backend/cuda/kernels/mis.cuh).  TEST INFRASTRUCTURE ONLY: tests/, smoke() and
 * tools/bench_mis.py load it (tests/greedy_oracle.py); the product never does.
 *
 * It includes the colouring checker (tests/gc_oracle.c) for its priority hash gc_hash
 * and its decreasing-priority order gc_key_desc, so both checkers sort vertices the
 * same way; the library built from this file exports orc_gc too.
 *
 * orc_mis: the greedy maximal independent set in decreasing priority
 * p(v) = (gc_hash(seed, v), v) order over the candidates (cand may be NULL: every
 * vertex; else the vertices with cand[v] != 0): member[v] = 1 iff v is a candidate
 * and no higher-priority candidate neighbour is a member.  The CSR's pattern must be
 * symmetric; self-loops are ignored.  Returns the size of the set; *depth (may be
 * NULL) = the synchronous Luby round count with these fixed priorities: a member's
 * round is 1 + the largest round among its higher-priority candidate neighbours, a
 * non-member candidate's the smallest round among its member neighbours, and depth
 * the largest round (0 without candidates). */
#include <limits.h>

#include "gc_oracle.c"

int orc_mis(int nrows, const int* rowptr, const int* colind, unsigned seed,
            const int* cand, int* member, int* depth);

int orc_mis(int nrows, const int* rowptr, const int* colind, unsigned seed,
            const int* cand, int* member, int* depth) {
  unsigned long long* order;
  int* round;
  int v, size = 0, deepest = 0;
  if (depth != NULL) *depth = 0;
  if (nrows <= 0) return 0;
  order = (unsigned long long*)malloc((size_t)nrows * sizeof(*order));
  round = (int*)calloc((size_t)nrows, sizeof(int));    /* 0: not decided yet */
  for (v = 0; v < nrows; ++v) {
    order[v] = ((unsigned long long)gc_hash(seed, (unsigned int)v) << 32) | (unsigned int)v;
    member[v] = 0;
  }
  qsort(order, (size_t)nrows, sizeof(*order), gc_key_desc);
  for (v = 0; v < nrows; ++v) {
    const int x = (int)(order[v] & 0xffffffffu);
    int e, in = 1, lv = 0, out = INT_MAX;
    if (cand != NULL && cand[x] == 0) continue;
    for (e = rowptr[x]; e < rowptr[x + 1]; ++e) {
      const int u = colind[e];
      if (round[u] == 0) continue;   /* lower priority, not a candidate, or x itself */
      if (member[u]) {
        in = 0;
        if (round[u] < out) out = round[u];
      }
      if (round[u] > lv) lv = round[u];
    }
    member[x] = in;
    round[x] = in ? lv + 1 : out;
    size += in;
    if (round[x] > deepest) deepest = round[x];
  }
  free(order);
  free(round);
  if (depth != NULL) *depth = deepest;
  return size;
}
