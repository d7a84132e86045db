/* The CPU label propagation the device cdlp is checked against: a plain restatement of
 * algorithm::cdlp (LDBC Graphalytics CDLP).  Test infrastructure written for this project.
 *
 * The arc i -> j when the CSR stores (i, j) and i != j.  L_0(v) = v.  Iteration k: M(v)
 * = the labels L_{k-1}(u) of v's out-neighbours and of its in-neighbours, an arc stored
 * both ways counted twice; L_k(v) = the smallest label of highest multiplicity in M(v),
 * L_{k-1}(v) when M(v) is empty.  Stops after max_iter iterations or after the first
 * that changes no label.  Counting uses one counter per label, reset through the list
 * of labels it touched, so an iteration costs one pass over the lists. */
#include <stdlib.h>
#include <string.h>

/* labels [n] receives L_T; *iterations = T; returns the number of distinct labels, -2
 * when out of memory. */
long long orc_cdlp(int n, const int* rp, const int* ci, int max_iter, int* labels,
                   int* iterations) {
  const long long nnz = n > 0 ? rp[n] : 0;
  const size_t nz = (size_t)(nnz > 0 ? nnz : 1), nv = (size_t)(n > 0 ? n : 1);
  int* cp = (int*)calloc(nv + 1, sizeof(int));        /* the in-lists (CSC) */
  int* ri = (int*)malloc(nz*sizeof(int));
  int* fill = (int*)malloc(nv*sizeof(int));
  int* prev = (int*)malloc(nv*sizeof(int));
  int* count = (int*)calloc(nv, sizeof(int));
  int* touched = (int*)malloc(2*nz*sizeof(int) + sizeof(int));
  if (!cp || !ri || !fill || !prev || !count || !touched) {
    free(cp); free(ri); free(fill); free(prev); free(count); free(touched);
    return -2;
  }
  for (long long k = 0; k < nnz; ++k) ++cp[ci[k] + 1];
  for (int i = 0; i < n; ++i) cp[i + 1] += cp[i];
  for (int i = 0; i < n; ++i) fill[i] = cp[i];
  for (int i = 0; i < n; ++i)
    for (int k = rp[i]; k < rp[i + 1]; ++k) ri[fill[ci[k]]++] = i;
  for (int i = 0; i < n; ++i) labels[i] = i;
  int t = 0;
  while (t < max_iter) {
    ++t;
    memcpy(prev, labels, (size_t)n*sizeof(int));
    long long changed = 0;
    for (int v = 0; v < n; ++v) {
      int m = 0;
      for (int k = rp[v]; k < rp[v + 1]; ++k)
        if (ci[k] != v && count[prev[ci[k]]]++ == 0) touched[m++] = prev[ci[k]];
      for (int k = cp[v]; k < cp[v + 1]; ++k)
        if (ri[k] != v && count[prev[ri[k]]]++ == 0) touched[m++] = prev[ri[k]];
      if (m == 0) continue;
      int best = touched[0], bc = count[touched[0]];
      for (int q = 0; q < m; ++q) {
        const int x = touched[q], c = count[x];
        if (c > bc || (c == bc && x < best)) { best = x; bc = c; }
        count[x] = 0;
      }
      changed += best != prev[v];
      labels[v] = best;
    }
    if (changed == 0) break;
  }
  *iterations = t;
  long long distinct = 0;
  memset(count, 0, nv*sizeof(int));
  for (int v = 0; v < n; ++v)
    if (count[labels[v]]++ == 0) ++distinct;
  free(cp); free(ri); free(fill); free(prev); free(count); free(touched);
  return distinct;
}
