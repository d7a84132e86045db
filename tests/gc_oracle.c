/* tests/gc_oracle.c — CPU greedy graph colouring, the checker of the device colouring
 * (backend/cuda/kernels/color.cuh).  TEST INFRASTRUCTURE ONLY: tests/, smoke() and
 * tools/bench_gc.py load it (tests/greedy_oracle.py); the product never does.
 *
 * Ours: the reference's SimpleReferenceGc orders vertices with std::mt19937 and cannot
 * pin a hashed order, so this restatement is pinned by properties instead
 * (tests/test_gc_oracle.py).
 *
 * orc_gc: greedy first-fit colouring in decreasing priority p(v) = (h(seed, v), v)
 * order, h(seed, v) = fmix32(v ^ (seed * 0x9E3779B9)) (murmur3 finaliser, 32-bit):
 * colors[v] = the smallest c >= 1 no higher-priority neighbour holds.  The CSR's
 * pattern must be symmetric; self-loops are ignored.  Returns the number of colours
 * (0 when nrows == 0); *depth (may be NULL) = the Jones-Plassmann round count,
 * 1 + the longest chain of higher-priority neighbours. */
#include <stdlib.h>

int orc_gc(int nrows, const int* rowptr, const int* colind, unsigned seed,
           int* colors, int* depth);

static unsigned int gc_hash(unsigned int seed, unsigned int v) {
  unsigned int x = v ^ (seed * 0x9E3779B9u);
  x ^= x >> 16; x *= 0x85EBCA6Bu;
  x ^= x >> 13; x *= 0xC2B2AE35u;
  x ^= x >> 16;
  return x;
}

static int gc_key_desc(const void* a, const void* b) {
  const unsigned long long x = *(const unsigned long long*)a;
  const unsigned long long y = *(const unsigned long long*)b;
  return x < y ? 1 : (x > y ? -1 : 0);
}

int orc_gc(int nrows, const int* rowptr, const int* colind, unsigned seed,
           int* colors, int* depth) {
  unsigned long long* order;
  int* stamp;
  int* level;
  int v, ncolors = 0, deepest = 0;
  if (depth != NULL) *depth = 0;
  if (nrows <= 0) return 0;
  order = (unsigned long long*)malloc((size_t)nrows * sizeof(*order));
  stamp = (int*)calloc((size_t)nrows + 2, sizeof(int));
  level = (int*)calloc((size_t)nrows, sizeof(int));
  for (v = 0; v < nrows; ++v) {
    order[v] = ((unsigned long long)gc_hash(seed, (unsigned int)v) << 32) | (unsigned int)v;
    colors[v] = 0;
  }
  qsort(order, (size_t)nrows, sizeof(*order), gc_key_desc);
  for (v = 0; v < nrows; ++v) {
    const int x = (int)(order[v] & 0xffffffffu);
    int e, c = 1, lv = 0;
    for (e = rowptr[x]; e < rowptr[x + 1]; ++e) {
      const int u = colind[e];
      if (colors[u] != 0) {          /* coloured before x: a higher-priority neighbour */
        stamp[colors[u]] = x + 1;
        if (level[u] > lv) lv = level[u];
      }
    }
    while (stamp[c] == x + 1) ++c;
    colors[x] = c;
    level[x] = lv + 1;
    if (c > ncolors) ncolors = c;
    if (lv + 1 > deepest) deepest = lv + 1;
  }
  free(order);
  free(stamp);
  free(level);
  if (depth != NULL) *depth = deepest;
  return ncolors;
}
