/* vw_ipmatch_oracle.c -- see vw_ipmatch_oracle.h.  Each function follows the reference's loop and its float / double types. */
#include "vw_ipmatch_oracle.h"

#include <float.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

float vwm_l2(const float* a, const float* b, int dim) {
  const float maxdist = FLT_MAX;
  float dist = 0.0f;
  for (int i = 0; i < dim; i++) {
    dist += (a[i] - b[i]) * (a[i] - b[i]);
    if (dist > maxdist) break;
  }
  return dist;
}

float vwm_hamming(const float* a, const float* b, int dim) {
  const float maxdist = FLT_MAX;
  float dist = 0.0f;
  int d = dim;
  const int num_64 = d / 8;
  d -= num_64 * 8;
  const int num_32 = d / 4;
  uint8_t* p1 = malloc(dim > 0 ? (size_t)dim : 1);
  uint8_t* p2 = malloc(dim > 0 ? (size_t)dim : 1);
  for (int k = 0; k < dim; ++k) {
    p1[k] = (uint8_t)(int)a[k];
    p2[k] = (uint8_t)(int)b[k];
  }
  int i = 0;
  for (int i64 = 0; i64 < num_64; ++i64) {
    uint64_t x, y;
    memcpy(&x, p1 + i, 8);
    memcpy(&y, p2 + i, 8);
    i += 8;
    dist += (float)(size_t)__builtin_popcountll(x ^ y);
    if (dist > maxdist) goto done;
  }
  for (int i32 = 0; i32 < num_32; ++i32) {
    uint32_t x, y;
    memcpy(&x, p1 + i, 4);
    memcpy(&y, p2 + i, 4);
    i += 4;
    dist += (float)(size_t)__builtin_popcount(x ^ y);
    if (dist > maxdist) goto done;
  }
  for (; i < dim; ++i) dist += (float)(size_t)__builtin_popcount((unsigned)(p1[i] ^ p2[i]));
done:
  free(p1);
  free(p2);
  return dist;
}

static int first_bad(const float* d, int n, int dim, long long* elem) {
  for (long long e = 0; e < (long long)n * dim; ++e)
    if (!(d[e] > -1.0f && d[e] < 256.0f)) { *elem = e; return 1; }
  return 0;
}

int vwm_match(int metric, const float* d1, const uint8_t* p1, int n1, const float* d2, const uint8_t* p2, int n2, int dim, double threshold,
              int32_t* index, double* first, double* second, int* bad_list, long long* bad_elem) {
  if (metric == 1) {
    if (8ll * dim > (1ll << 24)) return -4;
    if (n2 > 0 && first_bad(d1, n1, dim, bad_elem)) { *bad_list = 0; return -1; }
    if (n1 > 0 && first_bad(d2, n2, dim, bad_elem)) { *bad_list = 1; return -1; }
  }
  for (int i = 0; i < n1; i++) {
    double first_pick = 1e100, second_pick = 1e100;
    index[i] = -1;
    for (int j = 0; j < n2; j++) {
      if ((p1[i] != 0) != (p2[j] != 0)) continue;
      const float* a = d1 + (size_t)i * dim;
      const float* b = d2 + (size_t)j * dim;
      double distance = metric == 1 ? vwm_hamming(a, b, dim) : vwm_l2(a, b, dim);
      if (distance < first_pick) {
        index[i] = j;
        second_pick = first_pick;
        first_pick = distance;
      } else if (distance < second_pick) {
        second_pick = distance;
      }
    }
    if (first_pick > threshold * second_pick) index[i] = -1;
    if (first) first[i] = first_pick;
    if (second) second[i] = second_pick;
  }
  return 0;
}

/* a sorted array standing in for std::set<std::pair<float, float>> with the pair's operator< */
typedef struct { float a, b; } Pair;
static int pair_less(Pair x, Pair y) { return x.a < y.a || (!(y.a < x.a) && x.b < y.b); }
typedef struct { Pair* v; int n; } PairSet;
static int set_lower(const PairSet* s, Pair p) {
  int lo = 0, hi = s->n;
  while (lo < hi) {
    const int mid = (lo + hi) / 2;
    if (pair_less(s->v[mid], p)) lo = mid + 1; else hi = mid;
  }
  return lo;
}
static int set_find(const PairSet* s, Pair p) {
  const int k = set_lower(s, p);
  return k < s->n && !pair_less(p, s->v[k]);
}
static void set_insert(PairSet* s, Pair p) {
  const int k = set_lower(s, p);
  if (k < s->n && !pair_less(p, s->v[k])) return;
  memmove(s->v + k + 1, s->v + k, (size_t)(s->n - k) * sizeof(Pair));
  s->v[k] = p;
  s->n++;
}

int vwm_remove_duplicates(const float* xy1, const float* xy2, int n, int32_t* keep, int* n_kept) {
  for (int i = 0; i < 2 * n; ++i)
    if (isnan(xy1[i]) || isnan(xy2[i])) return -1;
  PairSet s1 = {malloc(sizeof(Pair) * (n > 0 ? n : 1)), 0}, s2 = {malloc(sizeof(Pair) * (n > 0 ? n : 1)), 0};
  int k = 0;
  for (int i = 0; i < n; i++) {
    const int j = n - i - 1;
    const Pair a = {xy1[2 * j], xy1[2 * j + 1]}, b = {xy2[2 * j], xy2[2 * j + 1]};
    if (set_find(&s1, a) || set_find(&s2, b)) continue;
    set_insert(&s1, a);
    set_insert(&s2, b);
    keep[k++] = j;
  }
  for (int i = 0; i < k / 2; ++i) {
    const int32_t t = keep[i];
    keep[i] = keep[k - 1 - i];
    keep[k - 1 - i] = t;
  }
  *n_kept = k;
  free(s1.v);
  free(s2.v);
  return 0;
}
