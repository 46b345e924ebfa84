/* vw_outlier_oracle.c -- see vw_outlier_oracle.h.  Built with the main oracle's flags (-O3 -msse4.1 -ffp-contract=off): the
 * float steps are float32 operations (x86-64 SSE, FLT_EVAL_METHOD 0), the double steps double, nothing is contracted.
 * One body per method serves both pixel types through the macros below; the type-specific steps are the difference
 * (*acc)[0] - (*col_acc)[0] and the length std::abs(dx) + std::abs(dy), both taken in the pixel type. */
#include "vw_outlier_oracle.h"

#include <math.h>
#include <stdlib.h>

static int clampo(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

static int cmp_double(const void* a, const void* b) {
  const double x = *(const double*)a, y = *(const double*)b;
  return x < y ? -1 : (x > y ? 1 : 0);
}

/* fabs((*acc)[0] - (*col_acc)[0]) and std::abs(v[0]) + std::abs(v[1]) in the pixel type, then as doubles */
static double absdiff_i(int32_t a, int32_t b) { return fabs((double)(a - b)); }
static double absdiff_f(float a, float b) { const float d = a - b; return fabs((double)d); }
static double len_i(int32_t x, int32_t y) { return (double)(abs(x) + abs(y)); }
static double len_f(float x, float y) { const float s = fabsf(x) + fabsf(y); return (double)s; }

/* the pixel at (x, y) of edge_extend(in, ConstantEdgeExtension()) */
#define AT(in, w, h, x, y) ((in)[(size_t)clampo((y), 0, (h) - 1) * (w) + clampo((x), 0, (w) - 1)])

#define OUTLIER_FUNCS(S, P)                                                                                               \
  /* RmOutliersUsingThreshFunc::operator() at (cx, cy) (DisparityMap.h:359-386) */                                       \
  static P thresh_at_##S(const P* in, int w, int h, int cx, int cy, int hx, int hy, double pt, double rt) {                \
    const P c = AT(in, w, h, cx, cy);                                                                                     \
    if (c.valid != 0) {                                                                                                   \
      int matched = 0, total = 0;                                                                                         \
      for (int yk = -hy; yk <= hy; ++yk)                                                                                  \
        for (int xk = -hx; xk <= hx; ++xk) {                                                                              \
          const P n = AT(in, w, h, cx + xk, cy + yk);                                                                     \
          if (n.valid != 0 && absdiff_##S(c.dx, n.dx) <= pt && absdiff_##S(c.dy, n.dy) <= pt) matched++;                  \
          total++;                                                                                                        \
        }                                                                                                                 \
      if (((double)matched / (double)total) < rt) { const P z = {0, 0, 0}; return z; }                                    \
    }                                                                                                                     \
    return c;                                                                                                             \
  }                                                                                                                       \
  /* RmOutliersUsingMeanFunc::operator() (:485-553).  len: scratch for (2hx+1)(2hy+1) doubles */                          \
  static P mean_at_##S(const P* in, int w, int h, int cx, int cy, int hx, int hy, double mdsq, double* len) {             \
    const P c = AT(in, w, h, cx, cy);                                                                                     \
    if (!(c.valid != 0)) return c;                                                                                        \
    size_t n = 0;                                                                                                         \
    for (int yk = -hy; yk <= hy; ++yk)                                                                                    \
      for (int xk = -hx; xk <= hx; ++xk) {                                                                                \
        const P q = AT(in, w, h, cx + xk, cy + yk);                                                                       \
        if (q.valid != 0) len[n++] = len_##S(q.dx, q.dy);                                                                 \
      }                                                                                                                   \
    qsort(len, n, sizeof(double), cmp_double);                                                                            \
    double cutoff = 0.0;                                                                                                  \
    if (n) cutoff = 2.0 * len[(int)(0.75 * n)];                                                                           \
    size_t matched = 0;                                                                                                   \
    double meanX = 0, meanY = 0;                                                                                          \
    for (int yk = -hy; yk <= hy; ++yk) {                                                                                  \
      int col = cx - hx;                                   /* col_acc */                                                 \
      for (int xk = -hx; xk <= hx; ++xk) {                                                                                \
        const P q = AT(in, w, h, col, cy + yk);                                                                           \
        if (q.valid != 0) {                                                                                               \
          const double val = len_##S(q.dx, q.dy);                                                                         \
          if (val > cutoff) continue;                      /* col_acc does not advance */                                \
          meanX += q.dx;                                                                                                  \
          meanY += q.dy;                                                                                                  \
          matched++;                                                                                                      \
        }                                                                                                                 \
        col++;                                                                                                            \
      }                                                                                                                   \
    }                                                                                                                     \
    double errorSq = mdsq + 1.0;                                                                                          \
    if (matched > 0) {                                                                                                    \
      meanX = meanX / (double)matched;                                                                                    \
      meanY = meanY / (double)matched;                                                                                    \
      const double thisX = c.dx, thisY = c.dy;                                                                            \
      errorSq = (thisX - meanX) * (thisX - meanX) + (thisY - meanY) * (thisY - meanY);                                    \
    }                                                                                                                     \
    if (errorSq > mdsq) { const P z = {0, 0, 0}; return z; }                                                              \
    return c;                                                                                                             \
  }                                                                                                                       \
  /* RmOutliersUsingStdDev::operator() (:647-723), with value vectors that hold every valid window pixel */               \
  static P stddev_at_##S(const P* in, int w, int h, int cx, int cy, int hx, int hy, double pt, double rt, double* xVals) { \
    const P c = AT(in, w, h, cx, cy);                                                                                     \
    if (!(c.valid != 0)) return c;                                                                                        \
    double* yVals = xVals + (size_t)(2 * hx + 1) * (2 * hy + 1);                                                          \
    size_t matched = 0;                                                                                                   \
    double meanX = 0, meanY = 0;                                                                                          \
    for (int yk = -hy; yk <= hy; ++yk)                                                                                    \
      for (int xk = -hx; xk <= hx; ++xk) {                                                                                \
        const P q = AT(in, w, h, cx + xk, cy + yk);                                                                       \
        if (q.valid != 0) {                                                                                               \
          xVals[matched] = q.dx;                                                                                          \
          yVals[matched] = q.dy;                                                                                          \
          meanX += q.dx;                                                                                                  \
          meanY += q.dy;                                                                                                  \
          matched++;                                                                                                      \
        }                                                                                                                 \
      }                                                                                                                   \
    if (matched == 0) { const P z = {0, 0, 0}; return z; }                                                                \
    meanX = meanX / (double)matched;                                                                                      \
    meanY = meanY / (double)matched;                                                                                      \
    double sumDiffX = 0, sumDiffY = 0;                                                                                    \
    for (size_t i = 0; i < matched; ++i) {                                                                                \
      const double diffX = xVals[i] - meanX, diffY = yVals[i] - meanY;                                                    \
      sumDiffX += diffX * diffX;                                                                                          \
      sumDiffY += diffY * diffY;                                                                                          \
    }                                                                                                                     \
    double stdDevX = sqrt(sumDiffX / (double)matched), stdDevY = sqrt(sumDiffY / (double)matched);                        \
    if (stdDevX < rt) stdDevX = rt;                                                                                       \
    if (stdDevY < rt) stdDevY = rt;                                                                                       \
    const double thisX = c.dx, thisY = c.dy;                                                                              \
    const double errorX = fabs(thisX - meanX), errorY = fabs(thisY - meanY);                                              \
    if ((errorX > pt * stdDevX) || (errorY > pt * stdDevY)) { const P z = {0, 0, 0}; return z; }                          \
    return c;                                                                                                             \
  }                                                                                                                       \
  static P pass1_at_##S(int method, const P* in, int w, int h, int cx, int cy, int hx, int hy, double pt, double rt,       \
                        double mdsq, double* scratch) {                                                                   \
    if (method == 0) return thresh_at_##S(in, w, h, cx, cy, hx, hy, pt, rt);                                              \
    if (method == 1) return mean_at_##S(in, w, h, cx, cy, hx, hy, mdsq, scratch);                                         \
    return stddev_at_##S(in, w, h, cx, cy, hx, hy, pt, rt, scratch);                                                      \
  }                                                                                                                       \
  /* rm_outliers_using_* (pass 1 over the edge-extended input) or disparity_cleanup_using_* (pass 1, then                 \
   * RmOutliersUsingThreshFunc(1, 1, 3.0, 0.2) over pass 1 WITHOUT a second edge extension: the border windows read pass 1 \
   * evaluated at out-of-image centres, Image/PerPixelAccessorViews.h:63-85) */                                           \
  static int filter_##S(int method, int cleanup, const P* in, int w, int h, int hx, int hy, double pt, double rt,         \
                        double mmd, P* out) {                                                                             \
    const double mdsq = mmd * mmd;                         /* m_max_mean_diffSq */                                       \
    double* scratch = (double*)malloc(2 * (size_t)(2 * hx + 1) * (2 * hy + 1) * sizeof(double));                          \
    if (!scratch) return -2;                                                                                              \
    if (!cleanup) {                                                                                                       \
      for (int y = 0; y < h; ++y)                                                                                         \
        for (int x = 0; x < w; ++x) out[(size_t)y * w + x] = pass1_at_##S(method, in, w, h, x, y, hx, hy, pt, rt, mdsq, scratch); \
    } else {                                                                                                              \
      const int pw = w + 2, ph = h + 2;                                                                                   \
      P* p1 = (P*)malloc((size_t)pw * ph * sizeof(P));                                                                    \
      if (!p1) { free(scratch); return -2; }                                                                              \
      for (int y = -1; y <= h; ++y)                                                                                       \
        for (int x = -1; x <= w; ++x)                                                                                     \
          p1[(size_t)(y + 1) * pw + (x + 1)] = pass1_at_##S(method, in, w, h, x, y, hx, hy, pt, rt, mdsq, scratch);      \
      for (int y = 0; y < h; ++y)                   /* every window lies inside p1: no clamping happens */               \
        for (int x = 0; x < w; ++x) out[(size_t)y * w + x] = thresh_at_##S(p1, pw, ph, x + 1, y + 1, 1, 1, 3.0, 0.20);   \
      free(p1);                                                                                                           \
    }                                                                                                                     \
    free(scratch);                                                                                                        \
    return 0;                                                                                                             \
  }

OUTLIER_FUNCS(i, vwo_outi_t)
OUTLIER_FUNCS(f, vwo_outf_t)

int vwo_outlier_filter(int method, int cleanup, int pixel_type, const void* in, int w, int h, int half_h, int half_v,
                       double pixel_threshold, double rejection_threshold, double max_mean_diff, void* out) {
  if (half_h <= 0 || half_v <= 0 || method < 0 || method > 2 || pixel_type < 0 || pixel_type > 1) return -1;
  if (w <= 0 || h <= 0) return 0;
  if (pixel_type == 0)
    return filter_i(method, cleanup != 0, (const vwo_outi_t*)in, w, h, half_h, half_v, pixel_threshold, rejection_threshold,
                    max_mean_diff, (vwo_outi_t*)out);
  return filter_f(method, cleanup != 0, (const vwo_outf_t*)in, w, h, half_h, half_v, pixel_threshold, rejection_threshold,
                  max_mean_diff, (vwo_outf_t*)out);
}
