/*
 * vw_smoothing_oracle.c -- CPU restatement of the disparity smoothing filters of Stereo/Algorithms.{h,cc}.
 * TEST INFRASTRUCTURE ONLY: see vw_smoothing_oracle.h.  Same build flags as the main oracle (oracle/Makefile):
 * -O3 -msse4.1 -ffp-contract=off, so no FMA contraction, like the reference's SSE build.
 *
 * Both disparity filters begin with
 * `disparity_out = disparity_in;`, the implicitly-declared copy assignment of ImageView
 * (Image/ImageView.h:95-148 declares no other non-template one), which shares the buffer: the
 * loops below therefore read and write ONE image, in raster order, exactly as the reference does.
 * Float disparity pixels are {dx, dy, valid} triples, pitch in pixels; valid means valid != 0.
 */
#include "vw_smoothing_oracle.h"
#include "vw_oracle.h"
#include <limits.h>
#include <math.h>
#include <stdlib.h>

static int clampi(int v, int lo, int hi) { return v < lo ? lo : (v > hi ? hi : v); }

static int cmp_double(const void* a, const void* b) {
  double x = *(const double*)a, y = *(const double*)b;
  return (x > y) - (x < y);
}

/* math::destructive_median (Math/Functors.h:393-398): sort, middle value or mean of the two */
double vwo_destructive_median(double* v, int n) {
  qsort(v, (size_t)n, sizeof(double), cmp_double);
  return n % 2 ? v[n / 2] : (v[n / 2 - 1] + v[n / 2]) / 2.0;
}

int vwo_disparity_median_filter(float* d, int w, int h, int pitch, int kernel_size) {
  int half = (kernel_size - 1) / 2;                                            /* :30 */
  if (kernel_size < 3) return 0;                                               /* :34-35 */
  int num = kernel_size * kernel_size;
  double* dx = (double*)malloc((size_t)num * sizeof(double));
  double* dy = (double*)malloc((size_t)num * sizeof(double));
  if (!dx || !dy) { free(dx); free(dy); return -2; }
  for (int row = half; row < h - half; ++row)                                  /* :38-39 */
    for (int col = half; col < w - half; ++col) {
      float* p = d + ((size_t)row * pitch + col) * 3;
      if (p[2] == 0.0f) continue;                                              /* :41-42 */
      int n = 0;
      for (int r = row - half; r <= row + half; ++r)                           /* :47-55 */
        for (int c = col - half; c <= col + half; ++c) {
          const float* q = d + ((size_t)r * pitch + c) * 3;
          if (q[2] != 0.0f) { dx[n] = q[0]; dy[n] = q[1]; ++n; }
        }
      if (n == 0) continue;
      double mx = vwo_destructive_median(dx, n), my = vwo_destructive_median(dy, n);
      p[0] = (float)mx; p[1] = (float)my; p[2] = 1.0f;                         /* :64 */
    }
  free(dx); free(dy);
  return 0;
}

/* texture_measure (Algorithms.h:144-209) of a plain float image: every pixel is valid, so the
 * window count is (2*half+1)^2.  dx / dy = derivative_filter(img, 1, 0) / (img, 0, 1)
 * (Image/Filter.h:304-308, Filter.tcc:91-118): kernel {0.5, 0, -0.5}, constant edge. */
int vwo_texture_measure(const float* img, int w, int h, int pitch, int kernel_size, double gradient_weight,
                        double stddev_weight, float* out) {
  if (w <= 0 || h <= 0 || kernel_size < 1) return -1;
  static const float dk[3] = {0.5f, 0.0f, -0.5f};
  float* dxi = (float*)malloc((size_t)w * h * sizeof(float));
  float* dyi = (float*)malloc((size_t)w * h * sizeof(float));
  if (!dxi || !dyi) { free(dxi); free(dyi); return -2; }
  vwo_separable_convolve(img, w, h, pitch, dk, 3, NULL, 0, 0, dxi);
  vwo_separable_convolve(img, w, h, pitch, NULL, 0, dk, 3, 0, dyi);
  int half = (kernel_size - 1) / 2;                                            /* :156 */
  for (int row = 0; row < h; ++row)                                            /* :167-168 */
    for (int col = 0; col < w; ++col) {
      double mean = 0, count = 0;                                              /* :176-187 */
      for (int r = row - half; r <= row + half; ++r)
        for (int c = col - half; c <= col + half; ++c) {
          mean += img[(size_t)clampi(r, 0, h - 1) * pitch + clampi(c, 0, w - 1)];
          count += 1.0;
        }
      mean /= count;
      double grad = 0, sd = 0;                                                 /* :189-198 */
      for (int r = row - half; r <= row + half; ++r)
        for (int c = col - half; c <= col + half; ++c) {
          size_t i = (size_t)clampi(r, 0, h - 1) * w + clampi(c, 0, w - 1);
          float g = fabsf(dxi[i]) + fabsf(dyi[i]);                             /* float add, then widened */
          grad += g;
          double e = img[(size_t)clampi(r, 0, h - 1) * pitch + clampi(c, 0, w - 1)] - mean;
          sd += e * e;                                                         /* pow(e, 2) */
        }
      grad = grad / (2.0 * count);                                             /* :200-204 */
      sd = sqrt(sd / count);
      out[(size_t)row * w + col] = (float)(grad * gradient_weight + sd * stddev_weight);
    }
  free(dxi); free(dyi);
  return 0;
}

/* texture_preserving_disparity_filter<float> (Algorithms.h:213-281); tex has the disparity's size */
int vwo_texture_preserving_disparity_filter(float* d, int w, int h, int pitch, const float* tex, int tpitch,
                                            float texture_max, int max_kernel_size) {
  float scale = max_kernel_size / texture_max;                                 /* :222 */
  if (max_kernel_size < 3 || texture_max <= 0) return 0;                       /* :228-229 */
  for (int row = 0; row < h; ++row)                                            /* :235-236 */
    for (int col = 0; col < w; ++col) {
      float* p = d + ((size_t)row * pitch + col) * 3;
      float t = tex[(size_t)row * tpitch + col];
      if (p[2] == 0.0f || t < 0) continue;                                     /* :240-241 */
      float adj = texture_max - t;                                             /* :243-245 */
      if (adj < 0) adj = 0;
      float f = floorf(adj * scale);
      /* int(floor(...)): out of range (NaN, inf) converts to INT_MIN on x86-64, which is skipped below */
      int k = (f >= -2147483648.0f && f < 2147483648.0f) ? (int)f : INT_MIN;   /* :246 */
      if (k % 2 == 0) k += 1;                                                  /* :247-248 */
      if (k < 3 || k > max_kernel_size) continue;                              /* :249-257 */
      int half = (k - 1) / 2;
      double sx = 0, sy = 0, count = 0;                                        /* :263-273 */
      for (int r = row - half; r <= row + half; ++r)
        for (int c = col - half; c <= col + half; ++c) {
          const float* q = d + ((size_t)clampi(r, 0, h - 1) * pitch + clampi(c, 0, w - 1)) * 3;
          if (q[2] != 0.0f) { sx += q[0]; sy += q[1]; count += 1.0; }
        }
      if (count < 1.0) continue;                                               /* :274-275 */
      p[0] = (float)(sx / count); p[1] = (float)(sy / count); p[2] = 1.0f;     /* :277 */
    }
  return 0;
}
