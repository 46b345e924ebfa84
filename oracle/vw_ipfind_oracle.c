/* vw_ipfind_oracle.c -- loop-for-loop restatement of ipfind's iagd + sgrad path; see vw_ipfind_oracle.h.
 * Citations are file:line under the reference's src/vw/. */
#include "vw_ipfind_oracle.h"
#include <math.h>
#include <stdlib.h>
#include <string.h>
#include <assert.h>

void vwf_free(void* p) { free(p); }

/* ---- normalize (Image/AutoNormalize.h:76-86, ChannelNormalizeFunctor Image/Algorithms.h:106-126) ---------------------- */
int vwf_normalize(const float* in, int w, int h, int has_nodata, double nodata, float* out) {
  const long long n = (long long)w * h;
  const float nd = (float)nodata;   /* CreatePixelMask<PixelGray<float>> holds the nodata value as a float */
  float mn = 0, mx = 0;
  int any = 0;
  for (long long k = 0; k < n; ++k) {
    const float v = in[k];
    if (!isfinite(v)) return VWF_EARG;
    if (has_nodata && v == nd) continue;
    if (!any) { mn = mx = v; any = 1; }           /* MinMaxAccumulator (Math/Functors.h:363-372) */
    else { if (v < mn) mn = v; if (mx < v) mx = v; }
  }
  if (!any) return n ? VWF_EARG : 0;              /* "MinMaxAccumulator: no valid samples" */
  const double ratio = mx == mn ? 0.0 : (1.0f - 0.0f) / (double)(mx - mn);
  for (long long k = 0; k < n; ++k) {
    const float v = in[k];
    out[k] = (has_nodata && v == nd) ? 0.0f : (float)((double)(v - mn) * ratio + 0.0f);
  }
  return 0;
}

/* ---- generate_gaussian_kernel (Image/Filter.tcc:37-80; vw::erf is ::erf outside WIN32, Math/Functions.h:180-200) ------ */
void vwf_gaussian_taps(double* k) {
  const int size = 9, center = 4;
  const double sigma = 2.0, z = 1 / (sqrt(2.0) * sigma);
  double sum = 0.0, tap;
  for (int i = 1; i <= center; ++i) {
    tap = erf((i + 0.5) * z) - erf((i - 0.5) * z);
    sum += tap;
    k[center + i] = k[center - i] = tap;
  }
  sum *= 2.0;
  tap = erf(0.5 * z) - erf(-0.5 * z);
  sum += tap;
  k[center] = tap;
  const double norm = 1.0 / sum;
  for (int i = 0; i < size; ++i) k[i] *= norm;
}

/* ---- OBALoG tables (InterestPoint/IntegralInterestOperator.cc:28-62), scales 0..7 ------------------------------------- */
static const double SIGMA[8] = {1.2, 1.5, 1.875, 2.34375, 2.9296875, 3.662109, 4.577636, 5.722046};
static const int BW[8][6] = {{11,7,5,3,3,1}, {13,9,7,5,3,1}, {17,11,9,5,5,3}, {21,13,11,7,7,3},
                             {27,17,13,9,9,5}, {33,21,17,11,11,5}, {41,27,21,13,13,7}, {51,33,27,17,17,7}};
static const int BH[8][6] = {{11,5,7,3,1,3}, {13,7,9,1,3,5}, {17,9,11,5,3,5}, {21,11,13,3,7,7},
                             {27,13,17,5,9,9}, {33,17,21,5,11,11}, {41,21,27,7,13,13}, {51,27,33,7,17,17}};
static const double BWT[8][6] = {
  {0.0006179999909,0.008283999749,0.008283999749,-0.03556599841,-0.05576400086,-0.05576400086},
  {0.0002659999882,0.004889999982,0.004889999982,-0.0221420005,-0.0488499999,-0.0221420005},
  {0.0002659424644,0.003207367443,0.003207367443,-0.001847865087,-0.022190776,-0.022190776},
  {0.000218920823,0.002005755751,0.002005755751,-0.01499466244,-0.0008247125278,-0.01499466244},
  {0.0001030362087,0.00137811946,0.00137811946,-0.009606413672,0.002226325845,-0.009606413672},
  {7.198028372e-05,0.0008259398524,0.0008259398524,-0.006072390568,-1.177469443e-06,-0.006072390568},
  {3.803569417e-05,0.0005251058097,0.0005251058097,-0.003885340628,0.0002823550512,-0.003885340628},
  {2.892054582e-05,0.0003287680581,0.0003287680581,-0.002447736656,-0.0002717150913,-0.002447736656}};

/* IntegralImage (InterestPoint/IntegralImage.h:41-91): (w+1) x (h+1), row-major, ((v + left) + up) - upleft */
static void integral(const float* src, int w, int h, long long sp, float* I) {
  const int iw = w + 1;
  for (int x = 0; x < iw; ++x) I[x] = 0;
  for (int y = 1; y <= h; ++y) I[(long long)y * iw] = 0;
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x) {
      float* p = I + (long long)(y + 1) * iw + (x + 1);
      *p = src[(long long)y * sp + x] + *(p - 1) + *(p - iw) - *(p - iw - 1);
    }
}

/* IntegralImage and BoxFilterView for any filter, exported for the reference's TestIntegral / TestBoxFilter pins */
void vwf_integral(const float* src, int w, int h, float* I) { integral(src, w, h, w, I); }
/* box_filter(integral, filter) of a w x h image (BoxFilter.h:48-114): nb boxes of start (sx, sy), size (bw, bh), float weight */
void vwf_box_filter(const float* I, int w, int h, int nb, const int* sx, const int* sy, const int* bw, const int* bh, const float* wt,
                    float* out) {
  int mx = 0;
  for (int b = 0; b < nb; ++b) { if (mx < bw[b]) mx = bw[b]; if (mx < bh[b]) mx = bh[b]; }
  const int pb = mx >> 1, iw = w + 1;
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x) {
      float result = 0;
      if (!(x < pb || x >= iw - pb - 1 || y < pb || y >= h + 1 - pb - 1))
        for (int b = 0; b < nb; ++b) {
          const int x0 = x + sx[b], y0 = y + sy[b];
          float box = 0;
          box += I[(long long)y0 * iw + x0];
          box -= I[(long long)y0 * iw + x0 + bw[b]];
          box -= I[(long long)(y0 + bh[b]) * iw + x0];
          box += I[(long long)(y0 + bh[b]) * iw + x0 + bw[b]];
          result += wt[b] * box;
        }
      out[(long long)y * w + x] = result;
    }
}

/* abs(box_filter(integral, scale s)) at (x, y) of a w x h tile (BoxFilter.h:48-114, IntegralInterestOperator.h:95-114) */
static float interest_at(const float* I, int w, int h, int s, int x, int y) {
  const int pb = BW[s][0] >> 1;   /* the largest box is the first: max_size >> 1 */
  if (x < pb || x >= w - pb || y < pb || y >= h - pb) return 0.0f;
  const int iw = w + 1;
  float result = 0;
  for (int b = 0; b < 6; ++b) {
    const int bw = BW[s][b], bh = BH[s][b];
    const int x0 = x - (bw >> 1), y0 = y - (bh >> 1);
    float box = 0;
    box += I[(long long)y0 * iw + x0];
    box -= I[(long long)y0 * iw + x0 + bw];
    box -= I[(long long)(y0 + bh) * iw + x0];
    box += I[(long long)(y0 + bh) * iw + x0 + bw];
    result += (float)BWT[s][b] * box;
  }
  return fabsf(result);
}

/* is_extrema (IntegralDetector.cc:106-134): strictly above all 26 neighbours */
static int is_extrema(const float* lo, const float* mid, const float* hi, int w, int x, int y) {
  const long long c = (long long)y * w + x;
  const float v = mid[c];
  if (v <= lo[c] || v <= hi[c]) return 0;
  for (int dy = -1; dy <= 1; ++dy)
    for (int dx = -1; dx <= 1; ++dx) {
      if (!dx && !dy) continue;
      const long long q = c + (long long)dy * w + dx;
      if (v <= lo[q] || v <= mid[q] || v <= hi[q]) return 0;
    }
  return 1;
}

/* OBALoGInterestOperator::threshold's Harris test (IntegralInterestOperator.h:123-153) on the interest image of scale m */
static int harris(const float* in, int w, int h, int ix, int iy, int m, const double* k) {
  const int step = (int)(float)SIGMA[m], offset = 4 * step;
  assert(ix - offset - 1 >= 0 && ix + offset + 1 < w && iy - offset - 1 >= 0 && iy + offset + 1 < h);
  float sxx = 0, syy = 0, sxy = 0;
  for (int y = iy - offset, jy = 0; y <= iy + offset; y += step, jy++)
    for (int x = ix - offset, jx = 0; x <= ix + offset; x += step, jx++) {
      const float Lx = in[(long long)y * w + x - 1] - in[(long long)y * w + x + 1];
      const float Ly = in[(long long)(y - 1) * w + x] - in[(long long)(y + 1) * w + x];
      const float weight = (float)(k[jx] * k[jy]);
      sxx += Lx * Lx * weight;
      syy += Ly * Ly * weight;
      sxy += Lx * Ly * weight;
    }
  const float trace = sxx + syy;
  const float det = sxx * syy - sxy * sxy;
  return (trace * trace) / det < 12;
}

/* std::list::sort with InterestPoint::operator< (descending interest), stable: a merge sort */
static void stable_sort_desc(vwf_point* a, long long n, vwf_point* tmp) {
  if (n < 2) return;
  const long long h = n / 2;
  stable_sort_desc(a, h, tmp);
  stable_sort_desc(a + h, n - h, tmp);
  long long i = 0, j = h, o = 0;
  while (i < h && j < n) tmp[o++] = (a[i].interest < a[j].interest) ? a[j++] : a[i++];
  while (i < h) tmp[o++] = a[i++];
  while (j < n) tmp[o++] = a[j++];
  memcpy(a, tmp, (size_t)n * sizeof *a);
}

/* IntegralAutoGainDetector::process_image (IntegralDetector.cc:264-370) on one tile; appends to *list */
static int process_tile(const float* img, long long pitch, int w, int h, int num_ip, const double* k, vwf_point** list, long long* n,
                        long long* cap, long long* stats) {
  float* I = malloc(sizeof(float) * (size_t)(w + 1) * (h + 1));
  float* in = malloc(sizeof(float) * (size_t)w * h * 8);
  if (!I || !in) { free(I); free(in); return VWF_EARG; }
  integral(img, w, h, pitch, I);
  for (int s = 0; s < 8; ++s)
    for (int y = 0; y < h; ++y)
      for (int x = 0; x < w; ++x) in[(long long)s * w * h + (long long)y * w + x] = interest_at(I, w, h, s, x, y);
  const long long start = *n;
  for (int m = 1; m <= 6; ++m) {
    const float* lo = in + (long long)(m - 1) * w * h, *mid = lo + (long long)w * h, *hi = mid + (long long)w * h;
    float imin = mid[0], imax = mid[0];   /* min_max_pixel_values of the whole interest image */
    for (long long q = 1; q < (long long)w * h; ++q) { if (mid[q] < imin) imin = mid[q]; if (imax < mid[q]) imax = mid[q]; }
    const float thr = (float)(imin + 0.001 * (imax - imin));
    for (int r = 1; r < h - 1; ++r)
      for (int c = 1; c < w - 1; ++c) {
        if (!is_extrema(lo, mid, hi, w, c, r)) continue;
        stats[1]++;
        const float v = mid[(long long)r * w + c];
        if (v < thr || !harris(mid, w, h, c, r, m, k)) continue;
        stats[2]++;
        if (*n == *cap) {
          *cap = *cap * 2 + 64;
          vwf_point* q = realloc(*list, sizeof(vwf_point) * (size_t)*cap);
          if (!q) { free(I); free(in); return VWF_EARG; }
          *list = q;
        }
        vwf_point p = {(float)c, (float)r, c, r, (float)SIGMA[m], v, 0.0f};
        (*list)[(*n)++] = p;
      }
  }
  const long long cnt = *n - start;
  if (num_ip > 0 && num_ip < cnt) {
    vwf_point* tmp = malloc(sizeof(vwf_point) * (size_t)cnt);
    if (!tmp) { free(I); free(in); return VWF_EARG; }
    stable_sort_desc(*list + start, cnt, tmp);
    free(tmp);
    *n = start + num_ip;
    stats[3]++;
  }
  free(I);
  free(in);
  return 0;
}

/* detect_interest_points (InterestPoint/DetectorBase.h:250-328): subdivide_bbox tiles in raster order */
int vwf_detect(const float* img, int w, int h, int tile_size, int ip_per_tile, vwf_point** out, long long* n, long long* stats) {
  const int ts = tile_size < 1024 ? 1024 : tile_size;
  double k[9];
  vwf_gaussian_taps(k);
  long long cap = 0;
  *out = NULL;
  *n = 0;
  for (int i = 0; i < 5; ++i) stats[i] = 0;
  for (int y0 = 0; y0 < h; y0 += ts)
    for (int x0 = 0; x0 < w; x0 += ts) {
      const int tw = w - x0 < ts ? w - x0 : ts, th = h - y0 < ts ? h - y0 : ts;
      int num_ip = 0;
      if (ip_per_tile > 0) {
        const double fraction = (double)tw * th / ((double)ts * ts);
        num_ip = (int)ceil(fraction * (double)ip_per_tile);
        if (num_ip < 1) num_ip = 1;
        if (num_ip > ip_per_tile) num_ip = ip_per_tile;
      }
      const long long s0 = *n;
      int rc = process_tile(img + (long long)y0 * w + x0, w, tw, th, num_ip, k, out, n, &cap, stats);
      if (rc) return rc;
      for (long long q = s0; q < *n; ++q) {   /* DetectorBase.h:231-236 */
        (*out)[q].x += x0; (*out)[q].ix += x0;
        (*out)[q].y += y0; (*out)[q].iy += y0;
      }
      stats[0]++;
    }
  return 0;
}

/* ---- remove_ip_near_nodata (InterestPoint/InterestPointUtils.h:45-82) --------------------------------------------------- */
long long vwf_remove_near_nodata(const float* raw, int w, int h, double nodata, int radius, vwf_point* pts, long long n) {
  const int bx0 = radius, by0 = radius, bx1 = w - radius, by1 = h - radius;
  long long o = 0;
  for (long long i = 0; i < n; ++i) {
    const vwf_point p = pts[i];
    if (!(p.ix >= bx0 && p.iy >= by0 && p.ix < bx1 && p.iy < by1)) continue;
    int bad = 0;
    for (int y = p.iy - radius; y <= p.iy + radius && !bad; ++y)
      for (int x = p.ix - radius; x <= p.ix + radius; ++x)
        if ((double)raw[(long long)y * w + x] == nodata) { bad = 1; break; }
    if (!bad) pts[o++] = p;
  }
  return o;
}

/* ---- describe_interest_points with SGradDescriptorGenerator (InterestPoint/Descriptor.h:202-355, 414-471) ---------------- */
static const int STRT[5] = {17, 15, 9, 6, 0}, BSZ[5] = {2, 4, 8, 10, 14}, BHF[5] = {1, 2, 4, 5, 7};

typedef struct { double a, b, c, d, ai, bi, ci, di, x, y; } affine;

/* get_support's AffineTransform (Descriptor.h:242-254, Math/Transform.h:310-339, the 2x2 inverse of Math/Matrix.h:2209-2216) */
static affine support_tx(float x, float y, float scale, double c, double s) {
  const float half = ((float)(42 - 1)) / 2.0f, scaling = 1.0f / scale;
  affine t;
  t.a = scaling * c; t.b = -scaling * s; t.c = scaling * s; t.d = scaling * c;
  t.x = scaling * (s * y - c * x) + half;
  t.y = -scaling * (s * x + c * y) + half;
  const double det = t.a * t.d - t.b * t.c;
  t.ai = t.d / det; t.bi = -t.b / det; t.ci = -t.c / det; t.di = t.a / det;
  return t;
}
static void reverse(const affine* t, double px, double py, double* rx, double* ry) {
  const double qx = px - t->x, qy = py - t->y;
  *rx = t->ai * qx + t->bi * qy;
  *ry = t->ci * qx + t->di * qy;
}

static int vw_floor(double v) { return (int)floor(v); }

/* the crop (x0, y0, cw, ch) of the zero-extended image, read with zero extension */
static float crop_px(const float* img, int w, int h, int x0, int y0, int cw, int ch, int i, int j) {
  if (i < 0 || j < 0 || i >= cw || j >= ch) return 0.0f;
  const int x = x0 + i, y = y0 + j;
  if (x < 0 || y < 0 || x >= w || y >= h) return 0.0f;
  return img[(long long)y * w + x];
}

/* BilinearInterpolation (Image/Interpolation.h:76-110) with real_type float */
static float bilinear(const float* img, int w, int h, int x0, int y0, int cw, int ch, double i, double j) {
  const int x = vw_floor(i), y = vw_floor(j);
  if ((double)x == i && (double)y == j) return crop_px(img, w, h, x0, y0, cw, ch, x, y);
  const float nx = (float)i - (float)x, ny = (float)j - (float)y;
  const float n1mx = 1.0f - nx, n1my = 1.0f - ny;
  float r = crop_px(img, w, h, x0, y0, cw, ch, x, y) * n1mx;
  r = r + crop_px(img, w, h, x0, y0, cw, ch, x + 1, y) * nx;
  r = r * n1my;
  float row = crop_px(img, w, h, x0, y0, cw, ch, x, y + 1) * n1mx;
  row = row + crop_px(img, w, h, x0, y0, cw, ch, x + 1, y + 1) * nx;
  return r + row * ny;
}

static void sgrad(const float* support, float* out) {
  float I[43 * 43];
  integral(support, 42, 42, 42, I);
  float sqr = 0;
  int f = 0;
  for (int s = 0; s < 5; ++s) {
    const float inv_bh2 = 1 / (float)(BHF[s] * BHF[s]);
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) {
        const int tx = STRT[s] + i * BSZ[s], ty = STRT[s] + j * BSZ[s], b = BHF[s];
        float q[4];
        const int x0s[4] = {tx, tx + b, tx, tx + b}, y0s[4] = {ty, ty, ty + b, ty + b};
        for (int k = 0; k < 4; ++k) {   /* IntegralBlock (InterestPoint/IntegralImage.cc:27-53) */
          const int x0 = x0s[k], y0 = y0s[k], x1 = x0 + b, y1 = y0 + b;
          float r = I[y0 * 43 + x0];
          r += I[y1 * 43 + x1];
          r -= I[y1 * 43 + x0];
          r -= I[y0 * 43 + x1];
          q[k] = r;
        }
        out[f] = (q[0] - q[2]) * inv_bh2; sqr += out[f] * out[f]; f++;
        out[f] = (q[1] - q[3]) * inv_bh2; sqr += out[f] * out[f]; f++;
        out[f] = (q[0] - q[1]) * inv_bh2; sqr += out[f] * out[f]; f++;
        out[f] = (q[2] - q[3]) * inv_bh2; sqr += out[f] * out[f]; f++;
      }
  }
  /* the unqualified sqrt resolves to ::sqrt(double) (vw/Math/Functions.h:167 over <cmath>): the quotient is a double */
  float inv = (float)(1.0f / sqrt((double)sqr));
  if (!isnormal(inv)) inv = 0.0f;
  for (int k = 0; k < VWF_DESC; ++k) out[k] *= inv;
}

static int in_tile(const vwf_point* p, int x0, int y0, int x1, int y1) {
  const int x = (int)p->x, y = (int)p->y;   /* IsInBBox: Vector2i(ip.x, ip.y) */
  return x >= x0 && y >= y0 && x < x1 && y < y1;
}

int vwf_describe(const float* img, int w, int h, int tile_size, vwf_point* pts, long long n, float* desc) {
  const int ts = tile_size < 1024 ? 1024 : tile_size;
  long long first = 0;
  float support[42 * 42];
  for (int ty = 0; ty < h; ty += ts)
    for (int tx = 0; tx < w; tx += ts) {
      const int x1 = tx + (w - tx < ts ? w - tx : ts), y1 = ty + (h - ty < ts ? h - ty : ts);
      /* std::partition over a std::list (bidirectional iterators: libstdc++'s swapping scan) */
      long long f = first, l = n;
      for (;;) {
        while (f != l && in_tile(&pts[f], tx, ty, x1, y1)) ++f;
        if (f == l) break;
        --l;
        while (f != l && !in_tile(&pts[l], tx, ty, x1, y1)) --l;
        if (f == l) break;
        vwf_point t = pts[f]; pts[f] = pts[l]; pts[l] = t;
        ++f;
      }
      const long long s0 = first, s1 = f;
      first = f;
      if (s0 == s1) continue;
      /* InterestPointDescriptionTask (Descriptor.h:259-301) */
      int bx0 = 0, by0 = 0, bx1 = 0, by1 = 0, have = 0;
      for (long long q = s0; q < s1; ++q) {
        const affine t = support_tx(pts[q].x, pts[q].y, pts[q].scale, cos(-pts[q].orientation), sin(-pts[q].orientation));
        double mnx = 0, mny = 0, mxx = 0, mxy = 0;
        const double cx[4] = {0, 41, 0, 41}, cy[4] = {0, 0, 41, 41};
        for (int c = 0; c < 4; ++c) {
          double rx, ry;
          reverse(&t, cx[c], cy[c], &rx, &ry);
          if (!c) { mnx = mxx = rx; mny = mxy = ry; continue; }
          if (rx > mxx) mxx = rx;
          if (rx < mnx) mnx = rx;
          if (ry > mxy) mxy = ry;
          if (ry < mny) mny = ry;
        }
        /* grow_bbox_to_int (Math/BBox.tcc:366-389), then BBox2i::grow(bbox) */
        const int ix0 = (int)floor(mnx), iy0 = (int)floor(mny), ix1 = (int)floor(mxx) + 1, iy1 = (int)floor(mxy) + 1;
        if (!have) { bx0 = ix0; by0 = iy0; bx1 = ix1; by1 = iy1; have = 1; continue; }
        const int gx[2] = {ix0, ix1}, gy[2] = {iy0, iy1};
        for (int c = 0; c < 2; ++c) {
          if (gx[c] > bx1) bx1 = gx[c];
          if (gx[c] < bx0) bx0 = gx[c];
          if (gy[c] > by1) by1 = gy[c];
          if (gy[c] < by0) by0 = gy[c];
        }
      }
      bx0 -= 1; by0 -= 1; bx1 += 1; by1 += 1;
      const int cw = bx1 - bx0, ch = by1 - by0;
      for (long long q = s0; q < s1; ++q) {
        pts[q].x -= bx0;
        pts[q].y -= by0;
        const affine t = support_tx(pts[q].x, pts[q].y, pts[q].scale, cos(-pts[q].orientation), sin(-pts[q].orientation));
        for (int j = 0; j < 42; ++j)
          for (int i = 0; i < 42; ++i) {
            double rx, ry;
            reverse(&t, i, j, &rx, &ry);
            support[j * 42 + i] = bilinear(img, w, h, bx0, by0, cw, ch, rx, ry);
          }
        sgrad(support, desc + q * VWF_DESC);
        pts[q].x += bx0;
        pts[q].y += by0;
      }
    }
  return first == n ? 0 : VWF_EARG;
}
