/* vw_sgm_oracle.c -- CPU restatement of Vision Workbench's SemiGlobalMatcher core (SURVEY.md section 8, row a10).
 *
 * TEST INFRASTRUCTURE ONLY (see oracle/vw_oracle.h): nothing under visionworkbench_b200/ may use it.
 *
 * Scope: vw::stereo::calc_disparity_sgm (Stereo/SGM.cc:167-230) -> SemiGlobalMatcher::semi_global_matching_func
 * (:2387-2448) with
 *   - CENSUS_TRANSFORM and TERNARY_CENSUS_TRANSFORM costs, kernel 3/5/7/9 (Image/CensusTransform.h:64-340,
 *     SGM.cc:39-73,1740-1873),
 *   - explicit penalties p1 / p2 (set_parameters, :77-160; <= 0 selects the defaults),
 *   - the same search box for every pixel (populate_constant_disp_bound_image, :231-239),
 *   - plain SGM accumulation along 8 directions (accum_sgm_multithread, :2462-2611; PixelPassTask, SGMAssist.h:691-832)
 *     with the SSE flavour of evaluate_path (:1014-1141, compute_path_internals_sse :950-990: unsigned 16-bit min,
 *     SATURATING add / subtract) -- the reference is built with SSE4.1, and the scalar flavour (:806-913) differs on overflow,
 *   - the integer winner of select_best_disparity (:1159-1288, including its tie-smoothing iterations that rewrite the
 *     accumulated costs) as used by create_disparity_view (:1290-1346),
 *   - the sub-pixel models of create_disparity_view_subpixel (:1402-1480,1497-1614), the 2-D parabola included.
 * Further down: the same pipeline with a search box per pixel (vwo_sgm_calc_disparity_bounds), the derivation of those
 * boxes from masks and the previous pyramid level (vwo_sgm_disp_bounds: populate_disp_bound_image / constrain_disp_bound_image,
 * :241-668) with the memory-limit retry loop over the conservation levels (:476-497), MGM accumulation
 * (vwo_mgm_calc_disparity_bounds), and the whole entry point (vwo_calc_disparity_sgm).  The R->L / filtering glue of
 * CorrelationView.cc:360-590 lives in vw_oracle.c.  Pinned by TestSGM.cxx:27-75 (> 99 % of the pixels equal the true
 * constant offset) on the reference's own fixture images, and, across the penalty range, by an independent numpy
 * restatement (tests/sgm_reference.py, tests/test_oracle_sgm_penalties.py); the sub-pixel stage has no known-answer test in
 * the reference (floats: tolerance 1e-5 on the GPU side).
 *
 * The accumulation order of the reference is thread dependent but irrelevant: every pixel lies on exactly one line per
 * direction and the per-line results are ADDED (uint16, wrapping) into the accumulation buffer (SGMAssist.h:790-815).
 */
#include "vw_oracle.h"
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef uint8_t cost_t;      /* SemiGlobalMatcher::CostType      (SGM.h:81) */
typedef uint16_t accum_t;    /* SemiGlobalMatcher::AccumCostType (SGM.h:82) */

/* vw::u8_convert (Image/ImageThresh.h:274-286): min/max stretch to 0..255, float arithmetic of ChannelNormalizeFunctor
 * (Image/Algorithms.h:106-126: float difference, double ratio), truncating cast */
static void u8_convert(const float* in, int w, int h, int pitch, uint8_t* out) {
  double mn = in[0], mx = in[0];
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x) { const double v = in[(size_t)y * pitch + x]; if (v < mn) mn = v; if (v > mx) mx = v; }
  if (mx == mn) mx = mn + 1.0;
  const float old_min = (float)mn, old_max = (float)mx, new_min = 0.0f, new_max = 255.0f;
  const double ratio = (old_max == old_min) ? 0.0 : (double)(new_max - new_min) / (double)(old_max - old_min);
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < w; ++x) {
      float v = in[(size_t)y * pitch + x];
      if (v < old_min) v = old_min;
      if (v > old_max) v = old_max;
      const float n = (float)((double)(v - old_min) * ratio + (double)new_min);
      out[(size_t)y * w + x] = (uint8_t)n;
    }
}

/* census signatures: only the SET of neighbours compared (strictly greater than the centre) matters for the Hamming
 * distance.  3x3/5x5/7x7: all neighbours (CensusTransform.h:64-110); 9x9: the 32 positions of :112-160. */
static const int C9_COLS[32] = {0, 4, 8, 1, 3, 5, 7, 2, 4, 6, 1, 4, 7, 0, 2, 3, 5, 6, 8, 1, 4, 7, 2, 4, 6, 1, 3, 5, 7, 0, 4, 8};
static const int C9_ROWS[32] = {0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 3, 3, 3, 4, 4, 4, 4, 4, 4, 5, 5, 5, 6, 6, 6, 7, 7, 7, 7, 8, 8, 8};

/* ternary census (Image/CensusTransform.h:167-340): 2 bits per neighbour: 00 below centre - t, 01 inside the band, 11 above
 * centre + t; 3x3 / 5x5: all neighbours in reverse raster order; 7x7: the custom 32-position pattern (:222-275); 9x9: the
 * same 32 positions as the binary 9x9 census (:277-340).  The reference stores the signatures in the integer type the BINARY
 * census of the same kernel uses, so the 48-bit ternary 5x5 signature is truncated to 32 bits (SGM.cc:1789-1803) -- kept. */
static const int T7_COLS[32] = {0, 2, 3, 4, 6, 1, 3, 5, 0, 2, 3, 4, 6, 0, 1, 2, 4, 5, 6, 0, 2, 3, 4, 6, 1, 3, 5, 0, 2, 3, 4, 6};
static const int T7_ROWS[32] = {0, 0, 0, 0, 0, 1, 1, 1, 2, 2, 2, 2, 2, 3, 3, 3, 3, 3, 3, 4, 4, 4, 4, 4, 5, 5, 5, 6, 6, 6, 6, 6};
static uint64_t census_value_ternary(const uint8_t* img, int w, int col, int row, int k, int thr) {
  const int hk = (k - 1) / 2;
  const int center = img[(size_t)row * w + col];
  const int lo = center - thr, hi = center + thr;
  uint64_t out = 0, addend = 1;
  if (k == 7 || k == 9) {
    const int* cs = k == 9 ? C9_COLS : T7_COLS;
    const int* rs = k == 9 ? C9_ROWS : T7_ROWS;
    for (int i = 0; i < 32; ++i) {
      const int val = img[(size_t)(row + rs[i] - hk) * w + (col + cs[i] - hk)];
      if (val >= lo) { out += addend; if (val > hi) out += addend * 2; }
      addend *= 4;
    }
    return out;
  }
  for (int r = row + hk; r >= row - hk; --r)
    for (int c = col + hk; c >= col - hk; --c) {
      if (r == row && c == col) continue;
      const int val = img[(size_t)r * w + c];
      if (val >= lo) { out += addend; if (val > hi) out += addend * 2; }
      addend *= 4;
    }
  if (k == 5) out &= 0xFFFFFFFFull;        /* ImageView<uint32> (SGM.cc:1789-1790) */
  if (k == 3) out &= 0xFFFFull;            /* uint16 (:1762) -- 16 bits, nothing is lost */
  return out;
}
uint64_t vwo_census_value(const uint8_t* img, int w, int col, int row, int k, int ternary, int thr);
static uint64_t census_value(const uint8_t* img, int w, int col, int row, int k) {
  const int hk = (k - 1) / 2;
  const int center = img[(size_t)row * w + col];
  uint64_t out = 0, addend = 1;
  if (k == 9) {
    for (int i = 0; i < 32; ++i) {
      if ((int)img[(size_t)(row + C9_ROWS[i] - 4) * w + (col + C9_COLS[i] - 4)] > center) out += addend;
      addend *= 2;
    }
    return out;
  }
  for (int r = row + hk; r >= row - hk; --r)
    for (int c = col + hk; c >= col - hk; --c) {
      if (r == row && c == col) continue;
      if ((int)img[(size_t)r * w + c] > center) out += addend;
      addend *= 2;
    }
  return out;
}
uint64_t vwo_census_value(const uint8_t* img, int w, int col, int row, int k, int ternary, int thr) {
  return ternary ? census_value_ternary(img, w, col, row, k, thr) : census_value(img, w, col, row, k);
}
static inline int popcount64(uint64_t v) { return __builtin_popcountll(v); }

static inline accum_t sat_add(accum_t a, accum_t b) { const unsigned s = (unsigned)a + b; return (accum_t)(s > 65535u ? 65535u : s); }
static inline accum_t sat_sub(accum_t a, accum_t b) { return (accum_t)(a > b ? a - b : 0); }
static inline accum_t min16(accum_t a, accum_t b) { return a < b ? a : b; }

typedef struct {
  int ndx, ndy, nd;          /* disparities: dx in [0, ndx), dy in [0, ndy) (min_disp = 0 in calc_disparity_sgm) */
  int p1, p2;
  int ow, oh, min_col, min_row;
  const uint8_t* left; int lw;
  const cost_t* cost;        /* [oh][ow][nd] */
  accum_t* accum;            /* [oh][ow][nd] */
  int* adj;                  /* [nd][8] (populate_adjacent_disp_lookup_table, :755-800) */
} Sgm;

/* one line of PixelPassTask::PixelPassDoWork (SGMAssist.h:705-774) starting at (c, r) going (sc, sr) */
static void sgm_line(const Sgm* s, int c, int r, int sc, int sr, accum_t* buf /* 2 * nd */) {
  const int nd = s->nd;
  accum_t* prior = buf;
  accum_t* cur = buf + nd;
  int last_val = -1;
  while (c >= 0 && c < s->ow && r >= 0 && r < s->oh) {
    const cost_t* local = s->cost + ((size_t)r * s->ow + c) * nd;
    const int cur_val = s->left[(size_t)(r + s->min_row) * s->lw + (c + s->min_col)];
    const int diff = abs(cur_val - last_val);
    if (last_val >= 0) {
      /* evaluate_path, SSE flavour (:1014-1141) */
      accum_t p2_mod = (accum_t)s->p2;
      if (diff > 0) p2_mod = (accum_t)(p2_mod / diff);
      if (p2_mod < s->p1) p2_mod = (accum_t)s->p1;
      accum_t min_prior = (accum_t)(255 + s->p2);                 /* get_bad_accum_val (SGM.h:240) */
      for (int d = 0; d < nd; ++d) if (prior[d] < min_prior) min_prior = prior[d];
      const accum_t dJ = (accum_t)(min_prior + p2_mod);           /* uint16 arithmetic of the reference (:1056) */
      for (int d = 0; d < nd; ++d) {
        const int* a = s->adj + (size_t)d * 8;
        accum_t m = min16(min16(min16(prior[a[0]], prior[a[1]]), min16(prior[a[2]], prior[a[3]])),
                          min16(min16(prior[a[4]], prior[a[5]]), min16(prior[a[6]], prior[a[7]])));
        accum_t res = sat_add(m, (accum_t)s->p1);
        res = min16(res, min16(prior[d], dJ));
        res = sat_add(res, (accum_t)local[d]);
        cur[d] = sat_sub(res, min_prior);
      }
    } else {
      for (int d = 0; d < nd; ++d) cur[d] = local[d];
    }
    accum_t* acc = s->accum + ((size_t)r * s->ow + c) * nd;      /* update_accum_buffer (SGMAssist.h:790-815) */
    for (int d = 0; d < nd; ++d) acc[d] = (accum_t)(acc[d] + cur[d]);
    accum_t* t = prior; prior = cur; cur = t;
    last_val = cur_val;
    c += sc; r += sr;
  }
}

/* select_best_disparity (:1159-1288): returns the index of the winner; may rewrite accum_vec (tie smoothing) */
static int select_best(accum_t* accum_vec, int width, int height, accum_t* buffer) {
  const int num = width * height;
  int min_count = 0, min_index = 0;
  accum_t min_val = 65535;
  for (int i = 0; i < num; ++i) {
    const accum_t v = accum_vec[i];
    buffer[i] = v;
    if (v == min_val) ++min_count;
    if (v < min_val) { min_index = i; min_val = v; min_count = 1; }
  }
  accum_t* input_array = accum_vec;
  accum_t* output_array = buffer;
  const double filter[3] = {1.0 / 3.0, 1.0 / 3.0, 1.0 / 3.0};
  int iter_count = 0, index = 0;
  while (min_count > 1) {
    accum_t* sw = input_array; input_array = output_array; output_array = sw;
    index = 0; min_count = 0; min_val = 65535; min_index = 0;
    for (int row = 0; row < height; ++row)
      for (int col = 0; col < width; ++col) {
        int mn = -1, mx = 1;
        double result = 0, weight_total = 0;
        if (iter_count < 5) {
          if (mn + col < 0) mn = 0;
          if (mx + col >= width) mx = 0;
          for (int k = mn; k <= mx; ++k) { const double wgt = filter[k + 1]; result += (double)input_array[index + k] * wgt; weight_total += wgt; }
        } else {
          if (mn + row < 0) mn = 0;
          if (mx + row >= height) mx = 0;
          for (int k = mn; k <= mx; ++k) { const double wgt = filter[k + 1]; result += (double)input_array[index + k * width] * wgt; weight_total += wgt; }
        }
        const accum_t v = (accum_t)round(result / weight_total);
        if (v == min_val) ++min_count;
        if (v < min_val) { min_index = index; min_val = v; min_count = 1; }
        output_array[index] = v;
        ++index;
      }
    if (++iter_count >= 6) break;
  }
  if (iter_count > 0 && iter_count % 2 == 0)
    for (int i = 0; i < index; ++i) input_array[i] = output_array[i];
  return min_index;
}

/* the 1-D sub-pixel models of SGM.cc:1402-1431 */
static double linear_fit(double x) { return x / 2.0; }
static double poly4_fit(double x) { return (x * x * x * x + x) / 4.0; }
static double cos_fit(double x) { const double PI = 3.14159265359; return (1 - cos(x * PI / 3.0)); }
static double lc_blend_fit(double x) {
  const double PI = 3.14159265359;
  const double factor = 1.195 - cos(x * (PI / 2.3));
  return cos_fit(x) * factor + linear_fit(x) * (1.0 - factor);
}
/* compute_subpixel_offset (:1445-1480) */
static double subpixel_offset(accum_t prev, accum_t center, accum_t next, int left_bound, int right_bound, int mode) {
  const double ld = (int)prev - (int)center, rd = (int)next - (int)center;
  if (rd == 0 && ld == 0) return 0;
  if (left_bound) return 0.5 * ((double)center / (double)next);            /* two_value_subpixel (:1440-1442) */
  if (right_bound) return -1.0 * (0.5 * ((double)center / (double)prev));
  double x = rd / ld, mult = -1.0;
  if (ld < rd) { x = ld / rd; mult = 1.0; }
  double value;
  switch (mode) {
    case 3: value = poly4_fit(x); break;
    case 4: value = cos_fit(x); break;
    case 5: value = lc_blend_fit(x); break;
    default: value = linear_fit(x); break;
  }
  return (value - 0.5) * mult;
}

/* ParabolaFit2d::find_peak (SGMAssist.h:36-134): the 6x9 pseudo-inverse is held in a Matrix<FLOAT,6,9> (:139) and multiplied
 * with the double z vector; the raw offset passes through a Vector2f (:116-117) before the erf correction. */
static int parabola_peak(double z1, double z2, double z3, double z4, double z5, double z6, double z7, double z8, double z9, double* dx, double* dy) {
  static const double pd[54] = {
     1.0/6, -1.0/3,  1.0/6,  1.0/6, -1.0/3,  1.0/6,   1.0/6, -1.0/3,  1.0/6,
     1.0/6,  1.0/6,  1.0/6, -1.0/3, -1.0/3, -1.0/3,   1.0/6,  1.0/6,  1.0/6,
     1.0/4,    0.0, -1.0/4,    0.0,    0.0,    0.0,  -1.0/4,    0.0,  1.0/4,
    -1.0/6,    0.0,  1.0/6, -1.0/6,    0.0,  1.0/6,  -1.0/6,    0.0,  1.0/6,
    -1.0/6, -1.0/6, -1.0/6,    0.0,    0.0,    0.0,   1.0/6,  1.0/6,  1.0/6,
    -1.0/9,  2.0/9, -1.0/9,  2.0/9,   5.0/9, 2.0/9,  -1.0/9,  2.0/9, -1.0/9 };
  const double z[9] = {z1, z2, z3, z4, z5, z6, z7, z8, z9};
  double vals[6];
  for (int i = 0; i < 6; ++i) {
    double acc = 0.0;                                              /* Math/Matrix.h product: sum of m(i,j) * v(j) in double */
    for (int j = 0; j < 9; ++j) acc += (double)(float)pd[i * 9 + j] * z[j];
    vals[i] = acc;
  }
  const double denom = 4.0 * vals[0] * vals[1] - (vals[2] * vals[2]);
  if (fabs(denom) < 0.01) return 0;
  const float ox = (float)((vals[2] * vals[4] - 2.0 * vals[1] * vals[3]) / denom);
  const float oy = (float)((vals[2] * vals[3] - 2.0 * vals[0] * vals[4]) / denom);
  const double sX = 0.34574, sY = 0.38944;
  double x = erf(ox / (sX * sqrt(2.0))) / 2.0, y = erf(oy / (sY * sqrt(2.0))) / 2.0;
  const double nrm = sqrt(x * x + y * y);
  if (nrm >= 0.5) { const double scale = nrm / 0.5; x /= scale; y /= scale; }
  *dx = x; *dy = y;
  return 1;
}

static int sgm_core(const float* left_f, int lw, int lh, int lpitch, const float* right_f, int rw, int rh, int rpitch,
                    int search_x, int search_y, int kernel_size, int p1, int p2, int* out, int* out_w, int* out_h,
                    int subpixel_mode, float* out_sub);

int vwo_sgm_calc_disparity(const float* left_f, int lw, int lh, int lpitch, const float* right_f, int rw, int rh, int rpitch,
                           int search_x, int search_y, int kernel_size, int p1, int p2, int* out, int* out_w, int* out_h) {
  return sgm_core(left_f, lw, lh, lpitch, right_f, rw, rh, rpitch, search_x, search_y, kernel_size, p1, p2, out, out_w, out_h, 0, NULL);
}
/* calc_disparity_sgm followed by create_disparity_view_subpixel on its (unfiltered) integer result (:1497-1614).
 * subpixel_mode: SgmSubpixelMode (SGM.h:93-99) 0 none, 2 linear, 3 poly4, 4 cosine, 5 lc_blend; 1 (2-D parabola) is not restated. */
int vwo_sgm_calc_disparity_subpixel(const float* left_f, int lw, int lh, int lpitch, const float* right_f, int rw, int rh, int rpitch,
                                    int search_x, int search_y, int kernel_size, int p1, int p2, int subpixel_mode,
                                    int* out, float* out_sub, int* out_w, int* out_h) {
  if (subpixel_mode == 1 || subpixel_mode < 0 || subpixel_mode > 5) return -2;
  return sgm_core(left_f, lw, lh, lpitch, right_f, rw, rh, rpitch, search_x, search_y, kernel_size, p1, p2, out, out_w, out_h, subpixel_mode, out_sub);
}

static int sgm_core(const float* left_f, int lw, int lh, int lpitch, const float* right_f, int rw, int rh, int rpitch,
                    int search_x, int search_y, int kernel_size, int p1, int p2, int* out, int* out_w, int* out_h,
                    int subpixel_mode, float* out_sub) {
  if (kernel_size != 3 && kernel_size != 5 && kernel_size != 7 && kernel_size != 9) return -2;     /* NoImplErr (:1885-1888) */
  if (search_x < 0 || search_y < 0) return -1;
  if (p1 <= 0) p1 = kernel_size == 3 ? 3 : kernel_size == 5 ? 15 : kernel_size == 7 ? 30 : 20;      /* set_parameters (:112-122) */
  if (p2 <= 0) p2 = kernel_size == 3 ? 70 : kernel_size == 5 ? 750 : kernel_size == 7 ? 1500 : 1000; /* (:141-151) */
  uint8_t* left = (uint8_t*)malloc((size_t)lw * lh);
  uint8_t* right = (uint8_t*)malloc((size_t)rw * rh);
  u8_convert(left_f, lw, lh, lpitch, left);
  u8_convert(right_f, rw, rh, rpitch, right);
  const int hk = (kernel_size - 1) / 2;
  Sgm s;
  s.ndx = search_x + 1; s.ndy = search_y + 1; s.nd = s.ndx * s.ndy; s.p1 = p1; s.p2 = p2;
  /* semi_global_matching_func (:2397-2420); min_disp = 0, max_disp = search */
  int min_row = hk, min_col = hk;
  int max_row = (lh - 1 - hk) < (rh - 1 - (hk + search_y)) ? (lh - 1 - hk) : (rh - 1 - (hk + search_y));
  int max_col = (lw - 1 - hk) < (rw - 1 - (hk + search_x)) ? (lw - 1 - hk) : (rw - 1 - (hk + search_x));
  if (max_row > lh - 1) max_row = lh - 1;
  if (max_col > lw - 1) max_col = lw - 1;
  s.ow = max_col - min_col + 1; s.oh = max_row - min_row + 1; s.min_col = min_col; s.min_row = min_row;
  *out_w = s.ow > 0 ? s.ow : 0; *out_h = s.oh > 0 ? s.oh : 0;
  if (s.ow <= 0 || s.oh <= 0) { free(left); free(right); return 0; }
  s.left = left; s.lw = lw;
  /* census images (:1740-1873) and Hamming costs (get_hamming_distance_costs, :39-73) */
  const int clw = lw - 2 * hk, clh = lh - 2 * hk, crw = rw - 2 * hk, crh = rh - 2 * hk;
  uint64_t* lc = (uint64_t*)malloc((size_t)clw * clh * 8);
  uint64_t* rc = (uint64_t*)malloc((size_t)crw * crh * 8);
  for (int r = 0; r < clh; ++r) for (int c = 0; c < clw; ++c) lc[(size_t)r * clw + c] = census_value(left, lw, c + hk, r + hk, kernel_size);
  for (int r = 0; r < crh; ++r) for (int c = 0; c < crw; ++c) rc[(size_t)r * crw + c] = census_value(right, rw, c + hk, r + hk, kernel_size);
  const size_t total = (size_t)s.ow * s.oh * s.nd;
  cost_t* cost = (cost_t*)malloc(total);
  accum_t* accum = (accum_t*)calloc(total, sizeof(accum_t));
  size_t ci = 0;
  for (int r = min_row; r <= max_row; ++r)
    for (int c = min_col; c <= max_col; ++c) {
      const int br = r - hk, bc = c - hk;
      for (int dy = 0; dy <= search_y; ++dy)
        for (int dx = 0; dx <= search_x; ++dx)
          cost[ci++] = (cost_t)popcount64(lc[(size_t)br * clw + bc] ^ rc[(size_t)(br + dy) * crw + (bc + dx)]);
    }
  s.cost = cost; s.accum = accum;
  /* adjacent-disparity table (:755-800) */
  s.adj = (int*)malloc((size_t)s.nd * 8 * sizeof(int));
  for (int dy = 0, d = 0; dy < s.ndy; ++dy) {
    const int yl = dy - 1 < 0 ? dy : dy - 1, ym = dy + 1 > search_y ? dy : dy + 1;
    for (int dx = 0; dx < s.ndx; ++dx, ++d) {
      const int xl = dx - 1 < 0 ? dx : dx - 1, xm = dx + 1 > search_x ? dx : dx + 1;
      int* a = s.adj + (size_t)d * 8;
      a[0] = yl * s.ndx + dx; a[1] = dy * s.ndx + xl; a[2] = dy * s.ndx + xm; a[3] = ym * s.ndx + dx;
      a[4] = yl * s.ndx + xl; a[5] = yl * s.ndx + xm; a[6] = ym * s.ndx + xl; a[7] = ym * s.ndx + xm;
    }
  }
  /* the eight directions of accum_sgm_multithread (:2462-2611): a line starts at every pixel whose predecessor is outside */
  static const int DIRS[8][2] = {{0, 1}, {0, -1}, {1, 0}, {-1, 0}, {1, 1}, {-1, 1}, {1, -1}, {-1, -1}};
  accum_t* buf = (accum_t*)malloc((size_t)2 * s.nd * sizeof(accum_t));
  for (int k = 0; k < 8; ++k) {
    const int sc = DIRS[k][0], sr = DIRS[k][1];
    for (int r = 0; r < s.oh; ++r)
      for (int c = 0; c < s.ow; ++c) {
        const int pc = c - sc, pr = r - sr;
        if (pc >= 0 && pc < s.ow && pr >= 0 && pr < s.oh) continue;
        sgm_line(&s, c, r, sc, sr, buf);
      }
  }
  /* create_disparity_view (:1290-1346) */
  accum_t* tmp = (accum_t*)malloc((size_t)s.nd * sizeof(accum_t));
  for (int j = 0; j < s.oh; ++j)
    for (int i = 0; i < s.ow; ++i) {
      const int idx = select_best(accum + ((size_t)j * s.ow + i) * s.nd, s.ndx, s.ndy, tmp);
      int* o = out + ((size_t)j * s.ow + i) * 3;
      o[1] = idx / s.ndx; o[0] = idx - o[1] * s.ndx; o[2] = 1;      /* disp_index_to_xy (:2737-2745), bounds = (0,0,sx,sy) */
    }
  if (out_sub) {                                                      /* create_disparity_view_subpixel (:1497-1614) */
    for (int j = 0; j < s.oh; ++j)
      for (int i = 0; i < s.ow; ++i) {
        const int* o = out + ((size_t)j * s.ow + i) * 3;
        float* f = out_sub + ((size_t)j * s.ow + i) * 3;
        const int dx = o[0], dy = o[1], width = s.ndx;
        f[2] = 1.0f;
        if (subpixel_mode == 0) { f[0] = (float)dx; f[1] = (float)dy; continue; }
        const int min_index = dy * width + dx;
        int x_left = -1, x_right = 1, y_up = -width, y_down = width;
        int lb = 0, rb = 0, tb = 0, bb = 0;
        if (dx == 0) { x_left = 0; lb = 1; }
        if (dx == search_x) { x_right = 0; rb = 1; }
        if (dy == 0) { y_up = 0; tb = 1; }
        if (dy == search_y) { y_down = 0; bb = 1; }
        const accum_t* av = accum + ((size_t)j * s.ow + i) * s.nd;
        const double ddx = subpixel_offset(av[min_index + x_left], av[min_index], av[min_index + x_right], lb, rb, subpixel_mode);
        const double ddy = subpixel_offset(av[min_index + y_up], av[min_index], av[min_index + y_down], tb, bb, subpixel_mode);
        f[0] = (float)(dx + ddx); f[1] = (float)(dy + ddy);          /* p_type(dx+delta_x, dy+delta_y): Vector2f from double */
      }
  }
  free(tmp); free(buf); free(s.adj); free(cost); free(accum); free(lc); free(rc); free(left); free(right);
  return 0;
}

/* ------------------------------------------------------------------------------------------------------------------------
 * The same pipeline with a search box PER PIXEL (m_disp_bound_image, SGM.h:303; consumed by get_hamming_distance_costs
 * :39-73, calc_main_buf_size :677-731, evaluate_path :1014-1141, create_disparity_view :1290-1346,
 * create_disparity_view_subpixel :1497-1614).  bounds: out_w * out_h quadruples {min_x, min_y, max_x, max_y} (inclusive,
 * inside [0, search]; max < min = "no search area", the pixel comes out invalid).  How the reference derives the boxes from
 * the previous pyramid level (populate_disp_bound_image / constrain_disp_bound_image, :241-675) is not restated yet: this
 * entry takes them as input, which is what the device kernels of round 2 will consume.
 * ---------------------------------------------------------------------------------------------------------------------- */
typedef struct {
  int ndx, ndy, nd, p1, p2, ow, oh, min_col, min_row, lw;
  const uint8_t* left;
  const int* bounds;       /* [oh][ow][4] */
  const size_t* starts;    /* m_buffer_starts (:684-692) */
  const cost_t* cost;
  accum_t* accum;
  const int* adj;
} SgmB;

static inline int nb_disp(const int* b) { return (b[2] < b[0] || b[3] < b[1]) ? 0 : (b[2] - b[0] + 1) * (b[3] - b[1] + 1); }   /* SGM.h:244-251 */

/* evaluate_path, SSE flavour (:1014-1141), for a pixel with box b whose predecessor has box bp and packed costs prior */
static void eval_path_bounds(const SgmB* s, const int* b, const int* bp, const accum_t* prior, const cost_t* local, accum_t* out, int diff,
                             accum_t* full_prior /* nd, all BAD on entry and on exit */) {
  const accum_t BAD = (accum_t)(255 + s->p2);
  accum_t p2_mod = (accum_t)s->p2;
  if (diff > 0) p2_mod = (accum_t)(p2_mod / diff);
  if (p2_mod < s->p1) p2_mod = (accum_t)s->p1;
  accum_t min_prior = BAD;
  int d = 0;
  for (int dy = bp[1]; dy <= bp[3]; ++dy)                           /* scatter the previous pixel's costs (:1037-1054) */
    for (int dx = bp[0]; dx <= bp[2]; ++dx, ++d) {
      if (prior[d] < min_prior) min_prior = prior[d];
      full_prior[dy * s->ndx + dx] = prior[d];
    }
  const accum_t dJ = (accum_t)(min_prior + p2_mod);
  int pd = 0;
  for (int dy = b[1]; dy <= b[3]; ++dy)
    for (int dx = b[0]; dx <= b[2]; ++dx, ++pd) {
      const int fd = dy * s->ndx + dx;
      const int* a = s->adj + (size_t)fd * 8;
      accum_t m = min16(min16(min16(full_prior[a[0]], full_prior[a[1]]), min16(full_prior[a[2]], full_prior[a[3]])),
                        min16(min16(full_prior[a[4]], full_prior[a[5]]), min16(full_prior[a[6]], full_prior[a[7]])));
      accum_t res = sat_add(m, (accum_t)s->p1);
      res = min16(res, min16(full_prior[fd], dJ));
      res = sat_add(res, (accum_t)local[pd]);
      out[pd] = sat_sub(res, min_prior);
    }
  for (int dy = bp[1]; dy <= bp[3]; ++dy)                           /* restore the flag value (:1131-1139) */
    for (int dx = bp[0]; dx <= bp[2]; ++dx) full_prior[dy * s->ndx + dx] = BAD;
}

static void sgm_line_bounds(const SgmB* s, int c, int r, int sc, int sr, accum_t* buf /* 2 * nd */, accum_t* full_prior /* nd, all BAD */) {
  accum_t* prior = buf;
  accum_t* cur = buf + s->nd;
  int last_val = -1;
  const int* bp = NULL;                     /* previous pixel's box */
  while (c >= 0 && c < s->ow && r >= 0 && r < s->oh) {
    const int* b = s->bounds + ((size_t)r * s->ow + c) * 4;
    const int n = nb_disp(b);
    const size_t st = s->starts[(size_t)r * s->ow + c];
    const cost_t* local = s->cost + st;
    const int cur_val = s->left[(size_t)(r + s->min_row) * s->lw + (c + s->min_col)];
    const int diff = abs(cur_val - last_val);
    if (last_val >= 0) eval_path_bounds(s, b, bp, prior, local, cur, diff, full_prior);
    else for (int d = 0; d < n; ++d) cur[d] = local[d];
    accum_t* acc = s->accum + st;
    for (int d = 0; d < n; ++d) acc[d] = (accum_t)(acc[d] + cur[d]);
    accum_t* t = prior; prior = cur; cur = t;
    bp = b;
    last_val = cur_val;
    c += sc; r += sr;
  }
}

/* MGM (accum_mgm_multithread, SGM.cc:2619-2700; SmoothPathAccumTask, SGMAssist.h:835-1239): eight full-image sweeps; in
 * each, a pixel's path cost is the (truncating) mean of evaluate_path from TWO predecessors, or its local cost on the
 * borders listed below; the sweep's result is added to the accumulation buffer (MultiAccumRowBuffer::add_lead_buffer_to_accum,
 * :357-387).  Both evaluations use the SAME grey-value difference, and get_path_pixel_diff (SGM.cc:2715-2721) looks at the
 * pixel OPPOSITE to the direction it is given -- kept as is. */
typedef struct { int p1c, p1r, p2c, p2r, dirx, diry; int need_r_gt0, need_r_lt, need_c_gt0, need_c_lt; int col_major, c_desc, r_desc; } MgmTask;
static const MgmTask MGM_TASKS[8] = {
  /* L  */ {-1, 0, 0, -1, -1, 0, 1, 0, 1, 0, 0, 0, 0},
  /* R  */ {1, 0, 0, 1, 1, 0, 0, 1, 0, 1, 0, 1, 1},
  /* TL */ {-1, -1, 1, -1, -1, -1, 1, 0, 1, 1, 0, 0, 0},
  /* BR */ {1, 1, -1, 1, 1, 1, 0, 1, 1, 1, 0, 1, 1},
  /* T  */ {0, -1, 1, 0, 0, -1, 1, 0, 0, 1, 1, 1, 0},
  /* B  */ {0, 1, -1, 0, 0, 1, 0, 1, 1, 0, 1, 0, 1},
  /* TR */ {1, -1, 1, 1, 1, -1, 1, 1, 0, 1, 1, 1, 0},
  /* BL */ {-1, 1, -1, -1, -1, 1, 1, 1, 1, 0, 1, 0, 1},
};
static void mgm_sweep(const SgmB* s, const MgmTask* t, accum_t* path /* ragged, like accum */, accum_t* tmp /* nd */, accum_t* full_prior) {
  const int last_c = s->ow - 1, last_r = s->oh - 1;
  const int n_outer = t->col_major ? s->ow : s->oh, n_inner = t->col_major ? s->oh : s->ow;
  for (int oo = 0; oo < n_outer; ++oo)
    for (int ii = 0; ii < n_inner; ++ii) {
      int c, r;
      if (t->col_major) { c = t->c_desc ? last_c - oo : oo; r = t->r_desc ? last_r - ii : ii; }
      else { r = t->r_desc ? last_r - oo : oo; c = t->c_desc ? last_c - ii : ii; }
      const size_t pix = (size_t)r * s->ow + c;
      const int* b = s->bounds + pix * 4;
      const int n = nb_disp(b);
      if (n == 0) continue;
      const cost_t* local = s->cost + s->starts[pix];
      accum_t* out = path + s->starts[pix];
      const int ok = (!t->need_r_gt0 || r > 0) && (!t->need_r_lt || r < last_r) && (!t->need_c_gt0 || c > 0) && (!t->need_c_lt || c < last_c);
      if (!ok) { for (int d = 0; d < n; ++d) out[d] = local[d]; continue; }
      const int a = s->left[(size_t)(r + s->min_row) * s->lw + (c + s->min_col)];
      const int bb = s->left[(size_t)(r - t->diry + s->min_row) * s->lw + (c - t->dirx + s->min_col)];
      const int diff = abs(a - bb);
      const size_t q1 = (size_t)(r + t->p1r) * s->ow + (c + t->p1c), q2 = (size_t)(r + t->p2r) * s->ow + (c + t->p2c);
      eval_path_bounds(s, b, s->bounds + q1 * 4, path + s->starts[q1], local, out, diff, full_prior);
      eval_path_bounds(s, b, s->bounds + q2 * 4, path + s->starts[q2], local, tmp, diff, full_prior);
      for (int d = 0; d < n; ++d) out[d] = (accum_t)(((int)out[d] + (int)tmp[d]) / 2);
    }
}

/* cost type of the current call: 0 = CENSUS_TRANSFORM, 1 = TERNARY_CENSUS_TRANSFORM (+ its threshold) */
static __thread int t_ternary = 0, t_ternary_thr = 5;
static int sgm_bounds_core(const float* left_f, int lw, int lh, int lpitch, const float* right_f, int rw, int rh, int rpitch,
                           int search_x, int search_y, int kernel_size, int p1, int p2, int subpixel_mode, const int* bounds,
                           int* out, float* out_sub, int* out_w, int* out_h, int use_mgm);
int vwo_sgm_calc_disparity_bounds(const float* left_f, int lw, int lh, int lpitch, const float* right_f, int rw, int rh, int rpitch,
                                  int search_x, int search_y, int kernel_size, int p1, int p2, int subpixel_mode, const int* bounds,
                                  int* out, float* out_sub, int* out_w, int* out_h) {
  return sgm_bounds_core(left_f, lw, lh, lpitch, right_f, rw, rh, rpitch, search_x, search_y, kernel_size, p1, p2, subpixel_mode, bounds, out, out_sub,
                         out_w, out_h, 0);
}
/* the same with MGM accumulation (use_mgm of calc_disparity_sgm) */
int vwo_mgm_calc_disparity_bounds(const float* left_f, int lw, int lh, int lpitch, const float* right_f, int rw, int rh, int rpitch,
                                  int search_x, int search_y, int kernel_size, int p1, int p2, int subpixel_mode, const int* bounds,
                                  int* out, float* out_sub, int* out_w, int* out_h) {
  return sgm_bounds_core(left_f, lw, lh, lpitch, right_f, rw, rh, rpitch, search_x, search_y, kernel_size, p1, p2, subpixel_mode, bounds, out, out_sub,
                         out_w, out_h, 1);
}
static int sgm_bounds_core(const float* left_f, int lw, int lh, int lpitch, const float* right_f, int rw, int rh, int rpitch,
                           int search_x, int search_y, int kernel_size, int p1, int p2, int subpixel_mode, const int* bounds,
                           int* out, float* out_sub, int* out_w, int* out_h, int use_mgm) {
  if (kernel_size != 3 && kernel_size != 5 && kernel_size != 7 && kernel_size != 9) return -2;
  if (search_x < 0 || search_y < 0 || !bounds) return -1;
  if (out_sub && (subpixel_mode < 0 || subpixel_mode > 5)) return -2;
  const int ternary = t_ternary, tern_thr = t_ternary_thr;
  if (!ternary) {                                                                           /* set_parameters (SGM.cc:106-157) */
    if (p1 <= 0) p1 = kernel_size == 3 ? 3 : kernel_size == 5 ? 15 : kernel_size == 7 ? 30 : 20;
    if (p2 <= 0) p2 = kernel_size == 3 ? 70 : kernel_size == 5 ? 750 : kernel_size == 7 ? 1500 : 1000;
  } else {
    if (p1 <= 0) p1 = kernel_size == 3 ? 12 : kernel_size == 5 ? 30 : 40;
    if (p2 <= 0) p2 = kernel_size == 3 ? 600 : kernel_size == 5 ? 1500 : 2000;
  }
  const int hk = (kernel_size - 1) / 2;
  SgmB s;
  s.ndx = search_x + 1; s.ndy = search_y + 1; s.nd = s.ndx * s.ndy; s.p1 = p1; s.p2 = p2; s.lw = lw;
  const int min_row = hk, min_col = hk;
  int max_row = (lh - 1 - hk) < (rh - 1 - (hk + search_y)) ? (lh - 1 - hk) : (rh - 1 - (hk + search_y));
  int max_col = (lw - 1 - hk) < (rw - 1 - (hk + search_x)) ? (lw - 1 - hk) : (rw - 1 - (hk + search_x));
  if (max_row > lh - 1) max_row = lh - 1;
  if (max_col > lw - 1) max_col = lw - 1;
  s.ow = max_col - min_col + 1; s.oh = max_row - min_row + 1; s.min_col = min_col; s.min_row = min_row;
  *out_w = s.ow > 0 ? s.ow : 0; *out_h = s.oh > 0 ? s.oh : 0;
  if (s.ow <= 0 || s.oh <= 0) return 0;
  const size_t npix = (size_t)s.ow * s.oh;
  for (size_t i = 0; i < npix; ++i) {
    const int* b = bounds + i * 4;
    if (nb_disp(b) && (b[0] < 0 || b[1] < 0 || b[2] > search_x || b[3] > search_y)) return -1;
  }
  uint8_t* left = (uint8_t*)malloc((size_t)lw * lh);
  uint8_t* right = (uint8_t*)malloc((size_t)rw * rh);
  u8_convert(left_f, lw, lh, lpitch, left);
  u8_convert(right_f, rw, rh, rpitch, right);
  s.left = left; s.bounds = bounds;
  size_t* starts = (size_t*)malloc(npix * sizeof(size_t));
  size_t total = 0;
  for (size_t i = 0; i < npix; ++i) { starts[i] = total; total += (size_t)nb_disp(bounds + i * 4); }
  if (total < 6) total = 6;                                            /* (:695-696) */
  s.starts = starts;
  const int clw = lw - 2 * hk, clh = lh - 2 * hk, crw = rw - 2 * hk, crh = rh - 2 * hk;
  uint64_t* lc = (uint64_t*)malloc((size_t)clw * clh * 8);
  uint64_t* rc = (uint64_t*)malloc((size_t)crw * crh * 8);
  for (int r = 0; r < clh; ++r) for (int c = 0; c < clw; ++c) lc[(size_t)r * clw + c] = vwo_census_value(left, lw, c + hk, r + hk, kernel_size, ternary, tern_thr);
  for (int r = 0; r < crh; ++r) for (int c = 0; c < crw; ++c) rc[(size_t)r * crw + c] = vwo_census_value(right, rw, c + hk, r + hk, kernel_size, ternary, tern_thr);
  cost_t* cost = (cost_t*)malloc(total);
  accum_t* accum = (accum_t*)calloc(total, sizeof(accum_t));
  size_t ci = 0;
  for (int r = min_row; r <= max_row; ++r)
    for (int c = min_col; c <= max_col; ++c) {
      const int br = r - hk, bc = c - hk;
      const int* b = bounds + ((size_t)(r - min_row) * s.ow + (c - min_col)) * 4;
      for (int dy = b[1]; dy <= b[3]; ++dy)
        for (int dx = b[0]; dx <= b[2]; ++dx)
          cost[ci++] = (cost_t)popcount64(lc[(size_t)br * clw + bc] ^ rc[(size_t)(br + dy) * crw + (bc + dx)]);
    }
  s.cost = cost; s.accum = accum;
  int* adj = (int*)malloc((size_t)s.nd * 8 * sizeof(int));
  for (int dy = 0, d = 0; dy < s.ndy; ++dy) {
    const int yl = dy - 1 < 0 ? dy : dy - 1, ym = dy + 1 > search_y ? dy : dy + 1;
    for (int dx = 0; dx < s.ndx; ++dx, ++d) {
      const int xl = dx - 1 < 0 ? dx : dx - 1, xm = dx + 1 > search_x ? dx : dx + 1;
      int* a = adj + (size_t)d * 8;
      a[0] = yl * s.ndx + dx; a[1] = dy * s.ndx + xl; a[2] = dy * s.ndx + xm; a[3] = ym * s.ndx + dx;
      a[4] = yl * s.ndx + xl; a[5] = yl * s.ndx + xm; a[6] = ym * s.ndx + xl; a[7] = ym * s.ndx + xm;
    }
  }
  s.adj = adj;
  static const int DIRS[8][2] = {{0, 1}, {0, -1}, {1, 0}, {-1, 0}, {1, 1}, {-1, 1}, {1, -1}, {-1, -1}};
  accum_t* buf = (accum_t*)malloc((size_t)2 * s.nd * sizeof(accum_t));
  accum_t* full_prior = (accum_t*)malloc((size_t)s.nd * sizeof(accum_t));
  for (int d = 0; d < s.nd; ++d) full_prior[d] = (accum_t)(255 + p2);
  if (!use_mgm) {
    for (int k = 0; k < 8; ++k) {
      const int sc = DIRS[k][0], sr = DIRS[k][1];
      for (int r = 0; r < s.oh; ++r)
        for (int c = 0; c < s.ow; ++c) {
          const int pc = c - sc, pr = r - sr;
          if (pc >= 0 && pc < s.ow && pr >= 0 && pr < s.oh) continue;
          sgm_line_bounds(&s, c, r, sc, sr, buf, full_prior);
        }
    }
  } else {
    accum_t* path = (accum_t*)malloc(total * sizeof(accum_t));
    for (int k = 0; k < 8; ++k) {
      memset(path, 0, total * sizeof(accum_t));
      mgm_sweep(&s, &MGM_TASKS[k], path, buf, full_prior);
      for (size_t i = 0; i < total; ++i) accum[i] = (accum_t)(accum[i] + path[i]);
    }
    free(path);
  }
  accum_t* tmp = (accum_t*)malloc((size_t)s.nd * sizeof(accum_t));
  for (int j = 0; j < s.oh; ++j)
    for (int i = 0; i < s.ow; ++i) {
      const size_t pix = (size_t)j * s.ow + i;
      const int* b = bounds + pix * 4;
      int* o = out + pix * 3;
      float* f = out_sub ? out_sub + pix * 3 : NULL;
      if (nb_disp(b) == 0) {                                          /* never valid (:1317-1321) */
        o[0] = o[1] = o[2] = 0;
        if (f) { f[0] = f[1] = f[2] = 0.0f; }
        continue;
      }
      const int width = b[2] - b[0] + 1, height = b[3] - b[1] + 1;
      accum_t* av = accum + starts[pix];
      const int idx = select_best(av, width, height, tmp);
      const int dyi = idx / width;
      const int dx = idx - dyi * width + b[0], dy = dyi + b[1];     /* disp_index_to_xy (:2737-2745) */
      o[0] = dx; o[1] = dy; o[2] = 1;
    }
  if (out_sub) {
    for (int j = 0; j < s.oh; ++j)
      for (int i = 0; i < s.ow; ++i) {
        const size_t pix = (size_t)j * s.ow + i;
        const int* b = bounds + pix * 4;
        const int* o = out + pix * 3;
        float* f = out_sub + pix * 3;
        if (!o[2]) continue;
        const int dx = o[0], dy = o[1], width = b[2] - b[0] + 1;
        f[2] = 1.0f;
        if (subpixel_mode == 0) { f[0] = (float)dx; f[1] = (float)dy; continue; }
        const int min_index = (dy - b[1]) * width + (dx - b[0]);
        int x_left = -1, x_right = 1, y_up = -width, y_down = width;
        int lb = 0, rb = 0, tb = 0, bb = 0;
        if (dx == b[0]) { x_left = 0; lb = 1; }
        if (dx == b[2]) { x_right = 0; rb = 1; }
        if (dy == b[1]) { y_up = 0; tb = 1; }
        if (dy == b[3]) { y_down = 0; bb = 1; }
        const accum_t* av = accum + starts[pix];
        double ddx, ddy;
        if (subpixel_mode == 1) {                                          /* SUBPIXEL_PARABOLA (:1566-1576) */
          if (!parabola_peak(av[min_index + x_left + y_up], av[min_index + y_up], av[min_index + x_right + y_up], av[min_index + x_left],
                             av[min_index], av[min_index + x_right], av[min_index + x_left + y_down], av[min_index + y_down],
                             av[min_index + x_right + y_down], &ddx, &ddy)) { f[0] = (float)dx; f[1] = (float)dy; continue; }
        } else {
          ddx = subpixel_offset(av[min_index + x_left], av[min_index], av[min_index + x_right], lb, rb, subpixel_mode);
          ddy = subpixel_offset(av[min_index + y_up], av[min_index], av[min_index + y_down], tb, bb, subpixel_mode);
        }
        f[0] = (float)(dx + ddx); f[1] = (float)(dy + ddy);
      }
  }
  free(tmp); free(full_prior); free(buf); free(adj); free(cost); free(accum); free(lc); free(rc); free(starts); free(left); free(right);
  return 0;
}

/* ------------------------------------------------------------------------------------------------------------------------
 * SemiGlobalMatcher::populate_disp_bound_image (SGM.cc:241-500) + one pass of constrain_disp_bound_image (:502-668): the
 * per-pixel search boxes from the masks and the previous (half-resolution) disparity.  min_disp = (0,0), max_disp =
 * (search_x, search_y) as set up by calc_disparity_sgm.  The reference retries conservation levels 0..3 until
 * calc_main_buf_size() fits --corr-memory-mb (:476-497, thread-count dependent); here the level is an input.
 *   prev      : pw x ph {dx, dy, valid} ints or NULL        lmask : ow x oh uint8 or NULL (must match the output size, :250-256)
 *   rmask     : rmw x rmh uint8 or NULL (>= output + search, :262-268)
 *   bounds    : ow x oh {min_x, min_y, max_x, max_y}; (0,0,-1,-1) = no search area
 * Returns 1 (go on), 0 (the reference returns an all-invalid disparity, :2430-2436), < 0 on bad arguments.
 * vw::BBox2i quirks that matter here (Math/BBox.tcc): grow(point) makes max = point (not + 1); empty() is
 * min >= max in ANY axis, so a box grown from identical points counts as empty; expand() ignores empty boxes.
 * ---------------------------------------------------------------------------------------------------------------------- */
typedef struct { int x0, y0, x1, y1; } IBox;
static const IBox IBOX_EMPTY = {2147483647, 2147483647, -2147483647 - 1, -2147483647 - 1};
static int ibox_empty(const IBox* b) { return b->x0 >= b->x1 || b->y0 >= b->y1; }
static void ibox_grow(IBox* b, int x, int y) { if (x > b->x1) b->x1 = x; if (x < b->x0) b->x0 = x; if (y > b->y1) b->y1 = y; if (y < b->y0) b->y0 = y; }
static void ibox_crop(IBox* b, const IBox* o) { if (b->x0 < o->x0) b->x0 = o->x0; if (b->x1 > o->x1) b->x1 = o->x1; if (b->y0 < o->y0) b->y0 = o->y0; if (b->y1 > o->y1) b->y1 = o->y1; }

int vwo_sgm_disp_bounds(const int* prev, int pw, int ph, const uint8_t* lmask, const uint8_t* rmask, int rmw, int rmh,
                        int ow, int oh, int search_x, int search_y, int buffer_x, int buffer_y, int conserve_level, int* bounds) {
  if (ow <= 0 || oh <= 0 || search_x < 0 || search_y < 0 || !bounds) return -1;
  const int ndx = search_x + 1, ndy = search_y + 1;
  if (rmask && !(rmw >= ow + ndx - 1 && rmh >= oh + ndy - 1)) return -3;               /* LogicErr (:262-268) */
  const int check_x_edge = ndx >= 10, check_y_edge = ndy >= 10;                          /* (:286-289) */
  uint8_t* full = (uint8_t*)calloc((size_t)ow * oh, 1);
  double area = 0, percent_trusted = 0, percent_masked = 0;
  int min_vr = 0, max_vr = 0;                                                            /* (:303-331) */
  if (rmask) {
    min_vr = rmh - 1;
    for (int c = 0; c < ow; ++c) {
      for (int i = rmh - 1; i > 0; --i) if (rmask[(size_t)i * rmw + c] > 0) { if (i > max_vr) max_vr = i; break; }
      for (int i = 0; i < rmh; ++i) if (rmask[(size_t)i * rmw + c] > 0) { if (i < min_vr) min_vr = i; break; }
    }
  }
  for (int r = 0; r < oh; ++r) {
    const int r_in = r / 2;
    int min_vc = -1, max_vc = -2;
    if (rmask) {                                                                         /* (:343-359) */
      for (int i = rmw - 1; i > 0; --i) if (rmask[(size_t)r * rmw + i] > 0) { max_vc = i; break; }
      if (max_vc > 0) for (int i = 0; i < rmw; ++i) if (rmask[(size_t)r * rmw + i] > 0) { min_vc = i; break; }
    }
    for (int c = 0; c < ow; ++c) {
      int* b = bounds + ((size_t)r * ow + c) * 4;
      if (lmask && lmask[(size_t)r * ow + c] == 0) { b[0] = 0; b[1] = 0; b[2] = -1; b[3] = -1; percent_masked += 1; continue; }
      int good = 0, dxs = 0, dys = 0;
      const int c_in = c / 2;
      if (prev && c_in < pw && r_in < ph) {                                              /* (:385-403) */
        const int* d = prev + ((size_t)r_in * pw + c_in) * 3;
        dxs = d[0] * 2; dys = d[1] * 2;
        const int on_edge = (check_x_edge && (dxs <= 0 || dxs >= search_x)) || (check_y_edge && (dys <= 0 || dys >= search_y));
        good = d[2] != 0 && !on_edge;
      }
      if (good) {                                                                        /* (:407-422) */
        b[0] = dxs - buffer_x; b[2] = dxs + buffer_x; b[1] = dys - buffer_y; b[3] = dys + buffer_y;
        if (b[0] < 0) b[0] = 0;
        if (b[1] < 0) b[1] = 0;
        if (b[2] > search_x) b[2] = search_x;
        if (b[3] > search_y) b[3] = search_y;
        percent_trusted += 1.0;
      } else {
        b[0] = 0; b[1] = 0; b[2] = search_x; b[3] = search_y;
        full[(size_t)r * ow + c] = 255;
      }
      if (rmask) {                                                                       /* (:431-452) */
        IBox v = {min_vc - c, min_vr - r, max_vc - c, max_vr - r};
        const IBox fo = {b[0], b[1], b[2], b[3]};
        ibox_crop(&v, &fo);
        if (v.x0 > v.x1 || v.y0 > v.y1) { b[0] = 0; b[1] = 0; b[2] = -1; b[3] = -1; percent_masked += 1; full[(size_t)r * ow + c] = 0; continue; }
        b[0] = v.x0; b[1] = v.y0; b[2] = v.x1; b[3] = v.y1;
      }
      area += (double)((b[3] - b[1] + 1) * (b[2] - b[0] + 1));
    }
  }
  const double num_pixels = (double)oh * ow;
  percent_masked /= num_pixels;
  percent_trusted /= num_pixels;
  /* constrain_disp_bound_image (:502-668) */
  const IBox max_range = {0, 0, search_x, search_y};
  int range = 10;
  if (conserve_level == 1) range = 25;
  if (conserve_level == 2) range = 3;
  if (conserve_level == 3) range = 0;
  if (prev) {
    for (int r = 0; r < oh; ++r) {
      int r0 = r - range, r1 = r + range;
      if (r0 < 0) r0 = 0;
      if (r1 >= oh) r1 = oh - 1;
      for (int c = 0; c < ow; ++c) {
        if (!full[(size_t)r * ow + c]) continue;
        int c0 = c - range, c1 = c + range;
        if (c0 < 0) c0 = 0;
        if (c1 >= ow) c1 = ow - 1;
        IBox nr = IBOX_EMPTY;
        for (int rs = r0; rs <= r1; ++rs)
          for (int cs = c0; cs <= c1; ++cs) {
            if (full[(size_t)rs * ow + cs]) continue;
            const int* v = bounds + ((size_t)rs * ow + cs) * 4;
            if (v[0] == 0 && v[1] == 0 && v[2] == -1 && v[3] == -1) continue;
            ibox_grow(&nr, v[0], v[1]);
            ibox_grow(&nr, v[2], v[3]);
          }
        int* b = bounds + ((size_t)r * ow + c) * 4;
        if (ibox_empty(&nr)) {
          if (conserve_level > 0) { b[0] = 0; b[1] = 0; b[2] = -1; b[3] = -1; }
          continue;
        }
        nr.x0 -= 2; nr.y0 -= 2; nr.x1 += 2; nr.y1 += 2;                                 /* expand(NEARBY_DISP_EXPANSION) */
        ibox_crop(&nr, &max_range);
        b[0] = nr.x0; b[1] = nr.y0; b[2] = nr.x1; b[3] = nr.y1;
      }
    }
  }
  free(full);
  area /= num_pixels;
  return !(area <= 0 || percent_masked >= 100);                                          /* (:664-666) */
}

/* ------------------------------------------------------------------------------------------------------------------------
 * The whole of vw::stereo::calc_disparity_sgm (SGM.cc:167-230) with its optional arguments: cost type (3 = CENSUS_TRANSFORM,
 * 4 = TERNARY_CENSUS_TRANSFORM, CostFunctions.h:143-149; anything else -> -4, the NoImplErr of :1888-1892), SGM / MGM,
 * sub-pixel mode, search buffer, masks, previous disparity and the memory-limit retry loop of populate_disp_bound_image
 * (:476-497; calc_main_buf_size :677-731 with `threads` = vw_settings().default_num_threads()).  bounds_io != NULL and
 * use_given_bounds != 0: take the boxes from there; otherwise the derived boxes are written there (if not NULL).
 * ---------------------------------------------------------------------------------------------------------------------- */
static int mem_fits(size_t main_buf, int ow, int oh, int search_x, int search_y, int use_mgm, int threads, double limit_mb) {
  if (main_buf < 6) main_buf = 6;
  const size_t nd = (size_t)(search_x + 1) * (search_y + 1);
  size_t small;
  if (use_mgm) {                                                    /* (:709-713), MultiAccumRowBuffer::multi_buf_size */
    size_t v = (size_t)oh * nd, h = (size_t)ow * nd;
    if (v > main_buf) v = main_buf;
    if (h > main_buf) h = main_buf;
    small = v * 4 + h * 4;
  } else {                                                          /* OneLineBuffer::one_buf_size (SGMAssist.h:565-583) */
    const int line = (int)(sqrt((double)(ow * ow + oh * oh)) + 1);
    size_t one = (size_t)line * nd;
    if (one > main_buf) one = main_buf;
    small = one * (size_t)threads;
  }
  const double mb = 1024.0 * 1024.0;
  return (double)main_buf * (3.0 / mb) + (double)small * (2.0 / mb) <= limit_mb;
}

int vwo_calc_disparity_sgm(const float* left_f, int lw, int lh, int lpitch, const float* right_f, int rw, int rh, int rpitch,
                           int search_x, int search_y, int kernel_size, int cost_type, int ternary_threshold, int p1, int p2, int use_mgm,
                           int subpixel_mode, int buffer_x, int buffer_y, double memory_limit_mb, int threads,
                           const uint8_t* lmask, const uint8_t* rmask, int rmw, int rmh, const int* prev, int pw, int ph,
                           int* bounds_io, int use_given_bounds, int* out, float* out_sub, int* out_w, int* out_h) {
  if (cost_type != 3 && cost_type != 4) return -4;
  if (kernel_size != 3 && kernel_size != 5 && kernel_size != 7 && kernel_size != 9) return -4;
  if (search_x < 0 || search_y < 0) return -1;
  const int hk = (kernel_size - 1) / 2;
  int max_row = (lh - 1 - hk) < (rh - 1 - (hk + search_y)) ? (lh - 1 - hk) : (rh - 1 - (hk + search_y));
  int max_col = (lw - 1 - hk) < (rw - 1 - (hk + search_x)) ? (lw - 1 - hk) : (rw - 1 - (hk + search_x));
  if (max_row > lh - 1) max_row = lh - 1;
  if (max_col > lw - 1) max_col = lw - 1;
  const int ow = max_col - hk + 1, oh = max_row - hk + 1;
  *out_w = ow > 0 ? ow : 0; *out_h = oh > 0 ? oh : 0;
  if (ow <= 0 || oh <= 0) return 0;
  const size_t npix = (size_t)ow * oh;
  int* bounds = (int*)malloc(npix * 4 * sizeof(int));
  int ok = 1;
  if (use_given_bounds && bounds_io) memcpy(bounds, bounds_io, npix * 4 * sizeof(int));
  else {
    ok = 0;
    for (int level = 0; level <= 3 && !ok; ++level) {
      const int rc = vwo_sgm_disp_bounds(prev, pw, ph, lmask, rmask, rmw, rmh, ow, oh, search_x, search_y, buffer_x, buffer_y, level, bounds);
      if (rc < 0) { free(bounds); return rc; }
      size_t total = 0;
      for (size_t i = 0; i < npix; ++i) total += (size_t)nb_disp(bounds + 4 * i);
      ok = mem_fits(total, ow, oh, search_x, search_y, use_mgm, threads, memory_limit_mb);
    }
    if (bounds_io) memcpy(bounds_io, bounds, npix * 4 * sizeof(int));
  }
  int rc = 0;
  if (!ok) {                                                        /* invalidate_mask(disparity) (:2430-2436) */
    memset(out, 0, npix * 3 * sizeof(int));
    if (out_sub) memset(out_sub, 0, npix * 3 * sizeof(float));
  } else {
    t_ternary = cost_type == 4; t_ternary_thr = ternary_threshold;
    int w2, h2;
    rc = sgm_bounds_core(left_f, lw, lh, lpitch, right_f, rw, rh, rpitch, search_x, search_y, kernel_size, p1, p2, subpixel_mode, bounds, out, out_sub,
                         &w2, &h2, use_mgm);
    t_ternary = 0; t_ternary_thr = 5;
  }
  free(bounds);
  return rc;
}
