/* vw_warp_oracle.c -- see vw_warp_oracle.h.  Types as in the reference: Vector2 is double, the bilinear real_type of a
 * float pixel is float, the bicubic result_type is double. */
#include "vw_warp_oracle.h"

#include <math.h>
#include <stddef.h>
#include <stdint.h>

typedef struct {
  const float* in;
  int w, h, edge;
} View;

/* math::impl::_floor / _round (Math/Functions.h:48-51, 74-81) */
static int32_t vw_floor(double val) {
  if (val < 0) {
    int32_t ival = (int32_t)val;
    if ((double)ival == val) return ival;
    return ival - 1;
  }
  return (int32_t)val;
}
static int32_t vw_round(double val) {
  if (val < 0) return (int32_t)(val - 0.5);
  return (int32_t)(val + 0.5);
}

/* EdgeExtensionView<ImageView<PixelGray<float>>, EdgeT>::operator()(i, j) */
static float edge_at(const View* v, int32_t i, int32_t j) {
  if (v->edge == 0) {
    if (i >= 0 && j >= 0 && i < v->w && j < v->h) return v->in[(size_t)j * v->w + i];
    return 0.0f;
  }
  return v->in[(size_t)((j < 0) ? 0 : (j >= v->h) ? (v->h - 1) : j) * v->w + ((i < 0) ? 0 : (i >= v->w) ? (v->w - 1) : i)];
}

static float bilinear(const View* v, double i, double j) {
  int32_t x = vw_floor(i), y = vw_floor(j);
  if (x == i && y == j) return edge_at(v, x, y);
  float normx = (float)i - (float)x, normy = (float)j - (float)y, norm1mx = 1 - normx, norm1my = 1 - normy;
  /* the accessor walks (x, y), (x + 1, y), advance(-1, 1) -> (x, y + 1), (x + 1, y + 1) */
  float result = edge_at(v, x, y) * norm1mx;
  result += edge_at(v, x + 1, y) * normx;
  result *= norm1my;
  float row = edge_at(v, x, y + 1) * norm1mx;
  row += edge_at(v, x + 1, y + 1) * normx;
  result += row * normy;
  return result;
}

static float bicubic(const View* v, double i, double j) {
  int32_t x = vw_floor(i), y = vw_floor(j);
  if (x == i && y == j) return edge_at(v, x, y);
  double normx = i - x, normy = j - y;
  double s0 = ((2 - normx) * normx - 1) * normx;  double t0 = ((2 - normy) * normy - 1) * normy;
  double s1 = (3 * normx - 5) * normx * normx + 2; double t1 = (3 * normy - 5) * normy * normy + 2;
  double s2 = ((4 - 3 * normx) * normx + 1) * normx; double t2 = ((4 - 3 * normy) * normy + 1) * normy;
  double s3 = (normx - 1) * normx * normx;         double t3 = (normy - 1) * normy * normy;
  double row, result;
  row = s0 * edge_at(v, x - 1, y - 1);
  row += s1 * edge_at(v, x, y - 1);
  row += s2 * edge_at(v, x + 1, y - 1);
  row += s3 * edge_at(v, x + 2, y - 1);
  result = t0 * row;
  row = s0 * edge_at(v, x - 1, y);
  row += s1 * edge_at(v, x, y);
  row += s2 * edge_at(v, x + 1, y);
  row += s3 * edge_at(v, x + 2, y);
  result += t1 * row;
  row = s0 * edge_at(v, x - 1, y + 1);
  row += s1 * edge_at(v, x, y + 1);
  row += s2 * edge_at(v, x + 1, y + 1);
  row += s3 * edge_at(v, x + 2, y + 1);
  result += t2 * row;
  row = s0 * edge_at(v, x - 1, y + 2);
  row += s1 * edge_at(v, x, y + 2);
  row += s2 * edge_at(v, x + 1, y + 2);
  row += s3 * edge_at(v, x + 2, y + 2);
  result += t3 * row;
  result *= 0.25;
  return (float)result;
}

void vww_transform(int kind, int interp, int edge, const double* m, const float* in, int w, int h, const float* disp, int dw, int dh,
                   int x0, int y0, float* out, int ow, int oh) {
  const View v = {in, w, h, edge};
  for (int jj = 0; jj < oh; ++jj)
    for (int ii = 0; ii < ow; ++ii) {
      const double pi = (double)(x0 + ii), pj = (double)(y0 + jj);
      double rx, ry;
      if (kind == 0) {
        double wz = m[6] * pi + m[7] * pj + m[8];
        rx = (m[0] * pi + m[1] * pj + m[2]) / wz;
        ry = (m[3] * pi + m[4] * pj + m[5]) / wz;
      } else {
        /* m_offset_image(p.x(), p.y()): NearestPixelInterpolation over ZeroEdgeExtension; p is integral */
        int32_t dx = vw_round(pi), dy = vw_round(pj);
        const float* d = (dx >= 0 && dy >= 0 && dx < dw && dy < dh) ? disp + 3 * ((size_t)dy * dw + dx) : NULL;
        if (!d || d[2] == 0.0f) { rx = -1; ry = pj; }
        else { rx = pi + d[0]; ry = pj + d[1]; }
      }
      float r = 0.0f;
      if (fabs(rx) < 1073741824.0 && fabs(ry) < 1073741824.0) {
        if (interp == 0) r = bilinear(&v, rx, ry);
        else if (interp == 1) r = bicubic(&v, rx, ry);
        else r = edge_at(&v, vw_round(rx), vw_round(ry));
      }
      out[(size_t)jj * ow + ii] = r;
    }
}
