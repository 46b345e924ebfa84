/* vw_dispmap_oracle.c -- see vw_dispmap_oracle.h.  Each function is written twice through a macro, once for int32 and once
 * for float pixels, with the reference's types: AccumulatorType is int64 for int32 and double for float
 * (Core/FundamentalTypes.h:111-122); Vector2 is double. */
#include "vw_dispmap_oracle.h"

#include <math.h>
#include <stddef.h>

typedef struct { int32_t x, y, v; } PixI;
typedef struct { float x, y, v; } PixF;

static int clampi(int a, int lo, int hi) { return a < lo ? lo : a > hi ? hi : a; }

/* CH: channel type, ACC: AccumulatorType<CH> */
#define DEFINE_DISPMAP(SUF, PIX, CH, ACC, ONE)                                                                            \
  /* m_child(i, j) of EdgeExtensionView<ViewT, ConstantEdgeExtension> */                                                   \
  static PIX at_##SUF(const PIX* in, int w, int h, int i, int j) { return in[(size_t)clampi(j, 0, h - 1) * w + clampi(i, 0, w - 1)]; } \
                                                                                                                          \
  static void subsample_##SUF(const PIX* in, int w, int h, PIX* out) {                                                    \
    const int ow = 1 + (w - 1) / 2, oh = 1 + (h - 1) / 2;                                                                 \
    for (int j = 0; j < oh; ++j)                                                                                          \
      for (int i = 0; i < ow; ++i) {                                                                                      \
        const int ci = i << 1, cj = j << 1;                                                                               \
        ACC bx = 0, by = 0, count = 0;                                                                                    \
        PIX p;                                                                                                            \
        /* buffer += k * bff_type(child): the child cast to the accumulator, then multiplied */                           \
        p = at_##SUF(in, w, h, ci, cj);         if (p.v) { count += 10; bx += 10 * (ACC)p.x; by += 10 * (ACC)p.y; }     \
        p = at_##SUF(in, w, h, ci + 1, cj);     if (p.v) { count += 5; bx += 5 * (ACC)p.x; by += 5 * (ACC)p.y; }        \
        p = at_##SUF(in, w, h, ci, cj + 1);     if (p.v) { count += 5; bx += 5 * (ACC)p.x; by += 5 * (ACC)p.y; }        \
        /* buffer += k * child: the product in the channel type, then widened */                                          \
        p = at_##SUF(in, w, h, ci - 1, cj);     if (p.v) { count += 5; bx += (CH)(5 * p.x); by += (CH)(5 * p.y); }      \
        p = at_##SUF(in, w, h, ci, cj - 1);     if (p.v) { count += 5; bx += (CH)(5 * p.x); by += (CH)(5 * p.y); }      \
        p = at_##SUF(in, w, h, ci + 1, cj + 1); if (p.v) { count += 2; bx += (CH)(2 * p.x); by += (CH)(2 * p.y); }      \
        p = at_##SUF(in, w, h, ci - 1, cj - 1); if (p.v) { count += 2; bx += (CH)(2 * p.x); by += (CH)(2 * p.y); }      \
        p = at_##SUF(in, w, h, ci - 1, cj + 1); if (p.v) { count += 2; bx += (CH)(2 * p.x); by += (CH)(2 * p.y); }      \
        p = at_##SUF(in, w, h, ci + 1, cj - 1); if (p.v) { count += 2; bx += (CH)(2 * p.x); by += (CH)(2 * p.y); }      \
        PIX r = {0, 0, 0};                                                                                                \
        if (count > 0) { r.x = (CH)(bx / (count * 2)); r.y = (CH)(by / (count * 2)); r.v = ONE; }                       \
        out[(size_t)j * ow + i] = r;                                                                                      \
      }                                                                                                                   \
  }                                                                                                                       \
                                                                                                                          \
  static void upsample_##SUF(const PIX* in, int w, int h, PIX* out) {                                                     \
    for (int j = 0; j < 2 * h; ++j)                                                                                       \
      for (int i = 0; i < 2 * w; ++i) {                                                                                   \
        const PIX p = in[(size_t)(j >> 1) * w + (i >> 1)];                                                                \
        PIX r;                                                                                                            \
        r.x = (CH)(p.x * 2); r.y = (CH)(p.y * 2); r.v = p.v ? ONE : 0;                                                    \
        out[(size_t)j * 2 * w + i] = r;                                                                                   \
      }                                                                                                                   \
  }                                                                                                                       \
                                                                                                                          \
  static int range_##SUF(const PIX* in, int w, int h, float* range) {                                                    \
    CH mn[2] = {0, 0}, mx[2] = {0, 0};                                                                                    \
    int valid = 0;                                                                                                        \
    for (int j = 0; j < h; ++j)                                                                                           \
      for (int i = 0; i < w; ++i) {                                                                                       \
        const PIX p = in[(size_t)j * w + i];                                                                              \
        if (!p.v) continue;                                                                                               \
        const CH a[2] = {p.x, p.y};                                                                                       \
        if (!valid) { mn[0] = mx[0] = a[0]; mn[1] = mx[1] = a[1]; valid = 1; continue; }                                  \
        for (int c = 0; c < 2; ++c) {                                                                                     \
          if (a[c] < mn[c]) mn[c] = a[c];                                                                                 \
          else if (a[c] > mx[c]) mx[c] = a[c];                                                                            \
        }                                                                                                                 \
      }                                                                                                                   \
    if (!valid) { range[0] = range[1] = range[2] = range[3] = 0.0f; return 0; }                                           \
    range[0] = (float)mn[0]; range[1] = (float)mn[1]; range[2] = (float)mx[0]; range[3] = (float)mx[1];                   \
    return 1;                                                                                                             \
  }                                                                                                                       \
                                                                                                                          \
  static void range_mask_##SUF(const PIX* in, int w, int h, const CH* mn, const CH* mx, PIX* out) {                        \
    for (int j = 0; j < h; ++j)                                                                                           \
      for (int i = 0; i < w; ++i) {                                                                                       \
        const PIX p = in[(size_t)j * w + i];                                                                              \
        PIX r = p;                                                                                                        \
        if (p.v) {                                                                                                        \
          const double lx = i, ly = j;                                                                                    \
          const CH m0 = (CH)(mx[0] - 1), m1 = (CH)(mx[1] - 1);                                                            \
          if (lx + p.x < mn[0] || lx + p.x >= m0 || ly + p.y < mn[0] || ly + p.y >= m1) {                                 \
            r.x = 0; r.y = 0; r.v = 0;                                                                                    \
          }                                                                                                               \
        }                                                                                                                 \
        out[(size_t)j * w + i] = r;                                                                                       \
      }                                                                                                                   \
  }                                                                                                                       \
                                                                                                                          \
  static void transform_##SUF(int mode, const double* m, int do_round, int sx0, int sy0, const PIX* in, int w, int h,       \
                              PIX* out) {                                                                                 \
    for (int j = 0; j < h; ++j)                                                                                           \
      for (int i = 0; i < w; ++i) {                                                                                       \
        const PIX p = in[(size_t)j * w + i];                                                                              \
        PIX r = {0, 0, 0};                                                                                                \
        if (mode == 0) {                                                                                                  \
          const double lx = i, ly = j;                                                                                    \
          const double px = lx + p.x, py = ly + p.y;                                                                      \
          const double ww = m[6] * px + m[7] * py + m[8];                                                                 \
          const double nx = (m[0] * px + m[1] * py + m[2]) / ww, ny = (m[3] * px + m[4] * py + m[5]) / ww;                \
          r.x = (CH)(nx - lx); r.y = (CH)(ny - ly); r.v = p.v ? ONE : 0;                                                  \
        } else if (p.v) {                                                                                                 \
          const double bx = (double)sx0 + (double)i, by = (double)sy0 + (double)j;                                        \
          const double ex = bx + p.x, ey = by + p.y;                                                                      \
          const double ww = m[6] * ex + m[7] * ey + m[8];                                                                 \
          const double tx = (m[0] * ex + m[1] * ey + m[2]) / ww, ty = (m[3] * ex + m[4] * ey + m[5]) / ww;                \
          double dx = tx - bx, dy = ty - by;                                                                              \
          if (do_round) { dx = round(dx); dy = round(dy); }                                                               \
          r.x = (CH)dx; r.y = (CH)dy; r.v = ONE;                                                                          \
        }                                                                                                                 \
        out[(size_t)j * w + i] = r;                                                                                       \
      }                                                                                                                   \
  }

DEFINE_DISPMAP(i, PixI, int32_t, int64_t, 1)
DEFINE_DISPMAP(f, PixF, float, double, 1.0f)

void vwd_subsample(int type, const void* in, int w, int h, void* out) {
  if (type == 0) subsample_i((const PixI*)in, w, h, (PixI*)out); else subsample_f((const PixF*)in, w, h, (PixF*)out);
}
void vwd_upsample(int type, const void* in, int w, int h, void* out) {
  if (type == 0) upsample_i((const PixI*)in, w, h, (PixI*)out); else upsample_f((const PixF*)in, w, h, (PixF*)out);
}
int vwd_range(int type, const void* in, int w, int h, float* range) {
  return type == 0 ? range_i((const PixI*)in, w, h, range) : range_f((const PixF*)in, w, h, range);
}
void vwd_range_mask(int type, const void* in, int w, int h, const void* min, const void* max, void* out) {
  if (type == 0) range_mask_i((const PixI*)in, w, h, (const int32_t*)min, (const int32_t*)max, (PixI*)out);
  else range_mask_f((const PixF*)in, w, h, (const float*)min, (const float*)max, (PixF*)out);
}
void vwd_transform(int type, int mode, const double* m9, int do_round, int sx0, int sy0, const void* in, int w, int h, void* out) {
  if (type == 0) transform_i(mode, m9, do_round, sx0, sy0, (const PixI*)in, w, h, (PixI*)out);
  else transform_f(mode, m9, do_round, sx0, sy0, (const PixF*)in, w, h, (PixF*)out);
}
