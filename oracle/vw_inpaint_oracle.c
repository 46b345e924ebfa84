/* vw_inpaint_oracle.c -- see vw_inpaint_oracle.h. */
#include "vw_inpaint_oracle.h"

#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct { int32_t dx, dy, valid; } PxI;
typedef struct { float dx, dy, valid; } PxF;

static int find(int* parent, int i) {
  while (parent[i] != i) { parent[i] = parent[parent[i]]; i = parent[i]; }
  return i;
}

/* channel c of tile pixel (x, y), as the stencil reads it */
static double child(int type, const void* t, int tw, int x, int y, int c) {
  if (type == 0) { const PxI* p = (const PxI*)t + (size_t)y * tw + x; return c ? (double)p->dy : (double)p->dx; }
  const PxF* p = (const PxF*)t + (size_t)y * tw + x;
  return c ? (double)p->dy : (double)p->dx;
}

/* InpaintTask::operator() (InpaintView.h:67-148) for one hole: lbl == root over [bx0, bx1) x [by0, by1) of the tile t.
 * The patched pixels are written into `res` (the tile's copy that the output window is read from). */
static int inpaint_blob(int type, const void* t, void* res, int tw, const int* lbl, int root, int bx0, int by0, int bx1, int by1) {
  const int cx0 = bx0 - 1, cy0 = by0 - 1, cw = bx1 - bx0 + 2, ch = by1 - by0 + 2;
  const size_t n = (size_t)cw * ch;
  unsigned char* mask = (unsigned char*)calloc(n, 1);
  int32_t* dist = (int32_t*)calloc(n, sizeof(int32_t));
  float* cf = (float*)malloc(n * 2 * sizeof(float));     /* cropped_copy, float pixels */
  int32_t* ci = (int32_t*)malloc(n * 2 * sizeof(int32_t)); /* cropped_copy, int32 pixels */
  for (int j = 0; j < ch; ++j)
    for (int i = 0; i < cw; ++i) {
      const size_t k = (size_t)j * cw + i;
      mask[k] = lbl[(size_t)(cy0 + j) * tw + cx0 + i] == root ? 255 : 0;
      for (int c = 0; c < 2; ++c) {
        if (type == 0) ci[2 * k + c] = (int32_t)child(type, t, tw, cx0 + i, cy0 + j, c);
        else cf[2 * k + c] = (float)child(type, t, tw, cx0 + i, cy0 + j, c);
      }
    }
  /* grassfire(mask) with borders (Grassfire.h:79-150); cw, ch >= 3 */
  for (int i = 0; i < cw; ++i) { dist[i] = mask[i] ? 1 : 0; dist[(size_t)(ch - 1) * cw + i] = mask[(size_t)(ch - 1) * cw + i] ? 1 : 0; }
  for (int j = 1; j < ch - 1; ++j) {
    const size_t r = (size_t)j * cw;
    dist[r] = mask[r] ? 1 : 0;
    for (int i = 1; i < cw - 1; ++i) {
      if (!mask[r + i]) dist[r + i] = 0;
      else {
        const int32_t a = dist[r + i - 1], b = dist[r + i - cw];
        dist[r + i] = 1 + (a < b ? a : b);
      }
    }
    dist[r + cw - 1] = mask[r + cw - 1] ? 1 : 0;
  }
  for (int j = ch - 2; j >= 1; --j)
    for (int i = cw - 2; i >= 1; --i) {
      const size_t k = (size_t)j * cw + i;
      if (dist[k] != 0) {
        const int32_t a = dist[k + 1], b = dist[k + cw], m = a < b ? a : b;
        if (m < dist[k]) dist[k] = m + 1;
      }
    }
  int dmax = 0;
  for (size_t k = 0; k < n; ++k) if (dist[k] > dmax) dmax = dist[k];
  /* processing order: d = 1..dmax, column-major */
  int* order = (int*)malloc(n * sizeof(int));
  size_t no = 0;
  for (int d = 1; d <= dmax; ++d)
    for (int i = 0; i < cw; ++i)
      for (int j = 0; j < ch; ++j)
        if (dist[(size_t)j * cw + i] == d) order[no++] = j * cw + i;
  static const int DX[8] = {-1, 0, 1, -1, 1, -1, 0, 1}, DY[8] = {-1, -1, -1, 0, 0, 1, 1, 1};
  static const double WT[8] = {.176765, .073235, .176765, .073235, .073235, .176765, .073235, .176765};
  const long sweeps = 10L * dmax * dmax;
  for (long s = 0; s < sweeps; ++s)
    for (size_t o = 0; o < no; ++o) {
      const int k = order[o];
      for (int c = 0; c < 2; ++c) {
        float sum = 0.0f; /* AccumulatorType() */
        for (int q = 0; q < 8; ++q) {
          const int kq = k + DY[q] * cw + DX[q];
          const double v = type == 0 ? (double)ci[2 * kq + c] : (double)cf[2 * kq + c];
          const double prod = WT[q] * v; /* ProductType<double, channel> is double */
          sum = (float)((double)sum + prod); /* float += double */
        }
        if (type == 0) ci[2 * k + c] = (int32_t)sum;
        else cf[2 * k + c] = sum;
      }
    }
  /* absorb the masked patch */
  for (int j = 0; j < ch; ++j)
    for (int i = 0; i < cw; ++i) {
      const size_t k = (size_t)j * cw + i;
      if (!mask[k]) continue;
      const size_t tk = (size_t)(cy0 + j) * tw + cx0 + i;
      if (type == 0) { PxI* p = (PxI*)res + tk; p->dx = ci[2 * k]; p->dy = ci[2 * k + 1]; p->valid = 1; }
      else { PxF* p = (PxF*)res + tk; p->dx = cf[2 * k]; p->dy = cf[2 * k + 1]; p->valid = 1.0f; }
    }
  free(mask); free(dist); free(cf); free(ci); free(order);
  return (int)sweeps;
}

int vwi_fill_holes_grass(int type, const void* in, int w, int h, int len, int x0, int y0, int ow, int oh, void* out, int* stats) {
  if (stats) stats[0] = stats[1] = stats[2] = 0;
  if (len < 0 || w <= 0 || h <= 0 || ow <= 0 || oh <= 0 || x0 < 0 || y0 < 0 || x0 > w - ow || y0 > h - oh) return -1;
  const size_t px = 12;
  /* biased_box = bbox.expand(len) cropped to the image */
  const long long tx0 = (long long)x0 - len < 0 ? 0 : (long long)x0 - len, ty0 = (long long)y0 - len < 0 ? 0 : (long long)y0 - len;
  const long long tx1 = (long long)x0 + ow + len > w ? w : (long long)x0 + ow + len;
  const long long ty1 = (long long)y0 + oh + len > h ? h : (long long)y0 + oh + len;
  const int tw = (int)(tx1 - tx0), th = (int)(ty1 - ty0);
  const size_t n = (size_t)tw * th;
  unsigned char* t = (unsigned char*)malloc(n * px);
  unsigned char* res = (unsigned char*)malloc(n * px);
  for (int y = 0; y < th; ++y)
    memcpy(t + (size_t)y * tw * px, (const unsigned char*)in + ((size_t)(ty0 + y) * w + tx0) * px, (size_t)tw * px);
  memcpy(res, t, n * px);
  /* 8-connected components of the invalid pixels (invert_mask(tile) is valid where the tile is not) */
  int* parent = (int*)malloc(n * sizeof(int));
  int* lbl = (int*)malloc(n * sizeof(int));
  for (size_t i = 0; i < n; ++i) parent[i] = (int)i;
#define INVALID(i) (type == 0 ? ((const PxI*)t)[i].valid == 0 : ((const PxF*)t)[i].valid == 0.0f)
  for (int y = 0; y < th; ++y)
    for (int x = 0; x < tw; ++x) {
      const int i = y * tw + x;
      if (!INVALID(i)) continue;
      static const int NX[4] = {-1, -1, 0, 1}, NY[4] = {0, -1, -1, -1};
      for (int k = 0; k < 4; ++k) {
        const int xx = x + NX[k], yy = y + NY[k];
        if (xx < 0 || xx >= tw || yy < 0) continue;
        if (!INVALID(yy * tw + xx)) continue;
        const int a = find(parent, i), b = find(parent, yy * tw + xx);
        if (a != b) parent[a > b ? a : b] = a > b ? b : a;
      }
    }
  /* per-root pixel count and half-open bounding box */
  int* size = (int*)calloc(n, sizeof(int));
  int* bb = (int*)malloc(n * 4 * sizeof(int));
  for (size_t i = 0; i < n; ++i) {
    lbl[i] = INVALID(i) ? find(parent, (int)i) : -1;
    bb[4 * i] = bb[4 * i + 1] = 0x7fffffff; bb[4 * i + 2] = bb[4 * i + 3] = -1;
  }
#undef INVALID
  for (int y = 0; y < th; ++y)
    for (int x = 0; x < tw; ++x) {
      const int r = lbl[(size_t)y * tw + x];
      if (r < 0) continue;
      size[r]++;
      int* b = bb + 4 * (size_t)r;
      if (x < b[0]) b[0] = x;
      if (y < b[1]) b[1] = y;
      if (x + 1 > b[2]) b[2] = x + 1;
      if (y + 1 > b[3]) b[3] = y + 1;
    }
  const int area = len * len;
  for (size_t r = 0; r < n; ++r) {
    if (size[r] == 0) continue;
    if (stats) stats[0]++;
    const int* b = bb + 4 * r;
    if (area > 0 && size[r] > area) continue;                 /* the max_area cull */
    if (b[2] - b[0] > len || b[3] - b[1] > len) continue;    /* wipe_big_blobs(len) */
    /* bbox.expand(1) must stay inside the tile: min >= 0 and max < cols / rows, max being half-open */
    if (b[0] - 1 < 0 || b[1] - 1 < 0 || b[2] + 1 >= tw || b[3] + 1 >= th) continue;
    const int sweeps = inpaint_blob(type, t, res, tw, lbl, (int)r, b[0], b[1], b[2], b[3]);
    if (stats) { stats[1]++; if (sweeps > stats[2]) stats[2] = sweeps; }
  }
  for (int y = 0; y < oh; ++y)
    memcpy((unsigned char*)out + (size_t)y * ow * px, res + ((size_t)(y0 - ty0 + y) * tw + (x0 - tx0)) * px, (size_t)ow * px);
  free(t); free(res); free(parent); free(lbl); free(size); free(bb);
  return 0;
}
