/* vw_epipolar_oracle.c -- see vw_epipolar_oracle.h.  The pinhole restatement of vw_triangulate_oracle.c (the camera inverse,
 * TsaiDistortionNorm, pixel_to_vector, dot_prod) and the interpolations and edge extensions of vw_warp_oracle.c are reused as
 * they are: both sources are included here, so their static functions are this file's too, and libvwepipolar.so carries
 * every vwt_ and vww_ entry point besides the ones below. */
#include "vw_triangulate_oracle.c"
#include "vw_warp_oracle.c"
#include "vw_epipolar_oracle.h"

/* Quaternion<double>(MatrixBase) (Math/Quaternion.h:211-252), then rotation_matrix() (:314-335) */
int vwt_quaternion_round_trip(const double R[9], double out[9], double quat[4]) {
  double d0 = R[0], d1 = R[4], d2 = R[8];
  double ww = 1.0 + d0 + d1 + d2;
  double xx = 1.0 + d0 - d1 - d2;
  double yy = 1.0 - d0 + d1 - d2;
  double zz = 1.0 - d0 - d1 + d2;
  double max = ww;
  if (xx > max) max = xx;
  if (yy > max) max = yy;
  if (zz > max) max = zz;
  double c[4];
  int branch;
  if (ww == max) {
    double w4 = sqrt(ww * 4.0);
    c[0] = w4 / 4;
    c[1] = (R[3 * 2 + 1] - R[3 * 1 + 2]) / w4;
    c[2] = (R[3 * 0 + 2] - R[3 * 2 + 0]) / w4;
    c[3] = (R[3 * 1 + 0] - R[3 * 0 + 1]) / w4;
    branch = 0;
  } else if (xx == max) {
    double x4 = sqrt(xx * 4.0);
    c[0] = (R[3 * 2 + 1] - R[3 * 1 + 2]) / x4;
    c[1] = x4 / 4;
    c[2] = (R[3 * 0 + 1] + R[3 * 1 + 0]) / x4;
    c[3] = (R[3 * 0 + 2] + R[3 * 2 + 0]) / x4;
    branch = 1;
  } else if (yy == max) {
    double y4 = sqrt(yy * 4.0);
    c[0] = (R[3 * 0 + 2] - R[3 * 2 + 0]) / y4;
    c[1] = (R[3 * 0 + 1] + R[3 * 1 + 0]) / y4;
    c[2] = y4 / 4;
    c[3] = (R[3 * 1 + 2] + R[3 * 2 + 1]) / y4;
    branch = 2;
  } else {
    double z4 = sqrt(zz * 4.0);
    c[0] = (R[3 * 1 + 0] - R[3 * 0 + 1]) / z4;
    c[1] = (R[3 * 0 + 2] + R[3 * 2 + 0]) / z4;
    c[2] = (R[3 * 1 + 2] + R[3 * 2 + 1]) / z4;
    c[3] = z4 / 4;
    branch = 3;
  }
  if (quat) memcpy(quat, c, sizeof c);
  double w = c[0], x = c[1], y = c[2], z = c[3];
  double w2 = w * w, x2 = x * x, y2 = y * y, z2 = z * z;
  double wx = w * x, wy = w * y, wz = w * z;
  double xy = x * y, yz = y * z, zx = z * x;
  out[3 * 0 + 0] = w2 + x2 - y2 - z2;
  out[3 * 1 + 1] = w2 - x2 + y2 - z2;
  out[3 * 2 + 2] = w2 - x2 - y2 + z2;
  out[3 * 0 + 1] = 2 * (xy - wz);
  out[3 * 0 + 2] = 2 * (zx + wy);
  out[3 * 1 + 2] = 2 * (yz - wx);
  out[3 * 1 + 0] = 2 * (xy + wz);
  out[3 * 2 + 0] = 2 * (zx - wy);
  out[3 * 2 + 1] = 2 * (yz + wx);
  return branch;
}

int vwt_epipolar(const vwt_pinhole* src0, const vwt_pinhole* src1, vwt_pinhole* dst0, vwt_pinhole* dst1) {
  double inv[9];
  int rc = vwt_camera_inverse(src0, inv);
  if (rc) return rc;
  rc = vwt_camera_inverse(src1, inv);
  if (rc) return rc;
  double rot0[9], rot1[9];
  vwt_quaternion_round_trip(src0->rotation, rot0, NULL);
  vwt_quaternion_round_trip(src1->rotation, rot1, NULL);
  const double* center0 = src0->center;
  const double* center1 = src1->center;
  double look0[3], look1[3];
  for (int i = 0; i < 3; ++i) { look0[i] = -1 * rot0[3 * i + 2]; look1[i] = -1 * rot1[3 * i + 2]; }
  double diff[3], u[3], mean_look[3], t1[3], temp[3], w[3], v[3];
  for (int i = 0; i < 3; ++i) diff[i] = center1[i] - center0[i];
  double nd = norm3(diff);
  for (int i = 0; i < 3; ++i) u[i] = (center1[i] - center0[i]) / nd;
  for (int i = 0; i < 3; ++i) mean_look[i] = (look0[i] + look1[i]) / 2.0;
  cross3(mean_look, u, t1);
  cross3(u, t1, temp);
  double nt = norm3(temp);
  for (int i = 0; i < 3; ++i) w[i] = temp[i] / nt;
  cross3(w, u, v);
  vwt_pinhole d;
  memset(&d, 0, sizeof d);
  double rot[9] = {u[0], -v[0], -w[0], u[1], -v[1], -w[1], u[2], -v[2], -w[2]};
  memcpy(d.rotation, rot, sizeof rot);
  d.fu = (src0->fu + src1->fu) / 2.0;
  d.fv = (src0->fv + src1->fv) / 2.0;
  d.cu = (src0->cu + src1->cu) / 2.0;
  d.cv = (src0->cv + src1->cv) / 2.0;
  d.pixel_pitch = (src0->pixel_pitch + src1->pixel_pitch) / 2.0;
  d.u_direction[0] = 1; d.v_direction[1] = 1; d.w_direction[2] = 1;
  d.lens = 0;
  *dst0 = d;
  *dst1 = d;
  memcpy(dst0->center, center0, sizeof d.center);
  memcpy(dst1->center, center1, sizeof d.center);
  return 0;
}

/* m_camera_matrix = m_intrinsics * m_extrinsics (PinholeModel.cc:565-603), row-major 3 x 4 */
int vwt_camera_matrix(const vwt_pinhole* cam, double P[12]) {
  double inv[9];
  int rc = vwt_camera_inverse(cam, inv);                 /* the asserts */
  if (rc) return rc;
  const double* uvw[3] = {cam->u_direction, cam->v_direction, cam->w_direction};
  double rt[9], nrt[9], extr[12], K[9] = {cam->fu, 0, cam->cu, 0, cam->fv, cam->cv, 0, 0, 1};
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) { rt[3 * r + c] = cam->rotation[3 * c + r]; nrt[3 * r + c] = -rt[3 * r + c]; }
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      double col[3] = {rt[c], rt[3 + c], rt[6 + c]};
      extr[4 * r + c] = dot3(uvw[r], col);
    }
  double m2[9];                                           /* uvwRotation * (-rotation_inverse), then times the center */
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      double col[3] = {nrt[c], nrt[3 + c], nrt[6 + c]};
      m2[3 * r + c] = dot3(uvw[r], col);
    }
  for (int r = 0; r < 3; ++r) extr[4 * r + 3] = dot3(m2 + 3 * r, cam->center);
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 4; ++c) {
      double col[3] = {extr[c], extr[4 + c], extr[8 + c]};
      P[4 * r + c] = dot3(K + 3 * r, col);
    }
  return 0;
}

/* TsaiLensDistortion::distorted_coordinates (LensDistortion.cc:345-369) */
static void tsai_distorted(const vwt_pinhole* cam, const double* p, double* out) {
  double focal[2] = {cam->fu, cam->fv}, offset[2] = {cam->cu, cam->cv};
  if (focal[0] < 1e-300 || focal[1] < 1e-300) { out[0] = out[1] = HUGE_VAL; return; }
  double dudv[2] = {p[0] - offset[0], p[1] - offset[1]};
  double p0[2] = {dudv[0] / focal[0], dudv[1] / focal[1]};
  double d[2];
  tsai_norm(p0, cam->lens_params, d);
  double dx = d[0], dy = d[1];
  dx = dx * focal[0] + offset[0];
  dy = dy * focal[1] + offset[1];
  out[0] = dx; out[1] = dy;
}

/* point_to_pixel (PinholeModel.cc:351-397) with m_camera_matrix P and m_inv_camera_transform inv: 0, or -4 (PointToPixelErr) */
static int point_to_pixel(const vwt_pinhole* cam, const double* P, const double* inv, const double* point, double* out) {
  double den = P[8] * point[0] + P[9] * point[1] + P[10] * point[2] + P[11];
  double pixel[2] = {(P[0] * point[0] + P[1] * point[1] + P[2] * point[2] + P[3]) / den,
                     (P[4] * point[0] + P[5] * point[1] + P[6] * point[2] + P[7]) / den};
  double dist[2] = {pixel[0], pixel[1]};
  if (cam->lens == 1) tsai_distorted(cam, pixel, dist);
  out[0] = dist[0] / cam->pixel_pitch;
  out[1] = dist[1] / cam->pixel_pitch;
  double pixel_vector[3], phys[3], d[3];
  pixel_to_vector(cam, inv, out, pixel_vector);
  for (int i = 0; i < 3; ++i) d[i] = point[i] - cam->center[i];
  double n = norm3(d);
  for (int i = 0; i < 3; ++i) phys[i] = d[i] / n;
  double e[3];
  for (int i = 0; i < 3; ++i) e[i] = pixel_vector[i] - phys[i];
  double diff = norm3(e);
  if (diff >= 0.01) {
    for (int i = 0; i < 3; ++i) e[i] = pixel_vector[i] + phys[i];
    diff = norm3(e);
  }
  if (diff >= 0.01 || diff != diff) return -4;
  return 0;
}

typedef struct { const vwt_pinhole* cam; double P[12], inv[9]; } Cam;

static int open_cam(const vwt_pinhole* p, Cam* c) {
  c->cam = p;
  int rc = vwt_camera_matrix(p, c->P);
  if (rc) return rc;
  return vwt_camera_inverse(p, c->inv);
}

int vwt_point_to_pixel(const vwt_pinhole* cam, const double point[3], double pix[2]) {
  Cam c;
  int rc = open_cam(cam, &c);
  if (rc) return rc;
  return point_to_pixel(cam, c.P, c.inv, point, pix);
}

/* CameraTransform<PinholeModel, PinholeModel>(src, dst)::forward / reverse (CameraTransform.h:52-74); -5 for the centers' VW_ASSERT */
static int centers_equal(const vwt_pinhole* a, const vwt_pinhole* b) {
  return a->center[0] == b->center[0] && a->center[1] == b->center[1] && a->center[2] == b->center[2];
}
static int map_pixel(const Cam* from, const Cam* to, const double* p, double* out) {
  double vec[3], pt[3];
  pixel_to_vector(from->cam, from->inv, p, vec);
  for (int i = 0; i < 3; ++i) pt[i] = vec[i] + from->cam->center[i];
  return point_to_pixel(to->cam, to->P, to->inv, pt, out);
}

int vwt_camera_transform_point(const vwt_pinhole* src, const vwt_pinhole* dst, int reverse, const double p[2], double out[2]) {
  Cam s, d;
  int rc = open_cam(src, &s);
  if (rc) return rc;
  rc = open_cam(dst, &d);
  if (rc) return rc;
  if (!centers_equal(src, dst)) return -5;
  return reverse ? map_pixel(&d, &s, p, out) : map_pixel(&s, &d, p, out);
}

int vwt_camera_reverse_window(const vwt_pinhole* src, const vwt_pinhole* dst, int x0, int y0, int ow, int oh, double* coords,
                              long long* first_fail) {
  Cam s, d;
  int rc = open_cam(src, &s);
  if (rc) return rc;
  rc = open_cam(dst, &d);
  if (rc) return rc;
  if (!centers_equal(src, dst)) return -5;
  *first_fail = -1;
  for (int j = 0; j < oh; ++j)
    for (int i = 0; i < ow; ++i) {
      long long k = (long long)j * ow + i;
      double p[2] = {(double)(x0 + i), (double)(y0 + j)};
      if (map_pixel(&d, &s, p, coords + 2 * k) && *first_fail < 0) *first_fail = k;
    }
  return *first_fail >= 0 ? -4 : 0;
}

/* BBox2f::grow (Math/BBox.tcc:82-97): double against float, float(point) stored */
static void grow(float* bb, const double* pt) {
  for (int i = 0; i < 2; ++i) {
    if (pt[i] > bb[2 + i]) bb[2 + i] = (float)pt[i];
    if (pt[i] < bb[i]) bb[i] = (float)pt[i];
  }
}

/* compute_transformed_bbox_fast (Image/Transform.h:271-315) through forward(); bbox = {min x, min y, max x, max y} */
static int transformed_bbox_fast(const Cam* s, const Cam* d, const int* roi, float* bbox, long long* fail_k) {
  const float big = (float)(2147483647 - 1);
  bbox[0] = bbox[1] = big;
  bbox[2] = bbox[3] = -big;
  double pt[2], out[2];
  long long k = 0;
  for (pt[0] = roi[0]; pt[0] < roi[2]; (pt[0])++, ++k) {
    pt[1] = roi[1];
    if (map_pixel(s, d, pt, out)) { *fail_k = k; return -4; }
    grow(bbox, out);
  }
  for (pt[0] = roi[0]; pt[0] < roi[2]; (pt[0])++, ++k) {
    pt[1] = roi[3] - 1;
    if (map_pixel(s, d, pt, out)) { *fail_k = k; return -4; }
    grow(bbox, out);
  }
  for (pt[1] = roi[1]; pt[1] < roi[3]; (pt[1])++, ++k) {
    pt[0] = roi[0];
    if (map_pixel(s, d, pt, out)) { *fail_k = k; return -4; }
    grow(bbox, out);
  }
  for (pt[1] = roi[1]; pt[1] < roi[3]; (pt[1])++, ++k) {
    pt[0] = roi[2] - 1;
    if (map_pixel(s, d, pt, out)) { *fail_k = k; return -4; }
    grow(bbox, out);
  }
  *fail_k = -1;
  return 0;
}

int vwt_transformed_bbox_fast(const vwt_pinhole* src, const vwt_pinhole* dst, const int roi[4], float bbox[4], long long* fail_k) {
  Cam s, d;
  int rc = open_cam(src, &s);
  if (rc) return rc;
  rc = open_cam(dst, &d);
  if (rc) return rc;
  if (!centers_equal(src, dst)) return -5;
  return transformed_bbox_fast(&s, &d, roi, bbox, fail_k);
}

/* resize_epipolar_cameras_to_fit (EpipolarUtils.cc:37-76); fail_k: the failing perimeter index, fail_cam its camera (0, 1) */
int vwt_resize_epipolar(const vwt_pinhole* cam1, const vwt_pinhole* cam2, vwt_pinhole* epi1, vwt_pinhole* epi2, const int roi1[4],
                        const int roi2[4], int size1[2], int size2[2], long long* fail_k, int* fail_cam) {
  Cam c1, c2, e1, e2;
  int rc;
  if ((rc = open_cam(cam1, &c1)) || (rc = open_cam(cam2, &c2)) || (rc = open_cam(epi1, &e1)) || (rc = open_cam(epi2, &e2))) return rc;
  if (!centers_equal(cam1, epi1) || !centers_equal(cam2, epi2)) return -5;
  float bb1[4], bb2[4];
  *fail_cam = 0;
  if ((rc = transformed_bbox_fast(&c1, &e1, roi1, bb1, fail_k))) return rc;
  *fail_cam = 1;
  if ((rc = transformed_bbox_fast(&c2, &e2, roi2, bb2, fail_k))) return rc;
  double min_col = bb2[0] < bb1[0] ? bb2[0] : bb1[0];   /* std::min(a, b): b < a ? b : a, in float */
  double min_row = bb2[1] < bb1[1] ? bb2[1] : bb1[1];
  double point_offset[2] = {epi1->cu, epi1->cv};
  double center_adjust[2] = {min_col * epi1->pixel_pitch, min_row * epi1->pixel_pitch};
  epi1->cu = point_offset[0] - center_adjust[0]; epi1->cv = point_offset[1] - center_adjust[1];
  epi2->cu = point_offset[0] - center_adjust[0]; epi2->cv = point_offset[1] - center_adjust[1];
  if ((rc = open_cam(epi1, &e1)) || (rc = open_cam(epi2, &e2))) return rc;
  *fail_cam = 0;
  if ((rc = transformed_bbox_fast(&c1, &e1, roi1, bb1, fail_k))) return rc;
  *fail_cam = 1;
  if ((rc = transformed_bbox_fast(&c2, &e2, roi2, bb2, fail_k))) return rc;
  size1[0] = (int)bb1[2]; size1[1] = (int)bb1[3];
  size2[0] = (int)bb2[2]; size2[1] = (int)bb2[3];
  return 0;
}

/* ---- camera_transform's interpolation stage ----------------------------------------------------------------------------- */

/* The interpolation stage of a transform at given reversed coordinates (coords: n (x, y) pairs), for transforms whose
 * reverse() is restated elsewhere (camera_transform: oracle/vw_triangulate_oracle.c); the same domain rule as vww_transform. */
void vww_sample(int interp, int edge, const float* in, int w, int h, const double* coords, long long n, float* out) {
  const View v = {in, w, h, edge};
  for (long long k = 0; k < n; ++k) {
    double rx = coords[2 * k], ry = coords[2 * k + 1];
    float r = 0.0f;
    if (fabs(rx) < 1073741824.0 && fabs(ry) < 1073741824.0) {
      if (interp == 0) r = bilinear(&v, rx, ry);
      else if (interp == 1) r = bicubic(&v, rx, ry);
      else r = edge_at(&v, vw_round(rx), vw_round(ry));
    }
    out[k] = r;
  }
}

/* PixelMask<float> {child, valid} (Image/PixelMask.h:52-116) */
typedef struct { float child, valid; } Mask;

/* EdgeExtensionView<ImageView<PixelMask<float>>, EdgeT>: 0 zero (PixelMask<float>() = {0, 0}), 1 constant, 2 value */
static Mask mask_at(const float* in, int w, int h, int edge, Mask value, int32_t i, int32_t j) {
  if (edge != 1) {
    if (i >= 0 && j >= 0 && i < w && j < h) { Mask m = {in[2 * ((size_t)j * w + i)], in[2 * ((size_t)j * w + i) + 1]}; return m; }
    if (edge == 0) { Mask z = {0.0f, 0.0f}; return z; }
    return value;
  }
  size_t k = (size_t)((j < 0) ? 0 : (j >= h) ? (h - 1) : j) * w + ((i < 0) ? 0 : (i >= w) ? (w - 1) : i);
  Mask m = {in[2 * k], in[2 * k + 1]};
  return m;
}

/* UnaryCompoundFunctor (PixelMask.h:499-534): result(func(arg[0])) is valid (1.0f), invalidated when !arg.valid() */
static Mask times(Mask a, float s) { Mask r = {a.child * s, 1.0f}; if (!a.valid) r.valid = 0.0f; return r; }
/* BinaryInPlaceCompoundFunctor (:410-445): func(arg1[0], arg2[0]), arg1 invalidated when !arg2.valid() */
static void plus_eq(Mask* a, Mask b) { a->child += b.child; if (!b.valid) a->valid = 0.0f; }

/* BilinearInterpolationImpl (Image/Interpolation.h:76-110) on PixelMask<float>: real_type float, result_type PixelMask<float>;
 * the integral shortcut is channel_cast_round_if_int<float> = compound_apply(ChannelCastFunctor), the UnaryCompoundFunctor
 * above */
static Mask bilinear_mask(const float* in, int w, int h, int edge, Mask value, double i, double j) {
  int32_t x = vw_floor(i), y = vw_floor(j);
  if (x == i && y == j) {
    Mask p = mask_at(in, w, h, edge, value, x, y);
    Mask r = {p.child, 1.0f};
    if (!p.valid) r.valid = 0.0f;
    return r;
  }
  float normx = (float)i - (float)x, normy = (float)j - (float)y, norm1mx = 1 - normx, norm1my = 1 - normy;
  Mask result = times(mask_at(in, w, h, edge, value, x, y), norm1mx);
  plus_eq(&result, times(mask_at(in, w, h, edge, value, x + 1, y), normx));
  result.child *= norm1my;                                /* UnaryInPlaceCompoundFunctor (:586-606): the child only */
  Mask row = times(mask_at(in, w, h, edge, value, x, y + 1), norm1mx);
  plus_eq(&row, times(mask_at(in, w, h, edge, value, x + 1, y + 1), normx));
  plus_eq(&result, times(row, normy));
  return result;
}

void vww_sample_masked(int edge, const float* edge_value, const float* in, int w, int h, const double* coords, long long n, float* out) {
  Mask value = {edge_value[0], edge_value[1]};
  for (long long k = 0; k < n; ++k) {
    double rx = coords[2 * k], ry = coords[2 * k + 1];
    Mask r = {0.0f, 0.0f};
    if (fabs(rx) < 1073741824.0 && fabs(ry) < 1073741824.0) r = bilinear_mask(in, w, h, edge, value, rx, ry);
    out[2 * k] = r.child;
    out[2 * k + 1] = r.valid;
  }
}
