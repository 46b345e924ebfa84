// cameras.cu -- the camera calls of the C ABI of include/vwb200.h: triangulation (K10), the epipolar rectification and
// camera_transform of pinhole pairs (K8), and the CAHV / CAHVOR cameras (K8, K10).  Each call checks its cameras, builds the
// device cameras on the host once, and stages its rasters through AbiCall.
//
// The host camera math is written with the primitives and vector helpers of pinhole.cuh and cahv.cuh, the same functions the
// kernels run.  On the host each primitive is one plain IEEE operation, and build.py compiles host code with
// -ffp-contract=off, so no product is fused with a sum into an FMA: every operation rounds as the reference's does.
#include "cahv.cuh"
#include <climits>
#include <cmath>
#include <cstring>
#include <utility>

using namespace vwb200;

extern "C" {

static void st3(double* p, V3 v) { p[0] = v.x; p[1] = v.y; p[2] = v.z; }

// ---- K10: triangulation (Stereo/StereoView.h, StereoModel.cc) through pinhole cameras ------------------------------------------
// The camera is built on the host once per call, in the reference's operation order.
static thread_local vwb200_triangulation_stats t_tri_stats = {0, 0, 0.0, 0.0, 0};

// vw::math::inverse (Math/Matrix.h:2218-2281) of a 3 x 3 matrix: LU with partial pivoting (the first largest |pivot|), then
// the lower and upper triangular solves on the permuted identity, in its loop order
static int lu_inverse3(const double* m, double* inv) {
  double b[9];
  std::memcpy(b, m, sizeof b);
  int pm[3] = {0, 1, 2};
  for (int i = 0; i < 3; ++i) {
    int p = i;
    double mx = -1;
    for (int k = i; k < 3; ++k)
      if (std::fabs(b[3 * k + i]) > mx) { mx = std::fabs(b[3 * k + i]); p = k; }
    if (b[3 * p + i] == 0.0) { set_error("Matrix is singular in inverse()"); return VWB200_EMATH; }
    if (p != i) {
      std::swap(pm[i], pm[p]);
      for (int c = 0; c < 3; ++c) std::swap(b[3 * i + c], b[3 * p + c]);
    }
    if (i != 2) {
      for (int k = i + 1; k < 3; ++k) b[3 * k + i] /= b[3 * i + i];
      for (int k = i + 1; k < 3; ++k)
        for (int c = i + 1; c < 3; ++c) b[3 * k + c] -= b[3 * k + i] * b[3 * i + c];
    }
  }
  for (int k = 0; k < 9; ++k) inv[k] = 0.0;
  for (int i = 0; i < 3; ++i) inv[3 * i + pm[i]] = 1.0;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) {
      const double t = inv[3 * i + j];
      if (t != 0.0)
        for (int k = i + 1; k < 3; ++k) inv[3 * k + j] -= b[3 * k + i] * t;
    }
  for (int i = 2; i >= 0; --i)
    for (int j = 2; j >= 0; --j) {
      const double t = inv[3 * i + j] /= b[3 * i + i];
      if (t != 0.0)
        for (int k = i - 1; k >= 0; --k) inv[3 * k + j] -= b[3 * k + i] * t;
    }
  return VWB200_OK;
}

// the argument checks of one camera (VWB200_EARG)
static int pinhole_check(const char* what, const vwb200_pinhole* p) {
  if (!p) { set_error("%s: null camera", what); return VWB200_EARG; }
  if (p->lens != VWB200_LENS_NULL && p->lens != VWB200_LENS_TSAI) { set_error("%s: unknown lens distortion %d", what, p->lens); return VWB200_EARG; }
  const int want = p->lens == VWB200_LENS_TSAI ? 5 : 0;
  if (p->num_lens_params != want) {
    set_error("%s: the %s lens distortion takes %d parameters, not %d", what, want ? "TSAI" : "NULL", want, p->num_lens_params);
    return VWB200_EARG;
  }
  return VWB200_OK;
}

// PinholeModel::rebuild_camera_matrix (PinholeModel.cc:553-605): the orthonormality asserts of u, v, w (VW_LINE_ASSERT throws
// LogicErr), then m_inv_camera_transform = inverse(uvw * transpose(R)) * inverse(K), each product a dot_prod from 0.0
static int pinhole_build(const char* what, const vwb200_pinhole& p, TriCam* c) {
  const V3 uvw[3] = {ld3(p.u_direction), ld3(p.v_direction), ld3(p.w_direction)};
  const bool ortho = dot3(uvw[0], uvw[1]) == 0 && dot3(uvw[0], uvw[2]) == 0 && dot3(uvw[1], uvw[2]) == 0 &&
                     std::fabs(norm3(uvw[0]) - 1) < 0.001 && std::fabs(norm3(uvw[1]) - 1) < 0.001 && std::fabs(norm3(uvw[2]) - 1) < 0.001;
  if (!ortho) { set_error("%s: the u, v, w coordinate frame is not orthonormal", what); return VWB200_ELOGIC; }
  double m[9], k[9] = {p.fu, 0, p.cu, 0, p.fv, p.cv, 0, 0, 1}, a[9], b[9];
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) m[3 * i + j] = dot3(uvw[i], ld3(p.rotation + 3 * j));       // row i of uvw . column j of R^T
  VWB_TRY(lu_inverse3(m, a));
  VWB_TRY(lu_inverse3(k, b));
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) c->inv[3 * i + j] = dot3(ld3(a + 3 * i), V3{b[j], b[3 + j], b[6 + j]});
  for (int q = 0; q < 3; ++q) c->c[q] = p.center[q];
  c->pitch = p.pixel_pitch;
  c->fu = p.fu; c->fv = p.fv; c->cu = p.cu; c->cv = p.cv;
  for (int q = 0; q < 5; ++q) c->k[q] = p.lens == VWB200_LENS_TSAI ? p.lens_params[q] : 0.0;
  c->tsai = p.lens == VWB200_LENS_TSAI;
  // m_camera_matrix = K * [uvw * transpose(R) | (uvw * (-transpose(R))) * C], every element a dot_prod from 0.0
  double e[12];
  for (int i = 0; i < 3; ++i) {
    double m2[3];
    for (int j = 0; j < 3; ++j) {
      e[4 * i + j] = m[3 * i + j];
      const double* r = p.rotation + 3 * j;
      m2[j] = dot3(uvw[i], V3{-r[0], -r[1], -r[2]});
    }
    e[4 * i + 3] = dot3(ld3(m2), ld3(p.center));
  }
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 4; ++j) c->P[4 * i + j] = dot3(ld3(k + 3 * i), V3{e[j], e[4 + j], e[8 + j]});
  return VWB200_OK;
}

// the five zeroed device statistics of one call
static int tri_stats_open(AbiCall& c, unsigned long long** d) {
  VWB_TRY(c.ar.alloc(d, 5));
  VWB_CUDA(cudaMemsetAsync(*d, 0, 5 * sizeof(unsigned long long), c.st));
  return VWB200_OK;
}

int vwb200_last_triangulation_stats(vwb200_triangulation_stats* out) { if (!out) return VWB200_EARG; *out = t_tri_stats; return VWB200_OK; }

// the raster checks of stereo_triangulate (after the cameras')
static int triangulate_args(const char* what, const void* disparity, int w, int h, ptrdiff_t pitch, int x0, int y0, int ow, int oh,
                            const double* xyz, ptrdiff_t xyz_pitch) {
  if (w <= 0 || h <= 0 || pitch < w) { set_error("%s: bad input size %d x %d, pitch %td", what, w, h, pitch); return VWB200_EARG; }
  if (ow <= 0 || oh <= 0 || xyz_pitch < ow) { set_error("%s: bad output size %d x %d, pitch %td", what, ow, oh, xyz_pitch); return VWB200_EARG; }
  if (x0 < 0 || y0 < 0 || x0 > w - ow || y0 > h - oh) {
    set_error("%s: the window (%d, %d, %d, %d) leaves the %d x %d input", what, x0, y0, ow, oh, w, h);
    return VWB200_EARG;
  }
  if (rasters_overlap(disparity, w, h, pitch, xyz, ow, oh, xyz_pitch, 12, 24)) { set_error("%s: xyz overlaps the disparity", what); return VWB200_EARG; }
  return VWB200_OK;
}

// the raster checks of StereoModel's image form (after the cameras')
static int model_points_args(const char* what, const float* disparity, int w, int h, ptrdiff_t pitch, const double* xyz, ptrdiff_t xyz_pitch,
                             const double* error, ptrdiff_t error_pitch) {
  if (w <= 0 || h <= 0 || pitch < w) { set_error("%s: bad input size %d x %d, pitch %td", what, w, h, pitch); return VWB200_EARG; }
  if (xyz_pitch < w || error_pitch < w) { set_error("%s: output pitches %td, %td are below the width %d", what, xyz_pitch, error_pitch, w); return VWB200_EARG; }
  if (rasters_overlap(disparity, w, h, pitch, xyz, w, h, xyz_pitch, 12, 24) || rasters_overlap(disparity, w, h, pitch, error, w, h, error_pitch, 12, 8) ||
      rasters_overlap(xyz, w, h, xyz_pitch, error, w, h, error_pitch, 24, 8)) {
    set_error("%s: the disparity, xyz and error rasters overlap", what);
    return VWB200_EARG;
  }
  return VWB200_OK;
}

int vwb200_universe_radius(const double* in, int w, int h, ptrdiff_t pitch, const double origin[3], double near_radius, double far_radius,
                           double* out, ptrdiff_t out_pitch, long long* rejected, long long* total, int on_device, void* stream) {
  const char* what = "UniverseRadius";
  if (!in || !out || !origin) { set_error("%s: null input, output or origin", what); return VWB200_EARG; }
  if (w <= 0 || h <= 0 || pitch < w || out_pitch < w) { set_error("%s: bad size %d x %d, pitches %td, %td", what, w, h, pitch, out_pitch); return VWB200_EARG; }
  if (!(near_radius >= 0 && far_radius >= 0)) { set_error("%s: radii must be >= 0.", what); return VWB200_EARG; }      // StereoView.h:160-163
  if (!(near_radius <= far_radius)) { set_error("%s: near radius must be <= far radius.", what); return VWB200_EARG; }
  if (!(out == in && out_pitch == pitch) && rasters_overlap(in, w, h, pitch, out, w, h, out_pitch, 24, 24)) {
    set_error("%s: out overlaps in (only out == in, with the same pitch, is allowed)", what);
    return VWB200_EARG;
  }
  VWB_TRY(ensure_device());
  AbiCall c;
  VWB_TRY(c.open(stream, on_device));
  const V3* din; ptrdiff_t dp;
  VWB_TRY(c.in((const V3*)in, w, h, pitch, on_device, &din, &dp));
  V3* dout; ptrdiff_t dop;
  VWB_TRY(c.out((V3*)out, w, h, out_pitch, on_device, &dout, &dop));
  unsigned long long* dst;
  VWB_TRY(tri_stats_open(c, &dst));
  VWB_TRY(universe_radius_launch((const double*)din, w, h, dp, origin, near_radius, far_radius, (double*)dout, dop, dst, c.st));
  unsigned long long s[5];
  VWB_CUDA(cudaMemcpyAsync(s, dst, sizeof s, cudaMemcpyDeviceToHost, c.st));
  VWB_TRY(c.finish());
  if (rejected) *rejected = (long long)s[0];
  if (total) *total = (long long)w * h;
  return VWB200_OK;
}

// ---- epipolar rectification (Camera/PinholeModel.cc:679-732, EpipolarUtils.cc:37-76, CameraTransform.h) -----------------------
// camera_pose().rotation_matrix(): Quaternion(R) (Math/Quaternion.h:211-252), branching on the largest of ww, xx, yy, zz, then
// rotation_matrix() (:314-335)
static void quaternion_round_trip(const double* R, double* out) {
  const double d0 = R[0], d1 = R[4], d2 = R[8];
  const double ww = 1.0 + d0 + d1 + d2, xx = 1.0 + d0 - d1 - d2, yy = 1.0 - d0 + d1 - d2, zz = 1.0 - d0 - d1 + d2;
  double mx = ww;
  if (xx > mx) mx = xx;
  if (yy > mx) mx = yy;
  if (zz > mx) mx = zz;
  double q[4];
  if (ww == mx) {
    const double w4 = std::sqrt(ww * 4.0);
    q[0] = w4 / 4; q[1] = (R[7] - R[5]) / w4; q[2] = (R[2] - R[6]) / w4; q[3] = (R[3] - R[1]) / w4;
  } else if (xx == mx) {
    const double x4 = std::sqrt(xx * 4.0);
    q[0] = (R[7] - R[5]) / x4; q[1] = x4 / 4; q[2] = (R[1] + R[3]) / x4; q[3] = (R[2] + R[6]) / x4;
  } else if (yy == mx) {
    const double y4 = std::sqrt(yy * 4.0);
    q[0] = (R[2] - R[6]) / y4; q[1] = (R[1] + R[3]) / y4; q[2] = y4 / 4; q[3] = (R[5] + R[7]) / y4;
  } else {
    const double z4 = std::sqrt(zz * 4.0);
    q[0] = (R[3] - R[1]) / z4; q[1] = (R[2] + R[6]) / z4; q[2] = (R[5] + R[7]) / z4; q[3] = z4 / 4;
  }
  const double w = q[0], x = q[1], y = q[2], z = q[3];
  const double w2 = w * w, x2 = x * x, y2 = y * y, z2 = z * z, wx = w * x, wy = w * y, wz = w * z, xy = x * y, yz = y * z, zx = z * x;
  out[0] = w2 + x2 - y2 - z2; out[4] = w2 - x2 + y2 - z2; out[8] = w2 - x2 - y2 + z2;
  out[1] = 2 * (xy - wz); out[2] = 2 * (zx + wy); out[5] = 2 * (yz - wx);
  out[3] = 2 * (xy + wz); out[6] = 2 * (zx - wy); out[7] = 2 * (yz + wx);
}

int vwb200_pinhole_epipolar(const vwb200_pinhole* cam0, const vwb200_pinhole* cam1, vwb200_pinhole* epi0, vwb200_pinhole* epi1) {
  const char* what = "epipolar";
  if (!epi0 || !epi1) { set_error("%s: null output camera", what); return VWB200_EARG; }
  VWB_TRY(pinhole_check(what, cam0));
  VWB_TRY(pinhole_check(what, cam1));
  TriCam t;
  VWB_TRY(pinhole_build(what, *cam0, &t));                  // the source cameras must be ones the reference can construct
  VWB_TRY(pinhole_build(what, *cam1, &t));
  double rot0[9], rot1[9];
  quaternion_round_trip(cam0->rotation, rot0);
  quaternion_round_trip(cam1->rotation, rot1);
  const V3 look0{-1 * rot0[2], -1 * rot0[5], -1 * rot0[8]}, look1{-1 * rot1[2], -1 * rot1[5], -1 * rot1[8]};
  const V3 mean{(look0.x + look1.x) / 2.0, (look0.y + look1.y) / 2.0, (look0.z + look1.z) / 2.0};
  const V3 u = normalize3(sub3(ld3(cam1->center), ld3(cam0->center)));
  const V3 w = normalize3(cross3(u, cross3(mean, u)));
  const V3 v = cross3(w, u);
  vwb200_pinhole e{};
  const double rot[9] = {u.x, -v.x, -w.x, u.y, -v.y, -w.y, u.z, -v.z, -w.z};      // the columns u, -v, -w
  std::memcpy(e.rotation, rot, sizeof rot);
  e.fu = (cam0->fu + cam1->fu) / 2.0; e.fv = (cam0->fv + cam1->fv) / 2.0;
  e.cu = (cam0->cu + cam1->cu) / 2.0; e.cv = (cam0->cv + cam1->cv) / 2.0;
  e.pixel_pitch = (cam0->pixel_pitch + cam1->pixel_pitch) / 2.0;
  e.u_direction[0] = e.v_direction[1] = e.w_direction[2] = 1.0;
  e.lens = VWB200_LENS_NULL;
  vwb200_pinhole e1 = e;                                    // the outputs may be the inputs
  std::memcpy(e.center, cam0->center, sizeof e.center);
  std::memcpy(e1.center, cam1->center, sizeof e.center);
  *epi0 = e;
  *epi1 = e1;
  return VWB200_OK;
}

struct MaskF { float v, valid; };                                // PixelMask<float>

// CameraTransform's VW_ASSERT (CameraTransform.h:53, 66): both cameras at one center
static int same_center(const char* what, const double* a, const double* b) {
  if (a[0] == b[0] && a[1] == b[1] && a[2] == b[2]) return VWB200_OK;
  set_error("%s: CameraTransformFunctor: Camera transformation require that the camera center is always the same for both cameras.", what);
  return VWB200_ELOGIC;
}

static int projection_error(const char* what, long long x, long long y) {
  set_error("%s: PinholeModel: Projection into pinhole camera is inaccurate. (first failing pixel (%lld, %lld))", what, x, y);
  return VWB200_EPROJECT;
}

// the perimeter index k of compute_transformed_bbox_fast over (x0, y0, x1, y1) as a pixel
static void perimeter_pixel(const int32_t* r, long long k, long long* x, long long* y) {
  const long long cw = (long long)r[2] - r[0], ch = (long long)r[3] - r[1];
  if (k < cw) { *x = r[0] + k; *y = r[1]; }
  else if (k < 2 * cw) { *x = r[0] + k - cw; *y = r[3] - 1LL; }
  else if (k < 2 * cw + ch) { *x = r[0]; *y = r[1] + k - 2 * cw; }
  else { *x = r[2] - 1LL; *y = r[1] + k - 2 * cw - ch; }
}

// both cameras' compute_transformed_bbox_fast through CameraTransform(cam, epi)::forward: bbox[cam] = {min x, min y, max x, max y}
static int epipolar_bboxes(AbiCall& c, const TriCam* cam, const TriCam* epi, const int32_t* const* roi, float (*bbox)[4]) {
  unsigned* keys;
  unsigned long long* fail;
  VWB_TRY(c.ar.alloc(&keys, 8));
  VWB_TRY(c.ar.alloc(&fail, 4));
  const float big = (float)(INT32_MAX - 1);                    // BBox2f's initial bounds (Math/BBox.tcc:38-45)
  const unsigned init[8] = {fkey(big), fkey(big), fkey(-big), fkey(-big), fkey(big), fkey(big), fkey(-big), fkey(-big)};
  const unsigned long long finit[4] = {0, ULLONG_MAX, 0, ULLONG_MAX};
  VWB_CUDA(cudaMemcpyAsync(keys, init, sizeof init, cudaMemcpyHostToDevice, c.st));
  VWB_CUDA(cudaMemcpyAsync(fail, finit, sizeof finit, cudaMemcpyHostToDevice, c.st));
  for (int i = 0; i < 2; ++i)
    VWB_TRY(camera_bbox_launch(cam[i], epi[i], roi[i][0], roi[i][1], roi[i][2], roi[i][3], keys + 4 * i, fail + 2 * i, c.st));
  unsigned k[8];
  unsigned long long f[4];
  VWB_CUDA(cudaMemcpyAsync(k, keys, sizeof k, cudaMemcpyDeviceToHost, c.st));
  VWB_CUDA(cudaMemcpyAsync(f, fail, sizeof f, cudaMemcpyDeviceToHost, c.st));
  VWB_CUDA(cudaStreamSynchronize(c.st));
  for (int i = 0; i < 2; ++i)
    if (f[2 * i]) {                                            // the reference throws at the first failing point of the first camera
      long long x, y;
      perimeter_pixel(roi[i], (long long)f[2 * i + 1], &x, &y);
      return projection_error("resize_epipolar_cameras_to_fit", x, y);
    }
  for (int i = 0; i < 8; ++i) bbox[i / 4][i % 4] = kfloat(k[i]);
  return VWB200_OK;
}

static int roi_check(const char* what, const int32_t* r) {
  if (!r) { set_error("%s: null ROI", what); return VWB200_EARG; }
  if (r[2] < r[0] || r[3] < r[1]) { set_error("%s: bad ROI (%d, %d, %d, %d)", what, r[0], r[1], r[2], r[3]); return VWB200_EARG; }
  return VWB200_OK;
}

int vwb200_resize_epipolar_cameras_to_fit(const vwb200_pinhole* cam1, const vwb200_pinhole* cam2, vwb200_pinhole* epi1, vwb200_pinhole* epi2,
                                          const int32_t roi1[4], const int32_t roi2[4], int32_t size1[2], int32_t size2[2], void* stream) {
  const char* what = "resize_epipolar_cameras_to_fit";
  if (!size1 || !size2) { set_error("%s: null output size", what); return VWB200_EARG; }
  VWB_TRY(pinhole_check(what, cam1));
  VWB_TRY(pinhole_check(what, cam2));
  VWB_TRY(pinhole_check(what, epi1));
  VWB_TRY(pinhole_check(what, epi2));
  VWB_TRY(roi_check(what, roi1));
  VWB_TRY(roi_check(what, roi2));
  TriCam cam[2], epi[2];
  VWB_TRY(pinhole_build(what, *cam1, &cam[0]));
  VWB_TRY(pinhole_build(what, *cam2, &cam[1]));
  VWB_TRY(pinhole_build(what, *epi1, &epi[0]));
  VWB_TRY(pinhole_build(what, *epi2, &epi[1]));
  VWB_TRY(same_center(what, cam[0].c, epi[0].c));
  VWB_TRY(same_center(what, cam[1].c, epi[1].c));
  VWB_TRY(ensure_device());
  AbiCall c;
  VWB_TRY(c.open(stream, 0));
  const int32_t* roi[2] = {roi1, roi2};
  float bb[2][4];
  VWB_TRY(epipolar_bboxes(c, cam, epi, roi, bb));
  // shift both principal points by the leftmost / uppermost corner (in CCD units), from epi1's offset (EpipolarUtils.cc:52-65)
  const double min_col = std::min(bb[0][0], bb[1][0]), min_row = std::min(bb[0][1], bb[1][1]);
  const double cu = epi1->cu - min_col * epi1->pixel_pitch, cv = epi1->cv - min_row * epi1->pixel_pitch;
  vwb200_pinhole e1 = *epi1, e2 = *epi2;
  e1.cu = e2.cu = cu;
  e1.cv = e2.cv = cv;
  VWB_TRY(pinhole_build(what, e1, &epi[0]));
  VWB_TRY(pinhole_build(what, e2, &epi[1]));
  VWB_TRY(epipolar_bboxes(c, cam, epi, roi, bb));
  VWB_TRY(c.finish());
  *epi1 = e1;
  *epi2 = e2;
  size1[0] = (int32_t)bb[0][2]; size1[1] = (int32_t)bb[0][3];    // Vector2i(bbox.max()): truncation toward zero
  size2[0] = (int32_t)bb[1][2]; size2[1] = (int32_t)bb[1][3];
  return VWB200_OK;
}

// the raster, pixel type, interpolation and edge checks of camera_transform (after the cameras'): VWB200_EARG, then
// VWB200_ENOIMPL for the combinations without a device form
static int camera_transform_args(const char* what, int pixel_type, int interp, int edge, const float* edge_value, const void* in, int w, int h,
                                 ptrdiff_t pitch, int x0, int y0, const void* out, int ow, int oh, ptrdiff_t opitch) {
  if (pixel_type != VWB200_PIXEL_GRAY_F32 && pixel_type != VWB200_PIXEL_MASK_F32) { set_error("%s: unknown pixel type %d", what, pixel_type); return VWB200_EARG; }
  if (interp != VWB200_INTERP_BILINEAR && interp != VWB200_INTERP_BICUBIC && interp != VWB200_INTERP_NEAREST) {
    set_error("%s: unknown interpolation %d", what, interp);
    return VWB200_EARG;
  }
  if (edge != VWB200_EDGE_ZERO && edge != VWB200_EDGE_CONSTANT && edge != VWB200_EDGE_VALUE) { set_error("%s: unknown edge extension %d", what, edge); return VWB200_EARG; }
  if (w <= 0 || h <= 0 || pitch < w) { set_error("%s: bad image size %d x %d, pitch %td", what, w, h, pitch); return VWB200_EARG; }
  if (ow <= 0 || oh <= 0 || opitch < ow) { set_error("%s: bad output size %d x %d, pitch %td", what, ow, oh, opitch); return VWB200_EARG; }
  if ((long long)x0 + ow - 1 > INT_MAX || (long long)y0 + oh - 1 > INT_MAX) {
    set_error("%s: the window (%d, %d, %d, %d) leaves the int32 pixel coordinates", what, x0, y0, ow, oh);
    return VWB200_EARG;
  }
  const bool masked = pixel_type == VWB200_PIXEL_MASK_F32;
  const size_t px = masked ? 8 : 4;
  if (rasters_overlap(in, w, h, pitch, out, ow, oh, opitch, px, px)) { set_error("%s: out overlaps the image", what); return VWB200_EARG; }
  if (edge == VWB200_EDGE_VALUE && !edge_value) { set_error("%s: ValueEdgeExtension needs an edge value", what); return VWB200_EARG; }
  if ((masked && interp != VWB200_INTERP_BILINEAR) || (!masked && edge == VWB200_EDGE_VALUE)) {
    set_error("%s: %s has no device form (PixelMask<float> takes bilinear interpolation, ValueEdgeExtension PixelMask<float> pixels)", what,
              masked ? "this interpolation of PixelMask<float> pixels" : "ValueEdgeExtension of float pixels");
    return VWB200_ENOIMPL;
  }
  return VWB200_OK;
}

// camera_transform's image and window, staged: float pixels, or {value, valid} pairs staged as such
static int camera_transform_stage(AbiCall& c, bool masked, const void* in, int w, int h, ptrdiff_t pitch, void* out, int ow, int oh, ptrdiff_t opitch,
                                  int on_device, const float** din, ptrdiff_t* dp, float** dout, ptrdiff_t* dop) {
  if (masked) {
    const MaskF* mi; MaskF* mo;
    VWB_TRY(c.in((const MaskF*)in, w, h, pitch, on_device, &mi, dp));
    VWB_TRY(c.out((MaskF*)out, ow, oh, opitch, on_device, &mo, dop));
    *din = (const float*)mi; *dout = (float*)mo;
    return VWB200_OK;
  }
  VWB_TRY(c.in((const float*)in, w, h, pitch, on_device, din, dp));
  return c.out((float*)out, ow, oh, opitch, on_device, dout, dop);
}

// ---- CAHV / CAHVOR cameras (Camera/CAHVModel.cc, CAHVORModel.cc, CameraTransform.h, StereoModel.cc:121-122) ---------------------
// linearize_camera evaluates the rays with cahv.cuh's cahv_pixel_to_vector, the function K8 and K10 run.
static int cahv_check(const char* what, const vwb200_cahv* c) {
  if (!c) { set_error("%s: null camera", what); return VWB200_EARG; }
  if (c->model != VWB200_CAMERA_CAHV && c->model != VWB200_CAMERA_CAHVOR) { set_error("%s: unknown camera model %d", what, c->model); return VWB200_EARG; }
  return VWB200_OK;
}

// ---- the pinhole and CAHV camera families ----------------------------------------------------------------------------------
// What stereo_triangulate, StereoModel and camera_transform need to know of a family: its C ABI and device cameras, the
// argument check, build (VWB200_ELOGIC / EMATH for a pinhole camera the reference cannot construct), the center, the statistic
// that receives the Newton iterations, and which camera_transform destinations have a device form.
struct PinholeFamily {
  using Abi = vwb200_pinhole;
  using Dev = TriCam;
  static constexpr auto check = pinhole_check;
  static constexpr auto build = pinhole_build;
  static const double* center(const TriCam& c) { return c.c; }
  static constexpr long long vwb200_triangulation_stats::*iterations = &vwb200_triangulation_stats::tsai_iterations;
  static int transform_dst(const char*, const vwb200_pinhole&) { return VWB200_OK; }
};
struct CahvFamily {
  using Abi = vwb200_cahv;
  using Dev = CahvCam;
  static constexpr auto check = cahv_check;
  static int build(const char*, const vwb200_cahv& c, CahvCam* d) {
    std::memcpy(d->C, c.C, sizeof d->C); std::memcpy(d->A, c.A, sizeof d->A); std::memcpy(d->H, c.H, sizeof d->H);
    std::memcpy(d->V, c.V, sizeof d->V); std::memcpy(d->O, c.O, sizeof d->O); std::memcpy(d->R, c.R, sizeof d->R);
    d->cahvor = c.model == VWB200_CAMERA_CAHVOR;
    d->flip = dot3(cross3(ld3(c.V), ld3(c.H)), ld3(c.A)) < 0.0;     // a left-handed camera, whose rays pixel_to_vector negates
    return VWB200_OK;
  }
  static const double* center(const CahvCam& c) { return c.C; }
  static constexpr long long vwb200_triangulation_stats::*iterations = &vwb200_triangulation_stats::cahvor_iterations;
  // K8 compiles the destination's ray without the CAHVOR Newton loop
  static int transform_dst(const char* what, const vwb200_cahv& c) {
    if (c.model == VWB200_CAMERA_CAHV) return VWB200_OK;
    set_error("%s: the destination camera must be CAHV (a CAHVOR one has no device form)", what);
    return VWB200_ENOIMPL;
  }
};

int vwb200_cahv_epipolar(const vwb200_cahv* cam0, const vwb200_cahv* cam1, vwb200_cahv* epi0, vwb200_cahv* epi1) {
  const char* what = "epipolar";
  if (!epi0 || !epi1) { set_error("%s: null output camera", what); return VWB200_EARG; }
  VWB_TRY(cahv_check(what, cam0));
  VWB_TRY(cahv_check(what, cam1));
  if (cam0->model != VWB200_CAMERA_CAHV || cam1->model != VWB200_CAMERA_CAHV) {
    set_error("%s: epipolar() takes CAHV cameras (linearize_camera takes a CAHVOR camera to one)", what);
    return VWB200_EARG;
  }
  const V3 A0 = ld3(cam0->A), H0 = ld3(cam0->H), V0 = ld3(cam0->V), A1 = ld3(cam1->A), H1 = ld3(cam1->H), V1 = ld3(cam1->V);
  const double hc = dot3(H0, A0) / 2.0 + dot3(H1, A1) / 2.0;
  const double vc = dot3(V0, A0) / 2.0 + dot3(V1, A1) / 2.0;
  const double hs = norm3(cross3(A0, H0)) / 2.0 + norm3(cross3(A1, H1)) / 2.0;
  const double vs = norm3(cross3(A0, V0)) / 2.0 + norm3(cross3(A1, V1)) / 2.0;
  const V3 app = add3(A0, A1);
  const V3 f = cross3(cross3(app, sub3(ld3(cam1->C), ld3(cam0->C))), app);
  const double nf = norm3(f);
  const V3 fs = dot3(f, H0) > 0 ? f : V3{-f.x, -f.y, -f.z};
  const V3 hp{fs.x * hs / nf, fs.y * hs / nf, fs.z * hs / nf};
  const V3 app2 = scale3(0.5, app);
  const double dh = dot3(app2, hp);
  const V3 a = normalize3(sub3(app2, V3{hp.x * dh / (hs * hs), hp.y * dh / (hs * hs), hp.z * dh / (hs * hs)}));
  const V3 t = cross3(a, hp);
  const V3 vp{t.x * vs / hs, t.y * vs / hs, t.z * vs / hs};
  vwb200_cahv e{};
  e.model = VWB200_CAMERA_CAHV;
  st3(e.A, a);
  st3(e.H, add3(hp, scale3(hc, a)));
  st3(e.V, add3(vp, scale3(vc, a)));
  vwb200_cahv e1 = e;                                            // the outputs may be the inputs
  std::memcpy(e.C, cam0->C, sizeof e.C);
  std::memcpy(e1.C, cam1->C, sizeof e1.C);
  *epi0 = e;
  *epi1 = e1;
  return VWB200_OK;
}

int vwb200_linearize_camera(const vwb200_cahv* cam, const int32_t cahvor_size[2], const int32_t cahv_size[2], vwb200_cahv* out) {
  const char* what = "linearize_camera";
  if (!cahvor_size || !cahv_size || !out) { set_error("%s: null size or output camera", what); return VWB200_EARG; }
  VWB_TRY(cahv_check(what, cam));
  if (cam->model != VWB200_CAMERA_CAHVOR) { set_error("%s: linearize_camera() takes a CAHVOR camera", what); return VWB200_EARG; }
  CahvCam c;                                                     // a copy: out may be cam
  VWB_TRY(CahvFamily::build(what, *cam, &c));
  const int ix = cahvor_size[0], iy = cahvor_size[1];
  // the landmarks around the perimeter; vpts[4] divides in int where vpts[1] divides in double, as the reference does
  const double hpts[6][2] = {{0, 0}, {0, (iy - 1) / 2.0}, {0, (double)(iy - 1)}, {(double)(ix - 1), 0}, {(double)(ix - 1), (iy - 1) / 2.0},
                             {ix - 1.0, iy - 1.0}};
  const double vpts[6][2] = {{0, 0}, {(ix - 1) / 2.0, 0}, {(double)(ix - 1), 0}, {0, (double)(iy - 1)}, {(double)((ix - 1) / 2), (double)(iy - 1)},
                             {ix - 1.0, iy - 1.0}};
  int iters = 0;
  const auto ray = [&](const double* pt) { return cahv_pixel_to_vector<true>(c, pt[0], pt[1], &iters); };
  V3 A{0.0, 0.0, 0.0};
  for (int k = 0; k < 6; ++k) A = add3(A, ray(vpts[k]));
  for (int k = 0; k < 6; ++k) A = add3(A, ray(hpts[k]));
  A = normalize3(A);
  const V3 r = cross3(normalize3(cross3(ld3(c.A), ld3(c.H))), A);
  const V3 dn = normalize3(cross3(A, r)), rt = normalize3(r);
  // the smallest |A x w| over the landmarks, w each ray with its component along n removed
  const auto min_sin = [&](const double (*pts)[2], V3 n) {
    double mn = 1;
    for (int k = 0; k < 6; ++k) {
      const V3 u3 = ray(pts[k]);
      const double sn = norm3(cross3(A, normalize3(sub3(u3, scale3(dot3(n, u3), n)))));
      if (mn > sn) mn = sn;
    }
    return mn;
  };
  const double hmin = min_sin(hpts, dn), vmin = min_sin(vpts, rt);
  // minfov: the smaller field of view
  const double ic[2] = {((double)cahv_size[0] - 1.0) / 2.0, ((double)cahv_size[1] - 1.0) / 2.0};
  const double ic2[2] = {ic[0] * ic[0], ic[1] * ic[1]};
  const double sf[2] = {std::sqrt(ic2[0] / (hmin * hmin) - ic2[0]), std::sqrt(ic2[1] / (vmin * vmin) - ic2[1])};
  vwb200_cahv o{};
  o.model = VWB200_CAMERA_CAHV;
  std::memcpy(o.C, c.C, sizeof o.C);
  st3(o.A, A);
  st3(o.H, add3(scale3(sf[0], rt), scale3(ic[0], A)));
  st3(o.V, add3(scale3(sf[1], dn), scale3(ic[1], A)));
  *out = o;
  return VWB200_OK;
}

int vwb200_pinhole_to_cahv(const vwb200_pinhole* pin, vwb200_cahv* out) {
  const char* what = "CAHVModel = PinholeModel";
  if (!out) { set_error("%s: null output camera", what); return VWB200_EARG; }
  VWB_TRY(pinhole_check(what, pin));
  if (pin->lens != VWB200_LENS_NULL) { set_error("%s: the pinhole has a lens distortion, which a CAHV camera cannot carry", what); return VWB200_EARG; }
  TriCam t;
  VWB_TRY(pinhole_build(what, *pin, &t));                        // a camera the reference can construct
  const double pitch = pin->pixel_pitch;
  if (pitch == 0) { set_error("%s: CAHVModel::operator=() input pinhole model has zero pitch!", what); return VWB200_EARG; }
  const double fH = pin->fu / pitch, fV = pin->fv / pitch, cH = pin->cu / pitch, cV = pin->cv / pitch;
  const double* R = pin->rotation;
  const auto rot = [&](const double* v) { return V3{dot3(ld3(R), ld3(v)), dot3(ld3(R + 3), ld3(v)), dot3(ld3(R + 6), ld3(v))}; };   // R * v
  const V3 Hv = rot(pin->u_direction), Vv = rot(pin->v_direction), A = rot(pin->w_direction);
  vwb200_cahv o{};
  o.model = VWB200_CAMERA_CAHV;
  std::memcpy(o.C, pin->center, sizeof o.C);
  st3(o.A, A);
  st3(o.H, add3(scale3(fH, Hv), scale3(cH, A)));
  st3(o.V, add3(scale3(fV, Vv), scale3(cV, A)));
  *out = o;
  return VWB200_OK;
}

// ---- stereo_triangulate, StereoModel and camera_transform through either camera family -----------------------------------
// The family bodies are templates, so they sit in an extern "C++" block.
extern "C++" {
template <class F>
static int stereo_triangulate_family(int pixel_type, const void* disparity, int w, int h, ptrdiff_t pitch, int x0, int y0, int ow, int oh,
                                     const typename F::Abi* cam1, const typename F::Abi* cam2, double angle_tol, double* xyz,
                                     ptrdiff_t xyz_pitch, int on_device, void* stream) {
  t_tri_stats = vwb200_triangulation_stats{};
  const char* what = "stereo_triangulate";
  if (!disparity || !xyz) { set_error("%s: null disparity or output", what); return VWB200_EARG; }
  if (pixel_type != VWB200_DISP_I32 && pixel_type != VWB200_DISP_F32) { set_error("%s: unknown pixel type %d", what, pixel_type); return VWB200_EARG; }
  VWB_TRY(F::check(what, cam1));
  VWB_TRY(F::check(what, cam2));
  VWB_TRY(triangulate_args(what, disparity, w, h, pitch, x0, y0, ow, oh, xyz, xyz_pitch));
  typename F::Dev c0, c1;
  VWB_TRY(F::build(what, *cam1, &c0));
  VWB_TRY(F::build(what, *cam2, &c1));
  const double tol = angle_tol > 0 ? angle_tol : 1e-4;            // are_nearly_parallel's (StereoModel.cc:81-83)
  VWB_TRY(ensure_device());
  AbiCall c;
  VWB_TRY(c.open(stream, on_device));
  V3* dxyz; ptrdiff_t dxp;
  VWB_TRY(c.out((V3*)xyz, ow, oh, xyz_pitch, on_device, &dxyz, &dxp));
  unsigned long long* dst;
  VWB_TRY(tri_stats_open(c, &dst));
  // only the window is read: stage that alone
  if (pixel_type == VWB200_DISP_I32) {
    const vwb200_dispi* din; ptrdiff_t dp;
    VWB_TRY(c.in((const vwb200_dispi*)disparity + (ptrdiff_t)y0 * pitch + x0, ow, oh, pitch, on_device, &din, &dp));
    VWB_TRY(stereo_triangulate_launch(din, dp, x0, y0, ow, oh, c0, c1, tol, (double*)dxyz, dxp, dst, c.st));
  } else {
    const DispF* din; ptrdiff_t dp;
    VWB_TRY(c.in((const DispF*)disparity + (ptrdiff_t)y0 * pitch + x0, ow, oh, pitch, on_device, &din, &dp));
    VWB_TRY(stereo_triangulate_launch(din, dp, x0, y0, ow, oh, c0, c1, tol, (double*)dxyz, dxp, dst, c.st));
  }
  unsigned long long s[5];
  VWB_CUDA(cudaMemcpyAsync(s, dst, sizeof s, cudaMemcpyDeviceToHost, c.st));
  VWB_TRY(c.finish());
  t_tri_stats.*F::iterations = (long long)s[4];
  return VWB200_OK;
}

template <class F>
static int stereo_model_points_family(const float* disparity, int w, int h, ptrdiff_t pitch, const typename F::Abi* cam1,
                                      const typename F::Abi* cam2, double angle_tol, double* xyz, ptrdiff_t xyz_pitch, double* error,
                                      ptrdiff_t error_pitch, int on_device, void* stream) {
  t_tri_stats = vwb200_triangulation_stats{};
  const char* what = "StereoModel";
  if (!disparity || !xyz || !error) { set_error("%s: null disparity or output", what); return VWB200_EARG; }
  VWB_TRY(F::check(what, cam1));
  VWB_TRY(F::check(what, cam2));
  VWB_TRY(model_points_args(what, disparity, w, h, pitch, xyz, xyz_pitch, error, error_pitch));
  typename F::Dev c0, c1;
  VWB_TRY(F::build(what, *cam1, &c0));
  VWB_TRY(F::build(what, *cam2, &c1));
  const double tol = angle_tol > 0 ? angle_tol : 1e-4;
  VWB_TRY(ensure_device());
  AbiCall c;
  VWB_TRY(c.open(stream, on_device));
  const DispF* din; ptrdiff_t dp;
  VWB_TRY(c.in((const DispF*)disparity, w, h, pitch, on_device, &din, &dp));
  V3* dxyz; ptrdiff_t dxp;
  VWB_TRY(c.out((V3*)xyz, w, h, xyz_pitch, on_device, &dxyz, &dxp));
  double* derr; ptrdiff_t dep;
  VWB_TRY(c.out(error, w, h, error_pitch, on_device, &derr, &dep));
  unsigned long long* dst;
  VWB_TRY(tri_stats_open(c, &dst));
  VWB_TRY(stereo_model_launch(din, w, h, dp, c0, c1, tol, (double*)dxyz, dxp, derr, dep, dst, c.st));
  unsigned long long s[5];
  VWB_CUDA(cudaMemcpyAsync(s, dst, sizeof s, cudaMemcpyDeviceToHost, c.st));
  VWB_TRY(c.finish());
  double sum, mx;
  std::memcpy(&sum, &s[0], sizeof sum);
  std::memcpy(&mx, &s[1], sizeof mx);
  t_tri_stats = vwb200_triangulation_stats{(long long)s[2], (long long)s[3], mx, sum, 0, 0};
  t_tri_stats.*F::iterations = (long long)s[4];
  return VWB200_OK;
}

template <class F>
static int camera_transform_family(const typename F::Abi* src, const typename F::Abi* dst, int pixel_type, int interp, int edge,
                                   const float* edge_value, const void* in, int w, int h, ptrdiff_t pitch, int x0, int y0, void* out, int ow,
                                   int oh, ptrdiff_t opitch, int on_device, void* stream) {
  const char* what = "camera_transform";
  if (!in || !out) { set_error("%s: null input or output", what); return VWB200_EARG; }
  VWB_TRY(F::check(what, src));
  VWB_TRY(F::check(what, dst));
  VWB_TRY(camera_transform_args(what, pixel_type, interp, edge, edge_value, in, w, h, pitch, x0, y0, out, ow, oh, opitch));
  VWB_TRY(F::transform_dst(what, *dst));
  const bool masked = pixel_type == VWB200_PIXEL_MASK_F32;
  const float ev[2] = {edge_value ? edge_value[0] : 0.0f, edge_value ? edge_value[1] : 0.0f};
  typename F::Dev s, d;
  VWB_TRY(F::build(what, *src, &s));
  VWB_TRY(F::build(what, *dst, &d));
  VWB_TRY(same_center(what, F::center(s), F::center(d)));
  VWB_TRY(ensure_device());
  AbiCall c;
  VWB_TRY(c.open(stream, on_device));
  const float* din; ptrdiff_t dp;
  float* dout; ptrdiff_t dop;
  VWB_TRY(camera_transform_stage(c, masked, in, w, h, pitch, out, ow, oh, opitch, on_device, &din, &dp, &dout, &dop));
  unsigned long long* fail;
  VWB_TRY(c.ar.alloc(&fail, 2));
  const unsigned long long finit[2] = {0, ULLONG_MAX};
  VWB_CUDA(cudaMemcpyAsync(fail, finit, sizeof finit, cudaMemcpyHostToDevice, c.st));
  VWB_TRY(camera_warp_launch(masked, interp, edge, ev, s, d, din, w, h, dp, x0, y0, dout, ow, oh, dop, fail, c.st));
  unsigned long long f[2];
  VWB_CUDA(cudaMemcpyAsync(f, fail, sizeof f, cudaMemcpyDeviceToHost, c.st));
  VWB_TRY(c.finish());
  if (f[0]) return projection_error(what, x0 + (long long)(f[1] % (unsigned long long)ow), y0 + (long long)(f[1] / (unsigned long long)ow));
  return VWB200_OK;
}
}  // extern "C++"

int vwb200_stereo_triangulate(int pixel_type, const void* disparity, int w, int h, ptrdiff_t pitch, int x0, int y0, int ow, int oh,
                              const vwb200_pinhole* cam1, const vwb200_pinhole* cam2, double angle_tol, double* xyz, ptrdiff_t xyz_pitch,
                              int on_device, void* stream) {
  return stereo_triangulate_family<PinholeFamily>(pixel_type, disparity, w, h, pitch, x0, y0, ow, oh, cam1, cam2, angle_tol, xyz, xyz_pitch,
                                                  on_device, stream);
}

int vwb200_cahv_stereo_triangulate(int pixel_type, const void* disparity, int w, int h, ptrdiff_t pitch, int x0, int y0, int ow, int oh,
                                   const vwb200_cahv* cam1, const vwb200_cahv* cam2, double angle_tol, double* xyz, ptrdiff_t xyz_pitch,
                                   int on_device, void* stream) {
  return stereo_triangulate_family<CahvFamily>(pixel_type, disparity, w, h, pitch, x0, y0, ow, oh, cam1, cam2, angle_tol, xyz, xyz_pitch,
                                               on_device, stream);
}

int vwb200_stereo_model_points(const float* disparity, int w, int h, ptrdiff_t pitch, const vwb200_pinhole* cam1,
                               const vwb200_pinhole* cam2, double angle_tol, double* xyz, ptrdiff_t xyz_pitch, double* error,
                               ptrdiff_t error_pitch, int on_device, void* stream) {
  return stereo_model_points_family<PinholeFamily>(disparity, w, h, pitch, cam1, cam2, angle_tol, xyz, xyz_pitch, error, error_pitch,
                                                   on_device, stream);
}

int vwb200_cahv_stereo_model_points(const float* disparity, int w, int h, ptrdiff_t pitch, const vwb200_cahv* cam1, const vwb200_cahv* cam2,
                                    double angle_tol, double* xyz, ptrdiff_t xyz_pitch, double* error, ptrdiff_t error_pitch, int on_device,
                                    void* stream) {
  return stereo_model_points_family<CahvFamily>(disparity, w, h, pitch, cam1, cam2, angle_tol, xyz, xyz_pitch, error, error_pitch, on_device,
                                                stream);
}

int vwb200_camera_transform(const vwb200_pinhole* src, const vwb200_pinhole* dst, int pixel_type, int interp, int edge, const float edge_value[2],
                            const void* in, int w, int h, ptrdiff_t pitch, int x0, int y0, void* out, int ow, int oh, ptrdiff_t opitch,
                            int on_device, void* stream) {
  return camera_transform_family<PinholeFamily>(src, dst, pixel_type, interp, edge, edge_value, in, w, h, pitch, x0, y0, out, ow, oh, opitch,
                                                on_device, stream);
}

int vwb200_cahv_camera_transform(const vwb200_cahv* src, const vwb200_cahv* dst, int pixel_type, int interp, int edge, const float edge_value[2],
                                 const void* in, int w, int h, ptrdiff_t pitch, int x0, int y0, void* out, int ow, int oh, ptrdiff_t opitch,
                                 int on_device, void* stream) {
  return camera_transform_family<CahvFamily>(src, dst, pixel_type, interp, edge, edge_value, in, w, h, pitch, x0, y0, out, ow, oh, opitch,
                                             on_device, stream);
}


}  // extern "C"
