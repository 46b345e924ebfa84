/* vw_triangulate_oracle.c -- see vw_triangulate_oracle.h.  Each function restates its reference counterpart in the same
 * operation order, one IEEE double operation per source operation (no FMA contraction). */
#include "vw_triangulate_oracle.h"

#include <float.h>
#include <math.h>
#include <string.h>

/* dot_prod: a sum from 0.0 */
static double dot3(const double* a, const double* b) {
  double r = 0.0;
  for (int i = 0; i < 3; ++i) r += a[i] * b[i];
  return r;
}
static double norm3(const double* a) { return sqrt(dot3(a, a)); }

int vwt_inverse3(const double m[9], double inv[9]) {
  double buf[9];
  size_t pm[3];
  memcpy(buf, m, sizeof buf);
  for (size_t i = 0; i < 3; ++i) pm[i] = i;
  for (size_t i = 0; i < 3; ++i) {
    /* index_norm_inf(subvector(column i, i, 3 - i)): the first largest magnitude */
    double maxval = -1;
    size_t idx = 0;
    for (size_t k = 0; k < 3 - i; ++k) {
      double a = fabs(buf[3 * (i + k) + i]);
      if (a > maxval) { maxval = a; idx = k; }
    }
    size_t i_norm_inf = i + idx;
    if (buf[3 * i_norm_inf + i] == 0.0) return -2;
    if (i_norm_inf != i) {
      size_t pbuf = pm[i];
      pm[i] = pm[i_norm_inf];
      pm[i_norm_inf] = pbuf;
      for (size_t c = 0; c < 3; ++c) {
        double t = buf[3 * i + c];
        buf[3 * i + c] = buf[3 * i_norm_inf + c];
        buf[3 * i_norm_inf + c] = t;
      }
    }
    if (i != 2) {
      for (size_t k = i + 1; k < 3; ++k) buf[3 * k + i] = buf[3 * k + i] / buf[3 * i + i];
      for (size_t k = i + 1; k < 3; ++k)
        for (size_t c = i + 1; c < 3; ++c) buf[3 * k + c] = buf[3 * k + c] - buf[3 * k + i] * buf[3 * i + c];
    }
  }
  for (int k = 0; k < 9; ++k) inv[k] = 0.0;
  for (size_t i = 0; i < 3; ++i) inv[3 * i + pm[i]] = 1.0;
  for (size_t i = 0; i < 3; ++i)
    for (size_t j = 0; j < 3; ++j) {
      double t = inv[3 * i + j];
      if (t != 0.0)
        for (size_t k = i + 1; k < 3; ++k) inv[3 * k + j] = inv[3 * k + j] - buf[3 * k + i] * t;
    }
  for (long i = 2; i >= 0; --i)
    for (long j = 2; j >= 0; --j) {
      double t = inv[3 * i + j] = inv[3 * i + j] / buf[3 * i + i];
      if (t != 0.0)
        for (long k = i - 1; k >= 0; --k) inv[3 * k + j] = inv[3 * k + j] - buf[3 * k + i] * t;
    }
  return 0;
}

int vwt_camera_inverse(const vwt_pinhole* cam, double inv[9]) {
  const double* u = cam->u_direction;
  const double* v = cam->v_direction;
  const double* w = cam->w_direction;
  if (!(dot3(u, v) == 0)) return -3;
  if (!(dot3(u, w) == 0)) return -3;
  if (!(dot3(v, w) == 0)) return -3;
  if (!(fabs(norm3(u) - 1) < 0.001)) return -3;
  if (!(fabs(norm3(v) - 1) < 0.001)) return -3;
  if (!(fabs(norm3(w) - 1) < 0.001)) return -3;
  const double* uvw[3] = {u, v, w};
  double rt[9], m[9], k[9], a[9], b[9];
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) rt[3 * r + c] = cam->rotation[3 * c + r];          /* transpose(m_rotation) */
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      double col[3] = {rt[c], rt[3 + c], rt[6 + c]};
      m[3 * r + c] = dot3(uvw[r], col);
    }
  k[0] = cam->fu; k[1] = 0; k[2] = cam->cu;
  k[3] = 0; k[4] = cam->fv; k[5] = cam->cv;
  k[6] = 0; k[7] = 0; k[8] = 1;
  int rc = vwt_inverse3(m, a);
  if (rc) return rc;
  rc = vwt_inverse3(k, b);
  if (rc) return rc;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) {
      double col[3] = {b[c], b[3 + c], b[6 + c]};
      inv[3 * r + c] = dot3(a + 3 * r, col);
    }
  return 0;
}

/* TsaiDistortionNorm (LensDistortion.cc:260-276) */
static void tsai_norm(const double* P, const double* d, double* out) {
  double x = P[0];
  double y = P[1];
  double k1 = d[0], k2 = d[1], p1 = d[2], p2 = d[3], k3 = d[4];
  double r2 = x * x + y * y;
  double rdist = 1.0 + k1 * r2 + k2 * r2 * r2 + k3 * r2 * r2 * r2;
  out[0] = x * rdist + (2.0 * p1 * x * y + p2 * (r2 + 2.0 * x * x));
  out[1] = y * rdist + (p1 * (r2 + 2.0 * y * y) + 2.0 * p2 * x * y);
}

/* TsaiDistortionJacobian (LensDistortion.cc:286-324) */
static void tsai_jacobian(const double* P, const double* d, double* J) {
  double x = P[0];
  double y = P[1];
  double k1 = d[0], k2 = d[1], p1 = d[2], p2 = d[3], k3 = d[4];
  double r2 = x * x + y * y;
  double dr2dx = 2.0 * x;
  double dr2dy = 2.0 * y;
  double rdist = 1.0 + k1 * r2 + k2 * r2 * r2 + k3 * r2 * r2 * r2;
  J[0] = rdist + x * (k1 * dr2dx + k2 * dr2dx * 2.0 * r2 + k3 * dr2dx * 3.0 * r2 * r2) + 2.0 * p1 * y + p2 * (dr2dx + 4.0 * x);
  J[1] = x * (k1 * dr2dy + k2 * dr2dy * 2.0 * r2 + k3 * dr2dy * 3.0 * r2 * r2) + 2.0 * p1 * x + p2 * dr2dy;
  J[2] = y * (k1 * dr2dx + k2 * dr2dx * 2.0 * r2 + k3 * dr2dx * 3.0 * r2 * r2) + (p1 * dr2dx + 2.0 * p2 * y);
  J[3] = rdist + y * (k1 * dr2dy + k2 * dr2dy * 2.0 * r2 + k3 * dr2dy * 3.0 * r2 * r2) + p1 * (dr2dy + 4.0 * y) + 2.0 * p2 * x;
}

static double norm2v(const double* v) { double r = 0.0; r += v[0] * v[0]; r += v[1] * v[1]; return sqrt(r); }

/* NewtonRaphson::solve (NewtonRaphson.cc:58-119) with the Tsai function and Jacobian */
static void newton_raphson(const double* dist, const double* guess, const double* outY, double step, double tol, double* res, int* exit_code,
                           int* iters) {
  (void)step;
  double X[2] = {guess[0], guess[1]};
  double bestX[2] = {X[0], X[1]};
  double best_err = DBL_MAX;
  int count = 1, maxTries = 20;
  *iters = 0;
  while (count < maxTries) {
    ++*iters;
    double f[2], F[2];
    tsai_norm(X, dist, f);
    F[0] = f[0] - outY[0];
    F[1] = f[1] - outY[1];
    if (isnan(norm2v(F))) { res[0] = bestX[0]; res[1] = bestX[1]; *exit_code = 2; return; }
    if (norm2v(F) < best_err) {
      best_err = norm2v(F);
      bestX[0] = X[0]; bestX[1] = X[1];
    }
    double J[4];
    tsai_jacobian(X, dist, J);
    double det = J[0] * J[3] - J[1] * J[2];
    if (fabs(det) < 1e-6 || isnan(det)) { res[0] = bestX[0]; res[1] = bestX[1]; *exit_code = 1; return; }
    double DX[2];
    DX[0] = (J[3] * F[0] - J[1] * F[1]) / det;
    DX[1] = (J[0] * F[1] - J[2] * F[0]) / det;
    X[0] = X[0] - DX[0];
    X[1] = X[1] - DX[1];
    if (norm2v(DX) < tol) { res[0] = X[0]; res[1] = X[1]; *exit_code = 0; return; }
    count++;
  }
  res[0] = bestX[0]; res[1] = bestX[1];
  *exit_code = 3;
}

int vwt_tsai_undistort(const vwt_pinhole* cam, const double p[2], double out[2], int* exit_code, int* iters) {
  double focal[2] = {cam->fu, cam->fv}, offset[2] = {cam->cu, cam->cv};
  *iters = 0;
  if (focal[0] < 1e-300 || focal[1] < 1e-300) { out[0] = out[1] = HUGE_VAL; *exit_code = 4; return 0; }
  double p0[2] = {(p[0] - offset[0]) / focal[0], (p[1] - offset[1]) / focal[1]};
  double U[2];
  newton_raphson(cam->lens_params, p0, p0, 1e-6, 1e-9, U, exit_code, iters);
  out[0] = U[0] * focal[0] + offset[0];
  out[1] = U[1] * focal[1] + offset[1];
  return 0;
}

static int pixel_to_vector(const vwt_pinhole* cam, const double* inv, const double* pix, double* dir) {
  double u[2] = {pix[0] * cam->pixel_pitch, pix[1] * cam->pixel_pitch};
  if (cam->lens == 1) {
    double o[2];
    int ex, it;
    vwt_tsai_undistort(cam, u, o, &ex, &it);
    u[0] = o[0]; u[1] = o[1];
  }
  double p[3] = {u[0], u[1], 1};
  double r[3];
  for (int i = 0; i < 3; ++i) r[i] = dot3(inv + 3 * i, p);
  double n = norm3(r);
  for (int i = 0; i < 3; ++i) dir[i] = r[i] / n;
  return 0;
}

int vwt_pixel_to_vector(const vwt_pinhole* cam, const double pix[2], double dir[3]) {
  double inv[9];
  int rc = vwt_camera_inverse(cam, inv);
  if (rc) return rc;
  return pixel_to_vector(cam, inv, pix, dir);
}

static void cross3(const double* a, const double* b, double* r) {
  r[0] = a[1] * b[2] - a[2] * b[1];
  r[1] = a[2] * b[0] - a[0] * b[2];
  r[2] = a[0] * b[1] - a[1] * b[0];
}

/* StereoModel::operator()(pixVec, errorVec) for two cameras with their inverse transforms */
static void model_point(const vwt_pinhole* const* cams, const double* const* invs, double angle_tol, const double* const* pix, double* result,
                        double* errorVec) {
  errorVec[0] = errorVec[1] = errorVec[2] = 0.0;
  result[0] = result[1] = result[2] = 0.0;
  double dirs[2][3], ctrs[2][3];
  int n = 0;
  for (int p = 0; p < 2; ++p) {
    const double* px = pix[p];
    if (px[0] != px[0] || px[1] != px[1] || (px[0] == -1e8 && px[1] == -1e8)) continue;
    pixel_to_vector(cams[p], invs[p], px, dirs[n]);
    memcpy(ctrs[n], cams[p]->center, sizeof ctrs[n]);
    ++n;
  }
  if (n < 2) return;
  double tol = 1e-4;
  if (angle_tol > 0) tol = angle_tol;
  int are_par = 1;
  if (1 - dot3(dirs[0], dirs[1]) >= tol) are_par = 0;
  if (are_par) return;
  /* triangulate_pair (StereoModel.cc:35-48) */
  double v12[3], v1[3], v2[3], d10[3], d01[3], cp1[3], cp2[3];
  cross3(dirs[0], dirs[1], v12);
  cross3(v12, dirs[0], v1);
  cross3(v12, dirs[1], v2);
  for (int i = 0; i < 3; ++i) { d10[i] = ctrs[1][i] - ctrs[0][i]; d01[i] = ctrs[0][i] - ctrs[1][i]; }
  double s1 = dot3(v2, d10) / dot3(v2, dirs[0]);
  double s2 = dot3(v1, d01) / dot3(v1, dirs[1]);
  for (int i = 0; i < 3; ++i) { cp1[i] = ctrs[0][i] + s1 * dirs[0][i]; cp2[i] = ctrs[1][i] + s2 * dirs[1][i]; }
  for (int i = 0; i < 3; ++i) { errorVec[i] = cp1[i] - cp2[i]; result[i] = 0.5 * (cp1[i] + cp2[i]); }
  int reflect = 0;
  for (int p = 0; p < 2; ++p) {
    double d[3] = {result[0] - ctrs[p][0], result[1] - ctrs[p][1], result[2] - ctrs[p][2]};
    if (dot3(d, dirs[p]) < 0) reflect = 1;
  }
  if (reflect)
    for (int i = 0; i < 3; ++i) result[i] = -result[i] + 2 * ctrs[0][i];
}

static int open_cams(const vwt_pinhole* cam1, const vwt_pinhole* cam2, double* inv1, double* inv2) {
  int rc = vwt_camera_inverse(cam1, inv1);
  if (rc) return rc;
  return vwt_camera_inverse(cam2, inv2);
}

int vwt_triangulate(const vwt_pinhole* cam1, const vwt_pinhole* cam2, double angle_tol, const double pix1[2], const double pix2[2],
                    double xyz[3], double err[3]) {
  double inv1[9], inv2[9];
  int rc = open_cams(cam1, cam2, inv1, inv2);
  if (rc) return rc;
  const vwt_pinhole* cams[2] = {cam1, cam2};
  const double* invs[2] = {inv1, inv2};
  const double* pix[2] = {pix1, pix2};
  model_point(cams, invs, angle_tol, pix, xyz, err);
  return 0;
}

int vwt_stereo_triangulate(int type, const void* disp, int w, int h, int x0, int y0, int ow, int oh, const vwt_pinhole* cam1,
                           const vwt_pinhole* cam2, double angle_tol, double* xyz) {
  if (x0 < 0 || y0 < 0 || ow < 0 || oh < 0 || x0 + ow > w || y0 + oh > h || (type != 0 && type != 1)) return -1;
  double inv1[9], inv2[9];
  int rc = open_cams(cam1, cam2, inv1, inv2);
  if (rc) return rc;
  const vwt_pinhole* cams[2] = {cam1, cam2};
  const double* invs[2] = {inv1, inv2};
  for (int j = y0; j < y0 + oh; ++j)
    for (int i = x0; i < x0 + ow; ++i) {
      double* o = xyz + 3 * ((size_t)(j - y0) * ow + (i - x0));
      size_t k = 3 * ((size_t)j * w + i);
      int valid;
      double dx, dy;
      if (type == 0) {
        const int* d = (const int*)disp + k;
        valid = d[2] != 0; dx = (double)d[0]; dy = (double)d[1];
      } else {
        const float* d = (const float*)disp + k;
        valid = d[2] != 0; dx = (double)d[0]; dy = (double)d[1];
      }
      if (!valid) { o[0] = o[1] = o[2] = 0.0; continue; }
      double left[2] = {(double)i, (double)j};
      double right[2] = {left[0] + dx, left[1] + dy};
      const double* pix[2] = {left, right};
      double err[3];
      model_point(cams, invs, angle_tol, pix, o, err);
    }
  return 0;
}

int vwt_stereo_model(const float* disp, int w, int h, const vwt_pinhole* cam1, const vwt_pinhole* cam2, double angle_tol, double* xyz,
                     double* err, double stats[4]) {
  double inv1[9], inv2[9];
  int rc = open_cams(cam1, cam2, inv1, inv2);
  if (rc) return rc;
  const vwt_pinhole* cams[2] = {cam1, cam2};
  const double* invs[2] = {inv1, inv2};
  double mean_error = 0.0, max_error = 0.0;
  long long point_count = 0, divergent = 0;
  for (int y = 0; y < h; y++)
    for (int x = 0; x < w; x++) {
      const float* d = disp + 3 * ((size_t)y * w + x);
      double* o = xyz + 3 * ((size_t)y * w + x);
      double* e = err + (size_t)y * w + x;
      if (d[2] != 0) {
        double left[2] = {(double)x, (double)y};
        double right[2] = {(double)(x + d[0]), (double)(y + d[1])};       /* int32 + float, in float */
        const double* pix[2] = {left, right};
        double ev[3];
        model_point(cams, invs, angle_tol, pix, o, ev);
        *e = norm3(ev);
        if (*e >= 0) {
          if (*e > max_error) max_error = *e;
          mean_error += *e;
          ++point_count;
        } else {
          o[0] = o[1] = o[2] = 0.0;
          divergent++;
        }
      } else {
        o[0] = o[1] = o[2] = 0.0;
        *e = 0;
      }
    }
  stats[0] = (double)point_count;
  stats[1] = (double)divergent;
  stats[2] = max_error;
  stats[3] = mean_error;
  return 0;
}

int vwt_universe_radius(const double* in, int w, int h, const double origin[3], double near_r, double far_r, double* out, long long counts[2]) {
  if (!(near_r >= 0 && far_r >= 0)) return -1;
  if (!(near_r <= far_r)) return -1;
  counts[0] = counts[1] = 0;
  for (size_t k = 0; k < (size_t)w * h; ++k) {
    const double* p = in + 3 * k;
    double* o = out + 3 * k;
    double px[3] = {p[0], p[1], p[2]};
    counts[1]++;
    if (!(px[0] == 0 && px[1] == 0 && px[2] == 0)) {
      double d[3] = {px[0] - origin[0], px[1] - origin[1], px[2] - origin[2]};
      double dist = norm3(d);
      if ((near_r != 0 && dist < near_r) || (far_r != 0 && dist > far_r)) {
        counts[0]++;
        o[0] = o[1] = o[2] = 0.0;
      } else {
        o[0] = px[0]; o[1] = px[1]; o[2] = px[2];
      }
    } else {
      o[0] = o[1] = o[2] = 0.0;
    }
  }
  return 0;
}
