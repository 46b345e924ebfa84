/* vw_cahv_oracle.c -- see vw_cahv_oracle.h.  It includes vw_epipolar_oracle.c (and through it the triangulation and warp
 * oracles) so that libvwcahv.so carries their entry points too, the interpolation stage and the pinhole camera included. */
#include "vw_epipolar_oracle.c"
#include "vw_cahv_oracle.h"

static int left_handed(const vwc_cahv* c) {
  double t[3];
  cross3(c->V, c->H, t);
  return dot3(t, c->A) < 0;
}

static void normalize3(const double* a, double* r) {
  double n = norm3(a);
  for (int i = 0; i < 3; ++i) r[i] = a[i] / n;
}

int vwc_pixel_to_vector(const vwc_cahv* c, const double pix[2], double dir[3], int* exit_code, int* iters) {
  if (c->model != 1 && c->model != 2) return -1;
  double f[3], g[3], t[3], rr[3];
  for (int i = 0; i < 3; ++i) { f[i] = c->V[i] - pix[1] * c->A[i]; g[i] = c->H[i] - pix[0] * c->A[i]; }
  cross3(f, g, t);
  normalize3(t, rr);
  if (left_handed(c))
    for (int i = 0; i < 3; ++i) rr[i] *= -1.0;
  if (exit_code) *exit_code = -1;
  if (c->model == 1) { memcpy(dir, rr, sizeof rr); return 0; }
  double omega = dot3(rr, c->O), lambda[3];
  for (int i = 0; i < 3; ++i) lambda[i] = rr[i] - omega * c->O[i];
  const double tau = dot3(lambda, lambda) / (omega * omega);
  const double k1 = 1 + c->R[0];
  const double k3 = c->R[1] * tau;
  const double k5 = c->R[2] * tau * tau;
  double u = 1.0 - (c->R[0] + k3 + k5);
  double du, poly, deriv;
  int code = 2;
  for (int i = 0;; i++) {
    if (i >= 20) break;
    if (iters) ++*iters;
    double u_2 = u * u;
    poly = ((k5 * u_2 + k3) * u_2 + k1) * u - 1;
    deriv = (5 * k5 * u_2 + 3 * k3) * u_2 + k1;
    if (deriv <= 0) { code = 1; break; }
    du = poly / deriv;
    u -= du;
    if (fabs(du) < 1.0e-6) { code = 0; break; }
  }
  if (exit_code) *exit_code = code;
  for (int i = 0; i < 3; ++i) t[i] = rr[i] - (1 - u) * lambda[i];
  normalize3(t, dir);
  return 0;
}

int vwc_point_to_pixel(const vwc_cahv* c, const double point[3], double pix[2]) {
  if (c->model != 1 && c->model != 2) return -1;
  double v[3];
  for (int i = 0; i < 3; ++i) v[i] = point[i] - c->C[i];
  if (c->model == 2) {
    double omega = dot3(v, c->O), lambda[3];
    for (int i = 0; i < 3; ++i) lambda[i] = v[i] - omega * c->O[i];
    double tau = dot3(lambda, lambda) / (omega * omega);
    double mu = c->R[0] + (c->R[1] * tau) + (c->R[2] * tau * tau);
    for (int i = 0; i < 3; ++i) v[i] = v[i] + mu * lambda[i];
  }
  double alpha = dot3(v, c->A);
  pix[0] = dot3(v, c->H) / alpha;
  pix[1] = dot3(v, c->V) / alpha;
  return 0;
}

int vwc_epipolar(const vwc_cahv* s0, const vwc_cahv* s1, vwc_cahv* d0, vwc_cahv* d1) {
  if (s0->model != 1 || s1->model != 1) return -1;
  double t[3];
  double hc = dot3(s0->H, s0->A) / 2.0 + dot3(s1->H, s1->A) / 2.0;
  double vc = dot3(s0->V, s0->A) / 2.0 + dot3(s1->V, s1->A) / 2.0;
  double n0, n1;
  cross3(s0->A, s0->H, t); n0 = norm3(t);
  cross3(s1->A, s1->H, t); n1 = norm3(t);
  double hs = n0 / 2.0 + n1 / 2.0;
  cross3(s0->A, s0->V, t); n0 = norm3(t);
  cross3(s1->A, s1->V, t); n1 = norm3(t);
  double vs = n0 / 2.0 + n1 / 2.0;
  double app[3], dc[3], f[3], hp[3], g[3], a[3], vp[3];
  for (int i = 0; i < 3; ++i) { app[i] = s0->A[i] + s1->A[i]; dc[i] = s1->C[i] - s0->C[i]; }
  cross3(app, dc, t);
  cross3(t, app, f);
  if (dot3(f, s0->H) > 0)
    for (int i = 0; i < 3; ++i) hp[i] = f[i] * hs / norm3(f);
  else
    for (int i = 0; i < 3; ++i) hp[i] = -f[i] * hs / norm3(f);
  for (int i = 0; i < 3; ++i) app[i] *= 0.5;
  for (int i = 0; i < 3; ++i) g[i] = hp[i] * dot3(app, hp) / (hs * hs);
  for (int i = 0; i < 3; ++i) t[i] = app[i] - g[i];
  normalize3(t, a);
  cross3(a, hp, t);
  for (int i = 0; i < 3; ++i) vp[i] = t[i] * vs / hs;
  vwc_cahv e;
  memset(&e, 0, sizeof e);
  e.model = 1;
  for (int i = 0; i < 3; ++i) { e.A[i] = a[i]; e.H[i] = hp[i] + hc * a[i]; e.V[i] = vp[i] + vc * a[i]; }
  vwc_cahv e1 = e;
  memcpy(e.C, s0->C, sizeof e.C);
  memcpy(e1.C, s1->C, sizeof e1.C);
  *d0 = e;
  *d1 = e1;
  return 0;
}

int vwc_linearize(const vwc_cahv* cam, const int in_size[2], const int out_size[2], vwc_cahv* out) {
  if (cam->model != 2) return -1;
  vwc_cahv c = *cam, o;
  memset(&o, 0, sizeof o);
  o.model = 1;
  memcpy(o.C, c.C, sizeof o.C);
  const int ix = in_size[0], iy = in_size[1];
  double hpts[6][2] = {{0, 0}, {0, (iy - 1) / 2.0}, {0, iy - 1}, {ix - 1, 0}, {ix - 1, (iy - 1) / 2.0}, {ix - 1.0, iy - 1.0}};
  double vpts[6][2] = {{0, 0}, {(ix - 1) / 2.0, 0}, {ix - 1, 0}, {0, iy - 1}, {(ix - 1) / 2, iy - 1}, {ix - 1.0, iy - 1.0}};
  double r[3], t[3], dn[3], rt[3];
  for (int k = 0; k < 6; ++k) { vwc_pixel_to_vector(&c, vpts[k], r, NULL, NULL); for (int i = 0; i < 3; ++i) o.A[i] += r[i]; }
  for (int k = 0; k < 6; ++k) { vwc_pixel_to_vector(&c, hpts[k], r, NULL, NULL); for (int i = 0; i < 3; ++i) o.A[i] += r[i]; }
  memcpy(t, o.A, sizeof t);
  normalize3(t, o.A);
  cross3(c.A, c.H, dn);
  cross3(dn, c.A, t);
  normalize3(t, rt);
  memcpy(t, dn, sizeof t);
  normalize3(t, dn);
  cross3(dn, o.A, rt);
  cross3(o.A, rt, t);
  normalize3(t, dn);
  memcpy(t, rt, sizeof t);
  normalize3(t, rt);
  double hmin = 1, hmax = -1, vmin = 1, vmax = -1;
  for (int k = 0; k < 6; ++k) {
    double u3[3], w3[3], d;
    vwc_pixel_to_vector(&c, hpts[k], u3, NULL, NULL);
    d = dot3(dn, u3);
    for (int i = 0; i < 3; ++i) t[i] = u3[i] - d * dn[i];
    normalize3(t, w3);
    cross3(o.A, w3, t);
    double sn = norm3(t);
    if (hmin > sn) hmin = sn;
    if (hmax < sn) hmax = sn;
  }
  for (int k = 0; k < 6; ++k) {
    double u3[3], w3[3], d;
    vwc_pixel_to_vector(&c, vpts[k], u3, NULL, NULL);
    d = dot3(rt, u3);
    for (int i = 0; i < 3; ++i) t[i] = u3[i] - d * rt[i];
    normalize3(t, w3);
    cross3(o.A, w3, t);
    double sn = norm3(t);
    if (vmin > sn) vmin = sn;
    if (vmax < sn) vmax = sn;
  }
  double ic[2] = {(out_size[0] - 1.0) / 2.0, (out_size[1] - 1.0) / 2.0};
  double ic2[2] = {ic[0] * ic[0], ic[1] * ic[1]};
  double sf[2] = {sqrt(ic2[0] / (hmin * hmin) - ic2[0]), sqrt(ic2[1] / (vmin * vmin) - ic2[1])};
  for (int i = 0; i < 3; ++i) {
    o.H[i] = sf[0] * rt[i] + ic[0] * o.A[i];
    o.V[i] = sf[1] * dn[i] + ic[1] * o.A[i];
  }
  *out = o;
  return 0;
}

int vwc_from_pinhole(const vwt_pinhole* p, vwc_cahv* out) {
  double inv[9];
  int rc = vwt_camera_inverse(p, inv);
  if (rc) return rc;
  if (p->lens != 0 || p->pixel_pitch == 0) return -1;
  double pitch = p->pixel_pitch;
  double fH = p->fu / pitch, fV = p->fv / pitch, cH = p->cu / pitch, cV = p->cv / pitch;
  double Hv[3], Vv[3], A[3];
  for (int i = 0; i < 3; ++i) {
    Hv[i] = dot3(p->rotation + 3 * i, p->u_direction);
    Vv[i] = dot3(p->rotation + 3 * i, p->v_direction);
    A[i] = dot3(p->rotation + 3 * i, p->w_direction);
  }
  memset(out, 0, sizeof *out);
  out->model = 1;
  for (int i = 0; i < 3; ++i) {
    out->C[i] = p->center[i];
    out->A[i] = A[i];
    out->H[i] = fH * Hv[i] + cH * A[i];
    out->V[i] = fV * Vv[i] + cV * A[i];
  }
  return 0;
}

int vwc_camera_reverse_window(const vwc_cahv* src, const vwc_cahv* dst, int x0, int y0, int ow, int oh, double* coords) {
  if (!(src->C[0] == dst->C[0] && src->C[1] == dst->C[1] && src->C[2] == dst->C[2])) return -5;
  for (int j = 0; j < oh; ++j)
    for (int i = 0; i < ow; ++i) {
      double p[2] = {(double)(x0 + i), (double)(y0 + j)}, v[3], pt[3];
      vwc_pixel_to_vector(dst, p, v, NULL, NULL);
      for (int k = 0; k < 3; ++k) pt[k] = v[k] + dst->C[k];
      vwc_point_to_pixel(src, pt, coords + 2 * ((size_t)j * ow + i));
    }
  return 0;
}

/* StereoModel::operator()(pixVec, errorVec) with CAHV / CAHVOR rays */
static void cahv_model_point(const vwc_cahv* const* cams, double angle_tol, const double* const* pix, double* result, double* errorVec,
                             long long* iters) {
  errorVec[0] = errorVec[1] = errorVec[2] = 0.0;
  result[0] = result[1] = result[2] = 0.0;
  double dirs[2][3], ctrs[2][3];
  int n = 0, it = 0;
  for (int p = 0; p < 2; ++p) {
    const double* px = pix[p];
    if (px[0] != px[0] || px[1] != px[1] || (px[0] == -1e8 && px[1] == -1e8)) continue;
    vwc_pixel_to_vector(cams[p], px, dirs[n], NULL, &it);
    memcpy(ctrs[n], cams[p]->C, sizeof ctrs[n]);
    ++n;
  }
  if (n < 2) return;
  if (iters) *iters += it;                   /* the passes of both rays of a pixel that is triangulated */
  double tol = 1e-4;
  if (angle_tol > 0) tol = angle_tol;
  if (!(1 - dot3(dirs[0], dirs[1]) >= tol)) return;
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

int vwc_stereo_triangulate(int type, const void* disp, int w, int h, int x0, int y0, int ow, int oh, const vwc_cahv* cam1, const vwc_cahv* cam2,
                           double angle_tol, double* xyz, long long* iters) {
  if (x0 < 0 || y0 < 0 || ow < 0 || oh < 0 || x0 + ow > w || y0 + oh > h || (type != 0 && type != 1)) return -1;
  const vwc_cahv* cams[2] = {cam1, cam2};
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
      cahv_model_point(cams, angle_tol, pix, o, err, iters);
    }
  return 0;
}

int vwc_stereo_model(const float* disp, int w, int h, const vwc_cahv* cam1, const vwc_cahv* cam2, double angle_tol, double* xyz, double* err,
                     double stats[4], long long* iters) {
  const vwc_cahv* cams[2] = {cam1, cam2};
  double mean_error = 0.0, max_error = 0.0;
  long long point_count = 0, divergent = 0;
  for (int y = 0; y < h; y++)
    for (int x = 0; x < w; x++) {
      const float* d = disp + 3 * ((size_t)y * w + x);
      double* o = xyz + 3 * ((size_t)y * w + x);
      double* e = err + (size_t)y * w + x;
      if (d[2] != 0) {
        double left[2] = {(double)x, (double)y};
        double right[2] = {(double)(x + d[0]), (double)(y + d[1])};
        const double* pix[2] = {left, right};
        double ev[3];
        cahv_model_point(cams, angle_tol, pix, o, ev, iters);
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
