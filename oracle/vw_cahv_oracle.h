/* vw_cahv_oracle.h -- CPU oracle of the CAHV and CAHVOR cameras, written loop for loop from the reference (test
 * infrastructure only):
 *   camera     CAHVModel::pixel_to_vector / point_to_pixel (Camera/CAHVModel.cc:167-185), CAHVORModel::pixel_to_vector /
 *              point_to_pixel without partial derivatives (CAHVORModel.cc:297-348, 431-448), epipolar(CAHV, CAHV)
 *              (CAHVModel.cc:297-337), linearize_camera (CAHVORModel.cc:460-547), CAHVModel = PinholeModel (CAHVModel.cc:64-99)
 *   transform  CameraTransform(src, dst)::reverse (Camera/CameraTransform.h:52-61) over a window; the interpolation stage is
 *              vww_sample / vww_sample_masked of vw_epipolar_oracle.c
 *   triangle   StereoView (form a) and StereoModel's image form (form b) (Stereo/StereoView.h:91-99, StereoModel.cc:35-147,
 *              254-309) with CAHV / CAHVOR rays
 * Cameras are vwc_cahv (the layout of vwb200_cahv).  Built with the reference's -O3 -msse4.1 and -ffp-contract=off. */
#ifndef VW_CAHV_ORACLE_H
#define VW_CAHV_ORACLE_H

#include "vw_epipolar_oracle.h"

typedef struct {
  int model;                                 /* 1 CAHV, 2 CAHVOR */
  double C[3], A[3], H[3], V[3], O[3], R[3];
} vwc_cahv;

/* pixel_to_vector(pix).  exit_code (CAHVOR): 0 |du| < 1e-6, 1 deriv <= 0, 2 the 20 passes ran out; -1 for CAHV.  iters:
 * the Newton passes (each computes poly and deriv). */
int vwc_pixel_to_vector(const vwc_cahv* cam, const double pix[2], double dir[3], int* exit_code, int* iters);
int vwc_point_to_pixel(const vwc_cahv* cam, const double point[3], double pix[2]);
/* epipolar(src0, src1, dst0, dst1): -1 unless both are CAHV */
int vwc_epipolar(const vwc_cahv* src0, const vwc_cahv* src1, vwc_cahv* dst0, vwc_cahv* dst1);
/* linearize_camera(cam, (ix, iy), (ox, oy)): -1 unless cam is CAHVOR */
int vwc_linearize(const vwc_cahv* cam, const int in_size[2], const int out_size[2], vwc_cahv* out);
/* CAHVModel = PinholeModel: -1 for a zero pixel pitch (ArgumentErr) or a lens, the pinhole's own codes otherwise */
int vwc_from_pinhole(const vwt_pinhole* pin, vwc_cahv* out);
/* reverse() of every pixel of the window (x0, y0, ow, oh) into coords (ow * oh pairs, row-major); -5 for different centers */
int vwc_camera_reverse_window(const vwc_cahv* src, const vwc_cahv* dst, int x0, int y0, int ow, int oh, double* coords);
/* form (a): as vwt_stereo_triangulate; iters (may be NULL) receives the Newton passes of both rays of every pixel whose two
 * pixels are usable (a pixel with one ray skipped is not triangulated, so its other ray is not counted) */
int vwc_stereo_triangulate(int type, const void* disp, int w, int h, int x0, int y0, int ow, int oh, const vwc_cahv* cam1, const vwc_cahv* cam2,
                           double angle_tol, double* xyz, long long* iters);
/* form (b): as vwt_stereo_model */
int vwc_stereo_model(const float* disp, int w, int h, const vwc_cahv* cam1, const vwc_cahv* cam2, double angle_tol, double* xyz, double* err,
                     double stats[4], long long* iters);

#endif
