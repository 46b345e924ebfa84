/* vw_triangulate_oracle.h -- CPU oracle of dense two-camera triangulation through pinhole cameras, written loop for loop from
 * the reference (test infrastructure only):
 *   camera     PinholeModel::rebuild_camera_matrix (Camera/PinholeModel.cc:553-605): the u, v, w orthonormality asserts, and
 *              inv = inverse(uvw * transpose(R)) * inverse(K) with vw::math::inverse (Math/Matrix.h:2218-2281, LU with partial
 *              pivoting) and dot_prod products (Math/Vector.h:1717-1726)
 *   ray        PinholeModel::pixel_to_vector (:422-430): undistort pix * pixel_pitch (NULL: identity; TSAI:
 *              Camera/LensDistortion.cc:258-400 through math::NewtonRaphson::solve, Math/NewtonRaphson.cc:58-119), then
 *              normalize(inv * (u, v, 1))
 *   point      StereoModel::operator()(pix1, pix2, errorVec) (Stereo/StereoModel.cc:35-48, 68-91, 97-147)
 *   form (a)   StereoView::operator() (Stereo/StereoView.h:91-99) over a window
 *   form (b)   StereoModel::operator()(ImageView<PixelMask<Vector2f>>, ImageView<double>&) (StereoModel.cc:254-309)
 *   radius     UniverseRadiusFunc::operator()(Vector3) (StereoView.h:172-186)
 * Built with the reference's -O3 -msse4.1 and -ffp-contract=off. */
#ifndef VW_TRIANGULATE_ORACLE_H
#define VW_TRIANGULATE_ORACLE_H

/* the layout of vwb200_pinhole (include/vwb200.h) */
typedef struct {
  double center[3];
  double rotation[9];
  double fu, fv, cu, cv;
  double u_direction[3], v_direction[3], w_direction[3];
  double pixel_pitch;
  int lens;                 /* 0 NULL, 1 TSAI */
  int num_lens_params;
  double lens_params[5];    /* k1, k2, p1, p2, k3 */
} vwt_pinhole;

/* Return codes: 0, -1 bad argument, -2 singular matrix (MathErr), -3 u, v, w not orthonormal (LogicErr). */

/* m_inv_camera_transform, row-major */
int vwt_camera_inverse(const vwt_pinhole* cam, double inv[9]);
/* vw::math::inverse of a row-major 3 x 3 matrix */
int vwt_inverse3(const double m[9], double inv[9]);
/* TsaiLensDistortion::undistorted_coordinates of p (already times pixel_pitch); exit: 0 converged (|DX| < tol), 1 |det| < 1e-6
 * or NaN det, 2 NaN |F|, 3 the 19 iterations ran out, 4 fu or fv < 1e-300; iters: the loop passes */
int vwt_tsai_undistort(const vwt_pinhole* cam, const double p[2], double out[2], int* exit_code, int* iters);
/* pixel_to_vector(pix) */
int vwt_pixel_to_vector(const vwt_pinhole* cam, const double pix[2], double dir[3]);
/* StereoModel(cam1, cam2, angle_tol)(pix1, pix2, errorVec) */
int vwt_triangulate(const vwt_pinhole* cam1, const vwt_pinhole* cam2, double angle_tol, const double pix1[2], const double pix2[2],
                    double xyz[3], double err[3]);
/* form (a): type 0 int32 / 1 float {dx, dy, valid} w x h dense disparity, window (x0, y0, ow, oh); xyz: ow * oh * 3 doubles */
int vwt_stereo_triangulate(int type, const void* disp, int w, int h, int x0, int y0, int ow, int oh, const vwt_pinhole* cam1,
                           const vwt_pinhole* cam2, double angle_tol, double* xyz);
/* form (b): xyz w * h * 3, err w * h; stats: points, divergent, max error, error sum (raster order) */
int vwt_stereo_model(const float* disp, int w, int h, const vwt_pinhole* cam1, const vwt_pinhole* cam2, double angle_tol, double* xyz,
                     double* err, double stats[4]);
/* UniverseRadiusFunc(origin, near, far) over w * h points; counts: rejected, total.  -1 for the reference's radius asserts. */
int vwt_universe_radius(const double* in, int w, int h, const double origin[3], double near_r, double far_r, double* out, long long counts[2]);

#endif
