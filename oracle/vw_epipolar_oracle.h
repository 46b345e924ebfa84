/* vw_epipolar_oracle.h -- CPU oracle of epipolar rectification of pinhole stereo pairs, written loop for loop from the reference
 * (test infrastructure only):
 *   epipolar   Quaternion(R).rotation_matrix() (Math/Quaternion.h:211-252, 314-335), epipolar() (Camera/PinholeModel.cc:679-732),
 *              m_camera_matrix (:553-605), point_to_pixel with its check (:351-397, Camera/LensDistortion.cc:345-369),
 *              CameraTransform forward / reverse (Camera/CameraTransform.h:52-74), compute_transformed_bbox_fast with BBox2f
 *              (Image/Transform.h:271-315, Math/BBox.tcc:38-97) and resize_epipolar_cameras_to_fit (Camera/EpipolarUtils.cc:37-76)
 *   sampling   the interpolation stage of camera_transform at given reversed coordinates, for PixelGray<float> (the
 *              interpolations and edges of vw_warp_oracle.c) and PixelMask<float> (bilinear, Image/Interpolation.h:75-110 on the
 *              PixelMask arithmetic of Image/PixelMask.h:321-626, zero / constant / value edges)
 * Cameras are vwt_pinhole (vw_triangulate_oracle.h).  Return codes: those of vw_triangulate_oracle.h, and -4 point_to_pixel's
 * check failed (PointToPixelErr), -5 a camera transform between cameras at different centers (LogicErr).  Built with the
 * reference's -O3 -msse4.1 and -ffp-contract=off. */
#ifndef VW_EPIPOLAR_ORACLE_H
#define VW_EPIPOLAR_ORACLE_H

#include "vw_triangulate_oracle.h"

/* the rotation of camera_pose(): returns the branch taken (0 ww, 1 xx, 2 yy, 3 zz); quat (may be NULL) receives w, x, y, z */
int vwt_quaternion_round_trip(const double R[9], double out[9], double quat[4]);
/* epipolar(src0, src1, dst0, dst1) */
int vwt_epipolar(const vwt_pinhole* src0, const vwt_pinhole* src1, vwt_pinhole* dst0, vwt_pinhole* dst1);
/* m_camera_matrix, row-major 3 x 4 */
int vwt_camera_matrix(const vwt_pinhole* cam, double P[12]);
/* point_to_pixel(point): pix is written also when the check fails (-4) */
int vwt_point_to_pixel(const vwt_pinhole* cam, const double point[3], double pix[2]);
/* CameraTransform(src, dst): forward (reverse == 0) or reverse of p */
int vwt_camera_transform_point(const vwt_pinhole* src, const vwt_pinhole* dst, int reverse, const double p[2], double out[2]);
/* reverse() of every pixel of the window (x0, y0, ow, oh) into coords (ow * oh pairs, row-major); -4 with *first_fail the
 * first failing row-major index (every pixel is still mapped) */
int vwt_camera_reverse_window(const vwt_pinhole* src, const vwt_pinhole* dst, int x0, int y0, int ow, int oh, double* coords,
                              long long* first_fail);
/* compute_transformed_bbox_fast(roi, CameraTransform(src, dst)): bbox {min x, min y, max x, max y}; -4 with *fail_k the
 * failing perimeter index */
int vwt_transformed_bbox_fast(const vwt_pinhole* src, const vwt_pinhole* dst, const int roi[4], float bbox[4], long long* fail_k);
/* resize_epipolar_cameras_to_fit: epi1, epi2 updated in place, sizes (width, height); -4 with the failing camera and index */
int vwt_resize_epipolar(const vwt_pinhole* cam1, const vwt_pinhole* cam2, vwt_pinhole* epi1, vwt_pinhole* epi2, const int roi1[4],
                        const int roi2[4], int size1[2], int size2[2], long long* fail_k, int* fail_cam);

/* The interpolation stage alone at n given reversed coordinates (x, y pairs): out[k] as vww_transform would give it for a
 * transform whose reverse() returned coords[k]; interp 0 bilinear, 1 bicubic, 2 nearest; edge 0 zero, 1 constant. */
void vww_sample(int interp, int edge, const float* in, int w, int h, const double* coords, long long n, float* out);
/* The same for PixelMask<float> {value, valid} images under bilinear interpolation with edge 0 Zero ({0, 0}), 1 Constant or
 * 2 ValueEdgeExtension(edge_value {value, valid}) (Image/EdgeExtension.h:66-76); out holds n {value, valid} pairs, {0, 0}
 * outside the domain. */
void vww_sample_masked(int edge, const float* edge_value, const float* in, int w, int h, const double* coords, long long n, float* out);

#endif
