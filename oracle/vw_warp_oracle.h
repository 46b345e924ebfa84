/* vw_warp_oracle.h -- CPU oracle of transform(image, tx, edge, interp) (src/vw/Image/Transform.h:485-601) on a float image
 * (PixelGray<float>), written loop for loop from the reference (test infrastructure only):
 *   TransformView::operator() (:362-365)          -> tx.reverse(Vector2(i, j))
 *     kind 0: HomographyTransform::reverse with the matrix given (inverse(H))   (Math/Transform.h:377-381)
 *     kind 1: DisparityTransform::reverse on a PixelMask<Vector2f> disparity   (Stereo/DisparityMap.h:1170-1187)
 *   InterpolationView::operator() (:258)          -> interp 0 Bilinear, 1 Bicubic, 2 NearestPixel (Image/Interpolation.h:75-225)
 *   EdgeExtensionView                              -> edge 0 Zero, 1 Constant (Image/EdgeExtension.tcc:47-61, 89-94)
 * out (ow x oh, dense) pixel (i, j) is the TransformView pixel (x0 + i, y0 + j).  A reversed coordinate that is not finite
 * or has |c| >= 2^30 gives 0.0f (the reference converts it out of int32 range, which is undefined).  in and the disparity
 * ({dx, dy, valid} floats, may be NULL for kind 0) are dense row-major.  Built with the reference's -O3 -msse4.1
 * -ffp-contract=off. */
#ifndef VW_WARP_ORACLE_H
#define VW_WARP_ORACLE_H

void vww_transform(int kind, int interp, int edge, const double* m9, const float* in, int w, int h, const float* disp, int dw, int dh,
                   int x0, int y0, float* out, int ow, int oh);

#endif
