/* vw_dispmap_oracle.h -- CPU oracle of the disparity resampling, range and transform operations of
 * src/vw/Stereo/DisparityMap.h, written loop for loop from the reference (test infrastructure only):
 *   vwd_subsample     DisparitySubsampleView over ConstantEdgeExtension        (:1251-1322)
 *   vwd_upsample      DisparityUpsampleView                                    (:1324-1358)
 *   vwd_range         get_disparity_range, PixelAccumulator<EWMinMaxAccumulator> (:48-66, Image/Statistics.h:193-223)
 *   vwd_range_mask    DisparityRangeMaskFunc                                   (:255-300)
 *   vwd_transform     mode 0: TransformDisparitiesFunc with the matrix HomographyTransform::reverse applies (:1016-1057)
 *                     mode 1: transform_disparities(do_round, subregion, T, disparity)                   (:1190-1224)
 * Pixels are {dx, dy, valid} triples of int32 (type 0, PixelMask<Vector2i>) or float (type 1, PixelMask<Vector2f>), dense
 * row-major.  Created pixels get valid = 1, invalid ones {0, 0, 0} (the valid words of the engine); passed-through pixels
 * are copied.  Built with the reference's -O3 -msse4.1 -ffp-contract=off. */
#ifndef VW_DISPMAP_ORACLE_H
#define VW_DISPMAP_ORACLE_H
#include <stdint.h>

void vwd_subsample(int type, const void* in, int w, int h, void* out);
void vwd_upsample(int type, const void* in, int w, int h, void* out);
/* range: min dx, min dy, max dx, max dy; returns 1 when a pixel was valid, 0 (and zeros) otherwise */
int vwd_range(int type, const void* in, int w, int h, float* range);
/* min / max: two int32 or two floats */
void vwd_range_mask(int type, const void* in, int w, int h, const void* min, const void* max, void* out);
void vwd_transform(int type, int mode, const double* m9, int do_round, int sx0, int sy0, const void* in, int w, int h, void* out);

#endif
