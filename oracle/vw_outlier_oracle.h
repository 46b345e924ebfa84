/* vw_outlier_oracle.h -- single-threaded C restatement of the neighbourhood outlier filters of Stereo/DisparityMap.h on
 * PixelMask<Vector2i> and PixelMask<Vector2f> disparities, written loop for loop from the reference (quirks kept):
 *   RmOutliersUsingThreshFunc (:318-387), RmOutliersUsingMeanFunc (:444-554), RmOutliersUsingStdDev (:600-724) and the
 *   composites rm_outliers_using_* / disparity_cleanup_using_* (:400-442, :567-598, :737-767).
 * Test infrastructure only. */
#ifndef VW_OUTLIER_ORACLE_H
#define VW_OUTLIER_ORACLE_H
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct { int32_t dx, dy, valid; } vwo_outi_t;
typedef struct { float dx, dy, valid; } vwo_outf_t;

/* method: 0 thresh, 1 mean, 2 stddev; cleanup: 0 rm_outliers_using_*, 1 disparity_cleanup_using_*; pixel_type: 0 int32,
 * 1 float.  in / out: dense w x h pixels, out separate from in.  Returns 0, -1 for a bad argument (half kernel <= 0,
 * unknown method or type), -2 when out of memory. */
int vwo_outlier_filter(int method, int cleanup, int pixel_type, const void* in, int w, int h, int half_h, int half_v,
                       double pixel_threshold, double rejection_threshold, double max_mean_diff, void* out);

#ifdef __cplusplus
}
#endif
#endif
