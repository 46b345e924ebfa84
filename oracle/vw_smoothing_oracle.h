/*
 * vw_smoothing_oracle.h -- CPU restatement ("oracle") of Vision Workbench's disparity smoothing filters
 * (Stereo/Algorithms.cc:26-67, Algorithms.h:144-281).  TEST INFRASTRUCTURE ONLY, like vw_oracle.h: the product
 * never links or calls it.  Built by oracle/smoothing.py into libvwsmoothing.so, which takes the separable convolution
 * of derivative_filter from libvworacle.so.
 *
 * The two disparity filters work IN PLACE and in raster order on d ({dx, dy, valid} float triples, pitch in pixels), as
 * the reference's shallow `disparity_out = disparity_in` makes them do.
 */
#ifndef VW_SMOOTHING_ORACLE_H
#define VW_SMOOTHING_ORACLE_H

#ifdef __cplusplus
extern "C" {
#endif

double vwo_destructive_median(double* v, int n);                    /* Math/Functors.h:393-398 (sorts v) */
int vwo_disparity_median_filter(float* d, int w, int h, int pitch, int kernel_size);
/* out is w x h, dense; kernel_size >= 1 */
int vwo_texture_measure(const float* img, int w, int h, int pitch, int kernel_size, double gradient_weight,
                        double stddev_weight, float* out);
int vwo_texture_preserving_disparity_filter(float* d, int w, int h, int pitch, const float* tex, int tpitch,
                                            float texture_max, int max_kernel_size);

#ifdef __cplusplus
}
#endif
#endif
