/* vw_ipfind_oracle.h -- CPU oracle of ipfind's default path (tools/ipfind.cc:253-401 with --interest-operator iagd and the
 * sgrad descriptor): normalize, IntegralAutoGainDetector through detect_interest_points, remove_ip_near_nodata and
 * SGradDescriptorGenerator through describe_interest_points.  Test infrastructure only; built with -ffp-contract=off. */
#pragma once
#include <stdint.h>

/* one interest point: the fields of vw::ip::InterestPoint the path reads or writes */
typedef struct { float x, y; int32_t ix, iy; float scale, interest, orientation; } vwf_point;

#define VWF_DESC 180
#define VWF_EARG (-1)   /* NaN / inf input, no valid pixel, a point outside the image's tiles */

/* normalize(image) or apply_mask(normalize(create_mask(image, nodata))) into out (w * h floats) */
int vwf_normalize(const float* in, int w, int h, int has_nodata, double nodata, float* out);
/* generate_gaussian_kernel(k, 2, 9) */
void vwf_gaussian_taps(double* k9);
/* detect_interest_points(image, IntegralAutoGainDetector(ip_per_tile), ip_per_tile) with default_tile_size tile_size.
 * *out is malloc'ed (vwf_free); stats5: tiles, raw extrema, kept after the thresholds, culled tiles, 0 */
int vwf_detect(const float* img, int w, int h, int tile_size, int ip_per_tile, vwf_point** out, long long* n, long long* stats5);
/* remove_ip_near_nodata(raw, nodata, list, radius) in place; returns the new count */
long long vwf_remove_near_nodata(const float* raw, int w, int h, double nodata, int radius, vwf_point* pts, long long n);
/* describe_interest_points(image, SGradDescriptorGenerator, list): reorders pts as std::partition does, writes the
 * descriptors (n * 180, in the new order) and the points' x / y as the crop round trip leaves them */
int vwf_describe(const float* img, int w, int h, int tile_size, vwf_point* pts, long long n, float* desc);
void vwf_free(void* p);
/* IntegralImage ((w+1) x (h+1)) and box_filter(integral, filter) of a w x h image, for the reference's unit-test pins */
void vwf_integral(const float* src, int w, int h, float* I);
void vwf_box_filter(const float* I, int w, int h, int nb, const int* sx, const int* sy, const int* bw, const int* bh, const float* wt,
                    float* out);
