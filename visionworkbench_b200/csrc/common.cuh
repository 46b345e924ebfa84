// common.cuh -- shared declarations for the vwb200 engine (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stddef.h>
#include <cstring>
#include <string>
#include <atomic>
#include <vector>
#include <algorithm>
#include "../../include/vwb200.h"

namespace vwb200 {

// SMs of the H100 SXM: persistent grids, their wave shaping and the per-CTA scratch carved for them are sized for it.
static constexpr int kNumSMs = 132;

// ---- error plumbing ---------------------------------------------------------------------
void set_error(const char* fmt, ...);
extern std::atomic<long long> g_launches;

#define VWB_CUDA(expr)                                                                      \
  do {                                                                                      \
    cudaError_t _e = (expr);                                                                \
    if (_e != cudaSuccess) {                                                                \
      ::vwb200::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e), __FILE__, __LINE__); \
      return VWB200_ECUDA;                                                                  \
    }                                                                                       \
  } while (0)

#define VWB_TRY(expr)                        \
  do {                                       \
    int _rc = (expr);                        \
    if (_rc != VWB200_OK) return _rc;        \
  } while (0)

#define VWB_LAUNCH_CHECK()                                                                  \
  do {                                                                                      \
    ::vwb200::g_launches.fetch_add(1, std::memory_order_relaxed);                           \
    cudaError_t _e = cudaGetLastError();                                                    \
    if (_e != cudaSuccess) {                                                                \
      ::vwb200::set_error("kernel launch failed: %s (%s:%d)", cudaGetErrorString(_e), __FILE__, __LINE__); \
      return VWB200_ECUDA;                                                                  \
    }                                                                                       \
  } while (0)

int ensure_device();   // VWB200_ENODEVICE when there is no CUDA device

// stream-ordered device buffers owned by one call
struct Arena {
  cudaStream_t st;
  std::vector<void*> ptrs;
  explicit Arena(cudaStream_t s) : st(s) {}
  ~Arena() { for (void* p : ptrs) cudaFreeAsync(p, st); }
  template <class T> int alloc(T** out, size_t n) {
    void* p = nullptr;
    cudaError_t e = cudaMallocAsync(&p, std::max<size_t>(n, 1) * sizeof(T), st);
    if (e != cudaSuccess) { set_error("cudaMallocAsync(%zu bytes) failed: %s", n * sizeof(T), cudaGetErrorString(e)); return VWB200_ENOMEM; }
    ptrs.push_back(p);
    *out = static_cast<T*>(p);
    return VWB200_OK;
  }
};

// an owned-or-borrowed stream
struct StreamGuard {
  cudaStream_t st = nullptr; bool own = false;
  // device-resident inputs are produced on the caller's stream: a NULL stream then means the legacy default stream
  // (which is what e.g. torch's default stream is), never a private one -- otherwise the kernels could start before the
  // producer of their inputs has finished.  Host-resident calls with no stream get a private non-blocking stream.
  int init(void* user, int device_resident = 0) {
    if (user) { st = static_cast<cudaStream_t>(user); return VWB200_OK; }
    if (device_resident) { st = cudaStreamLegacy; return VWB200_OK; }
    VWB_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    own = true;
    return VWB200_OK;
  }
  ~StreamGuard() { if (own && st) cudaStreamDestroy(st); }
};

// One call of the C ABI: its stream, its stream-ordered scratch, and the moves of the caller's rasters between the host and
// HBM.  Widths and pitches count elements of T (a float triple is 3 floats, a search box 4 int32).  finish() copies the
// staged outputs back and synchronises the stream: every call returns with its work done, device-resident calls included.
struct AbiCall {
  StreamGuard sg;
  Arena ar{nullptr};
  cudaStream_t st = nullptr;
  struct CopyBack { void* dst; size_t dpitch; const void* src; size_t row; int h; cudaMemcpyKind kind; const int* unless; };
  std::vector<CopyBack> backs;

  int open(void* stream, int device_resident) {
    VWB_TRY(sg.init(stream, device_resident));
    st = ar.st = sg.st;
    return VWB200_OK;
  }
  // an input: the caller's device raster, or a dense HBM copy of the host raster
  template <class T> int in(const T* src, int w, int h, ptrdiff_t pitch, int on_device, const T** dev, ptrdiff_t* dpitch) {
    if (on_device) { *dev = src; *dpitch = pitch; return VWB200_OK; }
    T* d;
    VWB_TRY(ar.alloc(&d, (size_t)w * h));
    VWB_CUDA(cudaMemcpy2DAsync(d, (size_t)w * sizeof(T), src, (size_t)pitch * sizeof(T), (size_t)w * sizeof(T), h, cudaMemcpyHostToDevice, st));
    *dev = d; *dpitch = w;
    return VWB200_OK;
  }
  // an output `user` (may be NULL: scratch only): the caller's device raster itself -- when `dense` asks for it, only if its
  // pitch is w -- or a dense HBM buffer that finish() copies to `user`, w elements per row so that the pitch padding is never
  // written, unless *unless is set by then.  The buffer starts as a copy of `init` (an in-out raster passes itself), which
  // lives where the call's inputs live.
  template <class T> int out(T* user, int w, int h, ptrdiff_t pitch, int on_device, T** dev, ptrdiff_t* dpitch, const T* init = nullptr,
                             ptrdiff_t ipitch = 0, bool dense = false, const int* unless = nullptr) {
    if (on_device && user && (!init || init == user) && (!dense || pitch == w)) { *dev = user; *dpitch = pitch; return VWB200_OK; }
    VWB_TRY(ar.alloc(dev, (size_t)w * h));
    *dpitch = w;
    const size_t row = (size_t)w * sizeof(T);
    if (init)
      VWB_CUDA(cudaMemcpy2DAsync(*dev, row, init, (size_t)ipitch * sizeof(T), row, h, on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyHostToDevice, st));
    if (user) backs.push_back(CopyBack{user, (size_t)pitch * sizeof(T), *dev, row, h, on_device ? cudaMemcpyDeviceToDevice : cudaMemcpyDeviceToHost, unless});
    return VWB200_OK;
  }
  int finish() {
    for (const CopyBack& b : backs)
      if (!b.unless || !*b.unless) VWB_CUDA(cudaMemcpy2DAsync(b.dst, b.dpitch, b.src, b.row, b.row, b.h, b.kind, st));
    VWB_CUDA(cudaStreamSynchronize(st));
    return VWB200_OK;
  }
};

// [a0, a1) and [b0, b1): the bytes of an w x h / ow x oh raster of `apx` / `bpx`-byte pixels (disparity pixels by default)
inline bool rasters_overlap(const void* a, int w, int h, ptrdiff_t ap, const void* b, int ow, int oh, ptrdiff_t bp, size_t apx = 12,
                            size_t bpx = 12) {
  if (w <= 0 || h <= 0 || ow <= 0 || oh <= 0) return false;
  const uintptr_t a0 = (uintptr_t)a, a1 = a0 + ((size_t)(h - 1) * ap + w) * apx;
  const uintptr_t b0 = (uintptr_t)b, b1 = b0 + ((size_t)(oh - 1) * bp + ow) * bpx;
  return a0 < b1 && b0 < a1;
}

// ---- order-preserving keys of floats (median select, outlier cutoff, bounding boxes) -----------------------------
// -0.0 sorts just below +0.0; NaN is outside the contract
__host__ __device__ __forceinline__ unsigned fkey(float f) {
#ifdef __CUDA_ARCH__
  const unsigned u = __float_as_uint(f);
#else
  unsigned u;
  std::memcpy(&u, &f, sizeof u);
#endif
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__host__ __device__ __forceinline__ float kfloat(unsigned k) {
  const unsigned u = (k & 0x80000000u) ? (k & 0x7FFFFFFFu) : ~k;
#ifdef __CUDA_ARCH__
  return __uint_as_float(u);
#else
  float f;
  std::memcpy(&f, &u, sizeof f);
  return f;
#endif
}

// ---- image descriptors (device pointers) ------------------------------------------------------
// float disparity pixel {dx, dy, valid} (PixelMask<Vector2f>); vwb200_dispi is the integer one
struct DispF { float dx, dy, valid; };
struct ImgF { const float* p; int w, h; ptrdiff_t pitch; };
struct ImgB { const uint8_t* p; int w, h; ptrdiff_t pitch; };

// A zone of the level loop (Stereo/CorrelationView.cc:607-648) or a whole calc_disparity call.
struct Zone {
  long long obase;   // element offset of the zone's output (0,0) in the output buffer
  int opitch;        // output row pitch (elements)
  int w, h;          // output size
  int lx, ly;        // left_region.min  (kernel-padded) in left image coordinates
  int rx, ry;        // right_region.min in right image coordinates
  int sx, sy;        // search volume
  int addx, addy;    // constant added to the children by the K1 epilogue (R->L pass: -search size)
  int nchunks;       // > 1: the disparity range is split over several CTAs (K1G_DCHUNK disparities each)
  int pad0;
  long long sbase;   // element offset of this zone's partial results in the scratch planes [chunk][h][w]
};
// One unit of work of the generic kernel: a TW x TH tile of a zone (x one chunk of its disparity range).
struct Tile { int zone; int tx, ty; int chunk; };

// ---- K1 generic (fp64, any float input, zones) --------------------------------------------
// cost: VWB200_* cost type.  inv_l / inv_r: for NCC, 1/boxsum(v^2) maps whose (0,0) sits at window
// origin (l_ox,l_oy) / (r_ox,r_oy) in image coordinates, pitch in elements.
struct NccMaps { const double* inv_l; int l_ox, l_oy, l_w, l_h; const double* inv_r; int r_ox, r_oy, r_w, r_h; };
// optional event pair recorded around the dominant kernel (kernel-only timing for the roofline)
struct KEvents { cudaEvent_t e0 = nullptr, e1 = nullptr; };
int k1_generic_launch(int cost, ImgF left, ImgF right, const Zone* d_zones, const Tile* d_tiles, int ntiles,
                      int kx, int ky, NccMaps ncc, vwb200_dispi* out, double* scratch_cost, int* scratch_idx, bool clamp_reads,
                      int stage_r_floats, cudaStream_t st, const KEvents* ev = nullptr,    // stage_r_floats: 0 = read through L1
                      const int* zone_gate = nullptr);                                     // != nullptr: only tiles of zones with gate[zone] != 0
bool k1_generic_can_stage(int kx, int ky, int sx, int sy, int nchunks);
long long k1_generic_stage_floats(int kx, int ky, int sx, int sy, int nchunks);
static constexpr int K1G_DCHUNK = 256;
// merge the per-chunk partial results of split zones (zone indices in d_split)
int k1_generic_merge_launch(int cost, const Zone* d_zones, const int* d_split, int nsplit, const double* scratch_cost,
                            const int* scratch_idx, vwb200_dispi* out, cudaStream_t st);
int k1_generic_tile_w(int kx);
int k1_generic_tile_h(int ky);
// ---- K1 zone-int (k1_zone_int.cu): the zone kernel in exact int32 for integer-valued imagery (level 0 of 8-bit rasters) ----
// range = vmax - vmin of both rasters; *ib_out = log2 of the disparities one warp covers (larger zones are split in chunks)
bool k1_zone_int_supported(int cost, int kx, int ky, long long range, int* ib_out);
int k1_zone_int_tile_w(int k);
int k1_zone_int_tile_h();
long long k1_zone_int_stage_u16(int k, int sx, int sy, int nchunks, int ib);
long long k1_zone_int_stage_max();
// zone_flag[zone] is set when a tile of the zone met a non-integer pixel (mean-filled masked pixels): the caller re-runs those
// zones through the fp64 zone kernel
int k1_zone_int_launch(int cost, ImgF left, ImgF right, const Zone* d_zones, const Tile* d_tiles, int ntiles, int k, float vmin, float vmax,
                       int warp_u16, vwb200_dispi* out, double* scratch_cost, int* scratch_idx, int* zone_flag, cudaStream_t st,
                       const KEvents* ev = nullptr);
// integer-valued rasters of a zone batch: enables the zone-int kernel in run_k1_zones.  checked: some pixels were replaced by
// a (non-integer) mean, zones that touch them fall back to the fp64 kernel
struct ZoneIntMode { bool on; float vmin, vmax; bool checked; };
// 1/boxsum(v*v) over window origins [ox0,ox0+ow) x [oy0,oy0+oh) with clamped (constant edge) reads.
int box_sq_inv_launch(ImgF img, int kx, int ky, int ox0, int oy0, int ow, int oh, double* out, cudaStream_t st);
// boxsum(v) (centred == 0) or boxsum((v - c)^2) (centred == 1) as int32 over the same window-origin domain (integer imagery)
int box_sum_i32_launch(ImgF img, int kx, int ky, int ox0, int oy0, int ow, int oh, int* out, cudaStream_t st, int centred = 0,
                       float c = 0.0f);
// left/right are whole images; the logical rasters start at (lox,loy) / (rox,roy) (constant edge extension outside),
// (addx,addy) is added to every output disparity (R->L pass of the level loop)
struct FastOrigin { int lox, loy, rox, roy, addx, addy; };
// NCC / wide-range SquaredCost on the exact-integer path with fp32 screening (k1_screen.cu)
int k1_screen_supported(int cost, int kx, int ky, int sx, int sy, float vmin, float vmax, bool integer_valued);
size_t k1_screen_workspace_bytes(int cost, int W, int H, int sx, int sy, int kx, int ky);
int k1_screen_launch(int cost, ImgF left, ImgF right, int W, int H, int sx, int sy, int kx, int ky, float vmin, float vmax,
                     vwb200_dispi* out, ptrdiff_t opitch, void* workspace, cudaStream_t st, const KEvents* ev = nullptr,
                     const FastOrigin* org = nullptr);
// ---- SemiGlobalMatcher (k5_sgm.cu, k5_sgm_paths.cu; declarations in k5_sgm.cuh) ---------------
// exact sequential re-evaluation of pixels flagged NaN by k1 (NCC zero-energy windows)
int k1_nan_fixup_launch(int cost, ImgF left, ImgF right, const Zone* d_zones, int nzones, int kx, int ky,
                        NccMaps ncc, vwb200_dispi* out, cudaStream_t st, int gridx = 8);

// left/right are whole images; the logical rasters start at (lox,loy) / (rox,roy) (constant edge extension outside),
// (addx,addy) is added to every output disparity (R->L pass of the level loop)
// ---- K1 fast (exact-integer path, single big zone) -------------------------------------------
// Returns VWB200_ENOIMPL if the configuration is outside what the fast path handles.
int k1_fast_supported(int cost, int kx, int ky, int sx, int sy, float vmin, float vmax, bool integer_valued);
int k1_fast_launch(int cost, ImgF left, ImgF right, int W, int H, int sx, int sy, int kx, int ky, float vmin, float vmax,
                   vwb200_dispi* out, ptrdiff_t opitch, void* workspace, size_t workspace_bytes, cudaStream_t st,
                   const KEvents* ev = nullptr, const struct FastOrigin* org = nullptr);
size_t k1_fast_workspace_bytes(int W, int H, int sx, int sy, int kx, int ky);
// min / max / integer-valuedness of an image (device reduction); result[0]=min,[1]=max,[2]=all-integers(1/0)
int image_stats_launch(ImgF img, float* d_result3, cudaStream_t st);

// ---- K2 pyramid ---------------------------------------------------------------------------------
int crop_extend_f32_launch(ImgF src, int x0, int y0, int w, int h, float* dst, ptrdiff_t dpitch, cudaStream_t st);
int crop_extend_u8_launch(ImgB src, int x0, int y0, int w, int h, int zero_outside, uint8_t* dst, ptrdiff_t dpitch, cudaStream_t st);
// masked mean over every 2nd pixel (CorrelationView.cc:133-136): d_acc = {double sum, double count}
int masked_mean_launch(ImgF img, ImgB mask, double* d_acc2, cudaStream_t st);
int mean_fill_launch(float* img, int w, int h, ptrdiff_t pitch, ImgB mask, const double* d_acc2, cudaStream_t st);
int mask_any_zero_launch(ImgB mask, int* d_flag, cudaStream_t st);      // *d_flag = 1 if the mask holds a zero (caller zeroes it)
int pyramid_down_launch(ImgF in, float* out, ptrdiff_t opitch, cudaStream_t st);
int subsample_mask_launch(ImgB in, uint8_t* out, ptrdiff_t opitch, cudaStream_t st);
// gaussian (separable, constant edge) into out via work; then Laplacian (mode 1) or img - g (mode 2)
int sepconv_launch(ImgF in, const float* d_taps, int n, float* work, float* out, cudaStream_t st);
int prefilter_final_launch(ImgF img, const float* g, int mode, float* out, cudaStream_t st);

// ---- K3 / K4 -------------------------------------------------------------------------------------
int consistency_launch(vwb200_dispi* l2r, int lw, int lh, ptrdiff_t lpitch, const vwb200_dispi* r2l, int rw, int rh,
                       ptrdiff_t rpitch, float thr, cudaStream_t st, int qax = 0, int qay = 0, float* diff = nullptr, ptrdiff_t dpitch = 0,
                       int dox = 0, int doy = 0);
int diff_invalidate_launch(const vwb200_dispi* disp, int w, int h, float* diff, ptrdiff_t dpitch, int dox, int doy, cudaStream_t st);
int sgm_finalize_launch(const float* sub, const vwb200_dispi* disp, int w, int ax, int ay, float* out, ptrdiff_t opitch_px, int ox, int oy,
                        int ow, int oh, cudaStream_t st);
// disparity_blob_filter; work: 2 * w * h ints
int blob_filter_launch(vwb200_dispi* d, int w, int h, int area, int* work, cudaStream_t st);
// pass 2 (1,1,3.0,0.20) reading the padded pass-1 buffer (w+2)x(h+2)
int cleanup_pass2_launch(const vwb200_dispi* p1, int w, int h, vwb200_dispi* out, cudaStream_t st);
int cleanup_pass2_launch(const DispF* p1, int w, int h, DispF* out, cudaStream_t st);
// pass 1 of rm_outliers_using_{thresh,mean,stddev} (method: VWB200_OUTLIERS_*) on either pixel type, evaluated over
// [x0,x0+ow) x [y0,y0+oh) of the constant-edge-extended input (row pitch ipitch); out has row pitch opitch.
// T = vwb200_dispi or DispF.
template <class T>
int outlier_pass1_launch(int method, const T* in, int w, int h, ptrdiff_t ipitch, int hx, int hy, double pt, double rt,
                         double max_mean_diff, int x0, int y0, int ow, int oh, T* out, ptrdiff_t opitch, cudaStream_t st);
int disparity_mask_launch(const vwb200_dispi* in, int w, int h, ImgB lmask, ImgB rmask, vwb200_dispi* out, cudaStream_t st);
// out[i] = {dx+ax, dy+ay, valid} as float triples (CorrelationView.cc:880-884)
int finalize_launch(const vwb200_dispi* in, int w, int h, int ax, int ay, float* out, ptrdiff_t opitch_px,
                    int ox, int oy, int ow, int oh, cudaStream_t st);

// ---- a11 ParabolaSubpixelView -------------------------------------------------------------------------
int disp_range_launch(const float* disp, int cols, int bx0, int by0, int bw, int bh, int* d_r5, cudaStream_t st);
int meansub_region_launch(const float* e, const float* g, int ew, int m, int w, int h, float* out, cudaStream_t st);
int log_region_launch(const float* g, int gw, int gx0, int gy0, int iw, int ih, int rx0, int ry0, int w, int h, float* out, cudaStream_t st);
int parabola_launch(const float* disp, int cols, int bx0, int by0, int bw, int bh, const float* L, int lw, const float* R, int rw,
                    int srx0, int sry0, int kx, int ky, float* out, cudaStream_t st);

// ---- disparity smoothing (k6_smoothing.cu) -----------------------------------------------------------
static constexpr int kSmoothMaxKernel = 31;   // largest kernel_size / max_kernel_size the smoothing kernels take
// in-place wavefront sweeps over W x H float disparity triples (pitch in pixels).  work: H + 2 ints of device scratch;
// *err_host receives (asynchronously, on st) 1 when the sweep stalled
int median_sweep_launch(float* d, int W, int H, ptrdiff_t pitch, int kernel_size, int* work, int* err_host, cudaStream_t st);
int texture_filter_sweep_launch(float* d, int W, int H, ptrdiff_t pitch, const float* tex, ptrdiff_t tpitch, float texture_max,
                                int max_kernel_size, int* work, int* err_host, cudaStream_t st);
int texture_measure_launch(ImgF img, int kernel_size, double gw, double sw, float* out, ptrdiff_t opitch, cudaStream_t st);

// ---- K7: disparity resampling, range and transforms (k7_dispmap.cu); T = vwb200_dispi or DispF, pitches in pixels ----------
// subsample: out is (1 + (w-1)/2) x (1 + (h-1)/2); upsample: out is 2w x 2h
template <class T> int dispmap_subsample_launch(const T* in, int w, int h, ptrdiff_t ip, T* out, ptrdiff_t op, cudaStream_t st);
template <class T> int dispmap_upsample_launch(const T* in, int w, int h, ptrdiff_t ip, T* out, ptrdiff_t op, cudaStream_t st);
// keys5: 5 x 8 bytes of device scratch; res5 (device): min x, min y, max x, max y, any valid pixel (1 / 0); w * h < 2^32
template <class T> int dispmap_range_launch(const T* in, int w, int h, ptrdiff_t ip, unsigned long long* keys5, float* res5, cudaStream_t st);
// min2 / max2: host pointers to two channel values each; out may be in (same pitch)
template <class T> int dispmap_range_mask_launch(const T* in, int w, int h, ptrdiff_t ip, const void* min2, const void* max2, T* out,
                                                 ptrdiff_t op, cudaStream_t st);
template <class T> int dispmap_transform_launch(int mode, const double* m9, int do_round, int sx0, int sy0, const T* in, int w, int h,
                                                ptrdiff_t ip, T* out, ptrdiff_t op, cudaStream_t st);

// ---- K8: transform(image, tx, edge, interp) of a float image over an output window (k8_warp.cu); pitches in elements ----------
// disp (DispF, dw x dh, pitch dp) is read for VWB200_WARP_DISPARITY only
int warp_launch(const vwb200_warp_params& p, const float* in, int w, int h, ptrdiff_t ip, const DispF* disp, int dw, int dh, ptrdiff_t dp,
                int x0, int y0, float* out, int ow, int oh, ptrdiff_t op, cudaStream_t st);
struct TriCam;
struct CahvCam;
// camera_transform (Camera/CameraTransform.h:43-183): reverse(p) = src.point_to_pixel(dst.pixel_to_vector(p) + C) between two
// pinhole cameras (Cam = TriCam), or from a CAHV or CAHVOR src into a CAHV dst (Cam = CahvCam).  masked: the pixels are
// PixelMask<float> {value, valid} float pairs (pitches in pairs; bilinear only, edge_value[2] for VWB200_EDGE_VALUE).
// fail (device, 0 and ULLONG_MAX on entry): [0] is set and [1] lowered to the row-major window index of every pixel whose
// point_to_pixel check fails (pinhole cameras only: the CAHV family has no check).
template <class Cam>
int camera_warp_launch(int masked, int interp, int edge, const float* edge_value, const Cam& src, const Cam& dst, const float* in, int w, int h,
                       ptrdiff_t ip, int x0, int y0, float* out, int ow, int oh, ptrdiff_t op, unsigned long long* fail, cudaStream_t st);
// compute_transformed_bbox_fast (Image/Transform.h:271-315) of the ROI (x0, y0, x1, y1) through CameraTransform(src, dst)::forward
// into keys4 (device, fkey of min x, min y, max x, max y; the caller seeds them with BBox2f's initial bounds); fail as above,
// with the perimeter index in the reference's loop order
int camera_bbox_launch(const TriCam& src, const TriCam& dst, int x0, int y0, int x1, int y1, unsigned* keys4, unsigned long long* fail,
                       cudaStream_t st);

// ---- K9: fill_holes_grass over an output window (k9_inpaint.cu); T = vwb200_dispi or DispF, pitches in pixels ---------------
// in and out are device rasters that do not overlap; stats are those of vwb200_last_fill_stats
template <class T> int fill_holes_grass_launch(const T* in, int w, int h, ptrdiff_t ip, int len, int x0, int y0, T* out, int ow, int oh,
                                               ptrdiff_t op, Arena& ar, cudaStream_t st, vwb200_fill_stats* stats);

// ---- K10: stereo triangulation (k10_triangulate.cu); pitches in pixels -----------------------------------------------------
// what PinholeModel::pixel_to_vector and camera_center need, built once per call by the host: the inverse camera transform
// (row-major), the center, the pixel pitch, the intrinsics the lens normalises by, and the Tsai parameters when tsai != 0;
// P is the 3 x 4 camera matrix K * [uvw * transpose(R) | uvw * (-transpose(R)) * C] (row-major) that point_to_pixel applies
struct TriCam { double inv[9], c[3], pitch, fu, fv, cu, cv, k[5]; int tsai; double P[12]; };
// what CAHVModel / CAHVORModel::pixel_to_vector, point_to_pixel and camera_center need (Camera/CAHVModel.cc:167-189,
// CAHVORModel.cc:297-350, 431-448): the six vectors (O and R unused unless cahvor), cahvor != 0 for the CAHVOR model, and
// flip != 0 where dot_prod(cross_prod(V, H), A) < 0 (the host evaluates it once per call in the reference's order)
struct CahvCam { double C[3], A[3], H[3], V[3], O[3], R[3]; int cahvor, flip; };
// Cam = TriCam (two pinhole cameras) or CahvCam (two CAHV or CAHVOR cameras, each independently).  stats: 5 x 8 bytes of
// zeroed device scratch -- [0] error sum (double), [1] max error (double bits), [2] points, [3] divergent, [4] the Newton
// iterations of both rays of every triangulated pixel (Tsai Newton-Raphson or CAHVOR Newton passes); form (a) fills [4] only.
// xyz pitches count {x, y, z} pixels.
template <class Cam, class T>
int stereo_triangulate_launch(const T* in, ptrdiff_t ip, int x0, int y0, int ow, int oh, const Cam& c0, const Cam& c1, double tol, double* xyz,
                              ptrdiff_t xp, unsigned long long* stats, cudaStream_t st);
template <class Cam>
int stereo_model_launch(const DispF* in, int w, int h, ptrdiff_t ip, const Cam& c0, const Cam& c1, double tol, double* xyz, ptrdiff_t xp,
                        double* err, ptrdiff_t ep, unsigned long long* stats, cudaStream_t st);
// in may be out (same pitch); *rejected (device) is added to
int universe_radius_launch(const double* in, int w, int h, ptrdiff_t ip, const double* origin, double near_r, double far_r, double* out,
                           ptrdiff_t op, unsigned long long* rejected, cudaStream_t st);

// ---- K11: exact interest point matching (k11_ipmatch.cu); descriptor pitches in floats --------------------------------------
// one query's summary over a set of candidates: the smallest distance, the lowest candidate index with it, and the
// second-smallest distance (equal to best when best occurs twice); +inf / INT_MAX for none
struct IpTop2 { float best; int j; float second; };
struct IpMatchInfo {
  int splits;                       // CTAs the candidate range was split over (0: no candidates)
  unsigned long long matches;       // valid once the stream has synchronised
  unsigned long long bad[2];        // Hamming: first invalid element index of desc1 / desc2 (row * dim + k), ~0 for none
};
// index / first / second: device outputs of n1 entries (first, second may be NULL).  Returns VWB200_EARG (with info->bad
// set, stream synchronised) when a Hamming descriptor holds a value outside (-1, 256) or NaN.
int ip_match_launch(int metric, const float* d1, ptrdiff_t p1, const uint8_t* pol1, int n1, const float* d2, ptrdiff_t p2,
                    const uint8_t* pol2, int n2, int dim, double threshold, int* index, double* first, double* second, Arena& ar,
                    cudaStream_t st, IpMatchInfo* info);

// ---- host-side restatement-free logic -----------------------------------------------------------
struct Box { int x0, y0, x1, y1; };
struct HostZone { Box img; Box disp; };
// quad-tree search-range refinement (behaviour of Stereo/Correlation.cc:139-328), host side.
void subdivide_regions_host(const vwb200_dispi* disp, int w, int h, int kx, int ky, std::vector<HostZone>& out);

}  // namespace vwb200
