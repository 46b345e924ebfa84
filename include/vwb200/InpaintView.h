// InpaintView.h -- C++ shim: fill_holes_grass(img, hole_fill_len) of Image/InpaintView.h:239-311 with the reference's
// parameter list, computed on the device through include/vwb200.h, for ImageView<PixelMask<Vector2i>> and
// ImageView<PixelMask<Vector2f>>.  Like the reference's FillHolesGrass it is a view: operator() throws NoImplErr, and
// prerasterize(bbox) fills the holes of the bbox grown by hole_fill_len, so the result depends on the bbox in the same way.
// Filled pixels carry the engine's valid word (1), not ChannelRange::max().  A negative hole_fill_len, one whose square
// overflows int32, and a bbox that leaves the image throw ArgumentErr where the reference does not check.
#pragma once
#include "DisparityResampling.h"

namespace vw {

template <class ImageT>
class B200FillHolesGrass : public ImageViewBase<B200FillHolesGrass<ImageT>> {
  ImageT m_img;
  int m_hole_fill_len;

public:
  typedef typename ImageT::pixel_type pixel_type;
  typedef pixel_type result_type;
  typedef ProceduralPixelAccessor<B200FillHolesGrass<ImageT>> pixel_accessor;

  B200FillHolesGrass(ImageT const& img, int hole_fill_len) : m_img(img), m_hole_fill_len(hole_fill_len) {}

  int cols() const { return m_img.cols(); }
  int rows() const { return m_img.rows(); }
  int planes() const { return 1; }
  pixel_accessor origin() const { return pixel_accessor(*this, 0, 0); }

  pixel_type operator()(double /*i*/, double /*j*/, int /*p*/ = 0) const {
    vw_throw(NoImplErr() << "FillHolesGrass::operator() is not implemented");
    return pixel_type();
  }

  typedef CropView<ImageView<pixel_type>> prerasterize_type;
  prerasterize_type prerasterize(BBox2i const& bbox) const {
    static_assert(sizeof(pixel_type) == 12, "disparity pixels must be {dx, dy, valid} triples of 4-byte values");
    ImageView<pixel_type> win(bbox.width(), bbox.height());
    stereo::b200_detail::check(vwb200_fill_holes_grass(stereo::b200_detail::DispPixel<pixel_type>::type, m_img.data(), m_img.cols(),
                                                       m_img.rows(), m_img.rstride(), m_hole_fill_len, bbox.min()[0], bbox.min()[1],
                                                       win.data(), win.cols(), win.rows(), win.rstride(), /*on_device=*/0, nullptr));
    return prerasterize_type(win, -bbox.min()[0], -bbox.min()[1], cols(), rows());
  }

  template <class DestT>
  void rasterize(DestT const& dest, BBox2i bbox) const { vw::rasterize(prerasterize(bbox), dest, bbox); }
};

template <class ImageT>
inline B200FillHolesGrass<ImageT> b200_fill_holes_grass(ImageT const& img, int hole_fill_len) {
  return B200FillHolesGrass<ImageT>(img, hole_fill_len);
}

}  // namespace vw
