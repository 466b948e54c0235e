// dfk_preprocess.h -- DeepFactors::PreprocessImage (core/deepfactors.cpp:634-680) and the image pyramid of
// UploadLiveFrame / Mapper::BuildKeyframe on top of dfk_preprocess_batch (include/dfk.h):
//   df::FramePreprocessor          owns a handle, the network camera, the number of levels and the normalisation switch
//     .Preprocess(frame, cam, out) one camera frame into the caller's device views
//     .Preprocess(frames, ...)     many frames in one call
//   df::ResizeViewport             PinholeCamera::ResizeViewport in the reference's fp32 arithmetic
// Cameras are df::PinholeCamera<float> (accessors, as in the rest of the facade) or DfkCamera.
// Frames are DEVICE uint8 x 3 views; the caller uploads them (PreprocessImage's cv::Mat lives on the host).
#ifndef DFK_PREPROCESS_H_
#define DFK_PREPROCESS_H_

#include <stdexcept>
#include <vector>

#include "dfk_facade.h"

namespace df
{

// pinhole_camera_impl.h:126-136: the camera of a frame of w x h pixels.  cam is a df::PinholeCamera<float> (or any
// camera with its accessors) or a DfkCamera.
template <typename CamT>
inline DfkCamera ResizeViewport(const CamT& camera, int w, int h)
{
  const DfkCamera cam = detail::Cam(camera);
  const float xr = static_cast<float>(w) / cam.width, yr = static_cast<float>(h) / cam.height;
  return DfkCamera{cam.fx * xr, cam.fy * yr, cam.u0 * xr, cam.v0 * yr, static_cast<float>(w), static_cast<float>(h)};
}

// The outputs of one frame, DEVICE views the caller owns: color (uint8 x 3) and gray (uint8) of the network camera's
// size, or ptr = nullptr when not wanted; levels[num_levels] float and grads[num_levels] 2-float (empty: no gradients)
struct PreprocessedFrame {
  DfkImage color{};
  DfkImage gray{};
  std::vector<DfkImage> levels;
  std::vector<DfkImage> grads;
};

class FramePreprocessor
{
public:
  // out_cam: the network camera (netcfg_.camera), whose width x height is the output size
  template <typename CamT>
  FramePreprocessor(const CamT& out_cam, int num_levels, bool normalize = false)
      : out_cam_(detail::Cam(out_cam)), num_levels_(num_levels), normalize_(normalize), h_(detail::MakeHandle())
  {
  }

  DfkHandle handle() const { return h_.get(); }
  void SetStream(void* stream) { detail::Check(h_.get(), dfk_set_stream(h_.get(), stream)); }
  int width() const { return static_cast<int>(out_cam_.width); }
  int height() const { return static_cast<int>(out_cam_.height); }
  int num_levels() const { return num_levels_; }

  // the item of one frame; src_cam is the camera at the frame's size (ResizeViewport)
  DfkPreprocessItem Item(const DfkImage& frame, const DfkCamera& src_cam, const PreprocessedFrame& out) const
  {
    if ((int)out.levels.size() != num_levels_ || (!out.grads.empty() && (int)out.grads.size() != num_levels_))
      throw std::invalid_argument("[FramePreprocessor] a frame needs num_levels level views (and gradient views)");
    return DfkPreprocessItem{frame, src_cam, out_cam_, out.color, out.gray, out.levels.empty() ? nullptr : out.levels.data(),
                             out.grads.empty() ? nullptr : out.grads.data(), normalize_ ? 1 : 0};
  }

  // one frame; stats_dev (DEVICE double[2], may be null) gets (mu, sigma) when normalising
  template <typename CamT>
  void Preprocess(const DfkImage& frame, const CamT& src_cam, const PreprocessedFrame& out, double* stats_dev = nullptr)
  {
    const DfkPreprocessItem it = Item(frame, detail::Cam(src_cam), out);
    detail::Check(h_.get(), dfk_preprocess_batch(h_.get(), &it, 1, num_levels_, stats_dev));
  }

  // many frames in one call; stats_dev (DEVICE double[n, 2], may be null)
  template <typename CamT>
  void Preprocess(const std::vector<DfkImage>& frames, const std::vector<CamT>& src_cams,
                  const std::vector<PreprocessedFrame>& outs, double* stats_dev = nullptr)
  {
    if (frames.size() != src_cams.size() || frames.size() != outs.size())
      throw std::invalid_argument("[FramePreprocessor] one camera and one output per frame");
    std::vector<DfkPreprocessItem> items;
    for (size_t i = 0; i < frames.size(); ++i) items.push_back(Item(frames[i], detail::Cam(src_cams[i]), outs[i]));
    detail::Check(h_.get(), dfk_preprocess_batch(h_.get(), items.data(), (int)items.size(), num_levels_, stats_dev));
  }

private:
  DfkCamera out_cam_;
  int num_levels_;
  bool normalize_;
  detail::HandlePtr h_;
};

}  // namespace df

#endif  // DFK_PREPROCESS_H_
