// dfk_matching.h -- the keypoint matching step of the reference's ReprojectionFactor (reprojection_factor.cpp:56-65)
// on top of dfk_hamming_match_batch / dfk_reprojection_match_batch (include/dfk.h):
//   df::Features                  the keypoints and descriptors of a keyframe, on the device (kf->features)
//   df::DMatch                    cv::DMatch's members (queryIdx, trainIdx, distance)
//   df::ReprojectionMatcher       owns a handle; MatchBatch / ReprojectionMatchesBatch run many factors in one call
//     .ReprojectionMatches        the constructor's three steps for one factor (BFMatcher, PruneMatchesEightPoint,
//                                 PruneMatchesByThreshold), as a std::vector<DMatch>
//     .PruneMatchesEightPoint     BFMatcher + RANSAC: the inliers in match (query) order, as features/matching.cpp:75-128
//   df::PruneMatchesByThreshold   features/matching.cpp:29-37 on the host: distance <= max_dist, sorted by (distance,
//                                 queryIdx), the order the device lists have
//   df::OrbDetector               the keypoints and descriptors themselves: OrbDetector(nfeatures, scale_factor, 1)
//     .DetectAndCompute           of features/feature_detection.h for one device image or a batch (dfk_orb_detect_batch)
//   df::OrbPyramidDetector        OrbDetector(nfeatures, scale_factor, nlevels) with any nlevels (rep_nlevels > 1)
//     .DetectAndCompute           likewise, through dfk_orb_detect_pyramid_batch
// The host-vector members copy their results back with the CUDA runtime; they exist where its header does.
#ifndef DFK_MATCHING_H_
#define DFK_MATCHING_H_

#include <algorithm>
#include <cstdint>
#include <limits>
#include <vector>

#include "dfk_facade.h"

namespace df
{

struct Features {
  const float* keypoints = nullptr;      // DEVICE [num, 2], keypoints[i].pt at level 0
  const uint8_t* descriptors = nullptr;  // DEVICE [num, descriptor_bytes], 16-byte aligned
  int num = 0;
  int descriptor_bytes = 32;             // 32 (ORB) or 64 (BRISK)
  DfkFeatureSet View() const { return DfkFeatureSet{keypoints, descriptors, num, descriptor_bytes}; }
};

struct DMatch {
  int queryIdx = -1, trainIdx = -1;
  float distance = 0.0f;
};

// ReprojectionFactor's matching arguments: rep_max_dist, rep_ransac_maxiters, rep_ransac_threshold
// (deepfactors_options.h:96-101) and PruneMatchesEightPoint's probability (matching.h:48-50)
struct MatchParams {
  float max_dist = 30.0f;
  int max_iterations = 1000;
  double threshold = 0.0001f;
  double probability = 0.99;
  uint64_t seed = 0;
};

// cv::DMatch::operator< orders by distance; ties here go to the lower queryIdx, as on the device
inline std::vector<DMatch> PruneMatchesByThreshold(std::vector<DMatch> matches, float max_dist)
{
  std::sort(matches.begin(), matches.end(), [](const DMatch& a, const DMatch& b) {
    return a.distance < b.distance || (a.distance == b.distance && a.queryIdx < b.queryIdx);
  });
  auto first_wrong = std::find_if(matches.begin(), matches.end(), [&](const DMatch& m) { return m.distance > max_dist; });
  return std::vector<DMatch>(matches.begin(), first_wrong);
}

class ReprojectionMatcher
{
public:
  ReprojectionMatcher() : h_(detail::MakeHandle()) {}

  DfkHandle handle() const { return h_.get(); }
  void SetStream(void* stream) { detail::Check(h_.get(), dfk_set_stream(h_.get(), stream)); }

  template <typename CamT>
  static DfkMatchItem Item(const Features& kf, const Features& fr, const CamT& cam, const MatchParams& p)
  {
    DfkMatchItem it{};
    it.query = kf.View();
    it.train = fr.View();
    it.cam = detail::Cam(cam);
    it.max_dist = p.max_dist;
    it.max_iterations = p.max_iterations;
    it.threshold = p.threshold;
    it.probability = p.probability;
    it.seed = p.seed;
    return it;
  }

  // dfk_hamming_match_batch: DEVICE output, (train, distance) per query of every item
  void MatchBatch(const std::vector<DfkMatchItem>& items, int32_t* matches_dev)
  {
    detail::Check(h_.get(), dfk_hamming_match_batch(h_.get(), items.data(), (int)items.size(), matches_dev));
  }

  // dfk_reprojection_match_batch: DEVICE outputs, (query, train, distance) rows, the counts, (best, inliers, evaluated)
  void ReprojectionMatchesBatch(const std::vector<DfkMatchItem>& items, int32_t* matches_dev, int32_t* counts_dev,
                                int32_t* ransac_dev = nullptr)
  {
    detail::Check(h_.get(), dfk_reprojection_match_batch(h_.get(), items.data(), (int)items.size(), matches_dev,
                                                         counts_dev, ransac_dev));
  }

#ifdef DFK_FACADE_CUDART
  // the three lines of ReprojectionFactor's constructor (reprojection_factor.cpp:56-65), for one factor
  template <typename CamT>
  std::vector<DMatch> ReprojectionMatches(const Features& kf, const Features& fr, const CamT& cam,
                                          const MatchParams& p = MatchParams())
  {
    return Run(Item(kf, fr, cam, p));
  }

  // BFMatcher + PruneMatchesEightPoint (matching.cpp:75-128): the best hypothesis' inliers in match order
  template <typename CamT>
  std::vector<DMatch> PruneMatchesEightPoint(const Features& kf, const Features& fr, const CamT& cam,
                                             const MatchParams& p = MatchParams())
  {
    DfkMatchItem it = Item(kf, fr, cam, p);
    it.max_dist = std::numeric_limits<float>::infinity();
    std::vector<DMatch> m = Run(it);
    std::sort(m.begin(), m.end(), [](const DMatch& a, const DMatch& b) { return a.queryIdx < b.queryIdx; });
    return m;
  }

private:
  std::vector<DMatch> Run(const DfkMatchItem& it)
  {
    const size_t n0 = (size_t)std::max(it.query.num, 0);
    int32_t* dev = nullptr;  // [n0 x 3 rows | count]
    if (cudaMalloc(&dev, sizeof(int32_t) * (3 * n0 + 1)) != cudaSuccess)
      throw std::runtime_error("[ReprojectionMatcher] device allocation failed");
    std::unique_ptr<int32_t, void (*)(int32_t*)> guard(dev, [](int32_t* q) { cudaFree(q); });
    std::vector<DfkMatchItem> items{it};
    ReprojectionMatchesBatch(items, dev, dev + 3 * n0);
    std::vector<int32_t> host(3 * n0 + 1);
    if (cudaMemcpyAsync(host.data(), dev, host.size() * sizeof(int32_t), cudaMemcpyDeviceToHost,
                        static_cast<cudaStream_t>(dfk_get_stream(h_.get()))) != cudaSuccess ||
        cudaStreamSynchronize(static_cast<cudaStream_t>(dfk_get_stream(h_.get()))) != cudaSuccess)
      throw std::runtime_error("[ReprojectionMatcher] result download failed");
    std::vector<DMatch> out((size_t)host[3 * n0]);
    for (size_t i = 0; i < out.size(); ++i) out[i] = DMatch{host[3 * i], host[3 * i + 1], (float)host[3 * i + 2]};
    return out;
  }
#endif

private:
  detail::HandlePtr h_;
};

// The reference's OrbDetector (features/feature_detection.h) on the device: cv::ORB::create(nfeatures, scale_factor,
// nlevels) with nlevels = 1 (rep_nlevels), through dfk_orb_detect_batch.  With one level cv::ORB ignores
// scale_factor; any other nlevels is rejected.  Keypoints come in the device order (response descending, then y,
// then x), as df::Features views.
class OrbDetector
{
public:
  explicit OrbDetector(int nfeatures = 500, float scale_factor = 1.2f, int nlevels = 1, int fast_threshold = 20)
      : nfeatures_(nfeatures), fast_threshold_(fast_threshold), h_(detail::MakeHandle())
  {
    if (nlevels != 1) throw std::invalid_argument("[OrbDetector] only nlevels = 1 (one pyramid level) is supported");
    (void)scale_factor;
  }

  DfkHandle handle() const { return h_.get(); }
  void SetStream(void* stream) { detail::Check(h_.get(), dfk_set_stream(h_.get(), stream)); }
  int nfeatures() const { return nfeatures_; }
  // rows reserved per image: ties at the response cut can add keypoints past nfeatures
  int capacity() const { return 2 * nfeatures_; }

  DfkOrbItem Item(const DfkImage& image) const { return DfkOrbItem{image, nfeatures_, fast_threshold_, capacity()}; }

  // dfk_orb_detect_batch into the caller's DEVICE buffers (rows at the prefix sums of the items' capacities)
  void DetectBatch(const std::vector<DfkOrbItem>& items, float* keypoints_dev, uint8_t* descriptors_dev,
                   float* angles_dev, float* responses_dev, int32_t* counts_dev)
  {
    detail::Check(h_.get(), dfk_orb_detect_batch(h_.get(), items.data(), (int)items.size(), keypoints_dev,
                                                 descriptors_dev, angles_dev, responses_dev, counts_dev));
  }

#ifdef DFK_FACADE_CUDART
  // FeatureDetector::DetectAndCompute for a device gray image: the features stay valid until the next detection
  Features DetectAndCompute(const DfkImage& image) { return DetectAndCompute(std::vector<DfkImage>{image})[0]; }

  // every image in one call; waits for the counts
  std::vector<Features> DetectAndCompute(const std::vector<DfkImage>& images)
  {
    const size_t n = images.size(), rows = n * (size_t)capacity();
    std::vector<DfkOrbItem> items;
    for (const DfkImage& im : images) items.push_back(Item(im));
    if (rows > rows_) {
      out_.reset();
      void* p = nullptr;  // [descriptors 32 per row | keypoints 2 floats per row | counts]
      if (cudaMalloc(&p, rows * 40 + 4 * n + 16) != cudaSuccess)
        throw std::runtime_error("[OrbDetector] device allocation failed");
      out_.reset(static_cast<uint8_t*>(p));
      rows_ = rows;
    }
    uint8_t* desc = out_.get();
    float* kp = reinterpret_cast<float*>(desc + 32 * rows_);
    int32_t* counts = reinterpret_cast<int32_t*>(kp + 2 * rows_);
    DetectBatch(items, kp, desc, nullptr, nullptr, counts);
    std::vector<int32_t> host(n);
    const cudaStream_t s = static_cast<cudaStream_t>(dfk_get_stream(h_.get()));
    if (cudaMemcpyAsync(host.data(), counts, n * sizeof(int32_t), cudaMemcpyDeviceToHost, s) != cudaSuccess ||
        cudaStreamSynchronize(s) != cudaSuccess)
      throw std::runtime_error("[OrbDetector] count download failed");
    std::vector<Features> out(n);
    for (size_t i = 0; i < n; ++i) {
      if (host[i] > capacity())
        throw std::runtime_error("[OrbDetector] more keypoints than the capacity (ties at the response cut)");
      const size_t o = i * (size_t)capacity();
      out[i] = Features{kp + 2 * o, desc + 32 * o, host[i], 32};
    }
    return out;
  }

private:
  struct Free {
    void operator()(uint8_t* p) const { cudaFree(p); }
  };
  std::unique_ptr<uint8_t, Free> out_;
  size_t rows_ = 0;
#endif

private:
  int nfeatures_, fast_threshold_;
  detail::HandlePtr h_;
};

// The reference's OrbDetector with a scale pyramid: cv::ORB::create(nfeatures, scale_factor, nlevels), 1 <= nlevels <=
// DFK_ORB_MAX_LEVELS, scale_factor > 1, through dfk_orb_detect_pyramid_batch.  Keypoints come at level 0 in the
// device order (levels ascending, each by response descending, then y, then x), as df::Features views.
class OrbPyramidDetector
{
public:
  explicit OrbPyramidDetector(int nfeatures = 500, float scale_factor = 1.2f, int nlevels = 8, int fast_threshold = 20)
      : nfeatures_(nfeatures), nlevels_(nlevels), fast_threshold_(fast_threshold), scale_factor_(scale_factor),
        h_(detail::MakeHandle())
  {
  }

  DfkHandle handle() const { return h_.get(); }
  void SetStream(void* stream) { detail::Check(h_.get(), dfk_set_stream(h_.get(), stream)); }
  int nfeatures() const { return nfeatures_; }
  int nlevels() const { return nlevels_; }
  float scale_factor() const { return scale_factor_; }
  // rows reserved per image: ties at the response cuts can add keypoints past nfeatures
  int capacity() const { return 2 * nfeatures_; }

  DfkOrbPyramidItem Item(const DfkImage& image) const
  {
    return DfkOrbPyramidItem{image, nfeatures_, scale_factor_, nlevels_, fast_threshold_, capacity()};
  }

  // dfk_orb_detect_pyramid_batch into the caller's DEVICE buffers (rows at the prefix sums of the items' capacities)
  void DetectBatch(const std::vector<DfkOrbPyramidItem>& items, float* keypoints_dev, uint8_t* descriptors_dev,
                   float* angles_dev, float* responses_dev, int32_t* octaves_dev, int32_t* counts_dev)
  {
    detail::Check(h_.get(), dfk_orb_detect_pyramid_batch(h_.get(), items.data(), (int)items.size(), keypoints_dev,
                                                         descriptors_dev, angles_dev, responses_dev, octaves_dev,
                                                         counts_dev));
  }

#ifdef DFK_FACADE_CUDART
  // FeatureDetector::DetectAndCompute for a device gray image: the features stay valid until the next detection
  Features DetectAndCompute(const DfkImage& image) { return DetectAndCompute(std::vector<DfkImage>{image})[0]; }

  // every image in one call; waits for the counts
  std::vector<Features> DetectAndCompute(const std::vector<DfkImage>& images)
  {
    const size_t n = images.size(), rows = n * (size_t)capacity();
    std::vector<DfkOrbPyramidItem> items;
    for (const DfkImage& im : images) items.push_back(Item(im));
    if (rows > rows_) {
      out_.reset();
      void* p = nullptr;  // [descriptors 32 per row | keypoints 2 floats per row | counts]
      if (cudaMalloc(&p, rows * 40 + 4 * n + 16) != cudaSuccess)
        throw std::runtime_error("[OrbPyramidDetector] device allocation failed");
      out_.reset(static_cast<uint8_t*>(p));
      rows_ = rows;
    }
    uint8_t* desc = out_.get();
    float* kp = reinterpret_cast<float*>(desc + 32 * rows_);
    int32_t* counts = reinterpret_cast<int32_t*>(kp + 2 * rows_);
    DetectBatch(items, kp, desc, nullptr, nullptr, nullptr, counts);
    std::vector<int32_t> host(n);
    const cudaStream_t s = static_cast<cudaStream_t>(dfk_get_stream(h_.get()));
    if (cudaMemcpyAsync(host.data(), counts, n * sizeof(int32_t), cudaMemcpyDeviceToHost, s) != cudaSuccess ||
        cudaStreamSynchronize(s) != cudaSuccess)
      throw std::runtime_error("[OrbPyramidDetector] count download failed");
    std::vector<Features> out(n);
    for (size_t i = 0; i < n; ++i) {
      if (host[i] > capacity())
        throw std::runtime_error("[OrbPyramidDetector] more keypoints than the capacity (ties at the response cuts)");
      const size_t o = i * (size_t)capacity();
      out[i] = Features{kp + 2 * o, desc + 32 * o, host[i], 32};
    }
    return out;
  }

private:
  struct Free {
    void operator()(uint8_t* p) const { cudaFree(p); }
  };
  std::unique_ptr<uint8_t, Free> out_;
  size_t rows_ = 0;
#endif

private:
  int nfeatures_, nlevels_, fast_threshold_;
  float scale_factor_;
  detail::HandlePtr h_;
};

}  // namespace df

#endif  // DFK_MATCHING_H_
