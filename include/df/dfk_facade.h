// dfk_facade.h -- header-only C++ facade that reproduces the reference's aligner API surface
// on top of the C ABI of libdfk.so (include/dfk.h).
//
// Same namespaces, class names, method names, argument order and result member names as
//   df::SfmAligner<Scalar,CS>      sources/cuda/cu_sfmaligner.h:50-97
//   df::SE3Aligner<Scalar>         sources/cuda/cu_se3aligner.h:38-86
//   df::SfmAlignerParams           sources/cuda/cu_sfmaligner.h:41-48
//   df::DenseSfmParams             sources/common/algorithm/dense_sfm.h:36-43
//   df::JTJJrReductionItem<T,NP>   sources/cuda/reduction_items.h:77-143
//   df::CorrespondenceReductionItem<T>   sources/cuda/reduction_items.h:35-71
//   df::UpdateDepth / SobelGradients / GaussianBlurDown / SquaredError   sources/cuda/cu_image_proc.h:27-44
// (jczarnowski/DeepFactors @ bffc78a).
//
// The reference's argument types come from Sophus, Eigen and VisionCore, none of which is a
// dependency of this repository.  The facade is therefore DUCK-TYPED: every method is a template
// over the argument types and only uses the members the real types have
//   pose      .data()                          -> const float*  (Sophus::SE3f: quaternion xyzw, translation)
//   code      .data()                          -> const float*  (Eigen::Matrix<float,CS,1>)
//   camera    .fx() .fy() .u0() .v0() .width() .height()       (df::PinholeCamera<float>)
//   image     .ptr() .pitch() .width() .height()               (vc::Image2DView / vc::Buffer2DView;
//                                                               pitch in BYTES, width in elements)
// so a build that does have those libraries passes its own objects straight through (see
// INTEGRATION.md), and a build without them uses the minimal stand-ins of df/dfk_standins.h.
// Results are returned by value like the reference; dense access goes through
// JtJ.toDenseMatrix(i, j) / JtJ.coeff() instead of an Eigen expression.
#ifndef DFK_FACADE_H_
#define DFK_FACADE_H_

#include <algorithm>
#include <array>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <utility>
#include <vector>

#include "../dfk.h"

// SfmAligner::EvaluateErrorBatch copies its results back with the CUDA runtime; it exists where the runtime's header does
#if __has_include(<cuda_runtime_api.h>)
#include <cuda_runtime_api.h>
#define DFK_FACADE_CUDART 1
#endif

namespace df
{

// ---------------------------------------------------------------------------------------------
// errors: the reference throws vc::CUDAException from CudaCheckLastError (launch_utils.h:26-32) and
// std::runtime_error (cu_sfmaligner.cpp:171-173); glog CHECKs abort.  Here everything is an exception.
// ---------------------------------------------------------------------------------------------
class CUDAException : public std::runtime_error
{
public:
  CUDAException(DfkStatus st, const std::string& msg) : std::runtime_error(msg), status(st) {}
  DfkStatus status;
};

namespace detail
{
inline void Check(DfkHandle h, DfkStatus st)
{
  if (st == DFK_OK) return;
  const char* m = dfk_last_error(h);
  throw CUDAException(st, (m && *m) ? std::string(m) : std::string(dfk_status_string(st)));
}

template <typename ImageT>
inline DfkImage View(const ImageT& img, unsigned floats_per_px)
{
  DfkImage v;
  v.ptr = const_cast<void*>(static_cast<const void*>(img.ptr()));
  v.pitch_bytes = img.pitch();
  // the reference views the code Jacobian as a (W*CS) x H float image (keyframe.h:52); gradients are
  // Eigen::Matrix<float,1,2> pixels.  `width` of the C ABI counts pixels.
  v.width = static_cast<uint32_t>(img.width() / (floats_per_px > 2 ? floats_per_px : 1));
  v.height = static_cast<uint32_t>(img.height());
  return v;
}

template <typename CamT>
inline DfkCamera Cam(const CamT& cam)
{
  return DfkCamera{static_cast<float>(cam.fx()), static_cast<float>(cam.fy()), static_cast<float>(cam.u0()),
                   static_cast<float>(cam.v0()), static_cast<float>(cam.width()), static_cast<float>(cam.height())};
}
// a DfkCamera passes through as it is
inline DfkCamera Cam(const DfkCamera& cam) { return cam; }

struct HandleDeleter {
  void operator()(DfkContext* h) const { dfk_destroy(h); }
};
using HandlePtr = std::unique_ptr<DfkContext, HandleDeleter>;

inline HandlePtr MakeHandle()
{
  DfkHandle h = nullptr;
  DfkStatus st = dfk_create(-1, &h);
  if (st != DFK_OK) throw CUDAException(st, "dfk_create failed: " + std::string(dfk_status_string(st)));
  // Ordering contract of the drop-in facade = the reference's: every launch goes to the LEGACY DEFAULT stream
  // (cu_sfmaligner.cpp:175-179 launches without a stream argument), so inputs an integrator produced asynchronously on
  // stream 0 (uploads, pyramid / network kernels) are complete before an aligner reads them.  A handle's own stream is
  // non-blocking and NOT ordered against stream 0; callers that want it (or their own stream) say so with SetStream.
  dfk_set_stream(h, nullptr);
  return HandlePtr(h);
}
}  // namespace detail

// ---------------------------------------------------------------------------------------------
// vc::types::SquareUpperTriangularMatrix<Scalar,NP> stand-in (VisionCore, not in tree): packed upper
// triangle, row major.
// ---------------------------------------------------------------------------------------------
template <typename Scalar, int NP>
struct SquareUpperTriangularMatrix {
  static constexpr int Size = NP * (NP + 1) / 2;
  std::array<Scalar, Size> coeff_{};

  std::array<Scalar, Size>& coeff() { return coeff_; }
  const std::array<Scalar, Size>& coeff() const { return coeff_; }
  static constexpr int Index(int i, int j) { return i * NP - (i * (i - 1)) / 2 + (j - i); }
  // element of the full symmetric matrix (toDenseMatrix()(i,j) in the reference)
  Scalar toDenseMatrix(int i, int j) const { return i <= j ? coeff_[Index(i, j)] : coeff_[Index(j, i)]; }
  // full symmetric NP x NP, row major
  std::vector<Scalar> toDenseMatrix() const
  {
    std::vector<Scalar> m(static_cast<size_t>(NP) * NP);
    for (int i = 0; i < NP; ++i)
      for (int j = 0; j < NP; ++j) m[static_cast<size_t>(i) * NP + j] = toDenseMatrix(i, j);
    return m;
  }
  SquareUpperTriangularMatrix& operator+=(const SquareUpperTriangularMatrix& o)
  {
    for (int i = 0; i < Size; ++i) coeff_[i] += o.coeff_[i];
    return *this;
  }
};

// reduction_items.h:35-71
template <typename Scalar>
struct CorrespondenceReductionItem {
  CorrespondenceReductionItem() : residual(0), inliers(0) {}
  CorrespondenceReductionItem operator+(const CorrespondenceReductionItem& rhs) const
  {
    CorrespondenceReductionItem r(*this);
    r += rhs;
    return r;
  }
  CorrespondenceReductionItem& operator+=(const CorrespondenceReductionItem& rhs)
  {
    residual += rhs.residual;
    inliers += rhs.inliers;
    return *this;
  }
  Scalar residual;
  std::size_t inliers;
};

// reduction_items.h:77-143
template <typename Scalar, int NP>
struct JTJJrReductionItem {
  typedef SquareUpperTriangularMatrix<Scalar, NP> HessianType;
  typedef std::array<Scalar, NP> JacobianType;
  JTJJrReductionItem() : residual(0), inliers(0) { Jtr.fill(Scalar(0)); }
  JTJJrReductionItem operator+(const JTJJrReductionItem& rhs) const
  {
    JTJJrReductionItem r(*this);
    r += rhs;
    return r;
  }
  JTJJrReductionItem& operator+=(const JTJJrReductionItem& rhs)
  {
    JtJ += rhs.JtJ;
    for (int i = 0; i < NP; ++i) Jtr[i] += rhs.Jtr[i];
    residual += rhs.residual;
    inliers += rhs.inliers;
    return *this;
  }
  HessianType JtJ;
  JacobianType Jtr;
  Scalar residual;
  std::size_t inliers;
};

// dense_sfm.h:36-43
struct DenseSfmParams {
  float huber_delta = 0.1f;
  float ocl_th = 1000;  // disabled by default
  float avg_dpt = 2.0f;
  float min_dpt = 0.0f;
  int valid_border = 2;
};

// cu_sfmaligner.h:41-48
struct SfmAlignerParams {
  DenseSfmParams sfmparams;
  int step_threads = 32;  // NOTE: threads must be a multiple of 32!
  int step_blocks = 11;
  int eval_threads = 224;
  int eval_blocks = 66;
};

// ---------------------------------------------------------------------------------------------
// df::SfmAligner<Scalar,CS>  (cu_sfmaligner.h:50-97)
// ---------------------------------------------------------------------------------------------
template <typename Scalar, int CS>
class SfmAligner
{
  static_assert(sizeof(Scalar) == sizeof(float), "only float is instantiated (cu_sfmaligner.cpp:209)");

public:
  typedef std::shared_ptr<SfmAligner<Scalar, CS>> Ptr;
  typedef JTJJrReductionItem<Scalar, 12 + CS> ReductionItem;
  typedef CorrespondenceReductionItem<Scalar> ErrorReductionItem;

  explicit SfmAligner(SfmAlignerParams params = SfmAlignerParams()) : params_(params), h_(detail::MakeHandle())
  {
    Upload();
  }
  virtual ~SfmAligner() {}

  template <typename SE3T, typename CamT, typename ImageBuffer, typename GradBuffer>
  ErrorReductionItem EvaluateError(const SE3T& pose0, const SE3T& pose1, const CamT& cam, const ImageBuffer& img0,
                                   const ImageBuffer& img1, const ImageBuffer& dpt0, const ImageBuffer& std0,
                                   const GradBuffer& grad1)
  {
    const DfkCamera c = detail::Cam(cam);
    const DfkImage i0 = detail::View(img0, 1), i1 = detail::View(img1, 1), d0 = detail::View(dpt0, 1);
    const DfkImage s0 = detail::View(std0, 1), g1 = detail::View(grad1, 2);
    ErrorReductionItem r;
    uint64_t inl = 0;
    detail::Check(h_.get(), dfk_sfm_evaluate_error(h_.get(), pose0.data(), pose1.data(), &c, &i0, &i1, &d0, &s0, &g1,
                                                   &r.residual, &inl));
    r.inliers = static_cast<std::size_t>(inl);
    return r;
  }

  template <typename SE3T, typename CodeT, typename CamT, typename ImageBuffer, typename GradBuffer>
  ReductionItem RunStep(const SE3T& pose0, const SE3T& pose1, const CodeT& code0, const CamT& cam,
                        const ImageBuffer& img0, const ImageBuffer& img1, const ImageBuffer& dpt0,
                        const ImageBuffer& std0, ImageBuffer& valid0, const ImageBuffer& prx0_jac,
                        const GradBuffer& grad1)
  {
    const DfkCamera c = detail::Cam(cam);
    const DfkImage i0 = detail::View(img0, 1), i1 = detail::View(img1, 1), d0 = detail::View(dpt0, 1);
    const DfkImage s0 = detail::View(std0, 1), v0 = detail::View(valid0, 1), g1 = detail::View(grad1, 2);
    const DfkImage jc = detail::View(prx0_jac, CS);
    ReductionItem r;
    uint64_t inl = 0;
    detail::Check(h_.get(), dfk_sfm_run_step(h_.get(), pose0.data(), pose1.data(), code0.data(), CS, &c, &i0, &i1, &d0,
                                              &s0, &v0, &jc, &g1, r.JtJ.coeff().data(), r.Jtr.data(), &r.residual,
                                              &inl));
    r.inliers = static_cast<std::size_t>(inl);
    return r;
  }

  // UpdateDepth + RunStep in one launch (what PhotometricFactor does back to back: UpdateDepthMaps,
  // photometric_factor.cpp:331-341, then RunAlignmentStep :267-274): dpt0 is decoded from prx_orig0 + prx0_jac * code0
  // inside the kernel, written to dpt0 (an output here) and used for the warp; the code Jacobian is read once.
  template <typename SE3T, typename CodeT, typename CamT, typename ImageBuffer, typename GradBuffer>
  ReductionItem RunStepDecodeDepth(const SE3T& pose0, const SE3T& pose1, const CodeT& code0, const CamT& cam,
                                   const ImageBuffer& img0, const ImageBuffer& img1, const ImageBuffer& prx_orig0,
                                   ImageBuffer& dpt0, ImageBuffer& valid0, const ImageBuffer& prx0_jac,
                                   const GradBuffer& grad1)
  {
    DfkSfmWorkItem w{};
    for (int k = 0; k < 7; ++k) {
      w.pose0[k] = pose0.data()[k];
      w.pose1[k] = pose1.data()[k];
    }
    w.cam = detail::Cam(cam);
    w.img0 = detail::View(img0, 1); w.img1 = detail::View(img1, 1); w.dpt0 = detail::View(dpt0, 1);
    w.valid0 = detail::View(valid0, 1); w.prx0_jac = detail::View(prx0_jac, CS); w.grad1 = detail::View(grad1, 2);
    w.prx_orig = detail::View(prx_orig0, 1);
    w.code = code0.data();
    std::vector<float> rec(DFK_SFM_RECORD_FLOATS(CS));
    detail::Check(h_.get(), dfk_sfm_run_step_batch_host(h_.get(), &w, 1, CS, rec.data()));
    ReductionItem r;
    constexpr int NP = 12 + CS, NH = NP * (NP + 1) / 2;
    for (int k = 0; k < NH; ++k) r.JtJ.coeff().data()[k] = rec[k];
    for (int k = 0; k < NP; ++k) r.Jtr.data()[k] = rec[NH + k];
    r.residual = rec[NH + NP];
    uint32_t bits;
    std::memcpy(&bits, &rec[NH + NP + 1], 4);
    r.inliers = bits;
    return r;
  }

#ifdef DFK_FACADE_CUDART
  // extension: the work item of one EvaluateError call, for EvaluateErrorBatch
  template <typename SE3T, typename CamT, typename ImageBuffer>
  static DfkSfmWorkItem ErrorItem(const SE3T& pose0, const SE3T& pose1, const CamT& cam, const ImageBuffer& img0,
                                  const ImageBuffer& img1, const ImageBuffer& dpt0)
  {
    DfkSfmWorkItem w{};
    for (int k = 0; k < 7; ++k) {
      w.pose0[k] = pose0.data()[k];
      w.pose1[k] = pose1.data()[k];
    }
    w.cam = detail::Cam(cam);
    w.img0 = detail::View(img0, 1); w.img1 = detail::View(img1, 1); w.dpt0 = detail::View(dpt0, 1);
    return w;
  }

  // extension: EvaluateError of many (pair, level) items in one launch (dfk_sfm_evaluate_error_batch), the error() half
  // of the PhotometricFactors of a window (photometric_factor.cpp:61-81); results in host memory after one synchronise.
  // Item i is bit for bit EvaluateError of that item alone.
  std::vector<ErrorReductionItem> EvaluateErrorBatch(const std::vector<DfkSfmWorkItem>& items)
  {
    std::vector<ErrorReductionItem> out(items.size());
    if (items.empty()) return out;
    const std::size_t bytes = sizeof(float) * 2 * items.size();
    float* dev = nullptr;
    if (cudaMalloc(reinterpret_cast<void**>(&dev), bytes) != cudaSuccess)
      throw std::runtime_error("[SfmAligner::EvaluateErrorBatch] device allocation failed");
    std::unique_ptr<float, cudaError_t (*)(void*)> guard(dev, cudaFree);
    detail::Check(h_.get(), dfk_sfm_evaluate_error_batch(h_.get(), items.data(), static_cast<int>(items.size()), dev));
    std::vector<float> host(2 * items.size());
    cudaStream_t s = static_cast<cudaStream_t>(dfk_get_stream(h_.get()));
    if (cudaMemcpyAsync(host.data(), dev, bytes, cudaMemcpyDeviceToHost, s) != cudaSuccess ||
        cudaStreamSynchronize(s) != cudaSuccess)
      throw std::runtime_error("[SfmAligner::EvaluateErrorBatch] result download failed");
    for (std::size_t i = 0; i < items.size(); ++i) {
      out[i].residual = host[2 * i];
      uint32_t bits;
      std::memcpy(&bits, &host[2 * i + 1], 4);
      out[i].inliers = bits;
    }
    return out;
  }
#endif

  void SetEvalThreadsBlocks(int threads, int blocks)
  {
    SfmAlignerParams p = params_;
    p.eval_threads = threads;
    p.eval_blocks = blocks;
    Upload(p);
  }
  void SetStepThreadsBlocks(int threads, int blocks)
  {
    SfmAlignerParams p = params_;
    p.step_threads = threads;
    p.step_blocks = blocks;
    Upload(p);
  }

  DfkHandle handle() const { return h_.get(); }  // extension: batched / asynchronous entry points of dfk.h
  // extension: launch on `stream` (a cudaStream_t; nullptr = the legacy default stream, the facade's default) or on the
  // handle's private non-blocking stream.  The caller then owns the ordering against its producers.
  void SetStream(void* stream) { detail::Check(h_.get(), dfk_set_stream(h_.get(), stream)); }
  void UseOwnStream() { detail::Check(h_.get(), dfk_use_own_stream(h_.get())); }

private:
  void Upload() { Upload(params_); }
  void Upload(const SfmAlignerParams& p)
  {
    DfkSfmAlignerParams c;
    c.sfmparams = DfkDenseSfmParams{p.sfmparams.huber_delta, p.sfmparams.ocl_th, p.sfmparams.avg_dpt,
                                    p.sfmparams.min_dpt, p.sfmparams.valid_border};
    c.step_threads = p.step_threads;
    c.step_blocks = p.step_blocks;
    c.eval_threads = p.eval_threads;
    c.eval_blocks = p.eval_blocks;
    detail::Check(h_.get(), dfk_sfm_set_params(h_.get(), &c));  // throws on threads % 32 != 0 / blocks > 1024
    params_ = p;
  }

  static const int max_blocks = 1024;
  SfmAlignerParams params_;
  detail::HandlePtr h_;
};

// ---------------------------------------------------------------------------------------------
// df::DepthAligner<Scalar, CS>  (cu_depthaligner.h:38-54)
// ---------------------------------------------------------------------------------------------
template <typename Scalar, int CS>
class DepthAligner
{
  static_assert(sizeof(Scalar) == sizeof(float), "only float is instantiated (cu_depthaligner.cpp:118)");

public:
  typedef std::shared_ptr<DepthAligner<Scalar, CS>> Ptr;
  typedef JTJJrReductionItem<Scalar, CS> ReductionItem;

  DepthAligner() : h_(detail::MakeHandle()) {}
  virtual ~DepthAligner() {}

  // cu_depthaligner.cpp:83-113; CodeT = Eigen::Matrix<Scalar,CS,1> (anything with data()), ImageBuffer = vc::Image2DView
  template <typename CodeT, typename ImageBuffer>
  ReductionItem RunStep(const CodeT& code, const ImageBuffer& target_dpt, const ImageBuffer& prx_orig,
                        const ImageBuffer& prx_jac)
  {
    const DfkImage t = detail::View(target_dpt, 1), p = detail::View(prx_orig, 1), j = detail::View(prx_jac, CS);
    ReductionItem r;
    uint64_t inl = 0;
    detail::Check(h_.get(), dfk_depth_run_step(h_.get(), code.data(), CS, &t, &p, &j, r.JtJ.coeff().data(), r.Jtr.data(),
                                               &r.residual, &inl));
    r.inliers = static_cast<std::size_t>(inl);
    return r;
  }
  DfkHandle handle() const { return h_.get(); }
  void SetStream(void* stream) { detail::Check(h_.get(), dfk_set_stream(h_.get(), stream)); }

private:
  detail::HandlePtr h_;
};

// ---------------------------------------------------------------------------------------------
// df::SE3Aligner<Scalar>  (cu_se3aligner.h:38-86)
// ---------------------------------------------------------------------------------------------
template <typename Scalar>
class SE3Aligner
{
  static_assert(sizeof(Scalar) == sizeof(float), "only float is instantiated (cu_se3aligner.cpp:179)");

public:
  typedef std::shared_ptr<SE3Aligner<Scalar>> Ptr;
  typedef JTJJrReductionItem<Scalar, 6> ReductionItem;
  typedef CorrespondenceReductionItem<Scalar> CorrespondenceItem;

  SE3Aligner() : h_(detail::MakeHandle()) {}
  virtual ~SE3Aligner() {}

  // Renders img0 from image img1 at pose T_01
  template <typename SE3T, typename CamT, typename ImageBuffer>
  CorrespondenceItem Warp(const SE3T& se3, const CamT& cam, const ImageBuffer& img0, const ImageBuffer& img1,
                          const ImageBuffer& dpt0, ImageBuffer& img2)
  {
    const DfkCamera c = detail::Cam(cam);
    const DfkImage i0 = detail::View(img0, 1), i1 = detail::View(img1, 1), d0 = detail::View(dpt0, 1);
    const DfkImage i2 = detail::View(img2, 1);
    CorrespondenceItem r;
    uint64_t inl = 0;
    detail::Check(h_.get(), dfk_se3_warp(h_.get(), se3.data(), &c, &i0, &i1, &d0, &i2, &r.residual, &inl));
    r.inliers = static_cast<std::size_t>(inl);
    return r;
  }

  template <typename SE3T, typename CamT, typename ImageBuffer, typename GradBuffer>
  ReductionItem RunStep(const SE3T& se3, const CamT& cam, const ImageBuffer& img0, const ImageBuffer& img1,
                        const ImageBuffer& dpt0, const GradBuffer& grad1)
  {
    const DfkCamera c = detail::Cam(cam);
    const DfkImage i0 = detail::View(img0, 1), i1 = detail::View(img1, 1), d0 = detail::View(dpt0, 1);
    const DfkImage g1 = detail::View(grad1, 2);
    ReductionItem r;
    uint64_t inl = 0;
    detail::Check(h_.get(), dfk_se3_run_step(h_.get(), se3.data(), &c, &i0, &i1, &d0, &g1, r.JtJ.coeff().data(),
                                              r.Jtr.data(), &r.residual, &inl));
    r.inliers = static_cast<std::size_t>(inl);
    return r;
  }

  DfkHandle handle() const { return h_.get(); }
  void SetStream(void* stream) { detail::Check(h_.get(), dfk_set_stream(h_.get(), stream)); }  // see SfmAligner::SetStream
  void UseOwnStream() { detail::Check(h_.get(), dfk_use_own_stream(h_.get())); }
  void SetHuberDelta(float val)
  {
    huber_delta_ = val;
    detail::Check(h_.get(), dfk_se3_set_huber_delta(h_.get(), val));
  }

  // The loop of CameraTracker::TrackFrame (core/system/camera_tracker.cpp:48-70) as ONE call: for level =
  // levels-1 .. 0, iterations_per_level[level] times { RunStep; update = -JtJ.ldlt().solve(Jtr); t += update.head<3>();
  // so3 = exp(update.tail<3>()) * so3 } with the solve and the retraction done on the device and a single read-back.
  // The pyramids are anything indexable by level (vc::RuntimeBufferPyramidManaged::operator[], std::vector of
  // views, SyncedBufferPyramid::GetGpuLevel results collected in a vector); camera_pyr[level] is the level's camera.
  // pose_ck is updated in place; returns {inliers / area, residual / inliers} of the last evaluated system, the two
  // numbers TrackFrame stores in inliers_ / error_ (:65-69).
  template <typename SE3T, typename CamPyr, typename ImagePyr0, typename ImagePyr1, typename DepthPyr, typename GradPyr>
  std::pair<float, float> TrackLevels(SE3T& pose_ck, const CamPyr& camera_pyr, const ImagePyr0& pyr_img0,
                                      const ImagePyr1& pyr_img1, const DepthPyr& pyr_dpt0, const GradPyr& pyr_grad1,
                                      const std::vector<int>& iterations_per_level)
  {
    std::vector<DfkTrackLevel> lv(iterations_per_level.size());
    for (std::size_t l = 0; l < lv.size(); ++l) {
      lv[l].cam = detail::Cam(camera_pyr[l]);
      lv[l].img0 = detail::View(pyr_img0[l], 1);
      lv[l].img1 = detail::View(pyr_img1[l], 1);
      lv[l].dpt0 = detail::View(pyr_dpt0[l], 1);
      lv[l].grad1 = detail::View(pyr_grad1[l], 2);
      lv[l].iterations = iterations_per_level[l];
    }
    float frac = 0.f, err = 0.f;
    detail::Check(h_.get(), dfk_se3_track(h_.get(), pose_ck.data(), lv.data(), static_cast<int>(lv.size()), &frac, &err,
                                          nullptr, nullptr, 0));
    return std::make_pair(frac, err);
  }

  // TrackLevels against many keyframes at once, the live frame (pyr_img1, pyr_grad1) shared: the loops of
  // DeepFactors::Relocalize (core/deepfactors.cpp:713-743) and of LoopDetector::DetectLoop's geometry check
  // (core/system/loop_detector.cpp:149-168) as ONE call.  kf_img_pyrs[n] / kf_dpt_pyrs[n] are keyframe n's pyramids,
  // poses_ck[n] its start pose (identity = what Reset does), updated in place.  Every Gauss-Newton iteration is one launch
  // for all keyframes.  Returns one {inliers / area, residual / inliers} per keyframe, bit for bit what TrackLevels gives
  // for that keyframe alone.
  template <typename SE3T, typename CamPyr, typename ImagePyrs0, typename ImagePyr1, typename DepthPyrs, typename GradPyr>
  std::vector<std::pair<float, float>> TrackLevelsBatch(std::vector<SE3T>& poses_ck, const CamPyr& camera_pyr,
                                                        const ImagePyrs0& kf_img_pyrs, const ImagePyr1& pyr_img1,
                                                        const DepthPyrs& kf_dpt_pyrs, const GradPyr& pyr_grad1,
                                                        const std::vector<int>& iterations_per_level)
  {
    const std::size_t n = poses_ck.size(), L = iterations_per_level.size();
    if (kf_img_pyrs.size() != n || kf_dpt_pyrs.size() != n)
      throw std::runtime_error("SE3Aligner::TrackLevelsBatch: one image and one depth pyramid per pose expected");
    std::vector<DfkTrackLevel> lv(n * L);
    std::vector<float> poses(n * 7);
    for (std::size_t k = 0; k < n; ++k) {
      for (std::size_t l = 0; l < L; ++l) {
        DfkTrackLevel& t = lv[k * L + l];
        t.cam = detail::Cam(camera_pyr[l]);
        t.img0 = detail::View(kf_img_pyrs[k][l], 1);
        t.img1 = detail::View(pyr_img1[l], 1);
        t.dpt0 = detail::View(kf_dpt_pyrs[k][l], 1);
        t.grad1 = detail::View(pyr_grad1[l], 2);
        t.iterations = iterations_per_level[l];
      }
      std::copy(poses_ck[k].data(), poses_ck[k].data() + 7, poses.begin() + 7 * k);
    }
    std::vector<float> frac(n, 0.f), err(n, 0.f);
    detail::Check(h_.get(), dfk_se3_track_batch(h_.get(), static_cast<int>(n), static_cast<int>(L), poses.data(),
                                                lv.data(), frac.data(), err.data(), nullptr));
    std::vector<std::pair<float, float>> stats(n);
    for (std::size_t k = 0; k < n; ++k) {
      std::copy(poses.begin() + 7 * k, poses.begin() + 7 * (k + 1), poses_ck[k].data());
      stats[k] = std::make_pair(frac[k], err[k]);
    }
    return stats;
  }

private:
  detail::HandlePtr h_;
  float huber_delta_ = 0.1f;
};

// ---------------------------------------------------------------------------------------------
// extension (no reference counterpart): a keyframe window problem and its Levenberg-Marquardt loop in the library
// (dfk_window_problem_*, dfk_window_lm).  The reference's integrator restages every factor on every ISAM2 iteration
// (mapper.cpp:518-519); here the items are staged once and only the state (poses and codes, fp64) changes.  RAII over
// the C object; every call runs on the handle given at construction (e.g. SfmAligner<float, CS>::handle()), whose
// sfmparams, Gram mode and SM limit at construction the problem keeps.  num_keyframes / num_frames are the window's.
// ---------------------------------------------------------------------------------------------
struct WindowError {  // window_opt.WindowError: each part summed in fp64 in factor order (buffer units)
  double energy = 0.0, photometric = 0.0, reprojection = 0.0, geometric = 0.0, priors = 0.0;
  int64_t no_inliers = 0, inliers = 0;
};

struct LMParams {  // window_opt.LMParams (the linearisation cache's eps has no counterpart: every factor is re-evaluated)
  int iterations = 10;
  double lambda_init = 1e-4, lambda_up = 10.0, lambda_down = 0.1, lambda_max = 1e6;
  bool fix_first_pose = true;
  double code_prior_weight = 0.0;
  bool use_error = false;  // evaluate E at every candidate, linearise accepted points only
};

struct LMTrace {  // window_opt.LMTrace
  std::vector<double> energy, lambda;
  std::vector<bool> accepted;
  int linearisations = 0, error_evaluations = 0;
};

// window_opt.LevelSchedule in the C ABI's terms (DfkLevelSchedule): pairs are the distinct window pairs of the dense
// items; error_pair / error_level empty: error item i follows dense item i; pair_remove_after empty: no pair leaves
struct LevelSchedule {
  std::vector<int32_t> iters, dense_level, error_pair, error_level, pair_steps_done;
  std::vector<uint8_t> pair_remove_after;
};
struct Isam2Params {  // window_opt.IncrementalOptimizer's parameters (dfk_window_problem_isam2_update)
  double relinearize_threshold = 0.05;
  int relinearize_skip = 1;
  double code_prior_weight = 0.0;
  bool fix_first_pose = true;
};
struct Isam2Result {  // gtsam::ISAM2Result's counts
  int variables_relinearized = 0, variables_reeliminated = 0, factors_relinearised = 0, first_column = 0;
  bool operator==(const Isam2Result& o) const
  {
    return variables_relinearized == o.variables_relinearized && variables_reeliminated == o.variables_reeliminated &&
           factors_relinearised == o.factors_relinearised && first_column == o.first_column;
  }
};

struct LevelTrace {  // DfkLevelTrace
  std::vector<double> switch_energy;
  std::vector<std::vector<int32_t>> pair_levels;  // [step][pair], -1: off
  std::vector<int32_t> pair_steps_done;
};

template <int CS>
class WindowProblem
{
public:
  WindowProblem(DfkHandle h, const DfkWindowProblemDesc& desc, int num_keyframes, int num_frames)
    : h_(h), K_(num_keyframes), F_(num_frames), nd_(desc.num_dense), ne_(desc.num_error)
  {
    if (!h || num_keyframes < 1 || num_frames < 0)
      throw std::invalid_argument("[WindowProblem] null handle / no keyframes / negative frame count");
    detail::Check(h_, dfk_window_problem_create(h_, &desc, &p_));
  }
  ~WindowProblem() { dfk_window_problem_destroy(h_, p_); }
  WindowProblem(const WindowProblem&) = delete;
  WindowProblem& operator=(const WindowProblem&) = delete;

  DfkWindowProblem* get() const { return p_; }

  // poses: (K + F) x 7 (keyframes, then frames; Sophus::SE3 data() order), codes: K x CS, host
  void SetState(const std::vector<double>& poses, const std::vector<double>& codes)
  {
    if (poses.size() != (size_t)(K_ + F_) * 7 || codes.size() != (size_t)K_ * CS)
      throw std::invalid_argument("[WindowProblem] the state is (K + F) x 7 pose and K x CS code doubles");
    detail::Check(h_, dfk_window_problem_set_state(h_, p_, poses.data(), codes.data()));
    detail::Check(h_, dfk_synchronize(h_));  // the host vectors may go away when this returns
  }
  void GetState(std::vector<double>& poses, std::vector<double>& codes) const
  {
    poses.resize((size_t)(K_ + F_) * 7);
    codes.resize((size_t)K_ * CS);
    detail::Check(h_, dfk_window_problem_get_state(h_, p_, poses.data(), codes.data()));
    detail::Check(h_, dfk_synchronize(h_));
  }
  // the window buffer at the state into window_dev (DEVICE, dfk_window_floats floats); asynchronous
  void Linearize(float* window_dev) { detail::Check(h_, dfk_window_problem_linearize(h_, p_, window_dev)); }
#ifdef DFK_FACADE_CUDART
  // the energy at the state without linearising; synchronous (one small read-back with the CUDA runtime)
  WindowError Error()
  {
    double* dev = nullptr;
    if (cudaMalloc(&dev, sizeof(double) * DFK_WINDOW_ERROR_DOUBLES) != cudaSuccess)
      throw std::runtime_error("[WindowProblem::Error] device allocation failed");
    double o[DFK_WINDOW_ERROR_DOUBLES] = {};
    DfkStatus st = dfk_window_problem_error(h_, p_, dev);
    if (st == DFK_OK) st = dfk_synchronize(h_);
    const cudaError_t e = st == DFK_OK ? cudaMemcpy(o, dev, sizeof(o), cudaMemcpyDeviceToHost) : cudaSuccess;
    cudaFree(dev);
    detail::Check(h_, st);
    if (e != cudaSuccess) throw std::runtime_error("[WindowProblem::Error] result download failed");
    WindowError r;
    r.energy = o[0]; r.photometric = o[1]; r.reprojection = o[2]; r.geometric = o[3]; r.priors = o[4];
    r.no_inliers = (int64_t)o[5]; r.inliers = (int64_t)o[6];
    return r;
  }
#endif
  // Levenberg-Marquardt from the state (dfk_window_lm); the state is the last accepted point afterwards
  LMTrace Optimize(const LMParams& p)
  {
    if (p.iterations < 0) throw std::invalid_argument("[WindowProblem::Optimize] iterations < 0");
    const DfkLMParams c{p.iterations, p.lambda_init, p.lambda_up, p.lambda_down, p.lambda_max, p.fix_first_pose ? 1 : 0,
                        p.code_prior_weight, p.use_error ? 1 : 0};
    std::vector<double> e(p.iterations + 1), lam(std::max(p.iterations, 1));
    std::vector<int32_t> acc(std::max(p.iterations, 1));
    DfkLMTrace t{e.data(), lam.data(), acc.data(), 0, 0, 0, 0};
    detail::Check(h_, dfk_window_lm(h_, p_, &c, &t));
    LMTrace r;
    r.energy.assign(e.begin(), e.begin() + t.num_energies);
    r.lambda.assign(lam.begin(), lam.begin() + t.num_steps);
    for (int i = 0; i < t.num_steps; ++i) r.accepted.push_back(acc[i] != 0);
    r.linearisations = t.linearisations;
    r.error_evaluations = t.error_evaluations;
    return r;
  }

  // the active dense and error items (dfk_window_problem_set_active); error_active empty: the dense mask, which needs
  // as many error as dense items.  The masks hold for Linearize, Error, Optimize and OptimizeLevels until the next call
  void SetActive(const std::vector<uint8_t>& dense_active, const std::vector<uint8_t>& error_active = {})
  {
    if (dense_active.size() != (size_t)nd_ || (!error_active.empty() && error_active.size() != (size_t)ne_))
      throw std::invalid_argument("[WindowProblem::SetActive] one byte per dense item and per error item");
    detail::Check(h_, dfk_window_problem_set_active(h_, p_, dense_active.data(),
                                                    error_active.empty() ? nullptr : error_active.data()));
  }
  // Levenberg-Marquardt coarse to fine (dfk_window_lm_levels); the problem keeps the masks of the last step
  LMTrace OptimizeLevels(const LMParams& p, const LevelSchedule& s, LevelTrace* lt = nullptr)
  {
    if (p.iterations < 0) throw std::invalid_argument("[WindowProblem::OptimizeLevels] iterations < 0");
    const size_t P = s.pair_steps_done.size();
    if (s.iters.empty() || s.dense_level.size() != (size_t)nd_ ||
        (!s.error_pair.empty() && s.error_pair.size() != (size_t)ne_) ||
        (!s.error_level.empty() && s.error_level.size() != (size_t)ne_) ||
        (!s.pair_remove_after.empty() && s.pair_remove_after.size() != P))
      throw std::invalid_argument("[WindowProblem::OptimizeLevels] schedule arrays of the wrong length");
    const DfkLMParams c{p.iterations, p.lambda_init, p.lambda_up, p.lambda_down, p.lambda_max, p.fix_first_pose ? 1 : 0,
                        p.code_prior_weight, p.use_error ? 1 : 0};
    const DfkLevelSchedule cs{(int32_t)s.iters.size(), s.iters.data(), s.dense_level.data(),
                              s.error_pair.empty() ? nullptr : s.error_pair.data(),
                              s.error_level.empty() ? nullptr : s.error_level.data(), (int32_t)P,
                              s.pair_steps_done.data(), s.pair_remove_after.empty() ? nullptr : s.pair_remove_after.data()};
    const int it = std::max(p.iterations, 1);
    std::vector<double> e(p.iterations + 1), lam(it), sw(it);
    std::vector<int32_t> acc(it), lv((size_t)it * std::max<size_t>(P, 1)), done(std::max<size_t>(P, 1));
    DfkLMTrace t{e.data(), lam.data(), acc.data(), 0, 0, 0, 0};
    DfkLevelTrace l{sw.data(), lv.data(), done.data(), 0};
    detail::Check(h_, dfk_window_lm_levels(h_, p_, &c, &cs, &t, &l));
    LMTrace r;
    r.energy.assign(e.begin(), e.begin() + t.num_energies);
    r.lambda.assign(lam.begin(), lam.begin() + t.num_steps);
    for (int i = 0; i < t.num_steps; ++i) r.accepted.push_back(acc[i] != 0);
    r.linearisations = t.linearisations;
    r.error_evaluations = t.error_evaluations;
    if (lt) {
      lt->switch_energy.assign(sw.begin(), sw.begin() + l.num_switches);
      lt->pair_levels.clear();
      for (int i = 0; i < t.num_steps; ++i) lt->pair_levels.emplace_back(lv.begin() + i * P, lv.begin() + (i + 1) * P);
      lt->pair_steps_done.assign(done.begin(), done.begin() + P);
    }
    return r;
  }

  // one ISAM2 update (dfk_window_problem_isam2_update): the state becomes theta_lin (+) delta; synchronous
  Isam2Result UpdateIncremental(const Isam2Params& p)
  {
    const DfkIsam2Params c = params(p);
    DfkIsam2Result r{};
    detail::Check(h_, dfk_window_problem_isam2_update(h_, p_, &c, &r));
    return Isam2Result{r.variables_relinearized, r.variables_reeliminated, r.factors_relinearised, r.first_column};
  }
  // theta_lin ((K + F) x 7, K x CS) and delta (K (6 + CS) + 6 F) of the last update, host
  void GetLinearization(std::vector<double>& poses, std::vector<double>& codes, std::vector<double>& delta) const
  {
    poses.resize((size_t)(K_ + F_) * 7);
    codes.resize((size_t)K_ * CS);
    delta.resize((size_t)K_ * (6 + CS) + 6 * (size_t)F_);
    detail::Check(h_, dfk_window_problem_get_linearization(h_, p_, poses.data(), codes.data(), delta.data()));
    detail::Check(h_, dfk_synchronize(h_));
  }
  // up to max_steps mapping steps (dfk_window_map_steps) with the works of s's pairs (read and written; empty: fresh
  // works); per step the ISAM2 counts, and in pair_levels every pair's factor level
  std::vector<Isam2Result> MappingSteps(const Isam2Params& p, const LevelSchedule& s, std::vector<DfkWorkState>& works,
                                        int max_steps, std::vector<std::vector<int>>* pair_levels = nullptr)
  {
    const size_t P = s.pair_remove_after.size();
    if (max_steps < 0 || s.iters.empty() || s.dense_level.size() != (size_t)nd_ ||
        (!s.error_pair.empty() && s.error_pair.size() != (size_t)ne_) ||
        (!s.error_level.empty() && s.error_level.size() != (size_t)ne_) || (!works.empty() && works.size() != P))
      throw std::invalid_argument("[WindowProblem::MappingSteps] schedule or works of the wrong length");
    const DfkIsam2Params c = params(p);
    const DfkLevelSchedule cs{(int32_t)s.iters.size(), s.iters.data(), s.dense_level.data(),
                              s.error_pair.empty() ? nullptr : s.error_pair.data(),
                              s.error_level.empty() ? nullptr : s.error_level.data(), (int32_t)P, nullptr,
                              P ? s.pair_remove_after.data() : nullptr};
    if (s.iters.size() > DFK_MAX_WORK_LEVELS)
      throw std::invalid_argument("[WindowProblem::MappingSteps] more than DFK_MAX_WORK_LEVELS levels");
    if (works.empty()) {  // fresh works: OptimizeWork's constructor
      DfkWorkState f{};
      f.active_level = (int32_t)s.iters.size() - 1;
      for (size_t l = 0; l < s.iters.size(); ++l) f.iters[l] = s.iters[l];
      f.first = 1;
      f.factor = -1;
      works.assign(P, f);
    }
    std::vector<DfkWorkState> w(works);
    w.resize(std::max<size_t>(P, 1));
    const size_t n = std::max(max_steps, 1);
    std::vector<int32_t> a(n), b(n), f(n), j(n), lv(n * std::max<size_t>(P, 1));
    DfkMapTrace t{a.data(), b.data(), f.data(), j.data(), lv.data(), 0};
    detail::Check(h_, dfk_window_map_steps(h_, p_, &c, &cs, w.data(), max_steps, &t));
    std::vector<Isam2Result> r;
    for (int i = 0; i < t.num_steps; ++i) r.push_back(Isam2Result{a[i], b[i], f[i], j[i]});
    if (pair_levels) {
      pair_levels->clear();
      for (int i = 0; i < t.num_steps; ++i) pair_levels->emplace_back(lv.begin() + i * P, lv.begin() + (i + 1) * P);
    }
    std::copy(w.begin(), w.begin() + P, works.begin());
    return r;
  }
  // continue old's ISAM2 run on this grown problem (dfk_window_problem_grow_from); set this problem's state first
  void GrowFrom(const WindowProblem& old, const std::vector<int32_t>& dense_of, const std::vector<int32_t>& rep_of,
                const std::vector<int32_t>& geo_of, const std::vector<int32_t>& frame_of)
  {
    if (dense_of.size() != (size_t)nd_ || frame_of.size() != (size_t)F_)
      throw std::invalid_argument("[WindowProblem::GrowFrom] one map entry per dense item and per frame");
    detail::Check(h_, dfk_window_problem_grow_from(h_, p_, old.p_, dense_of.data(), rep_of.data(), geo_of.data(),
                                                   frame_of.data()));
  }

private:
  static DfkIsam2Params params(const Isam2Params& p)
  {
    return DfkIsam2Params{p.relinearize_threshold, p.relinearize_skip, p.code_prior_weight, p.fix_first_pose ? 1 : 0};
  }
  DfkHandle h_;
  int K_, F_, nd_, ne_;
  DfkWindowProblem* p_ = nullptr;
};

// ---------------------------------------------------------------------------------------------
// cu_image_proc.h:27-44 free functions.  They use one process-wide handle (default stream semantics
// of the reference); pass an explicit handle to run them on another stream.
// ---------------------------------------------------------------------------------------------
namespace detail
{
inline DfkHandle DefaultHandle()
{
  static HandlePtr h = MakeHandle();
  return h.get();
}
}  // namespace detail

template <typename ImageBuf, typename GradBuf>
void SobelGradients(const ImageBuf& img, GradBuf& grad)
{
  const DfkImage i = detail::View(img, 1), g = detail::View(grad, 2);
  detail::Check(detail::DefaultHandle(), dfk_sobel_gradients(detail::DefaultHandle(), &i, &g));
  detail::Check(detail::DefaultHandle(), dfk_synchronize(detail::DefaultHandle()));  // launch_utils.h:28
}

template <typename ImageBuf>
void GaussianBlurDown(const ImageBuf& in, ImageBuf& out)
{
  const DfkImage i = detail::View(in, 1), o = detail::View(out, 1);
  detail::Check(detail::DefaultHandle(), dfk_gaussian_blur_down(detail::DefaultHandle(), &i, &o));
  detail::Check(detail::DefaultHandle(), dfk_synchronize(detail::DefaultHandle()));
}

template <typename ImageBuf>
float SquaredError(const ImageBuf& buf1, const ImageBuf& buf2)
{
  const DfkImage a = detail::View(buf1, 1), b = detail::View(buf2, 1);
  float out = 0.f;
  detail::Check(detail::DefaultHandle(), dfk_squared_error(detail::DefaultHandle(), &a, &b, &out));
  return out;
}

template <typename CodeT, typename ImageBuf>
void UpdateDepth(const CodeT& code, const ImageBuf& prx_orig, const ImageBuf& prx_jac, float avg_dpt, ImageBuf& dpt_out)
{
  const int cs = static_cast<int>(code.size());
  const DfkImage p = detail::View(prx_orig, 1), d = detail::View(dpt_out, 1);
  const DfkImage j = detail::View(prx_jac, static_cast<unsigned>(cs));
  detail::Check(detail::DefaultHandle(),
                dfk_update_depth(detail::DefaultHandle(), code.data(), cs, &p, &j, avg_dpt, &d));
  detail::Check(detail::DefaultHandle(), dfk_synchronize(detail::DefaultHandle()));
}

}  // namespace df

#endif  // DFK_FACADE_H_
