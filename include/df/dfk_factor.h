// dfk_factor.h -- the consumer side of the hot path, in C++: what df::PhotometricFactor does with an aligner result
// and how a window of such results becomes one set of normal equations.  Host-only, header-only, no GTSAM / Eigen.
//
//   LinearizePhotometric   PhotometricFactor::linearize + RunAlignmentStep's post-processing
//                          (sources/core/gtsam/photometric_factor.cpp:84-181, 223-293): the residual rescale
//                          res / inliers * W * H (:275-282; +inf when there is no overlap), JtJ cast to double, Jtr negated
//                          (:105-106), and the slicing into the HessianFactor blocks G11 G12 G13 G22 G23 G33 / g1 g2 g3
//                          (:126-161) in the aligner's column order [pose0 | pose1 | code0].
//   WindowSystem           the block-sparse -> dense normal equations of a keyframe window (SURVEY 8e): variables
//                          [pose_k (6) | code_k (C)] per keyframe; a pair (k0 -> k1) adds its pose0 / code0 blocks to
//                          keyframe k0's diagonal block, pose1 to k1's, and the pose0-pose1 / pose1-code0 couplings off the
//                          diagonal.  The buffer is what one NCCL all-reduce sums across ranks.
//   LinearizeReprojectionBatch
//                          many reprojection factors (loop closures, use_reprojection links) linearised in one launch
//                          straight into device records [A^T A | -A^T b | b^T b | inliers] (WindowSystem::AddUnscaled).
//   LinearizeSparseGeometricBatch
//                          many sparse geometric factors (use_geometric links) linearised in one launch into device
//                          records over [pose0 | pose1 | code0 | code1] (WindowSystem::AddGeometric).
//   DepthPriorFactor       DepthPriorFactor (depth_prior_factor.cpp:29-137): a keyframe code's pull towards a measured depth
//                          pyramid, every level linearised in one dfk_depth_prior_linearize_batch call
//                          (WindowSystem::AddDepthPrior, or dfk_window_add_depth_priors on the device).
//   LinearizeReprojection / LinearizeSparseGeometric
//                          the Jacobian rows of the two sparse factors (reprojection_factor.cpp:157-269,
//                          sparse_geometric_factor.cpp:157-271), evaluated on the device from the keyframes' GPU buffers;
//                          the caller copies the row blocks into gtsam::VerticalBlockMatrix Ab(0..) as the reference does.
// deepfactors_b200/factors.py is the Python mirror; tests/cpp/factor_test.cpp checks the two against each other.
#ifndef DFK_FACTOR_H_
#define DFK_FACTOR_H_

#include <cstddef>
#include <limits>
#include <utility>
#include <vector>

#include "dfk_facade.h"

namespace df
{

// row-major dense blocks, double like the reference's cast (photometric_factor.cpp:105)
template <int CS>
struct PhotometricBlocks {
  std::vector<double> G11, G12, G13, G22, G23, G33;  // 6x6, 6x6, 6xCS, 6x6, 6xCS, CSxCS
  std::vector<double> g1, g2, g3;                    // 6, 6, CS   (= -Jtr blocks)
  double f = 0.0;                                    // rescaled residual energy
};

template <int CS>
PhotometricBlocks<CS> LinearizePhotometric(const JTJJrReductionItem<float, 12 + CS>& sys, int width, int height)
{
  constexpr int NP = 12 + CS;
  PhotometricBlocks<CS> b;
  auto block = [&](int r0, int nr, int c0, int nc) {
    std::vector<double> m(static_cast<std::size_t>(nr) * nc);
    for (int r = 0; r < nr; ++r)
      for (int c = 0; c < nc; ++c) m[static_cast<std::size_t>(r) * nc + c] = static_cast<double>(sys.JtJ.toDenseMatrix(r0 + r, c0 + c));
    return m;
  };
  b.G11 = block(0, 6, 0, 6);
  b.G12 = block(0, 6, 6, 6);
  b.G13 = block(0, 6, 12, CS);
  b.G22 = block(6, 6, 6, 6);
  b.G23 = block(6, 6, 12, CS);
  b.G33 = block(12, CS, 12, CS);
  b.g1.resize(6);
  b.g2.resize(6);
  b.g3.resize(CS);
  for (int k = 0; k < 6; ++k) {
    b.g1[k] = -static_cast<double>(sys.Jtr[k]);
    b.g2[k] = -static_cast<double>(sys.Jtr[6 + k]);
  }
  for (int k = 0; k < CS; ++k) b.g3[k] = -static_cast<double>(sys.Jtr[12 + k]);
  static_assert(NP == 12 + CS, "column order [pose0 | pose1 | code0]");
  b.f = sys.inliers > 0 ? static_cast<double>(sys.residual) / static_cast<double>(sys.inliers) * width * height
                        : std::numeric_limits<double>::infinity();
  return b;
}

// Dense normal equations of a window of `num_keyframes` keyframes.
template <int CS>
class WindowSystem
{
public:
  static constexpr int Block = 6 + CS;
  explicit WindowSystem(int num_keyframes)
      : n_(num_keyframes), H_(static_cast<std::size_t>(dim()) * dim(), 0.0), g_(dim(), 0.0), f_(0.0)
  {
  }
  int dim() const { return n_ * Block; }
  double& H(int r, int c) { return H_[static_cast<std::size_t>(r) * dim() + c]; }
  double H(int r, int c) const { return H_[static_cast<std::size_t>(r) * dim() + c]; }
  std::vector<double>& H() { return H_; }
  std::vector<double>& g() { return g_; }
  const std::vector<double>& g() const { return g_; }
  double f() const { return f_; }

  // pair (k0 -> k1): keyframe k0 is warped into frame k1 (pose0 / code0 belong to k0, pose1 to k1)
  void Add(int k0, int k1, const JTJJrReductionItem<float, 12 + CS>& sys, int width, int height)
  {
    AddBlocks(k0, k1, sys);
    if (sys.inliers > 0) f_ += static_cast<double>(sys.residual) / static_cast<double>(sys.inliers) * width * height;
  }

  // a reprojection factor (k0 -> k1) as a record of LinearizeReprojectionBatch: same blocks, its residual b^T b enters f
  // as it is (no photometric rescale)
  void AddUnscaled(int k0, int k1, const JTJJrReductionItem<float, 12 + CS>& sys)
  {
    AddBlocks(k0, k1, sys);
    f_ += static_cast<double>(sys.residual);
  }

  // a sparse geometric factor (k0 -> k1) as a record of LinearizeSparseGeometricBatch, variables [pose0 | pose1 | code0 |
  // code1]: the blocks of all four (pose0 / code0 belong to k0, pose1 / code1 to k1) -- the HessianFactor over four
  // keys that replaces the JacobianFactor -- and f += b^T b
  void AddGeometric(int k0, int k1, const JTJJrReductionItem<float, 12 + 2 * CS>& sys)
  {
    const int off[4] = {k0 * Block, k1 * Block, k0 * Block + 6, k1 * Block + 6};  // pose0, pose1, code0, code1
    const int loc[4] = {0, 6, 12, 12 + CS};
    const int len[4] = {6, 6, CS, CS};
    for (int a = 0; a < 4; ++a) {
      for (int r = 0; r < len[a]; ++r) {
        g_[off[a] + r] -= static_cast<double>(sys.Jtr[loc[a] + r]);
        for (int b = 0; b < 4; ++b)
          for (int c = 0; c < len[b]; ++c)
            H(off[a] + r, off[b] + c) += static_cast<double>(sys.JtJ.toDenseMatrix(loc[a] + r, loc[b] + c));
      }
    }
    f_ += static_cast<double>(sys.residual);
  }

  // one level's record of DepthPriorFactor::Linearize on keyframe k ([JtJ packed upper | Jtr | residual | inliers],
  // DFK_DEPTH_RECORD_FLOATS(CS)): JtJ / sigma^2 to k's code block, -Jtr / sigma^2 to its code gradient and
  // residual / sigma^2 to f (f is twice the factor-graph error, as everywhere in this system)
  void AddDepthPrior(int k, const float* record, float sigma)
  {
    const double s2 = static_cast<double>(sigma) * static_cast<double>(sigma);
    const int o = k * Block + 6;
    int e = 0;
    for (int i = 0; i < CS; ++i)
      for (int j = i; j < CS; ++j, ++e) {
        H(o + i, o + j) += static_cast<double>(record[e]) / s2;
        if (j != i) H(o + j, o + i) += static_cast<double>(record[e]) / s2;
      }
    for (int i = 0; i < CS; ++i) g_[o + i] -= static_cast<double>(record[e + i]) / s2;
    f_ += static_cast<double>(record[e + CS]) / s2;
  }

private:
  void AddBlocks(int k0, int k1, const JTJJrReductionItem<float, 12 + CS>& sys)
  {
    const int off[3] = {k0 * Block, k1 * Block, k0 * Block + 6};  // pose0, pose1, code0
    const int loc[3] = {0, 6, 12};
    const int len[3] = {6, 6, CS};
    for (int a = 0; a < 3; ++a) {
      for (int r = 0; r < len[a]; ++r) {
        g_[off[a] + r] -= static_cast<double>(sys.Jtr[loc[a] + r]);
        for (int b = 0; b < 3; ++b)
          for (int c = 0; c < len[b]; ++c)
            H(off[a] + r, off[b] + c) += static_cast<double>(sys.JtJ.toDenseMatrix(loc[a] + r, loc[b] + c));
      }
    }
  }

  int n_;
  std::vector<double> H_, g_;
  double f_;
};

// contiguous, balanced shard of the pair list for `rank` (sizes differ by at most one): pairs shard across GPUs with
// no data-path collective, the window buffers of the ranks are summed by one all-reduce
// Rows of a JacobianFactor, row-major; `width` floats per row, the last one is b.
struct SparseRows {
  std::vector<float> rows;
  int num_rows = 0;
  int width = 0;
  float total_err = 0.0f;  // ReprojectionFactor: sum of squared unweighted errors (total_err_, reprojection_factor.cpp:242)
  int num_valid = 0;       // SparseGeometricFactor: rows that are not all zero
  const float* row(int i) const { return rows.data() + static_cast<std::size_t>(i) * width; }
};

// One factor of LinearizeReprojectionBatch: the arguments of LinearizeReprojection.  code0, query_xy and train_xy are
// read when LinearizeReprojectionBatch is called (not kept).
template <int CS, typename SE3T, typename CodeT, typename CamT, typename ImageBuffer>
DfkReprojectionItem ReprojectionItem(const SE3T& pose0, const SE3T& pose1, const CodeT& code0, const CamT& cam,
                                     const ImageBuffer& prx_orig, const ImageBuffer& prx_jac, int num_matches,
                                     const float* query_xy, const float* train_xy, float huber_delta, float sigma)
{
  DfkReprojectionItem it{};
  for (int k = 0; k < 7; ++k) {
    it.pose0[k] = pose0.data()[k];
    it.pose1[k] = pose1.data()[k];
  }
  it.cam = detail::Cam(cam);
  it.prx_orig = detail::View(prx_orig, 1);
  it.prx_jac = detail::View(prx_jac, CS);
  it.code = code0.data();
  it.num_matches = num_matches;
  it.query_xy = query_xy;
  it.train_xy = train_xy;
  it.cauchy_delta = huber_delta;
  it.sigma = sigma;
  return it;
}

// ReprojectionFactor::linearize (reprojection_factor.cpp:157-269): 2 rows per match,
// [dErr/dPose0 (6) | dErr/dPose1 (6) | dErr/dCode0 (CS) | b].  query_xy / train_xy: 2 floats per match (host);
// prx_orig / prx_jac: the keyframe's level-0 GPU views (kf->pyr_prx_orig.GetGpuLevel(0), kf->pyr_jac.GetGpuLevel(0)).
template <int CS, typename SE3T, typename CodeT, typename CamT, typename ImageBuffer>
SparseRows LinearizeReprojection(DfkHandle h, const SE3T& pose0, const SE3T& pose1, const CodeT& code0, const CamT& cam,
                                 const ImageBuffer& prx_orig, const ImageBuffer& prx_jac, int num_matches,
                                 const float* query_xy, const float* train_xy, float huber_delta, float sigma)
{
  const DfkReprojectionItem it = ReprojectionItem<CS>(pose0, pose1, code0, cam, prx_orig, prx_jac, num_matches, query_xy,
                                                      train_xy, huber_delta, sigma);
  SparseRows out;
  out.num_rows = 2 * num_matches;
  out.width = 13 + CS;
  out.rows.assign(static_cast<std::size_t>(out.num_rows) * out.width, 0.0f);
  detail::Check(h, dfk_reprojection_linearize(h, it.pose0, it.pose1, it.code, CS, &it.cam, &it.prx_orig, &it.prx_jac,
                                              it.num_matches, it.query_xy, it.train_xy, it.cauchy_delta, it.sigma,
                                              out.rows.data(), &out.total_err));
  return out;
}

// Many ReprojectionFactors linearised in one launch into normal-equation records (dfk_reprojection_linearize_batch):
// record i = [A^T A packed | -A^T b | b^T b | valid matches] of factor i's rows, in the RunStep record layout, at
// records_dev + i * DFK_SFM_RECORD_FLOATS(CS) (DEVICE).  Asynchronous on the handle's stream; what a window adds with
// WindowSystem::AddUnscaled, or dfk_window_assemble as an unscaled record (item size 0 x 0).
template <int CS>
void LinearizeReprojectionBatch(DfkHandle h, const std::vector<DfkReprojectionItem>& items, float* records_dev)
{
  detail::Check(h, dfk_reprojection_linearize_batch(h, items.data(), static_cast<int>(items.size()), CS, records_dev));
}

// One factor of LinearizeSparseGeometricBatch: the arguments of LinearizeSparseGeometric.  code0, code1 and points_xy
// are read when LinearizeSparseGeometricBatch is called (not kept).
template <int CS, typename SE3T, typename CodeT, typename CamT, typename ImageBuffer, typename GradBuffer>
DfkSparseGeometricItem SparseGeometricItem(const SE3T& pose0, const SE3T& pose1, const CodeT& code0, const CodeT& code1,
                                           const CamT& cam, const ImageBuffer& prx0_orig, const ImageBuffer& prx0_jac,
                                           const ImageBuffer& prx1_orig, const ImageBuffer& prx1_jac,
                                           const GradBuffer& dpt_grad1, int num_points, const int* points_xy,
                                           float huber_delta)
{
  DfkSparseGeometricItem it{};
  for (int k = 0; k < 7; ++k) {
    it.pose0[k] = pose0.data()[k];
    it.pose1[k] = pose1.data()[k];
  }
  it.cam = detail::Cam(cam);
  it.prx0_orig = detail::View(prx0_orig, 1);
  it.prx0_jac = detail::View(prx0_jac, CS);
  it.prx1_orig = detail::View(prx1_orig, 1);
  it.prx1_jac = detail::View(prx1_jac, CS);
  it.dpt_grad1 = detail::View(dpt_grad1, 2);
  it.code0 = code0.data();
  it.code1 = code1.data();
  it.num_points = num_points;
  it.points_xy = points_xy;
  it.huber_delta = huber_delta;
  return it;
}

// SparseGeometricFactor::linearize (sparse_geometric_factor.cpp:157-271): 1 row per sampled point,
// [dErr/dPose0 (6) | dErr/dPose1 (6) | dErr/dCode0 (CS) | dErr/dCode1 (CS) | b].  points_xy: 2 ints per point (host);
// the image arguments are the two keyframes' level-0 GPU views and kf1's depth gradient (2 floats per pixel).
template <int CS, typename SE3T, typename CodeT, typename CamT, typename ImageBuffer, typename GradBuffer>
SparseRows LinearizeSparseGeometric(DfkHandle h, const SE3T& pose0, const SE3T& pose1, const CodeT& code0, const CodeT& code1,
                                    const CamT& cam, const ImageBuffer& prx0_orig, const ImageBuffer& prx0_jac,
                                    const ImageBuffer& prx1_orig, const ImageBuffer& prx1_jac, const GradBuffer& dpt_grad1,
                                    int num_points, const int* points_xy, float huber_delta)
{
  const DfkSparseGeometricItem it = SparseGeometricItem<CS>(pose0, pose1, code0, code1, cam, prx0_orig, prx0_jac, prx1_orig,
                                                            prx1_jac, dpt_grad1, num_points, points_xy, huber_delta);
  SparseRows out;
  out.num_rows = num_points;
  out.width = 13 + 2 * CS;
  out.rows.assign(static_cast<std::size_t>(out.num_rows) * out.width, 0.0f);
  detail::Check(h, dfk_sparse_geometric_linearize(h, it.pose0, it.pose1, it.code0, it.code1, CS, &it.cam, &it.prx0_orig,
                                                  &it.prx0_jac, &it.prx1_orig, &it.prx1_jac, &it.dpt_grad1, it.num_points,
                                                  it.points_xy, it.huber_delta, out.rows.data(), &out.num_valid));
  return out;
}

// Many SparseGeometricFactors linearised in one launch into normal-equation records
// (dfk_sparse_geometric_linearize_batch): record i = [A^T A packed | -A^T b | b^T b | valid points] of factor i's rows
// over [pose0 | pose1 | code0 | code1], at records_dev + i * DFK_GEO_RECORD_FLOATS(CS) (DEVICE).  Asynchronous on the
// handle's stream; what a window adds with WindowSystem::AddGeometric, or dfk_window_assemble_geometric as a link.
template <int CS>
void LinearizeSparseGeometricBatch(DfkHandle h, const std::vector<DfkSparseGeometricItem>& items, float* records_dev)
{
  detail::Check(h, dfk_sparse_geometric_linearize_batch(h, items.data(), static_cast<int>(items.size()), CS,
                                                        records_dev));
}

inline void ShardPairs(std::size_t num_pairs, int world_size, int rank, std::size_t* begin, std::size_t* end)
{
  *begin = (num_pairs * static_cast<std::size_t>(rank)) / static_cast<std::size_t>(world_size);
  *end = (num_pairs * static_cast<std::size_t>(rank + 1)) / static_cast<std::size_t>(world_size);
}

// DepthPriorFactor (depth_prior_factor.cpp:29-137): keyframe `kf`'s code pulled towards a measured depth with standard
// deviation sigma.  levels[l] = (target depth, proximity, code Jacobian) GPU views of level l; the target pyramid is the
// caller's (the reference blurs it down once in its constructor: GaussianBlurDown, or dfk_build_image_pyramid).
// Linearize runs RunAlignment (:107-121) as one dfk_depth_prior_linearize_batch over the levels: record l is level l's
// DepthAligner::RunStep.  Error is the factor's error() (:62-76), 0.5 sum residual / sigma^2, from
// dfk_depth_prior_error_batch.  Unlike the reference, neither touches the keyframe's own depth (UpdateKfDepth).
template <int CS>
class DepthPriorFactor
{
public:
  struct Level {
    DfkImage target_dpt, prx_orig, prx_jac;
  };
  template <typename ImageBuffer>
  static Level MakeLevel(const ImageBuffer& target_dpt, const ImageBuffer& prx_orig, const ImageBuffer& prx_jac)
  {
    return Level{detail::View(target_dpt, 1), detail::View(prx_orig, 1), detail::View(prx_jac, CS)};
  }

  DepthPriorFactor(int kf, float sigma, std::vector<Level> levels) : kf_(kf), sigma_(sigma), levels_(std::move(levels)) {}
  int keyframe() const { return kf_; }
  float sigma() const { return sigma_; }
  int num_levels() const { return static_cast<int>(levels_.size()); }

  // the batch items at `code` (CS floats, read when the batch is called)
  std::vector<DfkDepthPriorItem> Items(const float* code) const
  {
    std::vector<DfkDepthPriorItem> out;
    for (const Level& l : levels_) out.push_back(DfkDepthPriorItem{l.target_dpt, l.prx_orig, l.prx_jac, code});
    return out;
  }
  // records_dev: DEVICE, num_levels() * DFK_DEPTH_RECORD_FLOATS(CS) floats.  Asynchronous on the handle's stream.
  void Linearize(DfkHandle h, const float* code, float* records_dev) const
  {
    const std::vector<DfkDepthPriorItem> it = Items(code);
    detail::Check(h, dfk_depth_prior_linearize_batch(h, it.data(), num_levels(), CS, records_dev));
  }
  // the error rows [residual | W * H (u32 bits)] of every level into out_dev (DEVICE, 2 * num_levels() floats), each
  // residual bit for bit the one of Linearize's record.  Asynchronous on the handle's stream.
  void ErrorRows(DfkHandle h, const float* code, float* out_dev) const
  {
    const std::vector<DfkDepthPriorItem> it = Items(code);
    detail::Check(h, dfk_depth_prior_error_batch(h, it.data(), num_levels(), CS, out_dev));
  }
  // error() from those rows copied to the host: 0.5 sum residual / sigma^2 over the levels
  double Error(const float* rows_host) const
  {
    const double s2 = static_cast<double>(sigma_) * static_cast<double>(sigma_);
    double e = 0.0;
    for (std::size_t l = 0; l < levels_.size(); ++l) e += static_cast<double>(rows_host[2 * l]) / s2;
    return 0.5 * e;
  }

private:
  int kf_;
  float sigma_;
  std::vector<Level> levels_;
};

}  // namespace df

#endif  // DFK_FACTOR_H_
