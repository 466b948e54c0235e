// dfk_window_lm.cu -- the small kernels of a window problem's Levenberg-Marquardt loop (dfk_window_problem_*,
// dfk_window_lm): everything between the factor batches that used to be host work.
//
//   repose    one launch: the pose- and code-dependent fields of every item of the problem from the fp64 state -- the
//             relative pose, its R and both 6x6 Jacobians (SfmItemDev, SparsePose) or q / t (EvalErrorDesc), and the
//             fp32 code slots (RunStep's fused decode, the sparse links, the depth decodes).  The poses and codes are
//             rounded to fp32 to nearest, as astype(np.float32) rounds them, and dfk_se3.cuh is the host staging's own
//             arithmetic, so every field is bit for bit what the batch calls stage from the same state.
//   retract   t += dt, q = normalize(exp(w) q), c += dc in fp64 (se3.retract / window_opt.apply_update)
//   deltas    Local(x0, x) = [t - t0 | log(R R0^T) | c - c0] of every frame prior and every keyframe-prior member
//   energy    one CTA: the window energy from the error outputs (each part summed sequentially in factor order, as
//             window_error_sum does) or from the buffer's f, plus the prior terms and the code prior
//   scatter   with an active subset (dfk_window_problem_set_active): the subset's records into their slots, zeros
//             into the inactive items' slots; with ISAM2's partial linearisation also "keep" for a valid record
//   relin     ISAM2's relinearisation check: theta_lin (+) delta_key for every key whose delta reaches the threshold
//   gather    a grown problem's kept records from the old problem's
//   diag max  max |d| of a buffer's diagonal over the kept variables (ISAM2's fixed diag_eps = 1e-12 of it)
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "dfk_internal.h"
#include "dfk_se3.cuh"

namespace dfk {
namespace {

__device__ void load_pose(const double* state, int slot, float p[7])
{
  for (int k = 0; k < 7; ++k) p[k] = __double2float_rn(state[(size_t)slot * 7 + k]);
}

__device__ void load_code(const double* codes, int slot, int C, float* dst)
{
  for (int c = threadIdx.x; c < C; c += blockDim.x) dst[c] = __double2float_rn(codes[(size_t)slot * C + c]);
}

__global__ void __launch_bounds__(64) window_repose_kernel(WindowReposeDev a)
{
  int b = blockIdx.x;
  const int C = a.code_size;
  const double* codes = a.state + (size_t)a.num_poses * 7;
  if (b < a.num_dense) {
    SfmItemDev& d = a.dense[b];
    const int4 s = a.dense_slots[b];
    if (threadIdx.x == 0) {
      float p0[7], p1[7];
      load_pose(a.state, s.x, p0);
      load_pose(a.state, s.y, p1);
      se3f::set_relative_pose_only(d, p1, p0);
    }
    load_code(codes, s.z, C, const_cast<float*>(d.code));
    return;
  }
  b -= a.num_dense;
  if (b < a.num_error) {
    EvalErrorDesc& d = a.error[b];
    const int4 s = a.error_slots[b];
    if (threadIdx.x == 0) {
      float p0[7], p1[7], p10[7];
      load_pose(a.state, s.x, p0);
      load_pose(a.state, s.y, p1);
      se3f::relative_pose(p1, p0, p10, nullptr, nullptr);
      for (int k = 0; k < 4; ++k) d.pc.q[k] = p10[k];
      for (int k = 0; k < 3; ++k) d.pc.t[k] = p10[4 + k];
    }
    return;
  }
  b -= a.num_error;
  if (b < a.num_rep) {
    ReprojItemDev& d = a.rep[b];
    const int4 s = a.rep_slots[b];
    if (threadIdx.x == 0) {
      float p0[7], p1[7];
      load_pose(a.state, s.x, p0);
      load_pose(a.state, s.y, p1);
      se3f::set_relative_pose_only(d.sp, p1, p0);
    }
    load_code(codes, s.z, C, const_cast<float*>(d.code));
    return;
  }
  b -= a.num_rep;
  if (b < a.num_geo) {
    GeoItemDev& d = a.geo[b];
    const int4 s = a.geo_slots[b];
    if (threadIdx.x == 0) {
      float p0[7], p1[7];
      load_pose(a.state, s.x, p0);
      load_pose(a.state, s.y, p1);
      se3f::set_relative_pose_only(d.sp, p1, p0);
    }
    load_code(codes, s.z, C, const_cast<float*>(d.code0));
    load_code(codes, s.w, C, const_cast<float*>(d.code1));
    return;
  }
  b -= a.num_geo;
  if (b < a.num_depth) load_code(codes, a.depth_slots[b].z, C, const_cast<float*>(a.depth[b].code));
}

// Sophus::SO3::exp as se3.so3_exp -> quaternion (x, y, z, w)
__device__ void so3_exp(const double w[3], double q[4])
{
  const double theta_sq = w[0] * w[0] + w[1] * w[1] + w[2] * w[2];
  const double theta = sqrt(theta_sq);
  double imag, real;
  if (theta < 1e-10) {
    imag = 0.5 - theta_sq / 48.0 + theta_sq * theta_sq / 3840.0;
    real = 1.0 - theta_sq / 8.0 + theta_sq * theta_sq / 384.0;
  } else {
    imag = sin(0.5 * theta) / theta;
    real = cos(0.5 * theta);
  }
  q[0] = imag * w[0]; q[1] = imag * w[1]; q[2] = imag * w[2]; q[3] = real;
}

__device__ void quat_mul_d(const double a[4], const double b[4], double o[4])
{
  o[0] = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1];
  o[1] = a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2];
  o[2] = a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0];
  o[3] = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
}

// se3.so3_log of a unit quaternion: the rotation vector, the half angle kept in (-pi/2, pi/2]
__device__ void so3_log(const double q[4], double out[3])
{
  const double n = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2]), w = q[3];
  double scale;
  if (n < 1e-10) scale = 2.0 / w - (2.0 / 3.0) * n * n / (w * w * w);
  else scale = 2.0 * (w != 0.0 ? atan(n / w) : 0.5 * M_PI) / n;
  out[0] = scale * q[0]; out[1] = scale * q[1]; out[2] = scale * q[2];
}

// one CTA per pose slot: keyframes take dx[k B ..], frames dx[K B + 6 f ..]; keyframes also retract their codes
__global__ void __launch_bounds__(128) window_retract_kernel(const double* __restrict__ in, double* __restrict__ out,
                                                             const double* __restrict__ dx, int K, int F, int C)
{
  const int s = blockIdx.x, B = 6 + C;
  const double* d = dx + (s < K ? (size_t)s * B : (size_t)K * B + 6 * (size_t)(s - K));
  if (threadIdx.x == 0) {
    const double* p = in + (size_t)s * 7;
    double e[4], q[4];
    so3_exp(d + 3, e);
    quat_mul_d(e, p, q);
    const double nrm = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
    double* o = out + (size_t)s * 7;
    for (int k = 0; k < 4; ++k) o[k] = q[k] / nrm;
    for (int k = 0; k < 3; ++k) o[4 + k] = p[4 + k] + d[k];
  }
  if (s < K) {
    const size_t c0 = (size_t)(K + F) * 7 + (size_t)s * C;
    for (int c = threadIdx.x; c < C; c += blockDim.x) out[c0 + c] = in[c0 + c] + d[6 + c];
  }
}

// one CTA per delta row r: keyframe ks[r] against x0 row r ([pose 7 | code C]), into delta[r B ..]
__global__ void __launch_bounds__(128) window_deltas_kernel(const double* __restrict__ state, int num_poses, int C,
                                                            const int* __restrict__ ks, const double* __restrict__ x0,
                                                            double* __restrict__ delta)
{
  const int r = blockIdx.x, k = ks[r], B = 6 + C;
  const double* p = state + (size_t)k * 7;
  const double* p0 = x0 + (size_t)r * (7 + C);
  double* o = delta + (size_t)r * B;
  if (threadIdx.x == 0) {
    const double q0i[4] = {-p0[0], -p0[1], -p0[2], p0[3]};
    double q[4];
    quat_mul_d(p, q0i, q);
    for (int i = 0; i < 3; ++i) o[i] = p[4 + i] - p0[4 + i];
    so3_log(q, o + 3);
  }
  const double* c = state + (size_t)num_poses * 7 + (size_t)k * C;
  for (int i = threadIdx.x; i < C; i += blockDim.x) o[6 + i] = c[i] - p0[7 + i];
}

constexpr int kEnergyThreads = 256;

// deterministic block sum (fixed tree); every thread gets the total
__device__ double block_sum(double v, double* sh)
{
  sh[threadIdx.x] = v;
  __syncthreads();
  for (int s = kEnergyThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] = __dadd_rn(sh[threadIdx.x], sh[threadIdx.x + s]);
    __syncthreads();
  }
  const double r = sh[0];
  __syncthreads();
  return r;
}

// f0 - 2 g^T d + d^T G d of the prior row [G (n x n) | g (n) | f0]
__device__ double prior_term(const double* row, const double* d, int n, double* sh)
{
  double dgd = 0.0, gd = 0.0;
  const double* g = row + (size_t)n * n;
  for (int i = threadIdx.x; i < n; i += kEnergyThreads) {
    const double* Gi = row + (size_t)i * n;
    double ri = 0.0;
    for (int j = 0; j < n; ++j) ri = __dadd_rn(ri, __dmul_rn(Gi[j], d[j]));
    dgd = __dadd_rn(dgd, __dmul_rn(d[i], ri));
    gd = __dadd_rn(gd, __dmul_rn(g[i], d[i]));
  }
  dgd = block_sum(dgd, sh);
  gd = block_sum(gd, sh);
  return __dadd_rn(__dsub_rn(row[(size_t)n * n + n], __dmul_rn(2.0, gd)), dgd);
}

__global__ void __launch_bounds__(kEnergyThreads) window_energy_kernel(WindowEnergyDev a)
{
  __shared__ double sh[kEnergyThreads];
  double priors = 0.0;
  for (int q = 0; q < a.num_frame_priors; ++q) {
    const double t = prior_term(a.frame_rows + (size_t)q * (a.B * a.B + a.B + 1), a.frame_delta + (size_t)q * a.B, a.B,
                                sh);
    priors = __dadd_rn(priors, t);
  }
  for (int q = 0; q < a.num_kf_priors; ++q) {
    const int n = (a.kf_mem_ptr[q + 1] - a.kf_mem_ptr[q]) * a.B;
    const double t = prior_term(a.kf_rows + a.kf_row_off[q], a.kf_delta + (size_t)a.kf_mem_ptr[q] * a.B, n, sh);
    priors = __dadd_rn(priors, t);
  }
  double cp = 0.0;
  if (a.code_prior_weight > 0.0) {
    double s = 0.0;
    for (int i = threadIdx.x; i < a.num_codes; i += kEnergyThreads) s = __dadd_rn(s, __dmul_rn(a.codes[i], a.codes[i]));
    cp = __dmul_rn(__dmul_rn(0.5, a.code_prior_weight), block_sum(s, sh));
  }
  if (threadIdx.x != 0) return;
  double phot = 0.0, rep = 0.0, geo = 0.0, E;
  double no_inl = 0.0, inl = 0.0;
  if (a.buf_f) {
    E = (double)*a.buf_f;
  } else {
    for (int i = 0; i < a.num_error; ++i) {
      const float2 o = a.err_out[i];
      const uint32_t n = __float_as_uint(o.y);
      if (n > 0) phot = __dadd_rn(phot, __dmul_rn(__ddiv_rn((double)o.x, (double)n), a.areas[i]));
      else no_inl += 1.0;
      inl += (double)n;
    }
    for (int i = 0; i < a.num_rep; ++i) rep = __dadd_rn(rep, (double)a.err_out[a.num_error + i].x);
    for (int i = 0; i < a.num_geo; ++i) geo = __dadd_rn(geo, (double)a.err_out[a.num_error + a.num_rep + i].x);
    E = __dadd_rn(__dadd_rn(__dadd_rn(phot, rep), geo), priors);
    if (a.num_depth_priors > 0) {  // prior by prior, level by level, after the other parts (window_opt.WindowError)
      double dep = 0.0;
      for (int q = 0; q < a.num_depth_priors; ++q) {
        const double s2 = __dmul_rn((double)a.depth_sigma[q], (double)a.depth_sigma[q]);
        for (int l = a.depth_level_ptr[q]; l < a.depth_level_ptr[q + 1]; ++l)
          dep = __dadd_rn(dep, __ddiv_rn((double)a.depth_err[l].x, s2));
      }
      *a.out_depth = dep;
      E = __dadd_rn(E, dep);
    }
  }
  double* o = a.out;
  o[0] = E; o[1] = phot; o[2] = rep; o[3] = geo; o[4] = priors; o[5] = no_inl; o[6] = inl;
  o[7] = __dadd_rn(E, cp);
}

// one CTA per record slot i: the active subset's record src[i], or an all-zero record for an inactive item (src[i] < 0)
__global__ void __launch_bounds__(256) window_scatter_records_kernel(const float* __restrict__ sub,
                                                                     const int* __restrict__ src, int rf,
                                                                     float* __restrict__ records)
{
  const int s = src[blockIdx.x];
  if (s == kKeepRecord) return;
  float* o = records + (size_t)blockIdx.x * rf;
  if (s < 0) {
    for (int k = threadIdx.x; k < rf; k += blockDim.x) o[k] = 0.0f;
    return;
  }
  const float* in = sub + (size_t)s * rf;
  for (int k = threadIdx.x; k < rf; k += blockDim.x) o[k] = in[k];
}

// one CTA per key (see launch_window_relinearize)
constexpr int kRelinThreads = 128;
__global__ void __launch_bounds__(kRelinThreads)
window_relinearize_kernel(const double* __restrict__ in, double* __restrict__ out, const double* __restrict__ delta,
                          int K, int F, int C, int check, double thr, int32_t* __restrict__ moved)
{
  __shared__ double red[kRelinThreads];
  __shared__ int any_nan;
  const int key = blockIdx.x, B = 6 + C;
  const bool is_code = key < 2 * K && (key & 1);
  const int slot = key < 2 * K ? key >> 1 : K + (key - 2 * K);  // pose slot (a keyframe or K + frame)
  const double* d = key < 2 * K ? delta + (size_t)(key >> 1) * B + (is_code ? 6 : 0)
                                : delta + (size_t)K * B + 6 * (size_t)(key - 2 * K);
  const int n = is_code ? C : 6;
  if (threadIdx.x == 0) any_nan = 0;
  __syncthreads();
  double m = 0.0;
  for (int i = threadIdx.x; i < n; i += kRelinThreads) {
    const double a = fabs(d[i]);
    if (a != a) any_nan = 1;
    m = fmax(m, a);
  }
  red[threadIdx.x] = m;
  __syncthreads();
  for (int s = kRelinThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] = fmax(red[threadIdx.x], red[threadIdx.x + s]);
    __syncthreads();
  }
  // numpy's max propagates a NaN, and NaN >= threshold is false
  const bool mv = check && !any_nan && red[0] >= thr;
  if (is_code) {
    const size_t c0 = (size_t)(K + F) * 7 + (size_t)(key >> 1) * C;
    for (int c = threadIdx.x; c < C; c += kRelinThreads) out[c0 + c] = mv ? in[c0 + c] + d[c] : in[c0 + c];
  } else if (threadIdx.x == 0) {
    const double* p = in + (size_t)slot * 7;
    double* o = out + (size_t)slot * 7;
    if (mv) {  // window_retract_kernel's arithmetic
      double e[4], q[4];
      so3_exp(d + 3, e);
      quat_mul_d(e, p, q);
      const double nrm = sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
      for (int k = 0; k < 4; ++k) o[k] = q[k] / nrm;
      for (int k = 0; k < 3; ++k) o[4 + k] = p[4 + k] + d[k];
    } else {
      for (int k = 0; k < 7; ++k) o[k] = p[k];
    }
  }
  if (threadIdx.x == 0) moved[key] = mv ? 1 : 0;
}

// one CTA per (new row, old row)
__global__ void __launch_bounds__(256) window_gather_records_kernel(const float* __restrict__ src, float* __restrict__ dst,
                                                                    const int2* __restrict__ map, int rf)
{
  const int2 m = map[blockIdx.x];
  for (int k = threadIdx.x; k < rf; k += blockDim.x) dst[(size_t)m.x * rf + k] = src[(size_t)m.y * rf + k];
}

// one CTA (see launch_window_diag_max)
constexpr int kDiagThreads = 256;
__global__ void __launch_bounds__(kDiagThreads)
window_diag_max_kernel(const float* __restrict__ buf, int K, int F, int C, size_t o_c, size_t o_f,
                       const int2* __restrict__ self_pairs, int num_self, double w, int fixed, double* out)
{
  __shared__ double red[kDiagThreads];
  const int B = 6 + C, n = K * B + 6 * F;
  double m = 0.0;
  for (int i = threadIdx.x; i < n; i += kDiagThreads) {
    if (i < fixed) continue;
    double d;
    if (i < K * B) {
      const int k = i / B, r = i - k * B;
      d = (double)buf[(size_t)k * B * B + (size_t)r * B + r];
      if (r < 6)
        for (int s = 0; s < num_self; ++s)
          if (self_pairs[s].y == k) {  // H += O, then H += O^T: the diagonal gets O(r, r) twice
            const double o = (double)buf[o_c + (size_t)self_pairs[s].x * 6 * B + (size_t)r * 6 + r];
            d = __dadd_rn(__dadd_rn(d, o), o);
          }
      if (r >= 6 && w > 0.0) d = __dadd_rn(d, w);
    } else {
      const int f = (i - K * B) / 6, r = i - K * B - 6 * f;
      d = (double)buf[o_f + 36 * (size_t)f + 7 * (size_t)r];
    }
    m = fmax(m, fabs(d));
  }
  red[threadIdx.x] = m;
  __syncthreads();
  for (int s = kDiagThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] = fmax(red[threadIdx.x], red[threadIdx.x + s]);
    __syncthreads();
  }
  if (threadIdx.x == 0) *out = red[0];
}

}  // namespace

cudaError_t launch_window_relinearize(const double* lin_in, double* lin_out, const double* delta, int K, int F, int C,
                                      bool check, double threshold, int32_t* moved, cudaStream_t stream)
{
  window_relinearize_kernel<<<2 * K + F, kRelinThreads, 0, stream>>>(lin_in, lin_out, delta, K, F, C, check ? 1 : 0,
                                                                     threshold, moved);
  return cudaGetLastError();
}

cudaError_t launch_window_gather_records(const float* src, float* dst, const int2* map, int n, int rf,
                                         cudaStream_t stream)
{
  if (n == 0) return cudaSuccess;
  window_gather_records_kernel<<<n, 256, 0, stream>>>(src, dst, map, rf);
  return cudaGetLastError();
}

cudaError_t launch_window_diag_max(const float* buf, int K, int F, int C, size_t coupling_off, size_t frame_off,
                                   const int2* self_pairs, int num_self, double w, bool fix_first_pose, double* out,
                                   cudaStream_t stream)
{
  window_diag_max_kernel<<<1, kDiagThreads, 0, stream>>>(buf, K, F, C, coupling_off, frame_off, self_pairs, num_self, w,
                                                          fix_first_pose ? 6 : 0, out);
  return cudaGetLastError();
}

cudaError_t launch_window_scatter_records(const float* sub, const int* src, int n, int rf, float* records,
                                          cudaStream_t stream)
{
  if (n == 0) return cudaSuccess;
  window_scatter_records_kernel<<<n, 256, 0, stream>>>(sub, src, rf, records);
  return cudaGetLastError();
}

cudaError_t launch_window_repose(const WindowReposeDev& a, cudaStream_t stream)
{
  const int n = a.num_dense + a.num_error + a.num_rep + a.num_geo + a.num_depth;
  if (n == 0) return cudaSuccess;
  window_repose_kernel<<<n, 64, 0, stream>>>(a);
  return cudaGetLastError();
}

cudaError_t launch_window_retract(const double* in, double* out, const double* dx, int K, int F, int C,
                                  cudaStream_t stream)
{
  window_retract_kernel<<<K + F, 128, 0, stream>>>(in, out, dx, K, F, C);
  return cudaGetLastError();
}

cudaError_t launch_window_deltas(const double* state, int num_poses, int C, int n, const int* ks, const double* x0,
                                 double* delta, cudaStream_t stream)
{
  if (n == 0) return cudaSuccess;
  window_deltas_kernel<<<n, 128, 0, stream>>>(state, num_poses, C, ks, x0, delta);
  return cudaGetLastError();
}

cudaError_t launch_window_energy(const WindowEnergyDev& a, cudaStream_t stream)
{
  window_energy_kernel<<<1, kEnergyThreads, 0, stream>>>(a);
  return cudaGetLastError();
}

}  // namespace dfk
