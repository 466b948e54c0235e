// dfk_api_window.cu -- C ABI of libdfk.so (see include/dfk.h), keyframe window: the window (create, assemble, priors,
// marginalisation, blanket), its solver, and the window problem with its Levenberg-Marquardt loops and ISAM2 steps.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <cmath>
#include <memory>
#include <new>
#include <string>
#include <vector>

#include "dfk.h"
#include "dfk_host.h"
#include "dfk_internal.h"
#include "dfk_levels.h"
#include "dfk_lm.h"
#include "dfk_works.h"

using namespace dfk;

// CSR adjacency of a keyframe window on the device (dfk_window_create)
struct DfkWindow {
  int device = 0;
  WindowDev dev{};
  // one allocation: the CSR lists kf0 | kf1 | pair | lk0 | lk1 (ptr | items each), frame_pair, the item areas, and with
  // keyframe priors their lists (KfPriorDev)
  DeviceBuf<unsigned char> blob;
  size_t floats = 0;
  // host copy of the structure, for dfk_window_solver_create and dfk_window_marginalize_keyframe
  std::vector<int> pair_k0, pair_k1, link_k0, link_k1, item_pair;
  // keyframe priors (dfk_window_create_priors): members prior_kf[prior_ptr[q] .. prior_ptr[q + 1]), the prior blocks
  // (blk_i < blk_j) and their device lists (KfPriorDev)
  std::vector<int> prior_ptr{0}, prior_kf, blk_i, blk_j;
  std::vector<long long> prior_off;  // doubles: start of prior q in a priors buffer; back() = the buffer's size
  KfPriorDev kp{};
};

// damped block-sparse Cholesky of one window (dfk_window_solver_create)
struct DfkWindowSolver {
  int device = 0;
  int num_vars = 0, code_size = 0, num_keyframes = 0;
  WindowSolverDev* dev = nullptr;
  ~DfkWindowSolver() { window_solver_destroy(dev); }
};

// ---------------------------------------------------------------------------------------------- window problem
// One window's every work item, planned and uploaded once (dfk_window_problem_create); the loop kernels of
// dfk_window_lm.cu re-pose them from the device state.  Everything the items point at that is not the caller's (code
// slots, ray tables, depth scratch of the error path) belongs to the problem.
struct DfkWindowProblem {
  int device = 0;
  const DfkWindow* w = nullptr;
  int K = 0, F = 0, C = 0, B = 0;
  float avg_dpt = 2.0f, huber_delta = 0.1f;  // the handle's sfmparams at create, like the dense items' (SfmItemDev)
  int nd = 0, nr = 0, ng = 0, ndep = 0, ne = 0, mf = 0, nkm = 0;  // items of each kind, frame priors, kf-prior members
  size_t S = 0;  // doubles of one state: (K + F) 7 + K C
  StepKernel step;
  SfmLaunchPlan plan;
  // one allocation: the parts create uploads, then the scratch (from dense_codes on, never uploaded)
  DeviceBuf<unsigned char> blob;
  Part<SfmItemDev> dense;
  Part<EvalErrorDesc> err;
  Part<double> areas;  // W * H of each error item
  Part<int4> dense_slots, err_slots, rep_slots, geo_slots, depth_slots;
  Part<DepthDecodeDesc> depth;
  Part<double> frows, kfrows, x0;  // prior rows, frozen points (frame priors, then kf members)
  Part<int> fp_lists;              // dfk_window_add_priors' CSR: ptr[K + 1] | prior indices
  Part<int> delta_kf;              // keyframe of every delta row
  Part<double> state;              // two states: [cur] the problem's, [1 - cur] an LM candidate
  Part<float> dense_codes, depth_codes;
  Part<double> delta;
  Part<float> err_out;             // (ne + nr + ng) x 2
  Part<unsigned char> small;       // the LM's read-back block [energy 8 | info | depth-prior energy], mirrored in
  Part<double> sm_energy, sm_depth_energy;  // small_host; these parts are offsets into it
  Part<int32_t> sm_info;
  PinnedBuf<unsigned char> small_host;
  DeviceBuf<unsigned char> depth_scratch;  // the depth items' decoded depths, one part each
  std::vector<DeviceBuf<float>> rays;
  DeviceBuf<unsigned char> rep, geo;  // the sparse batches' staged blocks
  Staged<DfkReprojectionItem> rep_st;
  Staged<DfkSparseGeometricItem> geo_st;
  int err_max_blocks = 1, err_rows = 0, depth_max_blocks = 1;
  int cur = 0;
  float* records = nullptr;
  float* geo_records = nullptr;
  WindowSolverDev* solver[2] = {nullptr, nullptr};  // [fix_first_pose]
  DeviceBuf<float> bufs;           // the LM's accepted and candidate window buffers
  int acc = 0;
  DeviceBuf<double> dx;
  // active subsets (dfk_window_problem_set_active): the create-time dense and error items with their slots and areas
  // are the templates a mask selects from; the selected items go to arrays of their own, so the full arrays stay as
  // create planned them and an all-active mask runs exactly the create-time launches
  std::vector<SfmItemDev> dense_tmpl;
  std::vector<EvalErrorDesc> err_tmpl;
  std::vector<int4> slots_tmpl;      // dense | error
  std::vector<double> areas_tmpl;
  bool sub_dense = false, sub_err = false;
  int nda = 0, nea = 0;              // active dense / error items while sub_dense / sub_err
  SfmLaunchPlan sub_plan;
  DeviceBuf<SfmItemDev> dense_sub;
  DeviceBuf<EvalErrorDesc> err_sub;
  DeviceBuf<int4> sub_slots;         // dense [0, nd) | error [nd, nd + ne)
  DeviceBuf<double> areas_sub;
  DeviceBuf<int> rec_src;            // record slot i <- subset record rec_src[i], -1: zeros
  DeviceBuf<float> sub_records;
  // depth priors (dfk_window_problem_set_depth_priors): ndp priors over ndpi (keyframe, level) items, staged once
  // ([descriptors | codes], the codes rewritten from the state before every batch), and the lists
  // [add CSR ptr K + 1 | prior indices ndp | level_ptr ndp + 1 | sigma ndp | keyframe of every item ndpi]
  int ndp = 0, ndpi = 0;
  DepthPriorStaged dp_st;
  DeviceBuf<unsigned char> dp, dp_lists;
  Part<int> dp_csr, dp_level_ptr, dp_kf;
  Part<float> dp_sigma;
  DeviceBuf<float> dp_partials, dp_records, dp_err;
  std::vector<int> dp_item_kf;       // the keyframe of every depth-prior item
  // ISAM2 (dfk_window_problem_isam2_update): two slots [theta_lin S | Delta K B + 6 F] doubles, [ic] the committed one
  // (an update writes the other and commits it when the solve succeeds), and the host's "linearised at theta_lin" flag
  // of every dense item, reprojection link, geometric link and depth-prior item
  DeviceBuf<double> isam;
  int ic = 0;
  bool isam_fresh = true;            // the next update starts from the state
  long long isam_updates = 0;
  double diag_eps = -1.0;            // fixed by the first update
  std::vector<uint8_t> lin_dense, lin_rep, lin_geo, lin_dp;
  std::vector<uint8_t> active;       // the dense mask of the last set_active
  std::vector<int4> rep_slots_h, geo_slots_h;
  std::vector<int> rep_size_h, geo_size_h;  // matches / points of every link (growth checks them)
  DeviceBuf<int2> gather;                    // dfk_window_problem_grow_from's (new row, old row) lists
  // the read-back block [diagonal max | moved flags 2 K + F | info] and its pinned mirror
  DeviceBuf<unsigned char> isam_small;
  PinnedBuf<unsigned char> isam_small_host;
  DeviceBuf<uint8_t> stale_dev;      // reprojection | geometric | depth-prior items
  DeviceBuf<int2> self_pairs;        // (pair, keyframe) of every pair (k, k)
  int num_self = -1;
  // the stale active dense items: their items, slots, tile plan and records, and every slot's source
  SfmLaunchPlan stale_plan;
  DeviceBuf<SfmItemDev> stale_items;
  DeviceBuf<int4> stale_slots;
  DeviceBuf<int> stale_src;
  DeviceBuf<float> stale_records;
  ~DfkWindowProblem()
  {
    window_solver_destroy(solver[0]);
    window_solver_destroy(solver[1]);
  }
  double* st(int i) const { return state.at(blob.ptr) + (size_t)i * S; }
  double* energy() const { return sm_energy.at(small.at(blob.ptr)); }
  int32_t* info() const { return sm_info.at(small.at(blob.ptr)); }
  double* depth_energy() const { return sm_depth_energy.at(small.at(blob.ptr)); }
  size_t delta_size() const { return (size_t)K * B + 6 * (size_t)F; }
  double* lin(int i) const { return isam.ptr + (size_t)i * (S + delta_size()); }
  double* isam_delta(int i) const { return lin(i) + S; }
  void clear_linearised()
  {
    std::fill(lin_dense.begin(), lin_dense.end(), 0);
    std::fill(lin_rep.begin(), lin_rep.end(), 0);
    std::fill(lin_geo.begin(), lin_geo.end(), 0);
    std::fill(lin_dp.begin(), lin_dp.end(), 0);
  }
};

namespace {

// One CSR list into ptr[keys + 1 + n], zero: ptr[keys + 1], then the items of each key in item order (the summation
// order of the gather kernels); an item whose key is outside [0, keys) is in no list
template <class KeyOf>
void fill_csr(int* ptr, int keys, int n, KeyOf key_of)
{
  for (int i = 0; i < n; ++i)
    if (key_of(i) < keys) ptr[key_of(i) + 1] += 1;
  for (int k = 0; k < keys; ++k) ptr[k + 1] += ptr[k];
  std::vector<int> next(ptr, ptr + keys);
  for (int i = 0; i < n; ++i)
    if (key_of(i) < keys) ptr[keys + 1 + next[key_of(i)]++] = i;
}

// The window buffer from the records: the assemble kernel, then the keyframe-prior blocks set to zero
// (dfk_window_add_keyframe_priors fills them)
DfkStatus assemble_window(DfkHandle h, const DfkWindow* w, const float* records, const float* geo_records, float* buf,
                          const char* what)
{
  DFK_CUDA(h, launch_window_assemble(w->dev, records, geo_records, buf, h->stream), what);
  h->launches += 1;
  if (w->kp.num_blocks > 0)
    DFK_CUDA(h, cudaMemsetAsync(buf + w->kp.block_off, 0, (w->floats - w->kp.block_off) * sizeof(float), h->stream), what);
  return DFK_OK;
}

WindowReposeDev repose_args(const DfkWindowProblem* p, const double* state)
{
  unsigned char* b = p->blob.ptr;
  WindowReposeDev a{};
  a.code_size = p->C;
  a.num_poses = p->K + p->F;
  a.state = state;
  a.dense = p->dense.at(b); a.dense_slots = p->dense_slots.at(b); a.num_dense = p->nd;
  a.error = p->err.at(b); a.error_slots = p->err_slots.at(b); a.num_error = p->ne;
  if (p->sub_dense) {
    a.dense = p->dense_sub.ptr; a.dense_slots = p->sub_slots.ptr; a.num_dense = p->nda;
  }
  if (p->sub_err) {
    a.error = p->err_sub.ptr; a.error_slots = p->sub_slots.ptr + p->nd; a.num_error = p->nea;
  }
  a.rep = p->rep_st.descs.at(p->rep.ptr); a.rep_slots = p->rep_slots.at(b); a.num_rep = p->nr;
  a.geo = p->geo_st.descs.at(p->geo.ptr); a.geo_slots = p->geo_slots.at(b); a.num_geo = p->ng;
  a.depth = p->depth.at(b); a.depth_slots = p->depth_slots.at(b); a.num_depth = p->ndep;
  return a;
}

// the depth priors' batch at `state`: the items' codes from the state, then the records (gram) or the error rows;
// stale (device, optional): only those items are written
DfkStatus problem_depth_priors(DfkHandle h, DfkWindowProblem* p, const double* state, bool gram, const char* what,
                               const uint8_t* stale = nullptr)
{
  DFK_CUDA(h, launch_depth_prior_codes(state + (size_t)(p->K + p->F) * 7, p->dp_kf.at(p->dp_lists.ptr), p->ndpi, p->C,
                                       p->dp_st.codes.at(p->dp.ptr), h->stream),
           what);
  DFK_CUDA(h, launch_depth_prior_batch(p->C, p->dp_st.descs.at(p->dp.ptr), p->ndpi, p->dp_st.max_parts, p->avg_dpt,
                                       p->dp_partials.ptr, gram ? p->dp_records.ptr : p->dp_err.ptr, gram, h->stream,
                                       stale),
           what);
  h->launches += 3;
  return DFK_OK;
}

DfkStatus problem_deltas(DfkHandle h, const DfkWindowProblem* p, const double* state)
{
  unsigned char* b = p->blob.ptr;
  DFK_CUDA(h, launch_window_deltas(state, p->K + p->F, p->C, p->mf + p->nkm, p->delta_kf.at(b), p->x0.at(b),
                                   p->delta.at(b), h->stream),
           "[WindowProblem] kernel launch failed");
  h->launches += (p->mf + p->nkm) > 0;
  return DFK_OK;
}

DfkStatus problem_finish(DfkHandle h, DfkWindowProblem* p, const double* state, float* buf, const uint8_t* dp_stale);

// the window buffer at state `state` into buf (dfk_window_problem_linearize).  Every record is rewritten, so no item
// is linearised at the ISAM2 theta_lin any more
DfkStatus problem_linearize(DfkHandle h, DfkWindowProblem* p, const double* state, float* buf)
{
  const char* what = "[WindowProblem::linearize] kernel launch failed";
  unsigned char* b = p->blob.ptr;
  p->clear_linearised();
  DFK_CUDA(h, launch_window_repose(repose_args(p, state), h->stream), what);
  h->launches += 1;
  const float avg = p->avg_dpt;
  if (p->sub_dense) {  // the active items only, then every record slot from the subset's records or zeros
    if (p->nda > 0) {
      DFK_CUDA(h, h->partials_dev.ensure((size_t)p->sub_plan.num_partials * p->step.pfloats),
               "[WindowProblem::linearize] scratch allocation failed");
      DFK_TRY(launch_step(h, p->step, p->C, p->dense_sub.ptr, p->nda, p->sub_plan, h->partials_dev.ptr,
                          p->sub_records.ptr));
    }
    DFK_CUDA(h, launch_window_scatter_records(p->sub_records.ptr, p->rec_src.ptr, p->nd, DFK_SFM_RECORD_FLOATS(p->C),
                                              p->records, h->stream),
             what);
    h->launches += 1;
  } else if (p->nd > 0) {
    DFK_CUDA(h, h->partials_dev.ensure((size_t)p->plan.num_partials * p->step.pfloats),
             "[WindowProblem::linearize] scratch allocation failed");
    DFK_TRY(launch_step(h, p->step, p->C, p->dense.at(b), p->nd, p->plan, h->partials_dev.ptr, p->records));
  }
  if (p->nr > 0) {
    const float2* q = p->rep_st.payload.at(p->rep.ptr);
    DFK_CUDA(h, launch_reprojection_records(p->C, p->rep_st.descs.at(p->rep.ptr), p->nr, q, q + p->rep_st.total, avg,
                                            p->records + (size_t)p->nd * DFK_SFM_RECORD_FLOATS(p->C), h->stream),
             what);
    h->launches += 1;
  }
  if (p->ng > 0) {
    DFK_CUDA(h, launch_sparse_geometric_records(p->C, p->geo_st.descs.at(p->geo.ptr), p->ng,
                                                p->geo_st.payload.at(p->geo.ptr), avg, p->geo_records, h->stream),
             what);
    h->launches += 1;
  }
  return problem_finish(h, p, state, buf, nullptr);
}

// the buffer from the records: the assembly, the frame and keyframe priors at `state`, then the depth priors (only the
// dp_stale items re-evaluated when given)
DfkStatus problem_finish(DfkHandle h, DfkWindowProblem* p, const double* state, float* buf, const uint8_t* dp_stale)
{
  const char* what = "[WindowProblem::linearize] kernel launch failed";
  unsigned char* b = p->blob.ptr;
  const DfkWindow* w = p->w;
  DFK_TRY(assemble_window(h, w, p->records, p->ng > 0 ? p->geo_records : nullptr, buf, what));
  DFK_TRY(problem_deltas(h, p, state));
  if (p->mf > 0) {
    DFK_CUDA(h, launch_window_add_priors(w->dev, p->mf, p->fp_lists.at(b), p->fp_lists.at(b) + p->K + 1, p->frows.at(b),
                                         p->delta.at(b), buf, h->stream),
             what);
    h->launches += 1;
  }
  if (w->kp.num_priors > 0) {
    DFK_CUDA(h, launch_window_add_keyframe_priors(w->dev, w->kp, p->kfrows.at(b), p->delta.at(b) + (size_t)p->mf * p->B,
                                                  buf, h->stream),
             what);
    h->launches += 1;
  }
  if (p->ndp > 0) {  // after the frame and keyframe priors, as SfmWindowProblem.linearise without an all-reduce
    DFK_TRY(problem_depth_priors(h, p, state, true, what, dp_stale));
    unsigned char* l = p->dp_lists.ptr;
    DFK_CUDA(h, launch_window_add_depth_priors(w->dev, p->ndp, p->dp_csr.at(l), p->dp_csr.at(l) + p->K + 1,
                                               p->dp_level_ptr.at(l), p->dp_sigma.at(l), p->dp_records.ptr, buf,
                                               h->stream),
             what);
    h->launches += 1;
  }
  return DFK_OK;
}

WindowEnergyDev energy_args(const DfkWindowProblem* p, const double* state, double w)
{
  unsigned char* b = p->blob.ptr;
  WindowEnergyDev a{};
  a.B = p->B;
  a.err_out = reinterpret_cast<const float2*>(p->err_out.at(b));
  a.areas = p->sub_err ? p->areas_sub.ptr : p->areas.at(b);
  a.num_error = p->sub_err ? p->nea : p->ne; a.num_rep = p->nr; a.num_geo = p->ng;
  a.num_frame_priors = p->mf; a.frame_rows = p->frows.at(b); a.frame_delta = p->delta.at(b);
  a.num_kf_priors = p->w->kp.num_priors; a.kf_rows = p->kfrows.at(b); a.kf_row_off = p->w->kp.off;
  a.kf_mem_ptr = p->w->kp.mem_ptr; a.kf_delta = p->delta.at(b) + (size_t)p->mf * p->B;
  a.codes = state + (size_t)(p->K + p->F) * 7;
  a.num_codes = p->K * p->C;
  a.code_prior_weight = w;
  a.num_depth_priors = p->ndp;
  if (p->ndp > 0) {
    a.depth_err = reinterpret_cast<const float2*>(p->dp_err.ptr);
    a.depth_level_ptr = p->dp_level_ptr.at(p->dp_lists.ptr);
    a.depth_sigma = p->dp_sigma.at(p->dp_lists.ptr);
    a.out_depth = p->depth_energy();
  }
  a.out = p->energy();
  return a;
}

// the energy at `state` without linearising into p->energy() (E + 1/2 w |c|^2 in slot 7)
DfkStatus problem_error(DfkHandle h, DfkWindowProblem* p, const double* state, double w)
{
  const char* what = "[WindowProblem::error] kernel launch failed";
  unsigned char* b = p->blob.ptr;
  DFK_CUDA(h, launch_window_repose(repose_args(p, state), h->stream), what);
  h->launches += 1;
  const float avg = p->avg_dpt;
  if (p->ndep > 0) {
    DFK_CUDA(h, launch_update_depth(p->C, p->depth.at(b), p->ndep, p->depth_max_blocks, avg, h->stream), what);
    h->launches += 1;
  }
  float* out = p->err_out.at(b);
  // with an active subset only its items are evaluated, and their rows come first (energy_args reads as many)
  const int ne = p->sub_err ? p->nea : p->ne;
  if (ne > 0) {
    const char* sw = "[WindowProblem::error] scratch allocation failed";
    DFK_CUDA(h, h->eval_partials.ensure((size_t)p->err_rows * 32), sw);
    DFK_TRY(ensure_tickets(h, h->eval_counters, (size_t)p->ne, sw, sw));
    DFK_CUDA(h, launch_eval_error(p->sub_err ? p->err_sub.ptr : p->err.at(b), ne, p->err_max_blocks,
                                        p->huber_delta, h->eval_partials.ptr, h->eval_counters.ptr, out, h->stream),
             what);
    h->launches += 1;
  }
  if (p->nr > 0) {
    const float2* q = p->rep_st.payload.at(p->rep.ptr);
    DFK_CUDA(h, launch_reprojection_error(p->C, p->rep_st.descs.at(p->rep.ptr), p->nr, q, q + p->rep_st.total, avg,
                                          out + 2 * (size_t)ne, h->stream),
             what);
    h->launches += 1;
  }
  if (p->ng > 0) {
    DFK_CUDA(h, launch_sparse_geometric_error(p->C, p->geo_st.descs.at(p->geo.ptr), p->ng,
                                              p->geo_st.payload.at(p->geo.ptr), avg, out + 2 * (size_t)(ne + p->nr),
                                              h->stream),
             what);
    h->launches += 1;
  }
  if (p->ndp > 0) DFK_TRY(problem_depth_priors(h, p, state, false, what));
  DFK_TRY(problem_deltas(h, p, state));
  DFK_CUDA(h, launch_window_energy(energy_args(p, state, w), h->stream), what);
  h->launches += 1;
  return DFK_OK;
}

// the active subsets of a validated mask (em: one byte per error item): the selected templates, their slots and the
// subset's tile plan, uploaded on the stream behind every launch still reading the previous ones.  The subset arrays
// are allocated once at full size, so no later mask reallocates an array a queued launch reads
DfkStatus problem_set_active(DfkHandle h, DfkWindowProblem* p, const uint8_t* dm, const uint8_t* em)
{
  const char* amsg = "[WindowProblem::set_active] allocation failed";
  const char* umsg = "[WindowProblem::set_active] upload failed";
  const int nd = p->nd, ne = p->ne;
  const bool all_d = std::all_of(dm, dm + nd, [](uint8_t v) { return v != 0; });
  for (int i = 0; i < nd; ++i) {
    // an item switched on or off holds another record than its last linearisation left: stale for ISAM2
    if (p->active[i] != (dm[i] != 0)) p->lin_dense[i] = 0;
    p->active[i] = dm[i] != 0;
  }
  const bool all_e = std::all_of(em, em + ne, [](uint8_t v) { return v != 0; });
  if (!all_d || !all_e) {
    DFK_CUDA(h, p->sub_slots.ensure((size_t)std::max(nd + ne, 1)), amsg);
    if (!all_d) {
      DFK_CUDA(h, p->dense_sub.ensure((size_t)std::max(nd, 1)), amsg);
      DFK_CUDA(h, p->rec_src.ensure((size_t)nd), amsg);
      DFK_CUDA(h, p->sub_records.ensure((size_t)nd * DFK_SFM_RECORD_FLOATS(p->C)), amsg);
    }
    if (!all_e) {
      DFK_CUDA(h, p->err_sub.ensure((size_t)std::max(ne, 1)), amsg);
      DFK_CUDA(h, p->areas_sub.ensure((size_t)std::max(ne, 1)), amsg);
    }
  }
  if (!all_d) {
    std::vector<SfmItemDev> items;
    std::vector<int4> sl;
    std::vector<int> src(nd, -1);
    for (int i = 0; i < nd; ++i)
      if (dm[i]) {
        src[i] = (int)items.size();
        items.push_back(p->dense_tmpl[i]);
        sl.push_back(p->slots_tmpl[i]);
      }
    plan_tiles(items.data(), (int)items.size(), p->step.max_ctas, &p->sub_plan);
    if (!items.empty()) {
      DFK_CUDA(h, cudaMemcpyAsync(p->dense_sub.ptr, items.data(), sizeof(SfmItemDev) * items.size(),
                                  cudaMemcpyHostToDevice, h->stream),
               umsg);
      DFK_CUDA(h, cudaMemcpyAsync(p->sub_slots.ptr, sl.data(), sizeof(int4) * sl.size(), cudaMemcpyHostToDevice,
                                  h->stream),
               umsg);
    }
    DFK_CUDA(h, cudaMemcpyAsync(p->rec_src.ptr, src.data(), sizeof(int) * nd, cudaMemcpyHostToDevice, h->stream), umsg);
    p->nda = (int)items.size();
  }
  if (!all_e) {
    std::vector<EvalErrorDesc> items;
    std::vector<int4> sl;
    std::vector<double> areas;
    for (int i = 0; i < ne; ++i)
      if (em[i]) {
        items.push_back(p->err_tmpl[i]);
        sl.push_back(p->slots_tmpl[nd + i]);
        areas.push_back(p->areas_tmpl[i]);
      }
    if (!items.empty()) {
      DFK_CUDA(h, cudaMemcpyAsync(p->err_sub.ptr, items.data(), sizeof(EvalErrorDesc) * items.size(),
                                  cudaMemcpyHostToDevice, h->stream),
               umsg);
      DFK_CUDA(h, cudaMemcpyAsync(p->sub_slots.ptr + nd, sl.data(), sizeof(int4) * sl.size(), cudaMemcpyHostToDevice,
                                  h->stream),
               umsg);
      DFK_CUDA(h, cudaMemcpyAsync(p->areas_sub.ptr, areas.data(), sizeof(double) * areas.size(),
                                  cudaMemcpyHostToDevice, h->stream),
               umsg);
    }
    p->nea = (int)items.size();
  }
  p->sub_dense = !all_d;
  p->sub_err = !all_e;
  return DFK_OK;
}

// dfk_window_lm's device half (the Ops of dfk_lm.h / dfk_levels.h): the state, buffers and solve of a problem
struct ProblemLMOps {
  DfkHandle h;
  DfkWindowProblem* p;
  const DfkLMParams* prm;
  WindowSolverDev* solver;
  size_t nf, f_off;
  double w;
  int cand() const { return 1 - p->cur; }
  float* buf(bool c) const { return p->bufs.ptr + (size_t)(c ? 1 - p->acc : p->acc) * nf; }
  DfkStatus linearize(bool c) { return problem_linearize(h, p, p->st(c ? cand() : p->cur), buf(c)); }
  DfkStatus energy(bool c, double* f)
  {
    const double* s = p->st(c ? cand() : p->cur);
    if (prm->use_error) {
      DFK_TRY(problem_error(h, p, s, w));
    } else {
      WindowEnergyDev a = energy_args(p, s, w);
      a.buf_f = buf(c) + f_off;
      a.num_frame_priors = a.num_kf_priors = 0;
      DFK_CUDA(h, launch_window_energy(a, h->stream), "[WindowLM] kernel launch failed");
      h->launches += 1;
    }
    double* e = p->sm_energy.at(p->small_host.ptr);
    DFK_TRY(download(h, e, p->energy(), 8 * sizeof(double), "[WindowLM] read-back failed", "[WindowLM] kernel failed"));
    *f = e[7];
    return DFK_OK;
  }
  DfkStatus solve(double lam, int* info)
  {
    DFK_CUDA(h, launch_window_solve(solver, buf(false), lam, w, p->st(p->cur) + (size_t)(p->K + p->F) * 7, p->dx.ptr,
                                    p->info(), h->stream, &h->launches, true),
             "[WindowLM] solve launch failed");
    int32_t* i = p->sm_info.at(p->small_host.ptr);
    DFK_TRY(download(h, i, p->info(), sizeof(int32_t), "[WindowLM] read-back failed", "[WindowLM] solve failed"));
    *info = *i;
    return DFK_OK;
  }
  DfkStatus retract()
  {
    DFK_CUDA(h, launch_window_retract(p->st(p->cur), p->st(cand()), p->dx.ptr, p->K, p->F, p->C, h->stream),
             "[WindowLM] kernel launch failed");
    h->launches += 1;
    return DFK_OK;
  }
  void accept()
  {
    p->cur = cand();
    p->acc = 1 - p->acc;
  }
};

// dfk_window_lm's checks of the parameters and trace, and the solver, buffers and Ops of a run
DfkStatus lm_setup(DfkHandle h, DfkWindowProblem* p, const DfkLMParams* prm, DfkLMTrace* tr, const char* name,
                   ProblemLMOps* ops)
{
  const std::string what = std::string("[") + name + "] ";
  if (!p || !prm || !tr || !tr->energy || (prm->iterations > 0 && (!tr->lambda || !tr->accepted)))
    return fail(h, DFK_ERR_INVALID_ARG, what + "null argument");
  if (p->device != h->device) return fail(h, DFK_ERR_INVALID_ARG, what + "problem and handle live on different devices");
  if (prm->iterations < 0 || !(std::isfinite(prm->lambda_init) && prm->lambda_init >= 0.0) ||
      !(std::isfinite(prm->code_prior_weight) && prm->code_prior_weight >= 0.0))
    return fail(h, DFK_ERR_INVALID_ARG, what + "iterations < 0, or lambda_init / code_prior_weight not finite and >= 0");
  if (!(std::isfinite(prm->lambda_up) && prm->lambda_up > 0.0) ||
      !(std::isfinite(prm->lambda_down) && prm->lambda_down > 0.0) || std::isnan(prm->lambda_max))
    return fail(h, DFK_ERR_INVALID_ARG, what + "lambda_up / lambda_down must be finite and > 0, lambda_max a number");
  const int fix = prm->fix_first_pose ? 1 : 0;
  const std::string amsg = what + "allocation failed";
  if (!p->solver[fix])
    DFK_CUDA(h, window_solver_create(p->K, p->C, p->F, p->w->pair_k0, p->w->pair_k1, p->w->link_k0, p->w->link_k1,
                                     p->w->blk_i, p->w->blk_j, p->w->kp.block_off, std::vector<int>(), &p->solver[0]),
             amsg.c_str());
  const size_t nf = p->w->floats, f_off = (size_t)p->K * p->B * (p->B + 1) + (size_t)p->w->dev.num_pairs * 6 * p->B;
  DFK_CUDA(h, p->bufs.ensure(2 * nf), amsg.c_str());
  DFK_CUDA(h, p->dx.ensure((size_t)p->K * p->B + 6 * (size_t)p->F), amsg.c_str());
  *ops = ProblemLMOps{h, p, prm, p->solver[fix], nf, f_off, prm->code_prior_weight};
  return DFK_OK;
}

// ------------------------------------------------------------------------------------------------------- ISAM2
DfkStatus isam2_check(DfkHandle h, const DfkWindowProblem* p, const DfkIsam2Params* prm, const std::string& what)
{
  if (!p || !prm) return fail(h, DFK_ERR_INVALID_ARG, what + "null argument");
  if (p->device != h->device) return fail(h, DFK_ERR_INVALID_ARG, what + "problem and handle live on different devices");
  if (prm->relinearize_skip < 1 || std::isnan(prm->relinearize_threshold) ||
      !(std::isfinite(prm->code_prior_weight) && prm->code_prior_weight >= 0.0))
    return fail(h, DFK_ERR_INVALID_ARG, what + "relinearize_skip must be >= 1, relinearize_threshold a number and "
                                               "code_prior_weight finite and >= 0");
  return DFK_OK;
}

// the buffers of the ISAM2 state and of a partial linearisation, allocated at their full sizes so that no later update
// reallocates what a queued launch reads; the solver of fix_first_pose; a fresh run starts from the state
DfkStatus isam2_setup(DfkHandle h, DfkWindowProblem* p, int fix, const char* amsg)
{
  const int K = p->K, F = p->F, nd = p->nd;
  DFK_CUDA(h, p->isam.ensure(2 * (p->S + p->delta_size())), amsg);
  DFK_CUDA(h, p->isam_small.ensure(sizeof(double) + (size_t)(2 * K + F + 1) * 4), amsg);
  DFK_CUDA(h, p->isam_small_host.ensure(sizeof(double) + (size_t)(2 * K + F + 1) * 4), amsg);
  DFK_CUDA(h, p->stale_dev.ensure((size_t)std::max(1, p->nr + p->ng + p->ndpi)), amsg);
  DFK_CUDA(h, p->stale_items.ensure((size_t)std::max(nd, 1)), amsg);
  DFK_CUDA(h, p->stale_slots.ensure((size_t)std::max(nd, 1)), amsg);
  DFK_CUDA(h, p->stale_src.ensure((size_t)std::max(nd, 1)), amsg);
  DFK_CUDA(h, p->stale_records.ensure((size_t)std::max(nd, 1) * DFK_SFM_RECORD_FLOATS(p->C)), amsg);
  DFK_CUDA(h, p->bufs.ensure(2 * p->w->floats), amsg);
  if (!p->solver[fix])
    DFK_CUDA(h, window_solver_create(K, p->C, F, p->w->pair_k0, p->w->pair_k1, p->w->link_k0, p->w->link_k1,
                                     p->w->blk_i, p->w->blk_j, p->w->kp.block_off, std::vector<int>(), &p->solver[0]),
             amsg);
  if (p->num_self < 0) {
    std::vector<int2> self;
    for (size_t q = 0; q < p->w->pair_k0.size(); ++q)
      if (p->w->pair_k0[q] == p->w->pair_k1[q]) self.push_back(make_int2((int)q, p->w->pair_k0[q]));
    DFK_CUDA(h, p->self_pairs.ensure(std::max<size_t>(1, self.size())), amsg);
    if (!self.empty())
      DFK_CUDA(h, cudaMemcpyAsync(p->self_pairs.ptr, self.data(), sizeof(int2) * self.size(), cudaMemcpyHostToDevice,
                                  h->stream),
               amsg);
    p->num_self = (int)self.size();
  }
  if (p->isam_fresh) {
    DFK_CUDA(h, cudaMemcpyAsync(p->lin(p->ic), p->st(p->cur), sizeof(double) * p->S, cudaMemcpyDeviceToDevice, h->stream),
             amsg);
    DFK_CUDA(h, cudaMemsetAsync(p->isam_delta(p->ic), 0, sizeof(double) * p->delta_size(), h->stream), amsg);
    p->clear_linearised();
    p->isam_updates = 0;
    p->diag_eps = -1.0;
    p->isam_fresh = false;
  }
  return DFK_OK;
}

// one IncrementalOptimizer.update() (dfk_window_problem_isam2_update's steps 1-6)
DfkStatus problem_isam2_update(DfkHandle h, DfkWindowProblem* p, const DfkIsam2Params* prm, DfkIsam2Result* res)
{
  const char* what = "[WindowProblem::isam2_update] kernel launch failed";
  const char* amsg = "[WindowProblem::isam2_update] allocation failed";
  const char* umsg = "[WindowProblem::isam2_update] upload failed";
  const int K = p->K, F = p->F, C = p->C, B = p->B, nd = p->nd, nr = p->nr, ng = p->ng, ndpi = p->ndpi;
  const int fix = prm->fix_first_pose ? 1 : 0;
  DFK_TRY(isam2_setup(h, p, fix, amsg));
  const int nxt = 1 - p->ic;
  const double* lin_in = p->lin(p->ic);
  double* lin = p->lin(nxt);
  double* delta = p->isam_delta(nxt);
  unsigned char* sd = p->isam_small.ptr;
  unsigned char* sh = p->isam_small_host.ptr;
  double* diag_dev = reinterpret_cast<double*>(sd);  // first: 8-byte aligned
  int32_t* moved_dev = reinterpret_cast<int32_t*>(sd + sizeof(double));
  int32_t* info_dev = moved_dev + 2 * K + F;
  // 1. the relinearisation check
  const bool check = (p->isam_updates + 1) % prm->relinearize_skip == 0;
  DFK_CUDA(h, launch_window_relinearize(lin_in, lin, p->isam_delta(p->ic), K, F, C, check, prm->relinearize_threshold,
                                        moved_dev, h->stream),
           what);
  h->launches += 1;
  std::vector<int32_t> moved(2 * K + F, 0);
  if (check) {
    DFK_TRY(download(h, sh, moved_dev, sizeof(int32_t) * moved.size(), "[WindowProblem::isam2_update] read-back failed",
                     "[WindowProblem::isam2_update] kernel failed"));
    memcpy(moved.data(), sh, sizeof(int32_t) * moved.size());
  }
  int num_moved = 0;
  for (int v : moved) num_moved += v;
  // 2. the stale items
  auto pose_moved = [&](int s) { return s >= 0 && moved[s < K ? 2 * s : 2 * K + (s - K)] != 0; };
  auto code_moved = [&](int c) { return c >= 0 && moved[2 * c + 1] != 0; };
  auto stale_of = [&](const int4& sl, uint8_t linearised) {
    return !linearised || pose_moved(sl.x) || pose_moved(sl.y) || code_moved(sl.z) || code_moved(sl.w);
  };
  std::vector<uint8_t> sd_dense(nd), sd_sparse(nr + ng + ndpi);
  for (int i = 0; i < nd; ++i) sd_dense[i] = stale_of(p->slots_tmpl[i], p->lin_dense[i]);
  for (int j = 0; j < nr; ++j) sd_sparse[j] = stale_of(p->rep_slots_h[j], p->lin_rep[j]);
  for (int j = 0; j < ng; ++j) sd_sparse[nr + j] = stale_of(p->geo_slots_h[j], p->lin_geo[j]);
  for (int j = 0; j < ndpi; ++j) sd_sparse[nr + ng + j] = !p->lin_dp[j] || code_moved(p->dp_item_kf[j]);
  // factors: the window pairs of the stale dense items, the stale links
  std::vector<int> pairs;
  for (int i = 0; i < nd; ++i)
    if (sd_dense[i]) pairs.push_back(p->w->item_pair[i]);
  std::sort(pairs.begin(), pairs.end());
  int factors = (int)(std::unique(pairs.begin(), pairs.end()) - pairs.begin());
  for (int j = 0; j < nr + ng; ++j) factors += sd_sparse[j];
  // 3. the stale items at theta_lin: the stale active dense items in record order, every slot's record source
  std::vector<SfmItemDev> items;
  std::vector<int4> sl;
  std::vector<int> src(nd);
  bool scatter = false;
  for (int i = 0; i < nd; ++i) {
    if (!p->active[i]) {
      src[i] = -1;
      scatter = true;
    } else if (sd_dense[i]) {
      src[i] = (int)items.size();
      items.push_back(p->dense_tmpl[i]);
      sl.push_back(p->slots_tmpl[i]);
      scatter = true;
    } else {
      src[i] = kKeepRecord;
    }
  }
  const int ns = (int)items.size();
  if (ns > 0) {
    plan_tiles(items.data(), ns, p->step.max_ctas, &p->stale_plan);
    DFK_CUDA(h, cudaMemcpyAsync(p->stale_items.ptr, items.data(), sizeof(SfmItemDev) * ns, cudaMemcpyHostToDevice,
                                h->stream),
             umsg);
    DFK_CUDA(h, cudaMemcpyAsync(p->stale_slots.ptr, sl.data(), sizeof(int4) * ns, cudaMemcpyHostToDevice, h->stream),
             umsg);
  }
  if (scatter)
    DFK_CUDA(h, cudaMemcpyAsync(p->stale_src.ptr, src.data(), sizeof(int) * nd, cudaMemcpyHostToDevice, h->stream), umsg);
  if (!sd_sparse.empty())
    DFK_CUDA(h, cudaMemcpyAsync(p->stale_dev.ptr, sd_sparse.data(), sd_sparse.size(), cudaMemcpyHostToDevice, h->stream),
             umsg);
  WindowReposeDev a = repose_args(p, lin);
  a.dense = p->stale_items.ptr; a.dense_slots = p->stale_slots.ptr; a.num_dense = ns;
  a.num_error = 0;
  a.num_depth = 0;
  DFK_CUDA(h, launch_window_repose(a, h->stream), what);
  h->launches += 1;
  if (ns > 0) {
    DFK_CUDA(h, h->partials_dev.ensure((size_t)p->stale_plan.num_partials * p->step.pfloats), amsg);
    DFK_TRY(launch_step(h, p->step, C, p->stale_items.ptr, ns, p->stale_plan, h->partials_dev.ptr,
                        p->stale_records.ptr));
  }
  if (scatter) {
    DFK_CUDA(h, launch_window_scatter_records(p->stale_records.ptr, p->stale_src.ptr, nd, DFK_SFM_RECORD_FLOATS(C),
                                              p->records, h->stream),
             what);
    h->launches += 1;
  }
  const float avg = p->avg_dpt;
  const bool any_rep = std::any_of(sd_sparse.begin(), sd_sparse.begin() + nr, [](uint8_t v) { return v != 0; });
  const bool any_geo = std::any_of(sd_sparse.begin() + nr, sd_sparse.begin() + nr + ng, [](uint8_t v) { return v != 0; });
  if (any_rep) {
    const float2* q = p->rep_st.payload.at(p->rep.ptr);
    DFK_CUDA(h, launch_reprojection_records(C, p->rep_st.descs.at(p->rep.ptr), nr, q, q + p->rep_st.total, avg,
                                            p->records + (size_t)nd * DFK_SFM_RECORD_FLOATS(C), h->stream,
                                            p->stale_dev.ptr),
             what);
    h->launches += 1;
  }
  if (any_geo) {
    DFK_CUDA(h, launch_sparse_geometric_records(C, p->geo_st.descs.at(p->geo.ptr), ng, p->geo_st.payload.at(p->geo.ptr),
                                                avg, p->geo_records, h->stream, p->stale_dev.ptr + nr),
             what);
    h->launches += 1;
  }
  float* buf = p->bufs.ptr;
  DFK_TRY(problem_finish(h, p, lin, buf, p->stale_dev.ptr + nr + ng));
  // 4. diag_eps, fixed by the first update
  if (p->diag_eps < 0.0) {
    const size_t o_c = (size_t)K * B * (B + 1);
    const size_t o_f = o_c + (size_t)p->w->dev.num_pairs * 6 * B + 2 + (size_t)p->w->dev.num_links * B * B;
    DFK_CUDA(h, launch_window_diag_max(buf, K, F, C, o_c, o_f, p->self_pairs.ptr, p->num_self, prm->code_prior_weight,
                                       fix != 0, diag_dev, h->stream),
             what);
    h->launches += 1;
    double mx = 0.0;
    DFK_TRY(download(h, &mx, diag_dev, sizeof(double), "[WindowProblem::isam2_update] read-back failed",
                     "[WindowProblem::isam2_update] kernel failed"));
    p->diag_eps = 1e-12 * mx;
  }
  // 5. the incremental solve from theta_lin
  int j0 = 0;
  DFK_CUDA(h, launch_window_solver_update(p->solver[fix], buf, prm->code_prior_weight, p->diag_eps,
                                          lin + (size_t)(K + F) * 7, delta, info_dev, h->stream, &h->launches, &j0,
                                          true),
           "[WindowProblem::isam2_update] solve failed");
  int32_t info = 0;
  DFK_TRY(download(h, sh, info_dev, sizeof(int32_t), "[WindowProblem::isam2_update] read-back failed",
                   "[WindowProblem::isam2_update] solve failed"));
  memcpy(&info, sh, sizeof(int32_t));
  const uint8_t now = info == 0 ? 1 : 0;  // a failed update leaves theta_lin: its records describe no linearisation
  for (int i = 0; i < nd; ++i)
    if (sd_dense[i]) p->lin_dense[i] = now;
  for (int j = 0; j < nr; ++j)
    if (sd_sparse[j]) p->lin_rep[j] = now;
  for (int j = 0; j < ng; ++j)
    if (sd_sparse[nr + j]) p->lin_geo[j] = now;
  for (int j = 0; j < ndpi; ++j)
    if (sd_sparse[nr + ng + j]) p->lin_dp[j] = now;
  if (info != 0)
    return fail(h, DFK_ERR_INVALID_ARG, "[WindowProblem::isam2_update] the window's system at theta_lin is not "
                                        "positive definite (info " + std::to_string(info) + ")");
  p->isam_updates += 1;
  p->ic = nxt;
  // 6. the estimate theta_lin (+) Delta
  DFK_CUDA(h, launch_window_retract(lin, p->st(p->cur), delta, K, F, C, h->stream), what);
  h->launches += 1;
  res->variables_relinearized = num_moved;
  res->variables_reeliminated = (K - j0) * B + 6 * F;
  res->factors_relinearised = factors;
  res->first_column = j0;
  return DFK_OK;
}

// the schedule's pairs and levels of the dense and error items (dfk_window_lm_levels and dfk_window_map_steps)
DfkStatus schedule_items(DfkHandle h, const DfkWindowProblem* p, const DfkLevelSchedule* sc, const std::string& what,
                         std::vector<int>& dpair, std::vector<int>& epair, std::vector<int>& elevel)
{
  const int nd = p->nd, ne = p->ne, L = sc->num_levels;
  if (L < 1 || !sc->iters || (nd > 0 && !sc->dense_level) || sc->num_pairs < 0)
    return fail(h, DFK_ERR_INVALID_ARG, what + "num_levels < 1, or null iters / dense_level");
  if (ne > 0 && ne != nd && (!sc->error_pair || !sc->error_level))
    return fail(h, DFK_ERR_INVALID_ARG, what + "error_pair and error_level are required when num_error != num_dense");
  for (int l = 0; l < L; ++l)
    if (sc->iters[l] < 0) return fail(h, DFK_ERR_INVALID_ARG, what + "iters[" + std::to_string(l) + "] < 0");
  // the schedule's pairs: the distinct window pairs of the dense items, in window order
  std::vector<int> ids;
  dpair.assign(nd, 0);
  for (int i = 0; i < nd; ++i) ids.push_back(p->w->item_pair[i]);
  std::sort(ids.begin(), ids.end());
  ids.erase(std::unique(ids.begin(), ids.end()), ids.end());
  if ((int)ids.size() != sc->num_pairs)
    return fail(h, DFK_ERR_INVALID_ARG, what + "num_pairs " + std::to_string(sc->num_pairs) + ", but the dense items" +
                                            " cover " + std::to_string(ids.size()) + " pairs");
  for (int i = 0; i < nd; ++i)
    dpair[i] = (int)(std::lower_bound(ids.begin(), ids.end(), p->w->item_pair[i]) - ids.begin());
  for (int i = 0; i < nd; ++i)
    if (sc->dense_level[i] < 0 || sc->dense_level[i] >= L)
      return fail(h, DFK_ERR_INVALID_ARG, what + "dense item " + std::to_string(i) + ": level outside [0, num_levels)");
  epair.assign(ne, 0);
  elevel.assign(ne, 0);
  for (int i = 0; i < ne; ++i) {
    epair[i] = sc->error_pair ? sc->error_pair[i] : dpair[i];
    elevel[i] = sc->error_level ? sc->error_level[i] : sc->dense_level[i];
    if (epair[i] < 0 || epair[i] >= sc->num_pairs || elevel[i] < 0 || elevel[i] >= L)
      return fail(h, DFK_ERR_INVALID_ARG, what + "error item " + std::to_string(i) + ": pair or level out of range");
  }
  return DFK_OK;
}

bool slot_ok(int s, int lo, int hi) { return s >= lo && s < hi; }

}  // namespace

extern "C" {

DfkStatus dfk_window_create(DfkHandle h, const DfkWindowDesc* d, DfkWindow** out)
{
  return dfk_window_create_geometric(h, d, 0, nullptr, nullptr, out);
}

DfkStatus dfk_window_create_geometric(DfkHandle h, const DfkWindowDesc* d, int L, const int32_t* link_k0,
                                      const int32_t* link_k1, DfkWindow** out)
{
  return dfk_window_create_frames(h, d, L, link_k0, link_k1, 0, out);
}

DfkStatus dfk_window_create_frames(DfkHandle h, const DfkWindowDesc* d, int L, const int32_t* link_k0,
                                   const int32_t* link_k1, int F, DfkWindow** out)
{
  return dfk_window_create_priors(h, d, L, link_k0, link_k1, F, 0, nullptr, nullptr, out);
}

DfkStatus dfk_window_create_priors(DfkHandle h, const DfkWindowDesc* d, int L, const int32_t* link_k0,
                                   const int32_t* link_k1, int F, int Q, const int32_t* prior_ptr,
                                   const int32_t* prior_kf, DfkWindow** out)
{
  return guarded(h, [&] {
    if (!d || !out || L < 0 || F < 0 || (L > 0 && (!link_k0 || !link_k1)) || Q < 0 ||
        (Q > 0 && (!prior_ptr || !prior_kf)))
      return fail(h, DFK_ERR_INVALID_ARG, "[Window] null argument");
    *out = nullptr;
    const int K = d->num_keyframes, P = d->num_pairs, n = d->num_items;
    if (K <= 0 || P <= 0 || n <= 0 || !d->pair_k0 || !d->pair_k1 || !d->item_pair || !d->item_width || !d->item_height)
      return fail(h, DFK_ERR_INVALID_ARG, "[Window] empty window / null index array");
    if (!dfk_sfm_supports_code_size(d->code_size))
      return fail(h, DFK_ERR_UNSUPPORTED, "[Window] no RunStep kernel for code size " + std::to_string(d->code_size));
    // pair_k1 in [K, K + F): frame pair_k1 - K, which must be k1 of exactly this one pair
    std::vector<int> frame_pair(F, -1);
    for (int p = 0; p < P; ++p) {
      if (d->pair_k0[p] < 0 || d->pair_k0[p] >= K || d->pair_k1[p] < 0 || d->pair_k1[p] >= K + F)
        return fail(h, DFK_ERR_INVALID_ARG, "[Window] pair " + std::to_string(p) + " names a keyframe outside the window");
      if (d->pair_k1[p] >= K) {
        if (frame_pair[d->pair_k1[p] - K] >= 0)
          return fail(h, DFK_ERR_INVALID_ARG, "[Window] frame " + std::to_string(d->pair_k1[p] - K) +
                                                  " is k1 of more than one pair");
        frame_pair[d->pair_k1[p] - K] = p;
      }
    }
    for (int f = 0; f < F; ++f)
      if (frame_pair[f] < 0)
        return fail(h, DFK_ERR_INVALID_ARG, "[Window] frame " + std::to_string(f) + " is k1 of no pair");
    for (int i = 0; i < n; ++i)
      // a record is scaled (W, H > 0: photometric) or unscaled (0, 0: reprojection)
      if (d->item_pair[i] < 0 || d->item_pair[i] >= P ||
          !((d->item_width[i] > 0 && d->item_height[i] > 0) || (d->item_width[i] == 0 && d->item_height[i] == 0)))
        return fail(h, DFK_ERR_INVALID_ARG, "[Window] record " + std::to_string(i) + " names a pair outside the window");
    for (int i = 0; i < n; ++i)
      if (d->pair_k1[d->item_pair[i]] >= K && d->item_width[i] == 0)
        return fail(h, DFK_ERR_INVALID_ARG, "[Window] record " + std::to_string(i) + " of a frame pair is unscaled");
    for (int l = 0; l < L; ++l) {
      if (link_k0[l] < 0 || link_k0[l] >= K || link_k1[l] < 0 || link_k1[l] >= K)
        return fail(h, DFK_ERR_INVALID_ARG, "[Window] link " + std::to_string(l) + " names a keyframe outside the window");
      if (link_k0[l] == link_k1[l])
        return fail(h, DFK_ERR_INVALID_ARG, "[Window] link " + std::to_string(l) + " ties a keyframe to itself");
    }
    // keyframe priors: non-empty ascending lists of distinct keyframes of the window
    if (Q > 0 && prior_ptr[0] != 0) return fail(h, DFK_ERR_INVALID_ARG, "[Window] prior_ptr[0] must be 0");
    for (int q = 0; q < Q; ++q) {
      if (prior_ptr[q + 1] <= prior_ptr[q])
        return fail(h, DFK_ERR_INVALID_ARG, "[Window] keyframe prior " + std::to_string(q) + " has no keyframe");
      for (int a = prior_ptr[q]; a < prior_ptr[q + 1]; ++a)
        if (prior_kf[a] < 0 || prior_kf[a] >= K || (a > prior_ptr[q] && prior_kf[a] <= prior_kf[a - 1]))
          return fail(h, DFK_ERR_INVALID_ARG, "[Window] keyframe prior " + std::to_string(q) +
                                                  " is not an ascending list of distinct keyframes of the window");
    }
    const int M = Q > 0 ? prior_ptr[Q] : 0;  // members of all priors
    // prior blocks: the distinct (i < j) of every prior, ascending; the entries of each keyframe and each block in
    // prior order
    std::vector<std::pair<int, int>> blocks;
    for (int q = 0; q < Q; ++q)
      for (int a = prior_ptr[q]; a < prior_ptr[q + 1]; ++a)
        for (int c = a + 1; c < prior_ptr[q + 1]; ++c) blocks.push_back({prior_kf[a], prior_kf[c]});
    std::sort(blocks.begin(), blocks.end());
    blocks.erase(std::unique(blocks.begin(), blocks.end()), blocks.end());
    const int NB = (int)blocks.size();
    std::vector<std::vector<int2>> kf_ent(K);
    std::vector<std::vector<int3>> blk_ent(NB);
    size_t num_blk_ent = 0;
    for (int q = 0; q < Q; ++q)
      for (int a = prior_ptr[q]; a < prior_ptr[q + 1]; ++a) {
        kf_ent[prior_kf[a]].push_back(make_int2(q, a - prior_ptr[q]));
        for (int c = a + 1; c < prior_ptr[q + 1]; ++c, ++num_blk_ent) {
          const int b = (int)(std::lower_bound(blocks.begin(), blocks.end(), std::make_pair(prior_kf[a], prior_kf[c])) -
                              blocks.begin());
          blk_ent[b].push_back(make_int3(q, a - prior_ptr[q], c - prior_ptr[q]));
        }
      }
    std::vector<long long> poff(Q + 1, 0);
    for (int q = 0; q < Q; ++q)
      poff[q + 1] = poff[q] + (long long)DFK_KF_PRIOR_DOUBLES(d->code_size, prior_ptr[q + 1] - prior_ptr[q]);
    // one CSR list per key kind (keyframe k0, frame k1, pair, and the links' keyframes), frame_pair, the item areas
    Staging s(h->staging);
    const Part<int> kf0 = s.add<int>(K + 1 + n), kf1 = s.add<int>(K + 1 + n), pair = s.add<int>(P + 1 + n);
    const Part<int> lk0 = s.add<int>(K + 1 + L), lk1 = s.add<int>(K + 1 + L), fr = s.add<int>(F);
    const Part<float> areas = s.add<float>(n);
    Part<int> mem_ptr, kf_ptr, blk_ptr;
    Part<int2> kfe;
    Part<int3> bke;
    Part<long long> off;
    if (Q > 0) {
      mem_ptr = s.add<int>(Q + 1); kf_ptr = s.add<int>(K + 1); blk_ptr = s.add<int>(NB + 1);
      kfe = s.add<int2>(M); bke = s.add<int3>(num_blk_ent); off = s.add<long long>(Q + 1);
    }
    unsigned char* hb = s.host();
    fill_csr(kf0.at(hb), K, n, [&](int i) { return d->pair_k0[d->item_pair[i]]; });
    // a frame pair's pose1 is the frame's: its items go to the frame's block, not to a keyframe's
    fill_csr(kf1.at(hb), K, n, [&](int i) { return d->pair_k1[d->item_pair[i]]; });
    fill_csr(pair.at(hb), P, n, [&](int i) { return d->item_pair[i]; });
    fill_csr(lk0.at(hb), K, L, [&](int l) { return link_k0[l]; });
    fill_csr(lk1.at(hb), K, L, [&](int l) { return link_k1[l]; });
    std::copy(frame_pair.begin(), frame_pair.end(), fr.at(hb));
    for (int i = 0; i < n; ++i) areas.at(hb)[i] = (float)d->item_width[i] * (float)d->item_height[i];
    if (Q > 0) {
      std::copy(prior_ptr, prior_ptr + Q + 1, mem_ptr.at(hb));
      int2* ke = kfe.at(hb);
      for (int k = 0; k < K; ++k) {
        kf_ptr.at(hb)[k + 1] = kf_ptr.at(hb)[k] + (int)kf_ent[k].size();
        ke = std::copy(kf_ent[k].begin(), kf_ent[k].end(), ke);
      }
      int3* be = bke.at(hb);
      for (int b = 0; b < NB; ++b) {
        blk_ptr.at(hb)[b + 1] = blk_ptr.at(hb)[b] + (int)blk_ent[b].size();
        be = std::copy(blk_ent[b].begin(), blk_ent[b].end(), be);
      }
      std::copy(poff.begin(), poff.end(), off.at(hb));
    }

    DeviceGuard guard(h->device);
    std::unique_ptr<DfkWindow> w(new (std::nothrow) DfkWindow());  // freed under the guard if the upload fails
    if (!w) return oom(h);
    w->device = h->device;
    const char* upload_failed = "[Window] index upload failed";
    // synchronous: the window may be used from any stream on its device
    DFK_CUDA(h, w->blob.ensure(s.bytes), upload_failed);
    DFK_CUDA(h, cudaMemcpy(w->blob.ptr, hb, s.bytes, cudaMemcpyHostToDevice), upload_failed);
    unsigned char* b = w->blob.ptr;
    w->dev.num_keyframes = K; w->dev.num_pairs = P; w->dev.num_items = n; w->dev.code_size = d->code_size;
    w->dev.kf0_ptr = kf0.at(b); w->dev.kf0_items = kf0.at(b) + K + 1;
    w->dev.kf1_ptr = kf1.at(b); w->dev.kf1_items = kf1.at(b) + K + 1;
    w->dev.pair_ptr = pair.at(b); w->dev.pair_items = pair.at(b) + P + 1;
    w->dev.item_area = areas.at(b);
    w->dev.num_links = L;
    w->dev.lk0_ptr = lk0.at(b); w->dev.lk0_links = lk0.at(b) + K + 1;
    w->dev.lk1_ptr = lk1.at(b); w->dev.lk1_links = lk1.at(b) + K + 1;
    w->dev.num_frames = F;
    w->dev.frame_pair = fr.at(b);
    const size_t B = 6 + (size_t)d->code_size;
    const size_t block_off = (size_t)K * (B * B + B) + (size_t)P * 6 * B + 2 + (size_t)L * B * B + (size_t)F * 42;
    w->floats = block_off + (size_t)NB * B * B;
    w->pair_k0.assign(d->pair_k0, d->pair_k0 + P);
    w->pair_k1.assign(d->pair_k1, d->pair_k1 + P);
    w->link_k0.assign(link_k0, link_k0 + L);
    w->link_k1.assign(link_k1, link_k1 + L);
    w->item_pair.assign(d->item_pair, d->item_pair + n);
    if (Q > 0) {
      w->prior_ptr.assign(prior_ptr, prior_ptr + Q + 1);
      w->prior_kf.assign(prior_kf, prior_kf + M);
      for (const auto& b : blocks) {
        w->blk_i.push_back(b.first);
        w->blk_j.push_back(b.second);
      }
      w->prior_off = poff;
      w->kp.num_priors = Q; w->kp.num_blocks = NB; w->kp.block_off = block_off;
      w->kp.mem_ptr = mem_ptr.at(b); w->kp.off = off.at(b);
      w->kp.kf_ptr = kf_ptr.at(b); w->kp.kf_ent = kfe.at(b);
      w->kp.blk_ptr = blk_ptr.at(b); w->kp.blk_ent = bke.at(b);
    }
    *out = w.release();
    return DFK_OK;
  });
}

DfkStatus dfk_window_destroy(DfkHandle /*h*/, DfkWindow* w)
{
  if (!w) return DFK_OK;
  DeviceGuard guard(w->device);
  delete w;
  return DFK_OK;
}

size_t dfk_window_floats(const DfkWindow* w) { return w ? w->floats : 0; }

DfkStatus dfk_window_assemble(DfkHandle h, const DfkWindow* w, const float* records_dev, float* window_dev)
{
  return guarded(h, [&] {
    if (!w || !records_dev || !window_dev) return fail(h, DFK_ERR_INVALID_ARG, "[Window] null argument");
    if (w->device != h->device) return fail(h, DFK_ERR_INVALID_ARG, "[Window] window and handle live on different devices");
    if (w->dev.num_links > 0)
      return fail(h, DFK_ERR_INVALID_ARG, "[Window] window has geometric links: assemble it with dfk_window_assemble_geometric");
    DeviceGuard guard(h->device);
    return assemble_window(h, w, records_dev, nullptr, window_dev, "[Window] kernel launch failed");
  });
}

DfkStatus dfk_window_assemble_geometric(DfkHandle h, const DfkWindow* w, const float* records_dev,
                                        const float* geo_records_dev, float* window_dev)
{
  return guarded(h, [&] {
    if (!w || !records_dev || !window_dev) return fail(h, DFK_ERR_INVALID_ARG, "[Window] null argument");
    if (w->device != h->device) return fail(h, DFK_ERR_INVALID_ARG, "[Window] window and handle live on different devices");
    if (w->dev.num_links > 0 && !geo_records_dev)
      return fail(h, DFK_ERR_INVALID_ARG, "[Window] window has geometric links but no geometric records");
    DeviceGuard guard(h->device);
    return assemble_window(h, w, records_dev, geo_records_dev, window_dev, "[Window] kernel launch failed");
  });
}

DfkStatus dfk_window_marginalize_frames(DfkHandle h, const DfkWindow* w, const float* records_dev, int n,
                                        const int32_t* frames_host, double* priors_dev, int32_t* info_dev)
{
  return guarded(h, [&] {
    if (!w || !records_dev || n < 0 || (n > 0 && (!frames_host || !priors_dev || !info_dev)))
      return fail(h, DFK_ERR_INVALID_ARG, "[Window::MarginalizeFrames] null argument");
    if (w->device != h->device)
      return fail(h, DFK_ERR_INVALID_ARG, "[Window::MarginalizeFrames] window and handle live on different devices");
    for (int i = 0; i < n; ++i)
      if (frames_host[i] < 0 || frames_host[i] >= w->dev.num_frames)
        return fail(h, DFK_ERR_INVALID_ARG, "[Window::MarginalizeFrames] frame " + std::to_string(frames_host[i]) +
                                                " is not a frame of the window");
    if (n == 0) return DFK_OK;
    DeviceGuard guard(h->device);
    const char* what = "[Window::MarginalizeFrames] index upload failed";
    DFK_CUDA(h, h->window_lists.ensure(n), what);
    // pageable source: staged before the call returns
    DFK_CUDA(h, cudaMemcpyAsync(h->window_lists.ptr, frames_host, sizeof(int) * n, cudaMemcpyHostToDevice, h->stream),
             what);
    DFK_CUDA(h, launch_window_marginalize_frames(w->dev, records_dev, n, h->window_lists.ptr, priors_dev, info_dev,
                                                 h->stream),
             "[Window::MarginalizeFrames] kernel launch failed");
    h->launches += 1;
    return DFK_OK;
  });
}

DfkStatus dfk_window_add_priors(DfkHandle h, const DfkWindow* w, int m, const int32_t* prior_kf_host,
                                const double* priors_dev, const double* delta_dev, float* window_dev)
{
  return guarded(h, [&] {
    if (!w || !window_dev || m < 0 || (m > 0 && (!prior_kf_host || !priors_dev || !delta_dev)))
      return fail(h, DFK_ERR_INVALID_ARG, "[Window::AddPriors] null argument");
    if (w->device != h->device)
      return fail(h, DFK_ERR_INVALID_ARG, "[Window::AddPriors] window and handle live on different devices");
    const int K = w->dev.num_keyframes;
    for (int i = 0; i < m; ++i)
      if (prior_kf_host[i] < 0 || prior_kf_host[i] >= K)
        return fail(h, DFK_ERR_INVALID_ARG, "[Window::AddPriors] prior " + std::to_string(i) +
                                                " names a keyframe outside the window");
    if (m == 0) return DFK_OK;
    // CSR of the priors per keyframe, in list order: ptr[K + 1] | indices[m]
    std::vector<int> lists(K + 1 + m, 0);
    fill_csr(lists.data(), K, m, [&](int i) { return prior_kf_host[i]; });
    DeviceGuard guard(h->device);
    const char* what = "[Window::AddPriors] index upload failed";
    DFK_CUDA(h, h->window_lists.ensure(lists.size()), what);
    DFK_CUDA(h, cudaMemcpyAsync(h->window_lists.ptr, lists.data(), sizeof(int) * lists.size(), cudaMemcpyHostToDevice,
                                h->stream),
             what);
    DFK_CUDA(h, launch_window_add_priors(w->dev, m, h->window_lists.ptr, h->window_lists.ptr + K + 1, priors_dev,
                                         delta_dev, window_dev, h->stream),
             "[Window::AddPriors] kernel launch failed");
    h->launches += 1;
    return DFK_OK;
  });
}

DfkStatus dfk_window_add_depth_priors(DfkHandle h, const DfkWindow* w, int m, const int32_t* prior_kf_host,
                                      const float* sigma_host, const int32_t* level_ptr_host, const float* records_dev,
                                      float* window_dev)
{
  return guarded(h, [&] {
    if (!w || !window_dev || m < 0 || (m > 0 && (!prior_kf_host || !sigma_host || !level_ptr_host || !records_dev)))
      return fail(h, DFK_ERR_INVALID_ARG, "[Window::AddDepthPriors] null argument");
    if (w->device != h->device)
      return fail(h, DFK_ERR_INVALID_ARG, "[Window::AddDepthPriors] window and handle live on different devices");
    if (!depth_supported(w->dev.code_size))
      return fail(h, DFK_ERR_UNSUPPORTED, "[Window::AddDepthPriors] code size not instantiated by the depth prior");
    const int K = w->dev.num_keyframes;
    if (m > 0 && level_ptr_host[0] != 0)
      return fail(h, DFK_ERR_INVALID_ARG, "[Window::AddDepthPriors] level_ptr[0] must be 0");
    for (int i = 0; i < m; ++i) {
      const std::string pre = "[Window::AddDepthPriors] prior " + std::to_string(i);
      if (prior_kf_host[i] < 0 || prior_kf_host[i] >= K)
        return fail(h, DFK_ERR_INVALID_ARG, pre + " names a keyframe outside the window");
      if (!std::isfinite(sigma_host[i]) || !(sigma_host[i] > 0.0f))
        return fail(h, DFK_ERR_INVALID_ARG, pre + ": sigma must be finite and > 0");
      if (level_ptr_host[i + 1] <= level_ptr_host[i])
        return fail(h, DFK_ERR_INVALID_ARG, pre + " has no records (level_ptr must increase)");
    }
    if (m == 0) return DFK_OK;
    // [CSR of the priors per keyframe: ptr[K + 1] | indices m] | level_ptr[m + 1] | sigma[m]
    Staging s(h->staging);
    const Part<int> csr_at = s.add<int>(K + 1 + m), lp_at = s.add<int>(m + 1);
    const Part<float> sg_at = s.add<float>(m);
    fill_csr(csr_at.at(s.host()), K, m, [&](int i) { return prior_kf_host[i]; });
    memcpy(lp_at.at(s.host()), level_ptr_host, sizeof(int) * (m + 1));
    memcpy(sg_at.at(s.host()), sigma_host, sizeof(float) * m);
    DeviceGuard guard(h->device);
    const char* what = "[Window::AddDepthPriors] index upload failed";
    DFK_CUDA(h, h->window_lists.ensure(s.bytes / sizeof(int)), what);
    DFK_CUDA(h, cudaMemcpyAsync(h->window_lists.ptr, s.host(), s.bytes, cudaMemcpyHostToDevice, h->stream), what);
    int* d = h->window_lists.ptr;
    DFK_CUDA(h, launch_window_add_depth_priors(w->dev, m, csr_at.at(d), csr_at.at(d) + K + 1, lp_at.at(d), sg_at.at(d),
                                               records_dev, window_dev, h->stream),
             "[Window::AddDepthPriors] kernel launch failed");
    h->launches += 1;
    return DFK_OK;
  });
}

DfkStatus dfk_window_add_keyframe_priors(DfkHandle h, const DfkWindow* w, const double* priors_dev,
                                         const double* delta_dev, float* window_dev)
{
  return guarded(h, [&] {
    if (!w || !window_dev) return fail(h, DFK_ERR_INVALID_ARG, "[Window::AddKeyframePriors] null argument");
    if (w->device != h->device)
      return fail(h, DFK_ERR_INVALID_ARG, "[Window::AddKeyframePriors] window and handle live on different devices");
    if (w->kp.num_priors == 0) return DFK_OK;
    if (!priors_dev || !delta_dev) return fail(h, DFK_ERR_INVALID_ARG, "[Window::AddKeyframePriors] null argument");
    DeviceGuard guard(h->device);
    DFK_CUDA(h, launch_window_add_keyframe_priors(w->dev, w->kp, priors_dev, delta_dev, window_dev, h->stream),
             "[Window::AddKeyframePriors] kernel launch failed");
    h->launches += 1;
    return DFK_OK;
  });
}

namespace {

// N(m): the keyframes that share a pair, a link or a keyframe prior with m, ascending
std::vector<int> window_blanket(const DfkWindow* w, int m)
{
  const int K = w->dev.num_keyframes;
  std::vector<char> in(K, 0);
  auto tie = [&](int a, int b) {
    if (a < K && b < K && (a == m || b == m)) in[a] = in[b] = 1;
  };
  for (size_t p = 0; p < w->pair_k0.size(); ++p) tie(w->pair_k0[p], w->pair_k1[p]);
  for (size_t l = 0; l < w->link_k0.size(); ++l) tie(w->link_k0[l], w->link_k1[l]);
  for (size_t q = 0; q + 1 < w->prior_ptr.size(); ++q) {
    const auto b = w->prior_kf.begin() + w->prior_ptr[q], e = w->prior_kf.begin() + w->prior_ptr[q + 1];
    if (std::find(b, e, m) != e)
      for (auto it = b; it != e; ++it) in[*it] = 1;
  }
  in[m] = 0;
  std::vector<int> out;
  for (int k = 0; k < K; ++k)
    if (in[k]) out.push_back(k);
  return out;
}

bool prior_contains(const DfkWindow* w, int q, int m)
{
  const auto b = w->prior_kf.begin() + w->prior_ptr[q], e = w->prior_kf.begin() + w->prior_ptr[q + 1];
  return std::find(b, e, m) != e;
}

}  // namespace

DfkStatus dfk_window_blanket(DfkHandle h, const DfkWindow* w, int m, int32_t* kf_out, int32_t* n)
{
  return guarded(h, [&] {
    if (!w || !kf_out || !n) return fail(h, DFK_ERR_INVALID_ARG, "[Window::Blanket] null argument");
    if (m < 0 || m >= w->dev.num_keyframes)
      return fail(h, DFK_ERR_INVALID_ARG, "[Window::Blanket] keyframe " + std::to_string(m) + " is not in the window");
    const std::vector<int> nb = window_blanket(w, m);
    std::copy(nb.begin(), nb.end(), kf_out);
    *n = (int32_t)nb.size();
    return DFK_OK;
  });
}

DfkStatus dfk_window_marginalize_keyframe(DfkHandle h, const DfkWindow* w, const float* records_dev,
                                          const float* geo_records_dev, int m, int num_frame_priors,
                                          const double* frame_priors_dev, const double* frame_delta_dev,
                                          const double* kf_priors_dev, const double* kf_delta_dev,
                                          double code_prior_weight, const double* code_m_host, double* prior_dev,
                                          int32_t* info_dev)
{
  return guarded(h, [&] {
    const char* what = "[Window::MarginalizeKeyframe] ";
    auto bad = [&](DfkStatus s, const std::string& msg) { return fail(h, s, what + msg); };
    if (!w || !records_dev || !prior_dev || !info_dev || num_frame_priors < 0 ||
        (num_frame_priors > 0 && (!frame_priors_dev || !frame_delta_dev)))
      return bad(DFK_ERR_INVALID_ARG, "null argument");
    if (w->device != h->device) return bad(DFK_ERR_INVALID_ARG, "window and handle live on different devices");
    const int K = w->dev.num_keyframes, C = w->dev.code_size, B = 6 + C;
    if (m < 0 || m >= K) return bad(DFK_ERR_INVALID_ARG, "keyframe " + std::to_string(m) + " is not in the window");
    if (w->dev.num_links > 0 && !geo_records_dev)
      return bad(DFK_ERR_INVALID_ARG, "window has geometric links but no geometric records");
    if (!(std::isfinite(code_prior_weight) && code_prior_weight >= 0.0))
      return bad(DFK_ERR_INVALID_ARG, "code_prior_weight must be finite and >= 0");
    if (code_prior_weight > 0.0 && !code_m_host) return bad(DFK_ERR_INVALID_ARG, "code_prior_weight > 0 needs m's code");
    for (size_t p = 0; p < w->pair_k0.size(); ++p)
      if (w->pair_k0[p] == m && w->pair_k1[p] >= K)
        return bad(DFK_ERR_INVALID_ARG, "keyframe " + std::to_string(m) + " still has tracked frames: marginalise them first");
    const int Q = w->kp.num_priors;
    std::vector<int> kq;  // the keyframe priors that contain m
    for (int q = 0; q < Q; ++q)
      if (prior_contains(w, q, m)) kq.push_back(q);
    if (!kq.empty() && (!kf_priors_dev || !kf_delta_dev))
      return bad(DFK_ERR_INVALID_ARG, "keyframe priors contain m but none were given");
    const std::vector<int> nb = window_blanket(w, m);
    const int n = (int)nb.size();
    if (n == 0) return bad(DFK_ERR_INVALID_ARG, "keyframe " + std::to_string(m) + " shares no factor with another");
    if (n > DFK_MAX_BLANKET)
      return bad(DFK_ERR_UNSUPPORTED, "blanket of " + std::to_string(n) + " keyframes (at most " +
                                          std::to_string(DFK_MAX_BLANKET) + ")");
    std::vector<int> loc(K, -1);
    loc[m] = 0;
    for (int i = 0; i < n; ++i) loc[nb[i]] = 1 + i;
    std::vector<KfMargRef> refs;
    for (size_t i = 0; i < w->item_pair.size(); ++i) {
      const int k0 = w->pair_k0[w->item_pair[i]], k1 = w->pair_k1[w->item_pair[i]];
      if (k1 < K && (k0 == m || k1 == m)) refs.push_back({0, (int)i, loc[k0], loc[k1]});
    }
    for (size_t l = 0; l < w->link_k0.size(); ++l)
      if (w->link_k0[l] == m || w->link_k1[l] == m) refs.push_back({1, (int)l, loc[w->link_k0[l]], loc[w->link_k1[l]]});
    for (int i = 0; i < num_frame_priors; ++i) refs.push_back({2, i, 0, 0});
    for (int q : kq) refs.push_back({3, q, 0, 0});
    const int T = n + 1 + n * (n + 1) / 2;
    std::vector<int> tasks;
    window_eliminate_first_tasks(n, tasks);
    const bool code = code_prior_weight > 0.0;
    // [refs | tile_row | tile_col | mem_loc | update tasks | code of m], and the workspace [tiles | rhs | f]
    Staging s(h->staging);
    const Part<KfMargRef> refs_at = s.add<KfMargRef>(refs.size());
    const Part<int> tr = s.add<int>(T), tc = s.add<int>(T), ml = s.add<int>(w->prior_kf.size());
    const Part<int> tk = s.add<int>(tasks.size());
    const Part<double> code_at = s.add<double>(code ? C : 0);
    unsigned char* hb = s.host();
    std::copy(refs.begin(), refs.end(), refs_at.at(hb));
    for (int t = 0; t <= n; ++t) tr.at(hb)[t] = t;  // tile_col 0
    for (int I = 1, t = n + 1; I <= n; ++I)
      for (int J = 1; J <= I; ++J, ++t) {
        tr.at(hb)[t] = I;
        tc.at(hb)[t] = J;
      }
    for (size_t a = 0; a < w->prior_kf.size(); ++a) ml.at(hb)[a] = loc[w->prior_kf[a]];
    std::copy(tasks.begin(), tasks.end(), tk.at(hb));
    if (code) memcpy(code_at.at(hb), code_m_host, C * sizeof(double));
    Layout ws;
    const Part<double> tiles = ws.add<double>((size_t)(T + 1) * B * B), rhs = ws.add<double>((size_t)(n + 1) * B);
    const Part<double> f = ws.add<double>(1);

    DeviceGuard guard(h->device);
    DFK_CUDA(h, h->marg_dev.ensure(ws.bytes), "[Window::MarginalizeKeyframe] scratch allocation failed");
    DFK_TRY(s.upload(h, h->marg_lists, what));  // pageable source: staged before the call returns
    unsigned char* li = h->marg_lists.ptr;
    KfMargDev md{};
    md.n = n;
    md.num_refs = (int)refs.size();
    md.refs = refs_at.at(li);
    md.tile_row = tr.at(li); md.tile_col = tc.at(li); md.mem_loc = ml.at(li);
    md.records = records_dev; md.geo = geo_records_dev;
    md.fpriors = frame_priors_dev; md.fdelta = frame_delta_dev;
    md.kpriors = kf_priors_dev; md.kdelta = kf_delta_dev;
    md.w = code_prior_weight; md.code = code_at.at(li);
    md.tiles = tiles.at(h->marg_dev.ptr); md.rhs = rhs.at(h->marg_dev.ptr); md.f = f.at(h->marg_dev.ptr);
    md.info = info_dev;
    const char* launch = "[Window::MarginalizeKeyframe] kernel launch failed";
    DFK_CUDA(h, launch_window_marg_gather(w->dev, w->kp, md, T, h->stream), launch);
    DFK_CUDA(h, launch_window_eliminate_first(C, n, md.tiles, md.rhs, info_dev, tk.at(li), (int)tasks.size() / 4,
                                              h->stream), launch);
    DFK_CUDA(h, launch_window_marg_finalize(C, md, T, prior_dev, h->stream), launch);
    h->launches += 4;
    return DFK_OK;
  });
}

DfkStatus dfk_window_solver_create(DfkHandle h, const DfkWindow* w, int num_fixed, const int32_t* fixed_vars,
                                   DfkWindowSolver** out)
{
  return dfk_window_solver_create_from(h, w, num_fixed, fixed_vars, nullptr, out);
}

DfkStatus dfk_window_solver_create_from(DfkHandle h, const DfkWindow* w, int num_fixed, const int32_t* fixed_vars,
                                        const DfkWindowSolver* prev, DfkWindowSolver** out)
{
  return guarded(h, [&] {
    if (!w || !out || num_fixed < 0 || (num_fixed > 0 && !fixed_vars))
      return fail(h, DFK_ERR_INVALID_ARG, "[WindowSolver] null argument");
    if (prev && prev->device != h->device)
      return fail(h, DFK_ERR_INVALID_ARG, "[WindowSolver] previous solver and handle live on different devices");
    if (prev && (prev->code_size != w->dev.code_size || prev->num_keyframes > w->dev.num_keyframes))
      return fail(h, DFK_ERR_INVALID_ARG, "[WindowSolver] the window does not extend the previous solver's: " +
                                              std::to_string(prev->num_keyframes) + " keyframes of code size " +
                                              std::to_string(prev->code_size) + " need a prefix of " +
                                              std::to_string(w->dev.num_keyframes) + " of size " +
                                              std::to_string(w->dev.code_size));
    if (!prev) *out = nullptr;
    if (w->device != h->device)
      return fail(h, DFK_ERR_INVALID_ARG, "[WindowSolver] window and handle live on different devices");
    const int K = w->dev.num_keyframes, C = w->dev.code_size, n = K * (6 + C);
    std::vector<int> fixed(fixed_vars, fixed_vars + num_fixed);
    std::vector<char> seen(n, 0);
    for (int q = 0; q < num_fixed; ++q) {
      if (fixed[q] < 0 || fixed[q] >= n)
        return fail(h, DFK_ERR_INVALID_ARG, "[WindowSolver] fixed variable " + std::to_string(fixed[q]) +
                                                " outside the window's " + std::to_string(n) + " variables");
      if (seen[fixed[q]]++)
        return fail(h, DFK_ERR_INVALID_ARG, "[WindowSolver] fixed variable " + std::to_string(fixed[q]) + " listed twice");
    }
    DeviceGuard guard(h->device);
    std::unique_ptr<DfkWindowSolver> s(new (std::nothrow) DfkWindowSolver());
    if (!s) return oom(h);
    s->device = h->device;
    s->num_vars = n; s->code_size = C; s->num_keyframes = K;
    DFK_CUDA(h, window_solver_create(K, C, w->dev.num_frames, w->pair_k0, w->pair_k1, w->link_k0, w->link_k1, w->blk_i,
                                     w->blk_j, w->kp.block_off, fixed, &s->dev),
             "[WindowSolver] workspace allocation failed");
    if (prev) {
      if (!window_solver_extends(prev->dev, s->dev))
        return fail(h, DFK_ERR_INVALID_ARG,
                    "[WindowSolver] the window fixes other variables among the previous solver's keyframes");
      int columns = 0;
      DFK_CUDA(h, window_solver_adopt(s->dev, prev->dev, h->stream, &columns),
               "[WindowSolver] copying the previous solver's factor failed");
    }
    *out = s.release();
    return DFK_OK;
  });
}

DfkStatus dfk_window_solver_update(DfkHandle h, DfkWindowSolver* s, const float* window_dev,
                                   const DfkWindowUpdateParams* p, const double* codes, double* dx_dev,
                                   int32_t* info_dev, int32_t* first_column)
{
  return guarded(h, [&] {
    if (!s || !window_dev || !p || !dx_dev || !info_dev || !first_column)
      return fail(h, DFK_ERR_INVALID_ARG, "[WindowSolver] null argument");
    if (s->device != h->device)
      return fail(h, DFK_ERR_INVALID_ARG, "[WindowSolver] solver and handle live on different devices");
    if (!(std::isfinite(p->diag_eps) && p->diag_eps >= 0.0))
      return fail(h, DFK_ERR_INVALID_ARG, "[WindowSolver] diag_eps must be finite and >= 0");
    if (!(std::isfinite(p->code_prior_weight) && p->code_prior_weight >= 0.0))
      return fail(h, DFK_ERR_INVALID_ARG, "[WindowSolver] code_prior_weight must be finite and >= 0");
    if (p->code_prior_weight > 0.0 && !codes)
      return fail(h, DFK_ERR_INVALID_ARG, "[WindowSolver] code_prior_weight > 0 needs the codes");
    DeviceGuard guard(h->device);
    int j0 = 0;
    DFK_CUDA(h, launch_window_solver_update(s->dev, window_dev, p->code_prior_weight, p->diag_eps, codes, dx_dev,
                                            info_dev, h->stream, &h->launches, &j0),
             "[WindowSolver] incremental update failed");
    *first_column = j0;
    return DFK_OK;
  });
}

DfkStatus dfk_window_solver_destroy(DfkHandle h, DfkWindowSolver* s)
{
  return guarded(h, [&] {
    if (!s) return DFK_OK;
    DeviceGuard guard(s->device);
    delete s;
    return DFK_OK;
  });
}

DfkStatus dfk_window_solver_tiles(DfkHandle h, const DfkWindowSolver* s, size_t* tiles)
{
  return guarded(h, [&] {
    if (!s || !tiles) return fail(h, DFK_ERR_INVALID_ARG, "[WindowSolver] null argument");
    *tiles = window_solver_tiles(s->dev);
    return DFK_OK;
  });
}

DfkStatus dfk_window_solve(DfkHandle h, const DfkWindowSolver* s, const float* window_dev, const DfkWindowSolveParams* p,
                           const double* codes, double* dx_dev, int32_t* info_dev)
{
  return guarded(h, [&] {
    if (!s || !window_dev || !p || !dx_dev || !info_dev)
      return fail(h, DFK_ERR_INVALID_ARG, "[WindowSolver] null argument");
    if (s->device != h->device)
      return fail(h, DFK_ERR_INVALID_ARG, "[WindowSolver] solver and handle live on different devices");
    if (!(std::isfinite(p->lambda) && p->lambda >= 0.0))
      return fail(h, DFK_ERR_INVALID_ARG, "[WindowSolver] lambda must be finite and >= 0");
    if (!(std::isfinite(p->code_prior_weight) && p->code_prior_weight >= 0.0))
      return fail(h, DFK_ERR_INVALID_ARG, "[WindowSolver] code_prior_weight must be finite and >= 0");
    if (p->code_prior_weight > 0.0 && !codes)
      return fail(h, DFK_ERR_INVALID_ARG, "[WindowSolver] code_prior_weight > 0 needs the codes");
    DeviceGuard guard(h->device);
    DFK_CUDA(h, launch_window_solve(s->dev, window_dev, p->lambda, p->code_prior_weight, codes, dx_dev, info_dev,
                                    h->stream, &h->launches),
             "[WindowSolver] kernel launch failed");
    return DFK_OK;
  });
}

// ---------------------------------------------------------------------------------------------- window problem
DfkStatus dfk_window_problem_create(DfkHandle h, const DfkWindowProblemDesc* d, DfkWindowProblem** out)
{
  return guarded(h, [&] {
    const std::string what = "[WindowProblem] ";
    if (!d || !out || !d->window) return fail(h, DFK_ERR_INVALID_ARG, what + "null argument");
    *out = nullptr;
    const DfkWindow* w = d->window;
    if (w->device != h->device) return fail(h, DFK_ERR_INVALID_ARG, what + "window and handle live on different devices");
    const int K = w->dev.num_keyframes, F = w->dev.num_frames, C = w->dev.code_size, B = 6 + C, NP = K + F;
    const int nd = d->num_dense, nr = d->num_reproj, ng = d->num_geo, ndep = d->num_depth, ne = d->num_error;
    const int mf = d->num_frame_priors, nkm = (int)w->prior_kf.size();
    if (nd < 0 || nr < 0 || ng < 0 || ndep < 0 || ne < 0 || mf < 0 || ne > 65535 || ndep > 65535)
      return fail(h, DFK_ERR_INVALID_ARG, what + "negative item count / more than 65535 error or depth items");
    if (nd + nr != w->dev.num_items || ng != w->dev.num_links)
      return fail(h, DFK_ERR_INVALID_ARG, what + "the items do not match the window's records (" +
                                              std::to_string(w->dev.num_items) + " records, " +
                                              std::to_string(w->dev.num_links) + " links)");
    if ((nd && (!d->dense || !d->dense_slots)) || (nr && (!d->reproj || !d->reproj_slots)) ||
        (ng && (!d->geo || !d->geo_slots || !d->geo_records_dev)) || (ndep && (!d->depth || !d->depth_slots)) ||
        (ne && (!d->error || !d->error_slots || !d->error_depth)) || !d->records_dev ||
        (mf && (!d->frame_prior_kf || !d->frame_prior_rows || !d->frame_prior_x0)) ||
        (w->kp.num_priors && (!d->kf_prior_rows || !d->kf_prior_x0)))
      return fail(h, DFK_ERR_INVALID_ARG, what + "null argument");
    // slots: pose slots name a keyframe or a frame, code slots a keyframe, an error item's depth slot a depth item.
    // Every kind checks its fields in this order
    enum { POSE0 = 1, POSE1 = 2, CODE0 = 4, CODE1 = 8, DEPTH = 16 };
    const char* const field_name[5] = {"pose0", "pose1", "code0", "code1", "depth"};
    const int field_end[5] = {NP, NP, K, K, ndep};
    struct Kind {
      const char* name;
      const DfkWindowItemSlots* slots;
      int n;
      int fields;
    };
    const Kind kinds[] = {{"dense", d->dense_slots, nd, POSE0 | POSE1 | CODE0},
                          {"reprojection", d->reproj_slots, nr, POSE0 | POSE1 | CODE0},
                          {"geometric", d->geo_slots, ng, POSE0 | POSE1 | CODE0 | CODE1},
                          {"depth", d->depth_slots, ndep, CODE0},
                          {"error", d->error_slots, ne, POSE0 | POSE1 | DEPTH}};
    for (const Kind& k : kinds)
      for (int i = 0; i < k.n; ++i) {
        const DfkWindowItemSlots& s = k.slots[i];
        const int v[5] = {s.pose0, s.pose1, s.code0, s.code1, (k.fields & DEPTH) ? d->error_depth[i] : 0};
        for (int f = 0; f < 5; ++f)
          if ((k.fields >> f & 1) && !slot_ok(v[f], 0, field_end[f]))
            return fail(h, DFK_ERR_INVALID_ARG, what + k.name + " item " + std::to_string(i) + ": " + field_name[f] +
                                                    " slot out of range");
      }
    for (int i = 0; i < mf; ++i)
      if (!slot_ok(d->frame_prior_kf[i], 0, K))
        return fail(h, DFK_ERR_INVALID_ARG, what + "frame prior " + std::to_string(i) + " names a keyframe outside the window");
    DeviceGuard guard(h->device);
    std::unique_ptr<DfkWindowProblem> p(new (std::nothrow) DfkWindowProblem());
    if (!p) return oom(h);
    p->device = h->device; p->w = w;
    p->K = K; p->F = F; p->C = C; p->B = B;
    p->nd = nd; p->nr = nr; p->ng = ng; p->ndep = ndep; p->ne = ne; p->mf = mf; p->nkm = nkm;
    p->S = (size_t)NP * 7 + (size_t)K * C;
    p->avg_dpt = h->params.sfmparams.avg_dpt;
    p->huber_delta = h->params.sfmparams.huber_delta;
    p->records = d->records_dev; p->geo_records = d->geo_records_dev;
    const char* amsg = "[WindowProblem] allocation failed";
    const size_t PD = DFK_PRIOR_DOUBLES(C), X = 7 + (size_t)C, nx = (size_t)mf + nkm;  // nx: frozen points
    // ---- one allocation: the parts create uploads, staged in a host image of the problem's own (the sparse batches
    // below stage through h->staging), then the scratch
    std::vector<unsigned char> image;
    Staging s(image);
    p->dense = s.add<SfmItemDev>(nd);
    p->err = s.add<EvalErrorDesc>(ne);
    p->areas = s.add<double>(ne);
    p->dense_slots = s.add<int4>(nd); p->err_slots = s.add<int4>(ne); p->rep_slots = s.add<int4>(nr);
    p->geo_slots = s.add<int4>(ng); p->depth_slots = s.add<int4>(ndep);
    p->depth = s.add<DepthDecodeDesc>(ndep);
    p->frows = s.add<double>(mf * PD);
    p->fp_lists = s.add<int>(mf > 0 ? K + 1 + mf : 0);
    p->kfrows = s.add<double>(w->kp.num_priors > 0 ? (size_t)w->prior_off.back() : 0);
    p->delta_kf = s.add<int>(nx);
    p->x0 = s.add<double>(nx * X);
    p->state = s.add<double>(2 * p->S);
    Layout scratch{s.bytes};
    p->dense_codes = scratch.add<float>((size_t)nd * C);
    p->depth_codes = scratch.add<float>((size_t)ndep * C);  // the repose kernel writes them from the state
    p->delta = scratch.add<double>(nx * B);
    p->err_out = scratch.add<float>(std::max<size_t>(1, 2 * (size_t)(ne + nr + ng)));
    Layout sm;
    p->sm_energy = sm.add<double>(8); p->sm_info = sm.add<int32_t>(1); p->sm_depth_energy = sm.add<double>(1);
    p->small = scratch.add<unsigned char>(sm.bytes);
    DFK_CUDA(h, p->blob.ensure(scratch.bytes), amsg);
    DFK_CUDA(h, p->small_host.ensure(sm.bytes), amsg);
    unsigned char *const hb = s.host(), *const db = p->blob.ptr;
    const std::vector<float> zero_code(std::max(C, 1), 0.0f);
    // ---- dense items: the batch's checks, kernel choice and tile plan, with a code slot of the problem's own each
    if (nd > 0) {
      std::vector<DfkSfmWorkItem> t(d->dense, d->dense + nd);
      for (auto& it : t) it.code = zero_code.data();
      DFK_TRY(choose_step_kernel(h, t.data(), nd, C, &p->step));
      SfmItemDev* items = p->dense.at(hb);
      DFK_TRY(build_items(h, t.data(), nd, C, p->step.tile_px, p->step.max_ctas, p->dense_codes.at(db), items, &p->plan));
      // ray tables of its own, not the handle's cache: the cache may flush (and free) its tables
      std::vector<const SfmItemDev*> owner;
      for (int i = 0; i < nd; ++i) {
        SfmItemDev& it = items[i];
        size_t r = 0;
        for (; r < owner.size(); ++r) {
          const SfmItemDev& o = *owner[r];
          if (o.fx == it.fx && o.fy == it.fy && o.u0 == it.u0 && o.v0 == it.v0 && o.width == it.width &&
              o.height == it.height)
            break;
        }
        if (r == owner.size()) {
          owner.push_back(&it);
          p->rays.emplace_back();
          DFK_CUDA(h, p->rays.back().ensure((size_t)it.width + it.height), amsg);
        }
        it.ray_tab = p->rays[r].ptr;
      }
      p->dense_tmpl.assign(items, items + nd);
    }
    // ---- sparse links: the batches' checks and staging, into blocks of the problem's own
    if (nr > 0) {
      std::vector<DfkReprojectionItem> t(d->reproj, d->reproj + nr);
      for (auto& it : t) it.code = zero_code.data();
      DFK_TRY(stage(h, what + "reprojection ", true, t.data(), nr, C, 0, h->staging, p->rep, &p->rep_st));
    }
    if (ng > 0) {
      std::vector<DfkSparseGeometricItem> t(d->geo, d->geo + ng);
      for (auto& it : t) it.code0 = it.code1 = zero_code.data();
      DFK_TRY(stage(h, what + "geometric ", true, t.data(), ng, C, 0, h->staging, p->geo, &p->geo_st));
    }
    // ---- the error path: depth decodes into scratch of the problem's own, and the error items reading it
    Layout dl;
    std::vector<Part<float>> dep(ndep);
    for (int i = 0; i < ndep; ++i) {
      const DfkDepthDecodeItem& it = d->depth[i];
      const uint32_t W = it.dpt.width, H = it.dpt.height;
      if (W == 0 || H == 0 || !img_ok(&it.prx_orig, W, H, 1) || !img_ok(&it.prx_jac, W, H, C))
        return fail(h, DFK_ERR_INVALID_ARG, what + "inconsistent image views in depth item " + std::to_string(i));
      dep[i] = dl.add<float>((size_t)W * H);
    }
    if (ndep > 0) {
      DFK_CUDA(h, p->depth_scratch.ensure(dl.bytes), amsg);
      for (int i = 0; i < ndep; ++i) {
        const DfkDepthDecodeItem& it = d->depth[i];
        set_depth_decode_desc(p->depth.at(hb)[i], it, C, p->depth_codes.at(db) + (size_t)i * C,
                              dep[i].at(p->depth_scratch.ptr), it.dpt.width, &p->depth_max_blocks);
      }
    }
    for (int i = 0; i < ne; ++i) {
      const DfkSfmWorkItem& it = d->error[i];
      const DfkDepthDecodeItem& dep_it = d->depth[d->error_depth[i]];
      const DfkImage dpt{dep[d->error_depth[i]].at(p->depth_scratch.ptr), (size_t)dep_it.dpt.width * 4,
                         dep_it.dpt.width, dep_it.dpt.height};
      const uint32_t W = it.img0.width, H = it.img0.height;
      if (it.code)
        return fail(h, DFK_ERR_INVALID_ARG, what + "error item " + std::to_string(i) +
                                                ": no fused depth decode (the depth comes from its depth item)");
      if (W == 0 || H == 0 || !img_ok(&it.img0, W, H, 1) || !img_ok(&it.img1, W, H, 1) || !img_ok(&dpt, W, H, 1))
        return fail(h, DFK_ERR_INVALID_ARG, what + "inconsistent image views in error item " + std::to_string(i));
      if (!cam_ok(&it.cam, W, H))
        return fail(h, DFK_ERR_INVALID_ARG, what + "camera viewport larger than the image views in error item " +
                                                std::to_string(i));
      const float ident[7] = {0, 0, 0, 1, 0, 0, 0};  // the repose kernel sets the relative pose
      set_eval_error_desc(p->err.at(hb)[i], it.cam, ident, it.img0, it.img1, dpt, &p->err_rows, &p->err_max_blocks);
      p->areas.at(hb)[i] = (double)W * (double)H;
    }
    p->err_tmpl.assign(p->err.at(hb), p->err.at(hb) + ne);
    p->areas_tmpl.assign(p->areas.at(hb), p->areas.at(hb) + ne);
    // ---- slots, one part per kind
    auto put_slots = [&](Part<int4> to, const DfkWindowItemSlots* sl, int n) {
      for (int i = 0; i < n; ++i) to.at(hb)[i] = make_int4(sl[i].pose0, sl[i].pose1, sl[i].code0, sl[i].code1);
    };
    put_slots(p->dense_slots, d->dense_slots, nd); put_slots(p->err_slots, d->error_slots, ne);
    put_slots(p->rep_slots, d->reproj_slots, nr); put_slots(p->geo_slots, d->geo_slots, ng);
    put_slots(p->depth_slots, d->depth_slots, ndep);
    p->slots_tmpl.assign(p->dense_slots.at(hb), p->dense_slots.at(hb) + nd);
    p->slots_tmpl.insert(p->slots_tmpl.end(), p->err_slots.at(hb), p->err_slots.at(hb) + ne);
    for (int j = 0; j < nr; ++j) p->rep_size_h.push_back(d->reproj[j].num_matches);
    for (int j = 0; j < ng; ++j) p->geo_size_h.push_back(d->geo[j].num_points);
    p->rep_slots_h.assign(p->rep_slots.at(hb), p->rep_slots.at(hb) + nr);
    p->geo_slots_h.assign(p->geo_slots.at(hb), p->geo_slots.at(hb) + ng);
    p->lin_dense.assign(nd, 0); p->lin_rep.assign(nr, 0); p->lin_geo.assign(ng, 0);
    p->active.assign(nd, 1);
    // ---- priors: rows, add_priors' lists, the keyframe of every delta row and the frozen points (frame priors, then
    // keyframe-prior members)
    if (mf > 0) {
      memcpy(p->frows.at(hb), d->frame_prior_rows, sizeof(double) * mf * PD);
      fill_csr(p->fp_lists.at(hb), K, mf, [&](int i) { return d->frame_prior_kf[i]; });
      std::copy(d->frame_prior_kf, d->frame_prior_kf + mf, p->delta_kf.at(hb));
      memcpy(p->x0.at(hb), d->frame_prior_x0, sizeof(double) * mf * X);
    }
    if (w->kp.num_priors > 0) {
      memcpy(p->kfrows.at(hb), d->kf_prior_rows, sizeof(double) * w->prior_off.back());
      std::copy(w->prior_kf.begin(), w->prior_kf.end(), p->delta_kf.at(hb) + mf);
      memcpy(p->x0.at(hb) + mf * X, d->kf_prior_x0, sizeof(double) * nkm * X);
    }
    // ---- state (zero codes, identity poses until set_state)
    for (int i = 0; i < 2 * NP; ++i) p->state.at(hb)[(size_t)(i / NP) * p->S + (size_t)(i % NP) * 7 + 3] = 1.0;
    DFK_TRY(s.upload(h, p->blob, what));
    if (nd > 0) {
      DFK_CUDA(h, launch_sfm_ray_tables(p->dense.at(db), nd, h->stream), "[WindowProblem] kernel launch failed");
      h->launches += 1;
    }
    // ---- the gauge solver
    const std::vector<int> gauge{0, 1, 2, 3, 4, 5};
    DFK_CUDA(h, window_solver_create(K, C, F, w->pair_k0, w->pair_k1, w->link_k0, w->link_k1, w->blk_i, w->blk_j,
                                     w->kp.block_off, gauge, &p->solver[1]),
             "[WindowProblem] solver workspace allocation failed");
    DFK_CUDA(h, cudaStreamSynchronize(h->stream), "[WindowProblem] upload failed");
    *out = p.release();
    return DFK_OK;
  });
}

DfkStatus dfk_window_problem_destroy(DfkHandle h, DfkWindowProblem* p)
{
  return guarded(h, [&] {
    if (!p) return DFK_OK;
    DeviceGuard guard(p->device);
    delete p;
    return DFK_OK;
  });
}

DfkStatus dfk_window_problem_set_state(DfkHandle h, DfkWindowProblem* p, const double* poses, const double* codes)
{
  return guarded(h, [&] {
    if (!p || !poses || (!codes && p->K * p->C > 0)) return fail(h, DFK_ERR_INVALID_ARG, "[WindowProblem] null argument");
    if (p->device != h->device) return fail(h, DFK_ERR_INVALID_ARG, "[WindowProblem] problem and handle live on different devices");
    DeviceGuard guard(h->device);
    const size_t np = (size_t)(p->K + p->F) * 7;
    DFK_CUDA(h, cudaMemcpyAsync(p->st(p->cur), poses, sizeof(double) * np, cudaMemcpyDefault, h->stream),
             "[WindowProblem] state copy failed");
    if (p->K * p->C > 0)
      DFK_CUDA(h, cudaMemcpyAsync(p->st(p->cur) + np, codes, sizeof(double) * (p->S - np), cudaMemcpyDefault, h->stream),
               "[WindowProblem] state copy failed");
    p->isam_fresh = true;
    return DFK_OK;
  });
}

DfkStatus dfk_window_problem_get_state(DfkHandle h, const DfkWindowProblem* p, double* poses, double* codes)
{
  return guarded(h, [&] {
    if (!p || !poses || (!codes && p->K * p->C > 0)) return fail(h, DFK_ERR_INVALID_ARG, "[WindowProblem] null argument");
    if (p->device != h->device) return fail(h, DFK_ERR_INVALID_ARG, "[WindowProblem] problem and handle live on different devices");
    DeviceGuard guard(h->device);
    const size_t np = (size_t)(p->K + p->F) * 7;
    DFK_CUDA(h, cudaMemcpyAsync(poses, p->st(p->cur), sizeof(double) * np, cudaMemcpyDefault, h->stream),
             "[WindowProblem] state copy failed");
    if (p->K * p->C > 0)
      DFK_CUDA(h, cudaMemcpyAsync(codes, p->st(p->cur) + np, sizeof(double) * (p->S - np), cudaMemcpyDefault, h->stream),
               "[WindowProblem] state copy failed");
    return DFK_OK;
  });
}

DfkStatus dfk_window_problem_linearize(DfkHandle h, DfkWindowProblem* p, float* window_dev)
{
  return guarded(h, [&] {
    if (!p || !window_dev) return fail(h, DFK_ERR_INVALID_ARG, "[WindowProblem::linearize] null argument");
    if (p->device != h->device) return fail(h, DFK_ERR_INVALID_ARG, "[WindowProblem] problem and handle live on different devices");
    DeviceGuard guard(h->device);
    return problem_linearize(h, p, p->st(p->cur), window_dev);
  });
}

DfkStatus dfk_window_problem_error(DfkHandle h, DfkWindowProblem* p, double* out_dev)
{
  return guarded(h, [&] {
    if (!p || !out_dev) return fail(h, DFK_ERR_INVALID_ARG, "[WindowProblem::error] null argument");
    if (p->device != h->device) return fail(h, DFK_ERR_INVALID_ARG, "[WindowProblem] problem and handle live on different devices");
    DeviceGuard guard(h->device);
    DFK_TRY(problem_error(h, p, p->st(p->cur), 0.0));
    DFK_CUDA(h, cudaMemcpyAsync(out_dev, p->energy(), sizeof(double) * DFK_WINDOW_ERROR_DOUBLES, cudaMemcpyDeviceToDevice,
                                h->stream),
             "[WindowProblem::error] copy failed");
    return DFK_OK;
  });
}

DfkStatus dfk_window_problem_error_ex(DfkHandle h, DfkWindowProblem* p, double* out_dev)
{
  return guarded(h, [&] {
    if (!p || !out_dev) return fail(h, DFK_ERR_INVALID_ARG, "[WindowProblem::error_ex] null argument");
    if (p->device != h->device) return fail(h, DFK_ERR_INVALID_ARG, "[WindowProblem] problem and handle live on different devices");
    DeviceGuard guard(h->device);
    DFK_TRY(problem_error(h, p, p->st(p->cur), 0.0));
    const char* what = "[WindowProblem::error_ex] copy failed";
    DFK_CUDA(h, cudaMemcpyAsync(out_dev, p->energy(), sizeof(double) * DFK_WINDOW_ERROR_DOUBLES, cudaMemcpyDeviceToDevice,
                                h->stream),
             what);
    if (p->ndp > 0)
      DFK_CUDA(h, cudaMemcpyAsync(out_dev + DFK_WINDOW_ERROR_DOUBLES, p->depth_energy(), sizeof(double),
                                  cudaMemcpyDeviceToDevice, h->stream),
               what);
    else
      DFK_CUDA(h, cudaMemsetAsync(out_dev + DFK_WINDOW_ERROR_DOUBLES, 0, sizeof(double), h->stream), what);
    return DFK_OK;
  });
}

DfkStatus dfk_window_problem_set_depth_priors(DfkHandle h, DfkWindowProblem* p, int m, const int32_t* prior_kf,
                                              const float* sigma, const int32_t* level_ptr,
                                              const DfkDepthPriorItem* items)
{
  return guarded(h, [&] {
    const char* what = "[WindowProblem::set_depth_priors] ";
    const std::string w(what);
    if (!p || m < 0 || (m > 0 && (!prior_kf || !sigma || !level_ptr || !items)))
      return fail(h, DFK_ERR_INVALID_ARG, w + "null argument");
    if (p->device != h->device) return fail(h, DFK_ERR_INVALID_ARG, "[WindowProblem] problem and handle live on different devices");
    if (m > 0 && level_ptr[0] != 0) return fail(h, DFK_ERR_INVALID_ARG, w + "level_ptr[0] must be 0");
    for (int i = 0; i < m; ++i) {
      const std::string pre = w + "prior " + std::to_string(i);
      if (prior_kf[i] < 0 || prior_kf[i] >= p->K) return fail(h, DFK_ERR_INVALID_ARG, pre + " names a keyframe outside the window");
      if (!std::isfinite(sigma[i]) || !(sigma[i] > 0.0f))
        return fail(h, DFK_ERR_INVALID_ARG, pre + ": sigma must be finite and > 0");
      if (level_ptr[i + 1] <= level_ptr[i] || level_ptr[i + 1] > 65535)
        return fail(h, DFK_ERR_INVALID_ARG, pre + " has no items (level_ptr must increase) or more than 65535 in all");
    }
    DeviceGuard guard(h->device);
    if (m == 0) {
      p->ndp = p->ndpi = 0;
      p->dp_item_kf.clear();
      p->lin_dp.clear();
      return DFK_OK;
    }
    const int n = level_ptr[m];
    // the items' views are checked as the batch checks them; their codes come from the state (slot = prior_kf)
    DepthPriorStaged st;
    DFK_TRY(stage_depth_prior(h, what, items, n, p->C, false, h->staging, p->dp, &st));
    // the lists, staged once the items' upload has read h->staging
    Staging s(h->staging);
    const Part<int> csr = s.add<int>(p->K + 1 + m), lp = s.add<int>(m + 1);
    const Part<float> sg = s.add<float>(m);
    const Part<int> kf = s.add<int>(n);
    fill_csr(csr.at(s.host()), p->K, m, [&](int i) { return prior_kf[i]; });
    memcpy(lp.at(s.host()), level_ptr, sizeof(int) * (m + 1));
    memcpy(sg.at(s.host()), sigma, sizeof(float) * m);
    for (int i = 0; i < m; ++i) std::fill(kf.at(s.host()) + level_ptr[i], kf.at(s.host()) + level_ptr[i + 1], prior_kf[i]);
    const char* amsg = "[WindowProblem::set_depth_priors] allocation failed";
    DFK_CUDA(h, p->dp_lists.ensure(s.bytes), amsg);
    DFK_CUDA(h, p->dp_partials.ensure((size_t)st.rows * depth_prior_partial_floats(p->C, true)), amsg);
    DFK_CUDA(h, p->dp_records.ensure((size_t)n * DFK_DEPTH_RECORD_FLOATS(p->C)), amsg);
    DFK_CUDA(h, p->dp_err.ensure((size_t)n * 2), amsg);
    DFK_TRY(s.upload(h, p->dp_lists, w));
    p->ndp = m;
    p->ndpi = n;
    p->dp_st = st;
    p->dp_csr = csr;
    p->dp_level_ptr = lp;
    p->dp_sigma = sg;
    p->dp_kf = kf;
    p->dp_item_kf.assign(kf.at(s.host()), kf.at(s.host()) + n);
    p->lin_dp.assign(n, 0);
    return DFK_OK;
  });
}

DfkStatus dfk_window_problem_retract(DfkHandle h, DfkWindowProblem* p, const double* dx_dev)
{
  return guarded(h, [&] {
    if (!p || !dx_dev) return fail(h, DFK_ERR_INVALID_ARG, "[WindowProblem::retract] null argument");
    if (p->device != h->device) return fail(h, DFK_ERR_INVALID_ARG, "[WindowProblem] problem and handle live on different devices");
    DeviceGuard guard(h->device);
    // into the other state, which then becomes the problem's
    DFK_CUDA(h, launch_window_retract(p->st(p->cur), p->st(1 - p->cur), dx_dev, p->K, p->F, p->C, h->stream),
             "[WindowProblem::retract] kernel launch failed");
    h->launches += 1;
    p->cur = 1 - p->cur;
    return DFK_OK;
  });
}

DfkStatus dfk_window_lm(DfkHandle h, DfkWindowProblem* p, const DfkLMParams* prm, DfkLMTrace* tr)
{
  return guarded(h, [&] {
    DeviceGuard guard(h->device);
    ProblemLMOps ops;
    DFK_TRY(lm_setup(h, p, prm, tr, "WindowLM", &ops));
    return lm_run(*prm, ops, tr);
  });
}

DfkStatus dfk_window_problem_set_active(DfkHandle h, DfkWindowProblem* p, const uint8_t* dense_active,
                                        const uint8_t* error_active)
{
  return guarded(h, [&] {
    const char* what = "[WindowProblem::set_active] ";
    if (!p || (p->nd > 0 && !dense_active) || (!error_active && p->ne != p->nd))
      return fail(h, DFK_ERR_INVALID_ARG, std::string(what) +
                                              "null argument (error_active may be NULL only when num_error == num_dense)");
    if (p->device != h->device)
      return fail(h, DFK_ERR_INVALID_ARG, "[WindowProblem] problem and handle live on different devices");
    DeviceGuard guard(h->device);
    return problem_set_active(h, p, dense_active, error_active ? error_active : dense_active);
  });
}

DfkStatus dfk_window_lm_levels(DfkHandle h, DfkWindowProblem* p, const DfkLMParams* prm, const DfkLevelSchedule* sc,
                               DfkLMTrace* tr, DfkLevelTrace* lt)
{
  return guarded(h, [&] {
    const std::string what = "[WindowLMLevels] ";
    if (!p || !sc) return fail(h, DFK_ERR_INVALID_ARG, what + "null argument");
    if (sc->num_pairs > 0 && !sc->pair_steps_done) return fail(h, DFK_ERR_INVALID_ARG, what + "null pair_steps_done");
    const int nd = p->nd, ne = p->ne;
    std::vector<int> dpair, epair, elevel;
    DFK_TRY(schedule_items(h, p, sc, what, dpair, epair, elevel));
    for (int q = 0; q < sc->num_pairs; ++q)
      if (sc->pair_steps_done[q] < 0)
        return fail(h, DFK_ERR_INVALID_ARG, what + "pair_steps_done[" + std::to_string(q) + "] < 0");
    DeviceGuard guard(h->device);
    struct LevelOps : ProblemLMOps {
      const DfkLevelSchedule* sc;
      const std::vector<int>* dpair;
      const std::vector<int>* epair;
      const std::vector<int>* elevel;
      std::vector<uint8_t> dm, em;
      DfkStatus set_levels(const int* lvl)
      {
        for (size_t i = 0; i < dm.size(); ++i) dm[i] = lvl[(*dpair)[i]] == sc->dense_level[i];
        for (size_t i = 0; i < em.size(); ++i) em[i] = lvl[(*epair)[i]] == (*elevel)[i];
        return problem_set_active(h, p, dm.data(), em.data());
      }
    } ops;
    DFK_TRY(lm_setup(h, p, prm, tr, "WindowLMLevels", &ops));
    ops.sc = sc;
    ops.dpair = &dpair;
    ops.epair = &epair;
    ops.elevel = &elevel;
    ops.dm.assign(nd, 1);
    ops.em.assign(ne, 1);
    return lm_levels_run(*prm, *sc, ops, tr, lt);
  });
}

DfkStatus dfk_window_problem_isam2_update(DfkHandle h, DfkWindowProblem* p, const DfkIsam2Params* prm,
                                          DfkIsam2Result* res)
{
  return guarded(h, [&] {
    const std::string what = "[WindowProblem::isam2_update] ";
    DFK_TRY(isam2_check(h, p, prm, what));
    if (!res) return fail(h, DFK_ERR_INVALID_ARG, what + "null argument");
    DeviceGuard guard(h->device);
    return problem_isam2_update(h, p, prm, res);
  });
}

DfkStatus dfk_window_problem_get_linearization(DfkHandle h, const DfkWindowProblem* p, double* lin_poses,
                                               double* lin_codes, double* delta)
{
  return guarded(h, [&] {
    const char* what = "[WindowProblem::get_linearization] copy failed";
    if (!p) return fail(h, DFK_ERR_INVALID_ARG, "[WindowProblem::get_linearization] null argument");
    if (p->device != h->device)
      return fail(h, DFK_ERR_INVALID_ARG, "[WindowProblem] problem and handle live on different devices");
    DeviceGuard guard(h->device);
    const size_t np = (size_t)(p->K + p->F) * 7;
    if (p->isam_fresh) {  // no update since create / set_state: the state, and zeros
      if (delta) {
        cudaPointerAttributes at{};
        DFK_CUDA(h, cudaPointerGetAttributes(&at, delta), what);
        if (at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged) {
          DFK_CUDA(h, cudaMemsetAsync(delta, 0, sizeof(double) * p->delta_size(), h->stream), what);
        } else {
          DFK_CUDA(h, cudaStreamSynchronize(h->stream), what);  // after any copy still writing it
          std::fill(delta, delta + p->delta_size(), 0.0);
        }
      }
      const double* st = p->st(p->cur);
      if (lin_poses) DFK_CUDA(h, cudaMemcpyAsync(lin_poses, st, sizeof(double) * np, cudaMemcpyDefault, h->stream), what);
      if (lin_codes && p->K * p->C > 0)
        DFK_CUDA(h, cudaMemcpyAsync(lin_codes, st + np, sizeof(double) * (p->S - np), cudaMemcpyDefault, h->stream),
                 what);
      return DFK_OK;
    }
    const double* lin = p->lin(p->ic);
    if (lin_poses)
      DFK_CUDA(h, cudaMemcpyAsync(lin_poses, lin, sizeof(double) * np, cudaMemcpyDefault, h->stream), what);
    if (lin_codes && p->K * p->C > 0)
      DFK_CUDA(h, cudaMemcpyAsync(lin_codes, lin + np, sizeof(double) * (p->S - np), cudaMemcpyDefault, h->stream), what);
    if (delta)
      DFK_CUDA(h, cudaMemcpyAsync(delta, p->isam_delta(p->ic), sizeof(double) * p->delta_size(), cudaMemcpyDefault,
                                  h->stream),
               what);
    return DFK_OK;
  });
}

DfkStatus dfk_window_problem_grow_from(DfkHandle h, DfkWindowProblem* pn, const DfkWindowProblem* po,
                                       const int32_t* dense_of, const int32_t* rep_of, const int32_t* geo_of,
                                       const int32_t* frame_of)
{
  return guarded(h, [&] {
    const std::string what = "[WindowProblem::grow_from] ";
    auto bad = [&](const std::string& m) { return fail(h, DFK_ERR_INVALID_ARG, what + m); };
    if (!pn || !po || pn == po) return bad("null argument, or the same problem twice");
    if ((pn->nd && !dense_of) || (pn->nr && !rep_of) || (pn->ng && !geo_of) || (pn->F && !frame_of))
      return bad("null map");
    if (pn->device != h->device || po->device != h->device)
      return bad("problems and handle live on different devices");
    if (po->isam_fresh) return bad("the old problem has no ISAM2 run to carry over");
    const int K0 = po->K, F0 = po->F, K = pn->K, F = pn->F, C = pn->C, B = pn->B;
    if (pn->C != po->C || K < K0)
      return bad("the new window must keep the old keyframes first, with the same code size");
    // frames: distinct old frames
    std::vector<char> used(F0, 0);
    for (int f = 0; f < F; ++f) {
      const int o = frame_of[f];
      if (o < -1 || o >= F0 || (o >= 0 && used[o]++)) return bad("frame_of[" + std::to_string(f) + "] is not a distinct old frame or -1");
    }
    // a new slot in terms of the old problem's slots: keyframes keep their index, a frame maps by frame_of, a new
    // keyframe or frame has no old slot
    auto pose_old = [&](int s) { return s < 0 ? -1 : s < K ? (s < K0 ? s : -2) : (frame_of[s - K] >= 0 ? K0 + frame_of[s - K] : -2); };
    auto code_old = [&](int c) { return c < 0 ? -1 : c < K0 ? c : -2; };
    auto same = [&](const int4& a, const int4& b) {
      return pose_old(a.x) == b.x && pose_old(a.y) == b.y && code_old(a.z) == b.z && code_old(a.w) == b.w;
    };
    struct Kind {
      const char* name;
      const int32_t* of;
      int n, n_old;
    };
    const Kind kinds[3] = {{"dense", dense_of, pn->nd, po->nd}, {"reprojection", rep_of, pn->nr, po->nr},
                           {"geometric", geo_of, pn->ng, po->ng}};
    std::vector<int2> rec_map, geo_map;
    for (int k = 0; k < 3; ++k) {
      std::vector<char> seen(kinds[k].n_old, 0);
      for (int i = 0; i < kinds[k].n; ++i) {
        const int o = kinds[k].of[i];
        const std::string it = std::string(kinds[k].name) + " item " + std::to_string(i);
        if (o == -1) continue;
        if (o < 0 || o >= kinds[k].n_old || seen[o]++) return bad(it + ": not a distinct old item or -1");
        bool ok;
        if (k == 0) {
          const SfmItemDev &a = pn->dense_tmpl[i], &b = po->dense_tmpl[o];
          ok = same(pn->slots_tmpl[i], po->slots_tmpl[o]) && a.width == b.width && a.height == b.height &&
               a.fx == b.fx && a.fy == b.fy && a.u0 == b.u0 && a.v0 == b.v0;
          rec_map.push_back(make_int2(i, o));
        } else if (k == 1) {
          ok = same(pn->rep_slots_h[i], po->rep_slots_h[o]) && pn->rep_size_h[i] == po->rep_size_h[o];
          rec_map.push_back(make_int2(pn->nd + i, po->nd + o));
        } else {
          ok = same(pn->geo_slots_h[i], po->geo_slots_h[o]) && pn->geo_size_h[i] == po->geo_size_h[o];
          geo_map.push_back(make_int2(i, o));
        }
        if (!ok) return bad(it + " does not read its old item's keys, or has another level or size");
      }
    }
    DeviceGuard guard(h->device);
    const char* amsg = "[WindowProblem::grow_from] allocation failed";
    // the solvers, grown from the old ones (dfk_window_solver_create_from's checks), before anything is written
    WindowSolverDev* grown[2] = {nullptr, nullptr};
    auto drop = [&] { window_solver_destroy(grown[0]); window_solver_destroy(grown[1]); };
    for (int fix = 0; fix < 2; ++fix) {
      if (!po->solver[fix]) continue;
      const std::vector<int> fixed = fix ? std::vector<int>{0, 1, 2, 3, 4, 5} : std::vector<int>();
      const cudaError_t e = window_solver_create(K, C, F, pn->w->pair_k0, pn->w->pair_k1, pn->w->link_k0,
                                                 pn->w->link_k1, pn->w->blk_i, pn->w->blk_j, pn->w->kp.block_off,
                                                 fixed, &grown[fix]);
      if (e != cudaSuccess) {
        drop();
        return cuda_fail(h, e, amsg);
      }
      if (!window_solver_extends(po->solver[fix], grown[fix])) {
        drop();
        return bad("the new window does not extend the old one's solver (keyframes, code size or fixed variables)");
      }
    }
    // the ISAM2 buffers of the new problem; its run continues the old one's
    pn->isam_fresh = false;
    DfkStatus st = isam2_setup(h, pn, 1, amsg);
    if (st == DFK_OK) {
      const cudaError_t e = pn->gather.ensure(std::max<size_t>(1, rec_map.size() + geo_map.size()));
      if (e != cudaSuccess) st = cuda_fail(h, e, amsg);
    }
    if (st != DFK_OK) {
      pn->isam_fresh = true;
      drop();
      return st;
    }
    for (int fix = 0; fix < 2; ++fix)
      if (grown[fix]) {
        int cols = 0;
        DFK_CUDA(h, window_solver_adopt(grown[fix], po->solver[fix], h->stream, &cols), amsg);
        window_solver_destroy(pn->solver[fix]);
        pn->solver[fix] = grown[fix];
        grown[fix] = nullptr;
      }
    const char* cmsg = "[WindowProblem::grow_from] copy failed";
    // the kept records, one gather launch per record buffer
    std::vector<int2> maps(rec_map);
    maps.insert(maps.end(), geo_map.begin(), geo_map.end());
    if (!maps.empty()) {
      DFK_CUDA(h, cudaMemcpyAsync(pn->gather.ptr, maps.data(), sizeof(int2) * maps.size(), cudaMemcpyHostToDevice,
                                  h->stream),
               cmsg);
      if (!rec_map.empty()) {
        DFK_CUDA(h, launch_window_gather_records(po->records, pn->records, pn->gather.ptr, (int)rec_map.size(),
                                                 DFK_SFM_RECORD_FLOATS(C), h->stream),
                 cmsg);
        h->launches += 1;
      }
      if (!geo_map.empty()) {
        DFK_CUDA(h, launch_window_gather_records(po->geo_records, pn->geo_records, pn->gather.ptr + rec_map.size(),
                                                 (int)geo_map.size(), DFK_GEO_RECORD_FLOATS(C), h->stream),
                 cmsg);
        h->launches += 1;
      }
    }
    // theta_lin and Delta: the old keyframes' and kept frames' from the old run, the new ones' from the new state
    const double *ol = po->lin(po->ic), *od = po->isam_delta(po->ic), *ns = pn->st(pn->cur);
    double *nl = pn->lin(pn->ic), *nd = pn->isam_delta(pn->ic);
    auto d2d = [&](double* dst, const double* src, size_t n) {
      return n ? cudaMemcpyAsync(dst, src, sizeof(double) * n, cudaMemcpyDeviceToDevice, h->stream) : cudaSuccess;
    };
    const size_t npn = (size_t)(K + F) * 7, npo = (size_t)(K0 + F0) * 7;
    DFK_CUDA(h, d2d(nl, ns, pn->S), cmsg);                                    // everything new from the state
    DFK_CUDA(h, d2d(nl, ol, (size_t)K0 * 7), cmsg);                          // old keyframe poses
    DFK_CUDA(h, d2d(nl + npn, ol + npo, (size_t)K0 * C), cmsg);              // old codes
    DFK_CUDA(h, cudaMemsetAsync(nd, 0, sizeof(double) * pn->delta_size(), h->stream), cmsg);
    DFK_CUDA(h, d2d(nd, od, (size_t)K0 * B), cmsg);                          // old keyframes' delta
    for (int f = 0; f < F; ++f)
      if (frame_of[f] >= 0) {
        DFK_CUDA(h, d2d(nl + (size_t)(K + f) * 7, ol + (size_t)(K0 + frame_of[f]) * 7, 7), cmsg);
        DFK_CUDA(h, d2d(nd + (size_t)K * B + 6 * f, od + (size_t)K0 * B + 6 * frame_of[f], 6), cmsg);
      }
    // the flags: kept items as they were, new items and the depth priors stale
    pn->clear_linearised();
    for (const int2& m : rec_map) {
      if (m.x < pn->nd) pn->lin_dense[m.x] = po->lin_dense[m.y];
      else pn->lin_rep[m.x - pn->nd] = po->lin_rep[m.y - po->nd];
    }
    for (const int2& m : geo_map) pn->lin_geo[m.x] = po->lin_geo[m.y];
    pn->isam_updates = po->isam_updates;
    pn->diag_eps = po->diag_eps;
    return DFK_OK;
  });
}

DfkStatus dfk_window_map_steps(DfkHandle h, DfkWindowProblem* p, const DfkIsam2Params* prm, const DfkLevelSchedule* sc,
                               DfkWorkState* works, int max_steps, DfkMapTrace* tr)
{
  return guarded(h, [&] {
    const std::string what = "[WindowMapSteps] ";
    DFK_TRY(isam2_check(h, p, prm, what));
    if (!sc) return fail(h, DFK_ERR_INVALID_ARG, what + "null argument");
    if (max_steps < 0) return fail(h, DFK_ERR_INVALID_ARG, what + "max_steps < 0");
    const int L = sc->num_levels, P = sc->num_pairs, nd = p->nd, ne = p->ne;
    if (L > DFK_MAX_WORK_LEVELS)
      return fail(h, DFK_ERR_INVALID_ARG, what + "more than DFK_MAX_WORK_LEVELS (" + std::to_string(DFK_MAX_WORK_LEVELS) +
                                              ") levels");
    std::vector<int> dpair, epair, elevel;
    DFK_TRY(schedule_items(h, p, sc, what, dpair, epair, elevel));
    std::vector<DfkWorkState> wk(P);
    for (int q = 0; q < P; ++q) {
      wk[q] = works ? works[q] : work_fresh(sc->iters, L);
      const DfkWorkState& w = wk[q];
      bool ok = w.active_level >= -2 && w.active_level < L && w.factor >= -1 && w.factor < L;
      for (int l = 0; l < L; ++l) ok = ok && w.iters[l] >= -1 && w.iters[l] <= sc->iters[l];
      if (!ok) return fail(h, DFK_ERR_INVALID_ARG, what + "work " + std::to_string(q) + " is not a state of its schedule");
    }
    DeviceGuard guard(h->device);
    std::vector<int> factor(P), prev(P);
    std::vector<uint8_t> dm(nd), em(ne);
    int step = 0;
    for (; step < max_steps && !works_empty(wk.data(), P); ++step) {
      for (int q = 0; q < P; ++q) prev[q] = wk[q].factor;
      works_step(wk.data(), P, sc->iters, sc->pair_remove_after, factor.data());
      for (int i = 0; i < nd; ++i) dm[i] = factor[dpair[i]] == sc->dense_level[i];
      for (int i = 0; i < ne; ++i) em[i] = factor[epair[i]] == elevel[i];
      DFK_TRY(problem_set_active(h, p, dm.data(), em.data()));
      // a pair whose factor changed holds a new factor: linearised at theta_lin.  Flags exist once an update ran
      if (!p->isam_fresh)
        for (int i = 0; i < nd; ++i)
          if (factor[dpair[i]] != prev[dpair[i]]) p->lin_dense[i] = 0;
      DfkIsam2Result r{};
      const DfkStatus st = problem_isam2_update(h, p, prm, &r);
      if (st != DFK_OK) {  // the steps before this one stand: hand back their works, so the run can continue
        if (tr) tr->num_steps = step;
        if (works) std::copy(wk.begin(), wk.end(), works);
        return st;
      }
      if (tr) {
        if (tr->variables_relinearized) tr->variables_relinearized[step] = r.variables_relinearized;
        if (tr->variables_reeliminated) tr->variables_reeliminated[step] = r.variables_reeliminated;
        if (tr->factors_relinearised) tr->factors_relinearised[step] = r.factors_relinearised;
        if (tr->first_column) tr->first_column[step] = r.first_column;
        if (tr->pair_levels) std::copy(factor.begin(), factor.end(), tr->pair_levels + (size_t)step * P);
      }
      if (r.variables_relinearized == 0) works_signal(wk.data(), P);
    }
    if (tr) tr->num_steps = step;
    if (works) std::copy(wk.begin(), wk.end(), works);
    return DFK_OK;
  });
}

}  // extern "C"
