// lins_seq.cu — sequence mode (include/lins_gpu.h: lins_gpu_seq_*): S running sequences advanced one scan per step with
// the whole per-scan chain of StateEstimator on the device:
//   predict x k (lins_seq_predict_kernel) -> processScan gate (host: it only reads cloud sizes) -> IESKF (the fused kernel,
//   one launch) -> divergence check (one D2H) -> estimateTransform loop per diverged sequence (lins_gpu.cu: icp_loop) ->
//   update / integrateTransformation / reset(1) / roll-pitch (lins_seq_post_kernel) -> transformToEnd (CSR kernel of
//   lins_gpu.cu) + the guarded map swap (a gather list: lins_ctx.hpp CopyList).
// Slots of a lins_gpu_seq_open run also initialise on the device (processPCL's status machine): the predict kernel
//   pre-integrates a slot's IMU rows between its first and second scan, the second scans' estimateTransform runs as ONE
//   batched icp_loop over all of them (lins_seq_icp_start_kernel sets its start poses), and lins_seq_init_kernel installs
//   the state of processFirstScan / processSecondScan.
// A run bound to the lockstep mappers (lins_gpu_seq_map_*) also keeps what each slot's scan_last_ would publish: the
//   outlier clouds of the step's scans (a stash), the published outlier cloud (a generation, like the maps), whether the
//   YZX clouds exist, and the global states (read back with the step's last synchronisation); lins_gpu_seq_map_step then
//   runs publishTopics and one lockstep mapper step on the device clouds.
// The filter algebra is lins_seq_step.cuh, shared with the CPU test.  Built with -fmad=false like the other bit-exact units.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <vector>

#include "../host/global_state_yzx.hpp"
#include "lins_ctx.hpp"
#include "lins_kernels.cuh"
#include "lins_seq_step.cuh"

using namespace lins_capi;
using lins_dev::BatchView;

namespace {

// what processImu does with a sequence's IMU rows this step (StateEstimator.hpp:242-270)
enum ImuUse : unsigned char { IMU_IGNORE = 0, IMU_PREDICT = 1, IMU_PREINTEGRATE = 2 };
// StateEstimator::FusionStatus
enum Fusion : int32_t { FUSION_INIT = 0, FUSION_FIRST_SCAN = 1, FUSION_RUNNING = 3 };

// One warp per sequence: the sequence's k StatePredictor::predict calls in order (kalman_filter.hpp:98-170), with its own
// constants k[s] / ik[s] (here and in the kernels below: the run's, or the slot's config).  The 18x18
// matrices live in shared memory; lane l owns the entries e = l, l + 32, ... of every matrix phase, each entry summed in
// the host's order.  A sequence in STATUS_FIRST_SCAN pre-integrates its rows instead (IntegrationBase::propagate, lane 0).
__global__ void __launch_bounds__(32) lins_seq_predict_kernel(double* __restrict__ filt, double* __restrict__ cov, double* __restrict__ imu_last,
                                                             const double* __restrict__ imu, const int* __restrict__ imu_off,
                                                             const unsigned char* __restrict__ use, double* __restrict__ pre,
                                                             const lins_seq::Consts* __restrict__ k, const lins_seq::InitConsts* __restrict__ ik) {
  const int s = blockIdx.x, lane = threadIdx.x;
  if (use[s] == IMU_IGNORE) return;
  const int m0 = imu_off[s], m1 = imu_off[s + 1];
  if (m0 == m1) return;
  if (use[s] == IMU_PREINTEGRATE) {
    if (lane == 0)
      for (int m = m0; m < m1; ++m) lins_seq::preint_propagate(pre + (size_t)s * 20, ik[s], imu[(size_t)m * 7], imu + (size_t)m * 7 + 1, imu + (size_t)m * 7 + 4);
    return;
  }
  __shared__ double P[324], Ft[324], F[324], FP[324], P2[324];
  __shared__ double st[20], al[3], gl[3];
  __shared__ lins_seq::PredictBlocks sb;  // R, va, aa of the sample being applied
  double* S = filt + (size_t)s * 20;
  double* C = cov + (size_t)s * 324;
  for (int e = lane; e < 324; e += 32) P[e] = C[e];
  if (lane < 20) st[lane] = S[lane];
  if (lane < 3) { al[lane] = imu_last[(size_t)s * 8 + lane]; gl[lane] = imu_last[(size_t)s * 8 + 3 + lane]; }
  __syncwarp();
  for (int m = m0; m < m1; ++m) {
    const double* smp = imu + (size_t)m * 7;
    const double dt = smp[0];
    if (lane == 0) {
      sb = lins_seq::predict_state(st, al, gl, dt, smp + 1, smp + 4);
      for (int i = 0; i < 3; ++i) { al[i] = smp[1 + i]; gl[i] = smp[4 + i]; }
    }
    __syncwarp();
    const lins_seq::PredictBlocks& b = sb;
    for (int e = lane; e < 324; e += 32) Ft[e] = lins_seq::ft_entry(b, e / 18, e % 18);
    __syncwarp();
    for (int e = lane; e < 324; e += 32) F[e] = lins_seq::f_entry(Ft, e / 18, e % 18, dt);
    __syncwarp();
    for (int e = lane; e < 324; e += 32) FP[e] = lins_seq::fp_entry(F, P, e / 18, e % 18);
    __syncwarp();
    for (int e = lane; e < 324; e += 32) {
      const int i = e / 18, j = e % 18;
      P2[e] = lins_seq::fpft_entry(FP, F, lins_seq::q_entry(b, k[s].noise, i, j, dt), i, j);
    }
    __syncwarp();
    for (int e = lane; e < 324; e += 32) { const int i = e / 18, j = e % 18; P[j * 18 + i] = 0.5 * (P2[i * 18 + j] + P2[j * 18 + i]); }
    __syncwarp();
  }
  for (int e = lane; e < 324; e += 32) C[e] = P[e];
  if (lane < 20) S[lane] = st[lane];
  if (lane < 3) { imu_last[(size_t)s * 8 + lane] = al[lane]; imu_last[(size_t)s * 8 + 3 + lane] = gl[lane]; }
}

// One thread per sequence that ran: filter_->update with the IESKF posterior (or, after divergence, the prior with
// estimateTransform's pose and the prior covariance), integrateTransformation, reset(1), calculateRPfromGravity +
// correctRollPitch (state_estimator.hpp:202-237).  lin receives linState_ (rn / qbn only after divergence, like the shim).
__global__ void lins_seq_post_kernel(int n, const unsigned char* __restrict__ status, const double* __restrict__ state_out,
                                     const double* __restrict__ cov_out, const double* __restrict__ icp_pose, double* __restrict__ filt,
                                     double* __restrict__ cov, double* __restrict__ glob, double* __restrict__ lin,
                                     const lins_seq::Consts* __restrict__ k) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n || (status[s] != LINS_SEQ_RAN && status[s] != LINS_SEQ_ICP)) return;
  double f[20];
  for (int i = 0; i < 20; ++i) f[i] = state_out[(size_t)s * 20 + i];
  double* L = lin + (size_t)s * 20;
  if (status[s] == LINS_SEQ_ICP) {
    const double* p = icp_pose + (size_t)s * 20;
    for (int i = 0; i < 10; ++i) if (i < 3 || i >= 6) { f[i] = p[i]; L[i] = p[i]; }
  } else {
    for (int i = 0; i < 20; ++i) L[i] = f[i];
  }
  double* P = cov + (size_t)s * 324;
  for (int e = 0; e < 324; ++e) P[e] = cov_out[(size_t)s * 324 + e];
  double* g = glob + (size_t)s * 20;
  lins_seq::integrate(g, f);
  lins_seq::reset1(f, P, k[s]);
  lins_seq::correct_roll_pitch(g, f);
  for (int i = 0; i < 19; ++i) filt[(size_t)s * 20 + i] = f[i];
}

// One thread per second scan: the start pose of its estimateTransform (processSecondScan's pl / ql) and a fresh loop state;
// every other sequence's loop state reads done, so the batched loop passes it over, and so does a second scan whose
// NUM_ITER (tune[s]) is 0: its loop runs no iteration.
__global__ void lins_seq_icp_start_kernel(int n, const unsigned char* __restrict__ status, const double* __restrict__ pre,
                                          double* __restrict__ icp_pose, lins_dev::IcpState* __restrict__ icp,
                                          const lins_dev::UnitTuning* __restrict__ tune) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const bool second = status[s] == LINS_SEQ_SECOND;
  lins_dev::IcpState& st = icp[s];
  for (int i = 0; i < 36; ++i) st.matP[i] = 0.0;
  st.iters = 0; st.converged = 0; st.pad = 0;
  st.done = second && tune[s].num_iter > 0 ? 0 : 1;
  if (second) lins_seq::second_scan_start(pre + (size_t)s * 20, icp_pose + (size_t)s * 20);
}

// One thread per sequence that initialised this step: processFirstScan (LINS_SEQ_FIRST) or the rest of processSecondScan
// after its estimateTransform (LINS_SEQ_SECOND; icp_pose holds the result).  imu: the step's processPCL samples, 6 per
// sequence.
__global__ void lins_seq_init_kernel(int n, const unsigned char* __restrict__ status, const double* __restrict__ imu,
                                     const double* __restrict__ icp_pose, double* __restrict__ pre, double* __restrict__ glob,
                                     double* __restrict__ filt, double* __restrict__ cov, double* __restrict__ lin,
                                     double* __restrict__ imu_last, const lins_seq::InitConsts* __restrict__ k) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const size_t o = (size_t)s * 20;
  double* il = imu_last + (size_t)s * 8;
  if (status[s] == LINS_SEQ_FIRST)
    lins_seq::first_scan(filt + o, cov + (size_t)s * 324, lin + o, pre + o, il, imu + (size_t)s * 6, k[s]);
  else if (status[s] == LINS_SEQ_SECOND)
    lins_seq::second_scan(glob + o, filt + o, cov + (size_t)s * 324, lin + o, il, pre + o, icp_pose + o, imu + (size_t)s * 6, k[s]);
}

// One warp per sequence s whose align[10 s + 9] != 0 (a tuned slot): alignIMUtoVehicle (Estimator.cpp:286-292) in place on
// its IMU values, acc_out = R^T acc and gyr_out = R^T gyr with R = align[10 s ..] (row-major, rpy2R(0, 0, yaw)): its rows
// imu[imu_off[s] .. imu_off[s + 1]) (dt, acc, gyr; dt stays) and, when scan_imu is set, its processPCL sample
// scan_imu[6 s ..] (acc, gyr).  out_j = (R_0j v_0 + R_1j v_1) + R_2j v_2, unfused (-fmad=false).
__global__ void __launch_bounds__(32) lins_seq_align_kernel(double* __restrict__ imu, const int* __restrict__ imu_off,
                                                            double* __restrict__ scan_imu, const double* __restrict__ align) {
  const int s = blockIdx.x, lane = threadIdx.x;
  const double* R = align + (size_t)s * 10;
  if (R[9] == 0.0) return;
  auto rot = [R](double* v) {
    const double x = v[0], y = v[1], z = v[2];
    for (int j = 0; j < 3; ++j) v[j] = (R[j] * x + R[3 + j] * y) + R[6 + j] * z;
  };
  for (int m = imu_off[s] + lane; m < imu_off[s + 1]; m += 32) { rot(imu + (size_t)m * 7 + 1); rot(imu + (size_t)m * 7 + 4); }
  if (scan_imu && lane == 0) { rot(scan_imu + (size_t)s * 6); rot(scan_imu + (size_t)s * 6 + 3); }
}

// One thread per sequence with mask[s] != 0 (every sequence for a null mask): the state of a new StateEstimator
__global__ void lins_seq_fresh_kernel(int n, const unsigned char* __restrict__ mask, double* __restrict__ glob, double* __restrict__ filt,
                                      double* __restrict__ cov, const lins_seq::InitConsts* __restrict__ k) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n || (mask && !mask[s])) return;
  lins_seq::fresh_slot(glob + (size_t)s * 20, filt + (size_t)s * 20, cov + (size_t)s * 324, k[s]);
}

static_assert(sizeof(lins_seq::Consts) == sizeof(SeqState::consts), "consts");
static_assert(sizeof(lins_seq::InitConsts) == sizeof(SeqState::init_consts), "init consts");

// noise, sq(init_pos_std) and pow(deg2rad(init_att_std), 2) of lins_seq_params (kalman_filter.hpp setNoise / reset(1))
void consts_of(double* out, const lins_seq_params* prm) {
  lins_seq::Consts k;
  for (int i = 0; i < 4; ++i) k.noise[i] = prm->noise[i];
  for (int i = 0; i < 3; ++i) {
    k.pos_var[i] = prm->init_pos_std[i] * prm->init_pos_std[i];                 // sq(init_pos_std)
    k.att_var[i] = std::pow(prm->init_att_std[i] * M_PI / 180.0, 2);            // pow(deg2rad(init_att_std), 2)
  }
  std::memcpy(out, &k, sizeof(k));
}

// the diagonal initializeCovariance installs (kalman_filter.hpp:197-209) and init_ba / init_bw
void init_consts_of(double* out, const lins_seq_params* prm, const lins_seq_init_params* ip) {
  lins_seq::InitConsts k;
  for (int i = 0; i < 3; ++i) {
    k.var[lins_seq::kPos + i] = prm->init_pos_std[i] * prm->init_pos_std[i];
    k.var[lins_seq::kVel + i] = ip->init_vel_std[i] * ip->init_vel_std[i];
    k.var[lins_seq::kAtt + i] = std::pow(prm->init_att_std[i] * M_PI / 180.0, 2);
    k.var[lins_seq::kAcc + i] = ip->init_acc_std[i] * ip->init_acc_std[i];
    k.var[lins_seq::kGyr + i] = ip->init_gyr_std[i] * ip->init_gyr_std[i];
    k.var[lins_seq::kGra + i] = 0.01;
    k.ba[i] = ip->init_ba[i];
    k.bw[i] = ip->init_bw[i];
  }
  std::memcpy(out, &k, sizeof(k));
}

constexpr size_t kNConsts = sizeof(SeqState::consts) / sizeof(double), kNInit = sizeof(SeqState::init_consts) / sizeof(double);

// Everything slot s reads: its config's and its tuning's values, else the run's open constants, the context's current
// lins_params (lins_gpu_set_params can change them between steps) and the call's feature params fp (null: feat is not
// filled).  Resolved again at every use, so an untuned slot follows the context.
struct SlotParams {
  double consts[kNConsts], init_consts[kNInit];  // lins_seq::Consts, InitConsts
  double period;                                  // SCAN_PERIOD
  FeatConsts feat;                                // the extraction of a _raw / _cloud2 step
  lins_dev::UnitTuning tune;
  double align[10];                               // alignIMUtoVehicle's R (row-major), then 1 = rotate the slot's IMU values
};

SlotParams slot_params(const lins_ctx* ctx, int s, const lins_feature_params* fp = nullptr) {
  const SeqState& q = ctx->seq;
  const SeqSlot& r = q.slot[s];
  const lins_params& p = ctx->prm;
  SlotParams o;
  if (r.cfg) {
    consts_of(o.consts, &r.cfg->filter);
    init_consts_of(o.init_consts, &r.cfg->filter, &r.cfg->init);
  } else {
    std::copy(q.consts, q.consts + kNConsts, o.consts);
    std::copy(q.init_consts, q.init_consts + kNInit, o.init_consts);
  }
  o.period = r.cfg ? r.cfg->scan_period : p.scan_period;
  if (fp) o.feat = feat_consts(r.cfg ? r.cfg->features : *fp, o.period);
  lins_dev::UnitTuning& t = o.tune;
  if (r.tune) {
    const lins_slot_tuning& u = r.tune->t;
    t.num_iter = u.num_iter; t.icp_freq = u.icp_freq; t.nearest_sq = u.nearest_feature_search_sq_dist;
    t.lidar_std = u.lidar_std; t.lidar_scale = u.lidar_scale;
  } else {
    t.num_iter = p.num_iter; t.icp_freq = p.icp_freq < 1 ? 1 : p.icp_freq; t.nearest_sq = p.nearest_feature_search_sq_dist;
    t.lidar_std = p.lidar_std; t.lidar_scale = p.lidar_scale;
  }
  std::fill(o.align, o.align + 10, 0.0);
  if (r.tune) { std::copy(r.tune->R, r.tune->R + 9, o.align); o.align[9] = 1.0; }
  return o;
}

}  // namespace

namespace lins_capi {

int check_open_run(lins_ctx* ctx, const char* entry, bool args_ok) {
  if (!ctx) return LINS_E_INVALID;
  const std::string e(entry);
  if (ctx->seq.n == 0) return fail(ctx, LINS_E_NOMAP, (e + ": no sequence run: call lins_gpu_seq_open").c_str());
  if (!args_ok) return fail(ctx, LINS_E_INVALID, (e + ": null argument").c_str());
  if (!ctx->seq.has_init) return fail(ctx, LINS_E_INVALID, (e + " needs a run opened by lins_gpu_seq_open").c_str());
  return LINS_OK;
}

int check_fresh(lins_ctx* ctx, int s, const char* entry) {
  if (ctx->seq.slot[s].fresh) return LINS_OK;
  return fail(ctx, LINS_E_INVALID, (std::string(entry) + ": a masked slot is not fresh (no step since open / restart)").c_str());
}

// every slot's device constants; then a synchronisation (the sources are pageable)
int upload_slot_consts(lins_ctx* ctx, int n) {
  SeqState& q = ctx->seq;
  std::vector<double> k(kNConsts * n), ik(kNInit * n);
  for (int s = 0; s < n; ++s) {
    const SlotParams p = slot_params(ctx, s);
    std::copy(p.consts, p.consts + kNConsts, &k[kNConsts * s]);
    std::copy(p.init_consts, p.init_consts + kNInit, &ik[kNInit * s]);
  }
  CK(q.slot_consts.reserve(k.size())); CK(q.slot_init_consts.reserve(ik.size()));
  CK(cudaMemcpyAsync(q.slot_consts.p, k.data(), sizeof(double) * k.size(), cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(q.slot_init_consts.p, ik.data(), sizeof(double) * ik.size(), cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  return LINS_OK;
}

}  // namespace lins_capi

namespace {

const lins_seq::Consts* slot_consts(const SeqState& q) { return reinterpret_cast<const lins_seq::Consts*>(q.slot_consts.p); }
const lins_seq::InitConsts* slot_init_consts(const SeqState& q) { return reinterpret_cast<const lins_seq::InitConsts*>(q.slot_init_consts.p); }

// alignIMUtoVehicle's R = rpy2R((0, 0, deg2rad(angle))) = Rz Ry Rx (math_utils.h:164-182), row-major, with the host's libm
void misalign_R(double angle, double* R) {
  const double y = angle * M_PI / 180.0, p = 0.0, r = 0.0;  // math_utils::deg2rad of (0, 0, angle)
  const double Rz[9] = {std::cos(y), -std::sin(y), 0, std::sin(y), std::cos(y), 0, 0, 0, 1};
  const double Ry[9] = {std::cos(p), 0., std::sin(p), 0., 1., 0., -std::sin(p), 0., std::cos(p)};
  const double Rx[9] = {1., 0., 0., 0., std::cos(r), -std::sin(r), 0., std::sin(r), std::cos(r)};
  auto mul = [](const double* A, const double* B, double* C) {
    for (int i = 0; i < 3; ++i)
      for (int j = 0; j < 3; ++j) C[3 * i + j] = (A[3 * i] * B[j] + A[3 * i + 1] * B[3 + j]) + A[3 * i + 2] * B[6 + j];
  };
  double T[9];
  mul(Rz, Ry, T);
  mul(T, Rx, R);
}

int launch_fresh(lins_ctx* ctx, SeqState& q, int n, const unsigned char* mask_dev) {
  lins_seq_fresh_kernel<<<(n + 127) / 128, 128, 0, ctx->stream>>>(n, mask_dev, q.glob.p, q.filt.p, q.cov.p, slot_init_consts(q));
  CK(cudaGetLastError());
  ctx->launches += 1;
  return LINS_OK;
}

// ---- slot lifecycle ------------------------------------------------------------------------------------------------------
// every per-slot buffer of a run of n slots; ns / nc: the surf / corner maps it starts with
int reserve_run(lins_ctx* ctx, SeqState& q, int n, size_t ns, size_t nc) {
  CK(q.filt.reserve((size_t)n * 20)); CK(q.cov.reserve((size_t)n * 324)); CK(q.glob.reserve((size_t)n * 20));
  CK(q.lin.reserve((size_t)n * 20)); CK(q.imu_last.reserve((size_t)n * 8)); CK(q.icp_pose.reserve((size_t)n * 20)); CK(q.icp.reserve(icp_state_bytes() * n));
  CK(q.run.results.reserve(n)); CK(q.run.reports.reserve(n));
  return reserve_maps(ctx, q.map, n, ns, nc);
}

// the host side of a run whose slots are in place: no step yet, every slot idle in the given fusion status
void install_run(SeqState& q, int n, bool has_init) {
  q.ev_valid = false;
  q.has_step = false;
  q.status.assign(n, LINS_SEQ_IDLE);
  q.has_init = has_init;
  q.fusion.assign(n, has_init ? FUSION_INIT : FUSION_RUNNING);
  q.n = n;
}

}  // namespace

namespace lins_capi {

// ---- map generations -----------------------------------------------------------------------------------------------------
// Where one (cloud, unit) range of the next generation comes from: a MapPiece (lins_ctx.hpp)

// g's device state for n units and current maps of ns / nc points
int reserve_maps(lins_ctx* ctx, MapGen& g, int n, size_t ns, size_t nc) {
  CK(g.cur[0].reserve(ns + 1)); CK(g.cur[1].reserve(nc + 1)); CK(g.cur[2].reserve(1)); CK(g.cur[3].reserve(1));
  for (Buf<float4>& b : g.nxt) CK(b.reserve(1));
  CK(g.dev.reserve(4 * (size_t)(n + 1) + (n + 3) / 4));
  return LINS_OK;
}

// queue the upload of h_off and h_stale (one H2D from a pageable copy: the driver stages it before the call returns)
cudaError_t queue_map_state(lins_ctx* ctx, MapGen& g) {
  std::vector<int> h(g.h_off.size() + (g.n + 3) / 4, 0);
  std::copy(g.h_off.begin(), g.h_off.end(), h.begin());
  std::memcpy(h.data() + g.h_off.size(), g.h_stale.data(), g.h_stale.size());
  return cudaMemcpyAsync(g.dev.p, h.data(), sizeof(int) * h.size(), cudaMemcpyHostToDevice, ctx->stream);
}

// cloud c (map_s, map_c, tree_s, tree_c) of unit s in the current generation
MapPiece current_piece(const MapGen& g, int c, int s) {
  const int N1 = g.n + 1;
  const int* mo = g.h_off.data();
  return MapPiece{g.cur[c].p + mo[c * N1 + s], mo[c * N1 + s + 1] - mo[c * N1 + s]};
}

// the map swap of updatePointCloud (:1151-1160) for unit s and its new clouds: they become its map; its 1-NN index is
// rebuilt on them iff corner >= 5 && surf >= 20 (not stale), else it stays on the clouds it was built on: the old map,
// or the older clouds of a unit that is already stale
MapRefresh refresh_maps(const MapGen& g, int s, MapPiece surf, MapPiece corner) {
  MapRefresh r{{surf, corner, MapPiece{}, MapPiece{}}, 0};
  if (corner.len >= 5 && surf.len >= 20) return r;  // :1156-1157
  const int from = g.h_stale[s] ? 2 : 0;
  r.next[2] = current_piece(g, from, s);
  r.next[3] = current_piece(g, from + 1, s);
  r.stale = 1;
  return r;
}

// The next generation from next[4 * s + c], unit s's cloud c: fills h_noff, reserves nxt and appends the copies that fill
// it, in unit order, to `copies`
int build_next_maps(lins_ctx* ctx, MapGen& g, const std::vector<MapPiece>& next, std::vector<DevCopy>& copies) {
  const int n = g.n, N1 = n + 1;
  g.h_noff.assign(4 * (size_t)N1, 0);
  int* no = g.h_noff.data();
  for (int s = 0; s < n; ++s)
    for (int c = 0; c < 4; ++c) no[c * N1 + s + 1] = no[c * N1 + s] + next[4 * (size_t)s + c].len;
  for (int c = 0; c < 4; ++c) CK(g.nxt[c].reserve((size_t)no[(c + 1) * N1 - 1] + 1));
  for (int s = 0; s < n; ++s)
    for (int c = 0; c < 4; ++c) {
      const MapPiece& p = next[4 * (size_t)s + c];
      if (p.len) copies.push_back(DevCopy{p.src, g.nxt[c].p + no[c * N1 + s], p.len, 0});
    }
  return LINS_OK;
}

// the next generation becomes the current one (whatever fills it has been queued)
void swap_maps(MapGen& g) {
  for (int c = 0; c < 4; ++c) std::swap(g.cur[c], g.nxt[c]);
  g.h_off.swap(g.h_noff);
}

}  // namespace lins_capi

namespace {

// ---- a step ----------------------------------------------------------------------------------------------------------------
// What every step entry checks before anything runs: the run, n_seq and n_scans (the number of scans d carries), the IMU
// rows, and scan_imu while a present slot initialises
template <typename Desc>
int check_step(lins_ctx* ctx, const Desc* d, int n_scans, const double* scan_imu) {
  if (!ctx) return LINS_E_INVALID;
  SeqState& q = ctx->seq;
  const int n = q.n;
  if (n == 0) return fail(ctx, LINS_E_NOMAP, "lins_gpu_seq_begin has not been called");
  if (!d || d->n_seq != n || n_scans != n) return fail(ctx, LINS_E_INVALID, "n_seq differs from the hand-over's");
  if (q.pub.bound && q.pub.pending) return fail(ctx, LINS_E_INVALID, "the last step's lins_gpu_seq_map_step has not run");
  q.pub.dev_outliers = false;  // (until a projection stashes them)
  if (d->imu_off) { const int rc = check_csr(ctx, d->imu_off, n, d->imu, "bad imu offsets / samples"); if (rc != LINS_OK) return rc; }
  else if (d->imu) return fail(ctx, LINS_E_INVALID, "imu without imu_off");
  if (!scan_imu)
    for (int s = 0; s < n; ++s)
      if ((!d->present || d->present[s]) && q.fusion[s] != FUSION_RUNNING)
        return fail(ctx, LINS_E_INVALID, "scan_imu is required while a present slot is initialising");
  return LINS_OK;
}

// Query compaction: the surf / corner queries of the step's clouds (q.up.qs / qc at offs[0] / offs[1]) of the slots whose
// status is `code`, packed from off[0] / off[N1] on (set by the caller).  Fills the rest of off (2 x (n + 1)), appends
// their copies to `copies` with each destination (cloud, offset) in `to`, and returns the largest per-slot total.
int compact_queries(const SeqState& q, const int32_t* const offs[4], int32_t code, std::vector<int>& off, std::vector<DevCopy>& copies,
                    std::vector<std::pair<int, int>>& to) {
  const int n = q.n, N1 = n + 1;
  int max_q = 0;
  for (int s = 0; s < n; ++s) {
    const bool take = q.status[s] == code;
    const int nq[2] = {take ? offs[0][s + 1] - offs[0][s] : 0, take ? offs[1][s + 1] - offs[1][s] : 0};
    for (int c = 0; c < 2; ++c) {
      off[c * N1 + s + 1] = off[c * N1 + s] + nq[c];
      if (nq[c]) { copies.push_back(DevCopy{(c ? q.up.qc.p : q.up.qs.p) + offs[c][s], nullptr, nq[c], 0}); to.emplace_back(c, off[c * N1 + s]); }
    }
    max_q = std::max(max_q, nq[0] + nq[1]);
  }
  return max_q;
}

// the phases of a step after its input is validated and uploaded (seq_step_run)
int seq_step_phases(lins_ctx* ctx, const lins_seq_step_desc* d, const int32_t* const offs[4], const double* scan_imu) {
  SeqState& q = ctx->seq;
  const int n = q.n;
  int rc = LINS_OK;

  // ---- host bookkeeping: who runs, the compacted queries, the next maps (all from sizes the host knows) --------------
  std::vector<int32_t>& status = q.status;
  const int N1 = n + 1;
  if (q.pub.bound) q.pub.fusion_before = q.fusion;  // (publishTopics' rule reads the status before the scan)
  std::vector<MapPiece> next(4 * (size_t)n);
  std::vector<unsigned char> new_stale(q.map.h_stale);
  std::vector<unsigned char> imu_use(n, IMU_IGNORE);
  int n_run = 0, n_init = 0, n_second = 0;
  for (int s = 0; s < n; ++s) {
    const bool present = !d->present || d->present[s];
    const int nsl = offs[2][s + 1] - offs[2][s], ncl = offs[3][s + 1] - offs[3][s];
    const int32_t fs = q.fusion[s];
    if (present) q.slot[s].fresh = false;
    if (!present) status[s] = LINS_SEQ_IDLE;
    else if (fs == FUSION_RUNNING) status[s] = (ncl <= 5 || nsl <= 10) ? LINS_SEQ_SKIPPED : LINS_SEQ_RAN;  // :436-440
    else if (ncl < 10 || nsl < 100) status[s] = LINS_SEQ_INIT_WAIT;  // processFirstScan / processSecondScan (:331-336, :379-384)
    else status[s] = fs == FUSION_INIT ? LINS_SEQ_FIRST : LINS_SEQ_SECOND;
    if (present) imu_use[s] = fs == FUSION_RUNNING ? IMU_PREDICT : fs == FUSION_FIRST_SCAN ? IMU_PREINTEGRATE : IMU_IGNORE;
    const bool ran = status[s] == LINS_SEQ_RAN;
    const bool init = status[s] == LINS_SEQ_FIRST || status[s] == LINS_SEQ_SECOND;
    n_run += ran;
    n_init += init;
    n_second += status[s] == LINS_SEQ_SECOND;
    // map swap (refresh_maps).  A first scan's clouds become the map as they are (setInputCloud, :363-364) and a second
    // scan's like a running one's: both pass the guard after the init gate.
    MapPiece* p = &next[4 * (size_t)s];  // map_s, map_c, tree_s, tree_c
    if (ran || init) {
      const MapRefresh m = refresh_maps(q.map, s, MapPiece{q.up.ts.p + offs[2][s], nsl}, MapPiece{q.up.tc.p + offs[3][s], ncl});
      std::copy(m.next, m.next + 4, p);
      new_stale[s] = m.stale;
    } else {
      for (int c = 0; c < 4; ++c) p[c] = current_piece(q.map, c, s);
    }
  }
  // the IESKF's queries, then the second scans' after them in the compacted buffers, with offsets of their own (init_off):
  // the IESKF launch sees no query of theirs, the estimateTransform loop none of the IESKF's.  One gather list: the
  // query copies (the first n_qcopies), then the map refresh's.
  std::vector<DevCopy> copies;
  std::vector<std::pair<int, int>> qto;  // destination of each query copy: (cloud, offset), resolved once the buffers exist
  std::vector<int> run_off(2 * (size_t)N1, 0), init_off(2 * (size_t)N1, 0);
  const int max_q = compact_queries(q, offs, LINS_SEQ_RAN, run_off, copies, qto);
  for (int c = 0; c < 2; ++c) init_off[c * N1] = run_off[c * N1 + N1 - 1];
  const int max_init_q = compact_queries(q, offs, LINS_SEQ_SECOND, init_off, copies, qto);
  const int n_qcopies = (int)copies.size();

  // ---- allocations ------------------------------------------------------------------------------------------------
  Resident& r = q.run;
  r.n = n; r.nqs = init_off[N1 - 1]; r.nqc = init_off[2 * N1 - 1]; r.max_q = max_q;
  r.nts = q.map.h_off[N1 - 1]; r.ntc = q.map.h_off[2 * N1 - 1];
  CK(r.qs.reserve(r.nqs + 1)); CK(r.qc.reserve(r.nqc + 1)); CK(r.qs_off.reserve(N1)); CK(r.qc_off.reserve(N1));
  rc = reserve_outputs(ctx, r, true, false);
  if (rc != LINS_OK) return rc;
  CK(r.h_off.reserve(4 * (size_t)N1));
  if (n_init) { CK(q.init_off.reserve(2 * (size_t)N1)); CK(q.scan_imu.reserve((size_t)n * 6)); CK(q.h_scan_imu.reserve((size_t)n * 6)); }
  // (pre and init_icp are lins_gpu_seq_open's: they keep their contents from step to step)
  rc = build_next_maps(ctx, q.map, next, copies);
  if (rc != LINS_OK) return rc;
  const size_t n_imu = d->imu_off ? (size_t)d->imu_off[n] : 0;
  CK(q.imu.reserve(7 * n_imu + 1)); CK(q.imu_off.reserve(N1)); CK(q.h_imu.reserve(7 * n_imu + 1)); CK(q.h_imu_off.reserve(N1));
  CK(q.status_d.reserve(3 * (size_t)n)); CK(q.h_status.reserve(3 * (size_t)n));
  CK(q.period.reserve(n)); CK(q.h_period.reserve(n));
  CK(q.unit_tune.reserve(n)); CK(q.h_unit_tune.reserve(n));
  const bool any_tuned = std::any_of(q.slot.begin(), q.slot.end(), [](const SeqSlot& x) { return x.tune.has_value(); });
  const bool align = any_tuned && (n_imu || n_init);  // (a run without a tuned slot launches what it launched before)
  if (align) { CK(q.align.reserve(10 * (size_t)n)); CK(q.h_align.reserve(10 * (size_t)n)); }
  const int n_copies = (int)copies.size();
  if ((rc = q.copies.reserve(ctx, n_copies)) != LINS_OK) return rc;
  CK(q.prior_state.reserve((size_t)n * 20)); CK(q.prior_cov.reserve((size_t)n * 324));
  CK(q.icp_ind_s.reserve(3 * r.nqs + 4)); CK(q.icp_ind_c.reserve(2 * r.nqc + 4));
  float4* qdst[2] = {r.qs.p, r.qc.p};
  for (int i = 0; i < n_qcopies; ++i) copies[i].dst = qdst[qto[i].first] + qto[i].second;

  // ---- uploads: IMU, status, copy lists, compacted query offsets ---------------------------------------------------
  if (d->imu_off) std::memcpy(q.h_imu_off.p, d->imu_off, sizeof(int) * N1);
  else std::memset(q.h_imu_off.p, 0, sizeof(int) * N1);
  if (n_imu) std::memcpy(q.h_imu.p, d->imu, sizeof(double) * 7 * n_imu);
  for (int s = 0; s < n; ++s) {
    const SlotParams p = slot_params(ctx, s);
    q.h_status.p[s] = (unsigned char)status[s]; q.h_status.p[2 * n + s] = imu_use[s]; q.h_period.p[s] = p.period; q.h_unit_tune.p[s] = p.tune;
    if (align) std::copy(p.align, p.align + 10, q.h_align.p + 10 * (size_t)s);
  }
  std::memcpy(r.h_off.p, run_off.data(), sizeof(int) * 2 * N1);
  std::memcpy(r.h_off.p + 2 * N1, init_off.data(), sizeof(int) * 2 * N1);
  if (n_imu) CK(cudaMemcpyAsync(q.imu.p, q.h_imu.p, sizeof(double) * 7 * n_imu, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(q.imu_off.p, q.h_imu_off.p, sizeof(int) * N1, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(q.status_d.p, q.h_status.p, n, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(q.status_d.p + 2 * n, q.h_status.p + 2 * n, n, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(q.period.p, q.h_period.p, sizeof(double) * n, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(q.unit_tune.p, q.h_unit_tune.p, sizeof(lins_dev::UnitTuning) * n, cudaMemcpyHostToDevice, ctx->stream));
  if (align) CK(cudaMemcpyAsync(q.align.p, q.h_align.p, sizeof(double) * 10 * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  if ((rc = q.copies.stage(ctx, copies.data(), n_copies, 0)) != LINS_OK) return rc;
  CK(cudaMemcpyAsync(r.qs_off.p, r.h_off.p, sizeof(int) * N1, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(r.qc_off.p, r.h_off.p + N1, sizeof(int) * N1, cudaMemcpyHostToDevice, ctx->stream));
  if (n_init) {
    std::memcpy(q.h_scan_imu.p, scan_imu, sizeof(double) * 6 * (size_t)n);  // (validated: non-null when a slot initialises)
    CK(cudaMemcpyAsync(q.scan_imu.p, q.h_scan_imu.p, sizeof(double) * 6 * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(q.init_off.p, r.h_off.p + 2 * N1, sizeof(int) * 2 * N1, cudaMemcpyHostToDevice, ctx->stream));
  }

  // ---- 1. IMU propagation (StatePredictor::predict; the pre-integration of a slot between its first and second scan) --
  for (cudaEvent_t& e : q.ev) if (!e) CK(cudaEventCreate(&e));
  q.ev_valid = false;
  CK(cudaEventRecord(q.ev[0], ctx->stream));
  const lins_seq::Consts* k = slot_consts(q);
  const lins_seq::InitConsts* ik = slot_init_consts(q);
  if (align) {  // the tuned slots' IMU values into the vehicle frame (imuCallback) before anything reads them
    lins_seq_align_kernel<<<n, 32, 0, ctx->stream>>>(q.imu.p, q.imu_off.p, n_init ? q.scan_imu.p : nullptr, q.align.p);
    CK(cudaGetLastError());
    ctx->launches += 1;
  }
  if (n_imu) {
    lins_seq_predict_kernel<<<n, 32, 0, ctx->stream>>>(q.filt.p, q.cov.p, q.imu_last.p, q.imu.p, q.imu_off.p, q.status_d.p + 2 * n, q.pre.p, k, ik);
    CK(cudaGetLastError());
    ctx->launches += 1;
  }
  // the prior of this step's IESKF (also what lins_gpu_seq_download_ieskf returns)
  CK(cudaMemcpyAsync(q.prior_state.p, q.filt.p, sizeof(double) * 20 * (size_t)n, cudaMemcpyDeviceToDevice, ctx->stream));
  CK(cudaMemcpyAsync(q.prior_cov.p, q.cov.p, sizeof(double) * 324 * (size_t)n, cudaMemcpyDeviceToDevice, ctx->stream));
  CK(cudaEventRecord(q.ev[1], ctx->stream));
  if (n_run == 0 && n_init == 0) {  // nothing passed the gate: the maps stay, nothing else to do
    for (int e = 2; e < 5; ++e) CK(cudaEventRecord(q.ev[e], ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    for (int s = 0; s < n; ++s) if (status[s] == LINS_SEQ_INIT_WAIT) q.fusion[s] = FUSION_INIT;
    q.ev_valid = true;
    q.has_step = true;
    q.h_run_off.swap(run_off);
    return LINS_OK;
  }

  // ---- 2. IESKF over every sequence; those that do not run have no queries ------------------------------------------
  if ((rc = q.copies.launch(ctx, 0, n_qcopies)) != LINS_OK) return rc;
  BatchView bv;
  std::memset(&bv, 0, sizeof(bv));
  bv.n_scans = n;
  bv.qs = r.qs.p; bv.qs_off = r.qs_off.p; bv.qc = r.qc.p; bv.qc_off = r.qc_off.p;
  map_targets(bv, q.map);
  bv.unit_period = q.period.p;
  bv.unit_tune = q.unit_tune.p;
  bv.state_in = q.prior_state.p; bv.cov_in = q.prior_cov.p; bv.state_out = r.state_out.p; bv.cov_out = r.cov_out.p;
  bv.results = r.results.p; bv.reports = r.reports.p;
  bv.ind_s = r.ind_s.p; bv.ind_c = r.ind_c.p; bv.az_s = r.az_s.p; bv.az_c = r.az_c.p;
  bv.accum = r.accum.p; bv.work_counter = r.counter.p;
  bv.qtile = fused_qtile(r.max_q);
  if (n_run) {
    rc = fused_ieskf_launch(ctx, r, bv);
    if (rc != LINS_OK) return rc;
  }
  CK(cudaEventRecord(q.ev[2], ctx->stream));

  // ---- 3. divergence: one D2H of the result records -----------------------------------------------------------------
  bool any_icp = false;
  if (n_run) {
    CK(r.h_results.reserve(n));
    CK(cudaMemcpyAsync(r.h_results.p, r.results.p, sizeof(lins_scan_result) * n, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
  }
  for (int s = 0; s < n && n_run; ++s) {
    if (status[s] != LINS_SEQ_RAN || !(r.h_results.p[s].flags & 2u)) continue;
    // estimateTransform from the prior's pose (performIESKF's "Using ICP Method" branch, StateEstimator.hpp:585-592)
    status[s] = LINS_SEQ_ICP;
    q.h_status.p[s] = LINS_SEQ_ICP;
    any_icp = true;
    CK(cudaMemcpyAsync(q.icp_pose.p + (size_t)s * 20, q.prior_state.p + (size_t)s * 20, sizeof(double) * 20, cudaMemcpyDeviceToDevice, ctx->stream));
    BatchView u = bv;
    u.n_scans = 1;
    u.qs_off += s; u.qc_off += s; u.ts_off += s; u.tc_off += s; u.nn_s_off += s; u.nn_c_off += s; u.nn_stale += s; u.unit_period += s; u.unit_tune += s;
    u.cov_in += (size_t)s * 324; u.state_out += (size_t)s * 20; u.cov_out += (size_t)s * 324; u.results += s; u.reports = nullptr;
    u.accum += (size_t)s * 32;
    u.ind_s = q.icp_ind_s.p; u.ind_c = q.icp_ind_c.p;  // (the IESKF's IDs stay readable)
    u.qtile = fused_qtile((run_off[s + 1] - run_off[s]) + (run_off[N1 + s + 1] - run_off[N1 + s]));
    lins_dev::IcpState* icp = reinterpret_cast<lins_dev::IcpState*>(q.icp.p) + s;
    CK(cudaMemsetAsync(icp, 0, icp_state_bytes(), ctx->stream));
    rc = icp_loop(ctx, r, u, q.icp_pose.p + (size_t)s * 20, icp, q.h_unit_tune.p[s].num_iter);
    if (rc != LINS_OK) return rc;
  }
  if (any_icp) CK(cudaMemcpyAsync(q.status_d.p, q.h_status.p, n, cudaMemcpyHostToDevice, ctx->stream));

  // ---- 3b. the second scans' estimateTransform (processSecondScan), all in one loop: each from its pre-integrated pose
  // against its first scan's map; the IESKF's sequences read done and are passed over --------------------------------
  lins_dev::IcpState* init_icp = reinterpret_cast<lins_dev::IcpState*>(q.init_icp.p);
  if (n_second) {
    lins_seq_icp_start_kernel<<<(n + 127) / 128, 128, 0, ctx->stream>>>(n, q.status_d.p, q.pre.p, q.icp_pose.p, init_icp, q.unit_tune.p);
    CK(cudaGetLastError());
    ctx->launches += 1;
    BatchView u = bv;
    u.qs_off = q.init_off.p; u.qc_off = q.init_off.p + N1;
    u.reports = nullptr;
    u.ind_s = q.icp_ind_s.p; u.ind_c = q.icp_ind_c.p;
    u.qtile = fused_qtile(max_init_q);
    int n_iter = 0;  // (the largest NUM_ITER of the second scans)
    for (int s = 0; s < n; ++s) if (status[s] == LINS_SEQ_SECOND) n_iter = std::max(n_iter, q.h_unit_tune.p[s].num_iter);
    rc = icp_loop(ctx, r, u, q.icp_pose.p, init_icp, n_iter);
    if (rc != LINS_OK) return rc;
  }
  CK(cudaEventRecord(q.ev[3], ctx->stream));

  // ---- 4. update, integrateTransformation, reset(1), roll / pitch; processFirstScan / the rest of processSecondScan ---
  if (n_run) {
    lins_seq_post_kernel<<<(n + 127) / 128, 128, 0, ctx->stream>>>(n, q.status_d.p, r.state_out.p, r.cov_out.p, q.icp_pose.p, q.filt.p, q.cov.p,
                                                                     q.glob.p, q.lin.p, k);
    CK(cudaGetLastError());
    ctx->launches += 1;
  }
  if (n_init) {
    lins_seq_init_kernel<<<(n + 127) / 128, 128, 0, ctx->stream>>>(n, q.status_d.p, q.scan_imu.p, q.icp_pose.p, q.pre.p, q.glob.p, q.filt.p,
                                                                     q.cov.p, q.lin.p, q.imu_last.p, ik);
    CK(cudaGetLastError());
    ctx->launches += 1;
  }

  // ---- 5. transformToEnd of the new less-* clouds + the guarded map swap (a first scan's clouds stay as they are) ------
  unsigned char* run_mask = q.status_d.p + n;
  for (int s = 0; s < n; ++s)
    q.h_status.p[n + s] = status[s] == LINS_SEQ_RAN || status[s] == LINS_SEQ_ICP || status[s] == LINS_SEQ_SECOND ? 1 : 0;
  CK(cudaMemcpyAsync(run_mask, q.h_status.p + n, n, cudaMemcpyHostToDevice, ctx->stream));
  rc = transform_to_end(ctx, q.up.ts.p, q.up.ts_off.p, n, q.lin.p, run_mask, q.period.p);
  if (rc == LINS_OK) rc = transform_to_end(ctx, q.up.tc.p, q.up.tc_off.p, n, q.lin.p, run_mask, q.period.p);
  if (rc == LINS_OK) rc = q.copies.launch(ctx, n_qcopies, n_copies - n_qcopies);
  if (rc != LINS_OK) return rc;
  swap_maps(q.map);
  q.map.h_stale = new_stale;
  CK(queue_map_state(ctx, q.map));
  CK(cudaEventRecord(q.ev[4], ctx->stream));
  if (q.pub.bound) CK(cudaMemcpyAsync(q.pub.h_glob.p, q.glob.p, sizeof(double) * 20 * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));  // (the two sources above are pageable and change with the next step)
  for (int s = 0; s < n; ++s) {  // processPCL's status transitions (:294-307)
    if (status[s] == LINS_SEQ_INIT_WAIT) q.fusion[s] = FUSION_INIT;
    else if (status[s] == LINS_SEQ_FIRST) q.fusion[s] = FUSION_FIRST_SCAN;
    else if (status[s] == LINS_SEQ_SECOND) q.fusion[s] = FUSION_RUNNING;
  }
  q.ev_valid = true;
  q.has_step = true;
  q.h_run_off.swap(run_off);
  return LINS_OK;
}

// The part of a step after its input is validated and uploaded.  From here on the sequences' state changes: a failure ends
// the run (lins_gpu.h), the context stays usable.
int seq_step_run(lins_ctx* ctx, const lins_seq_step_desc* d, const int32_t* const offs[4], const double* scan_imu) {
  const int rc = seq_step_phases(ctx, d, offs, scan_imu);
  if (rc != LINS_OK) ctx->seq.n = 0;
  else if (ctx->seq.pub.bound) ctx->seq.pub.pending = true;
  return rc;
}

// The rest of a step whose features were extracted into ctx->feat (scan s's clouds at f.out[k] + src_off[s], counts read
// back): the present slots' features -> the step's four clouds (q.up, lins_seq_step_desc order), dense in slot order,
// then the sequence step.
int step_from_features(lins_ctx* ctx, const uint8_t* pres, const double* imu, const int32_t* imu_off, const int32_t* src_off,
                       const double* scan_imu) {
  SeqState& q = ctx->seq;
  const int n = q.n, N1 = n + 1;
  FeatState& f = ctx->feat;
  Resident& r = q.up;
  std::vector<int32_t> off(4 * (size_t)N1, 0);
  r.max_q = 0;
  for (int s = 0; s < n; ++s) {
    const bool present = !pres || pres[s];
    for (int k = 0; k < 4; ++k) off[k * N1 + s + 1] = off[k * N1 + s] + (present ? f.h_counts.p[5 * s + k] : 0);
    r.max_q = std::max(r.max_q, (off[s + 1] - off[s]) + (off[N1 + s + 1] - off[N1 + s]));
  }
  r.n = n; r.nqs = off[N1 - 1]; r.nqc = off[2 * N1 - 1]; r.nts = off[3 * N1 - 1]; r.ntc = off[4 * N1 - 1];
  CK(r.qs.reserve(r.nqs + 1)); CK(r.qc.reserve(r.nqc + 1)); CK(r.ts.reserve(r.nts + 1)); CK(r.tc.reserve(r.ntc + 1));
  CK(r.qs_off.reserve(N1)); CK(r.qc_off.reserve(N1)); CK(r.ts_off.reserve(N1)); CK(r.tc_off.reserve(N1));
  CK(r.h_off.reserve(4 * (size_t)N1));
  float4* dst[4] = {r.qs.p, r.qc.p, r.ts.p, r.tc.p};
  int* doff[4] = {r.qs_off.p, r.qc_off.p, r.ts_off.p, r.tc_off.p};
  std::vector<DevCopy> copies;
  for (int k = 0; k < 4; ++k)
    for (int s = 0; s < n; ++s) {
      const int len = off[k * N1 + s + 1] - off[k * N1 + s];
      if (len) copies.push_back(DevCopy{f.out[k].p + src_off[s], dst[k] + off[k * N1 + s], len, 0});
    }
  int rc = f.copies.reserve(ctx, copies.size());
  if (rc == LINS_OK) rc = f.copies.stage(ctx, copies.data(), (int)copies.size(), 0);
  if (rc != LINS_OK) return rc;
  std::memcpy(r.h_off.p, off.data(), sizeof(int) * off.size());
  for (int k = 0; k < 4; ++k) CK(cudaMemcpyAsync(doff[k], r.h_off.p + (size_t)k * N1, sizeof(int) * N1, cudaMemcpyHostToDevice, ctx->stream));
  if ((rc = f.copies.launch(ctx, 0, (int)copies.size())) != LINS_OK) return rc;
  lins_seq_step_desc sd;
  std::memset(&sd, 0, sizeof(sd));
  sd.n_seq = n; sd.present = pres; sd.imu = imu; sd.imu_off = imu_off; sd.point_format = LINS_POINTS_XYZI32;
  const int32_t* offs[4] = {&off[0], &off[N1], &off[2 * N1], &off[3 * N1]};
  return seq_step_run(ctx, &sd, offs, scan_imu);
}

// The rest of a step whose sweeps' projection (with the NaN removal) is queued in ctx->proj at the raw offsets src_off:
// the extraction on the projection's output where it lies (each scan's segmented count as its extent; line_num: the
// ring stride, the table's largest line_num, whose extra rings are empty), one D2H + synchronisation for the counts before
// the sequences change, then step_from_features.
int step_from_projection(lins_ctx* ctx, const uint8_t* pres, const double* imu, const int32_t* imu_off, int line_num,
                         const lins_feature_params* fp, const int32_t* src_off, const double* scan_imu) {
  SeqState& q = ctx->seq;
  const int n = q.n;
  ProjState& pr = ctx->proj;
  SeqPubState& pb = q.pub;
  // a bound run keeps the outlier clouds: their counts join the extraction's read-back
  if (pb.bound) CK(cudaMemcpyAsync(pb.h_proj_counts.p, pr.counts.p, sizeof(int) * 2 * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  FeatInputs in;
  in.n = n; in.line_num = line_num; in.total = src_off[n];
  in.pts = pr.seg.p; in.off = pr.up.qs_off.p; in.count = pr.counts.p; in.count_stride = 2;
  in.ground = pr.ground.p; in.col = pr.col.p; in.range = pr.range.p; in.ring = pr.ring.p; in.ori = pr.ori.p;
  std::vector<FeatConsts> k(n);
  for (int s = 0; s < n; ++s) k[s] = slot_params(ctx, s, fp).feat;
  int rc = features_launch(ctx, k.data(), in);
  if (rc != LINS_OK) return rc;
  if (pb.bound) {  // the stash: every slot's outlier cloud, device to device (an absent slot's sweep projected empty)
    pb.h_stash_off.assign((size_t)n + 1, 0);
    for (int s = 0; s < n; ++s) pb.h_stash_off[s + 1] = pb.h_stash_off[s] + pb.h_proj_counts.p[2 * s + 1];
    CK(pb.stash.reserve((size_t)pb.h_stash_off[n] + 1));
    std::vector<DevCopy> copies;
    for (int s = 0; s < n; ++s) {
      const int no = pb.h_stash_off[s + 1] - pb.h_stash_off[s];
      if (no) copies.push_back(DevCopy{pr.outl.p + src_off[s], pb.stash.p + pb.h_stash_off[s], no, 0});
    }
    if ((rc = pb.copies.reserve(ctx, copies.size())) != LINS_OK) return rc;
    if ((rc = pb.copies.stage(ctx, copies.data(), (int)copies.size(), 0)) != LINS_OK) return rc;
    if ((rc = pb.copies.launch(ctx, 0, (int)copies.size())) != LINS_OK) return rc;
    pb.dev_outliers = true;
  }
  return step_from_features(ctx, pres, imu, imu_off, src_off, scan_imu);
}

// ---- the publish step of a bound run ---------------------------------------------------------------------------------
// publishTopics' rule (Estimator.cpp:254-284): a slot publishes after every scan of an estimator that was initialised
// before it, i.e. present with a status other than STATUS_INIT before the step
bool publishes(int32_t status, int32_t fusion_before) {
  return status != LINS_SEQ_IDLE && fusion_before != FUSION_INIT;
}
// updatePointCloud ran: the scan was accepted (SECOND / RAN / ICP)
bool accepted(int32_t status) { return status == LINS_SEQ_SECOND || status == LINS_SEQ_RAN || status == LINS_SEQ_ICP; }

// lins_gpu_seq_map_step on a checked call: the estimator side (outlier stash and generation, YZX flags, poses) is
// committed, then one lockstep mapper step of the publishing slots on the device clouds
int seq_map_run(lins_ctx* ctx, const lins_seq_map_desc* d, lins_mapper_report* reps, uint8_t* published) {
  SeqState& q = ctx->seq;
  SeqPubState& pb = q.pub;
  const int n = q.n;
  CK(cudaSetDevice(ctx->device));
  std::vector<uint8_t> pub(n, 0);
  for (int s = 0; s < n; ++s) pub[s] = publishes(q.status[s], pb.fusion_before[s]) ? 1 : 0;
  // a caller's outlier clouds into the stash (the last step ended with a synchronisation: the staging is free)
  if (!pb.dev_outliers) {
    const int total = d->outlier_off[n];
    pb.h_stash_off.assign(d->outlier_off, d->outlier_off + n + 1);
    CK(pb.stash.reserve((size_t)total + 1)); CK(pb.h_stash.reserve((size_t)total + 1));
    if (total) {
      pack_into(pb.h_stash.p, d->outlier, total);
      CK(cudaMemcpyAsync(pb.stash.p, pb.h_stash.p, sizeof(float4) * total, cudaMemcpyHostToDevice, ctx->stream));
    }
  }
  // updatePointCloud of the accepted scans (their YZX clouds and pose); processFirstScan's fresh scan_last_
  for (int s = 0; s < n; ++s) {
    const int32_t st = q.status[s];
    SeqSlot& r = q.slot[s];
    if (st == LINS_SEQ_FIRST) r.yzx = false;
    if (!accepted(st)) continue;
    r.yzx = true;
    const double* g = pb.h_glob.p + 20 * (size_t)s;  // rn = g[0..2], qbn = g[6..9]
    lins::global_state_yzx(g, g + 6, r.pose, r.pose + 3);
  }
  // the next outlier generation: an accepted scan's outliers, a slot without YZX clouds none, else the kept ones
  const int N1 = n + 1;
  pb.h_noutl_off.assign(N1, 0);
  std::vector<MapPiece> next(n);
  for (int s = 0; s < n; ++s) {
    if (!q.slot[s].yzx) next[s] = MapPiece{};
    else if (accepted(q.status[s])) next[s] = MapPiece{pb.stash.p + pb.h_stash_off[s], pb.h_stash_off[s + 1] - pb.h_stash_off[s]};
    else next[s] = MapPiece{pb.outl.p + pb.h_outl_off[s], pb.h_outl_off[s + 1] - pb.h_outl_off[s]};
    pb.h_noutl_off[s + 1] = pb.h_noutl_off[s] + next[s].len;
  }
  CK(pb.noutl.reserve((size_t)pb.h_noutl_off[n] + 1));
  std::vector<DevCopy> copies;
  for (int s = 0; s < n; ++s)
    if (next[s].len) copies.push_back(DevCopy{next[s].src, pb.noutl.p + pb.h_noutl_off[s], next[s].len, 0});
  int rc = pb.copies.reserve(ctx, copies.size());
  if (rc == LINS_OK) rc = pb.copies.stage(ctx, copies.data(), (int)copies.size(), 0);
  if (rc == LINS_OK) rc = pb.copies.launch(ctx, 0, (int)copies.size());
  if (rc != LINS_OK) return rc;
  std::swap(pb.outl, pb.noutl);
  pb.h_outl_off.swap(pb.h_noutl_off);
  pb.pending = false;
  if (published) std::copy(pub.begin(), pub.end(), published);

  // the mapping nodes' inputs: scan_last_'s less-sharp / less-flat clouds are the slot's current maps, in XYZ order.
  // The fusion node handles the odometry before the mapping node's cycle for this scan ends (DESIGN.md §4.13).
  std::vector<MapPiece> dev(3 * (size_t)n);
  std::vector<double> quat(4 * (size_t)n), pos(3 * (size_t)n);
  for (int s = 0; s < n; ++s) {
    std::memset(&pb.fused[s], 0, sizeof(pb.fused[s]));
    if (!pub[s]) continue;
    const SeqSlot& r = q.slot[s];
    if (r.yzx) {
      dev[3 * s + 0] = current_piece(q.map, 1, s);
      dev[3 * s + 1] = current_piece(q.map, 0, s);
      dev[3 * s + 2] = MapPiece{pb.outl.p + pb.h_outl_off[s], pb.h_outl_off[s + 1] - pb.h_outl_off[s]};
    }
    std::copy(r.pose, r.pose + 3, &pos[3 * (size_t)s]);
    std::copy(r.pose + 3, r.pose + 7, &quat[4 * (size_t)s]);
    mapper_node_fuse(ctx->mappers.node[s], d->time[s], r.pose + 3, r.pose, pb.fused[s]);
  }
  lins_mappers_desc md;
  std::memset(&md, 0, sizeof(md));
  md.n_slots = n; md.present = pub.data(); md.time = d->time; md.quat = quat.data(); md.pos = pos.data();
  std::vector<double> period(n);
  for (int s = 0; s < n; ++s) period[s] = slot_params(ctx, s).period;
  return mappers_step(ctx, ctx->mappers, &md, reps, dev.data(), period.data());
}

}  // namespace

extern "C" {

int lins_gpu_seq_begin(lins_ctx* ctx, const lins_seq_params* prm, const lins_seq_begin_desc* d) {
  if (!ctx) return LINS_E_INVALID;
  if (!prm || !d || d->n_seq < 1) return fail(ctx, LINS_E_INVALID, "bad sequence hand-over");
  if (!d->filter_state || !d->filter_cov || !d->global_state || !d->imu_last) return fail(ctx, LINS_E_INVALID, "null hand-over state");
  const int n = d->n_seq;
  int rc = check_csr(ctx, d->surf_map_off, n, d->surf_map, "bad surf map offsets / cloud");
  if (rc == LINS_OK) rc = check_csr(ctx, d->corner_map_off, n, d->corner_map, "bad corner map offsets / cloud");
  if (rc != LINS_OK) return rc;
  if (d->point_format != LINS_POINTS_XYZI32 && d->point_format != LINS_POINTS_PACKED16) return fail(ctx, LINS_E_INVALID, "bad point_format");
  CK(cudaSetDevice(ctx->device));
  SeqState& q = ctx->seq;
  q.n = 0;  // (until the hand-over is in place)
  q.pub.bound = false;
  // the maps go through the batch uploader as the target clouds of n units without queries
  std::vector<int32_t> zeros(n + 1, 0);
  const lins_point* pts[4] = {nullptr, nullptr, d->surf_map, d->corner_map};
  const int32_t* offs[4] = {zeros.data(), zeros.data(), d->surf_map_off, d->corner_map_off};
  rc = upload_clouds(ctx, q.up, n, pts, offs, d->point_format);
  if (rc != LINS_OK) return rc;
  const size_t ns = d->surf_map_off[n], nc = d->corner_map_off[n];
  rc = reserve_run(ctx, q, n, ns, nc);
  if (rc != LINS_OK) return rc;
  if (ns) CK(cudaMemcpyAsync(q.map.cur[0].p, q.up.ts.p, sizeof(float4) * ns, cudaMemcpyDeviceToDevice, ctx->stream));
  if (nc) CK(cudaMemcpyAsync(q.map.cur[1].p, q.up.tc.p, sizeof(float4) * nc, cudaMemcpyDeviceToDevice, ctx->stream));
  std::vector<double> st((size_t)n * 20), gl((size_t)n * 20), il((size_t)n * 8);
  pad_states(st.data(), d->filter_state, n);
  pad_states(gl.data(), d->global_state, n);
  copy_rows(il.data(), 8, d->imu_last, 6, n);
  q.map.reset(n);
  std::memcpy(&q.map.h_off[0], d->surf_map_off, sizeof(int) * (n + 1));
  std::memcpy(&q.map.h_off[n + 1], d->corner_map_off, sizeof(int) * (n + 1));
  CK(cudaMemcpyAsync(q.filt.p, st.data(), sizeof(double) * st.size(), cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(q.lin.p, st.data(), sizeof(double) * st.size(), cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(q.glob.p, gl.data(), sizeof(double) * gl.size(), cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(q.imu_last.p, il.data(), sizeof(double) * il.size(), cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(q.cov.p, d->filter_cov, sizeof(double) * 324 * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  CK(queue_map_state(ctx, q.map));
  CK(cudaStreamSynchronize(ctx->stream));  // (the sources above are pageable host memory)
  consts_of(q.consts, prm);
  std::fill(q.init_consts, q.init_consts + kNInit, 0.0);  // (a hand-over does not initialise)
  q.slot.assign(n, SeqSlot());
  if ((rc = upload_slot_consts(ctx, n)) != LINS_OK) return rc;
  // result records / reports read as zero until a step has run a sequence's IESKF
  CK(cudaMemsetAsync(q.run.results.p, 0, sizeof(lins_scan_result) * n, ctx->stream));
  CK(cudaMemsetAsync(q.run.reports.p, 0, sizeof(lins_report) * n, ctx->stream));
  install_run(q, n, false);
  return LINS_OK;
}

int lins_gpu_seq_open(lins_ctx* ctx, const lins_seq_params* prm, const lins_seq_init_params* ip, int32_t n_seq) {
  if (!ctx) return LINS_E_INVALID;
  if (!prm || !ip || n_seq < 1) return fail(ctx, LINS_E_INVALID, "bad lins_gpu_seq_open arguments");
  CK(cudaSetDevice(ctx->device));
  SeqState& q = ctx->seq;
  q.n = 0;  // (until the slots are in place)
  q.pub.bound = false;
  const int n = n_seq;
  int rc = reserve_run(ctx, q, n, 0, 0);  // (no maps)
  if (rc != LINS_OK) return rc;
  CK(q.pre.reserve((size_t)n * 20)); CK(q.init_icp.reserve(icp_state_bytes() * n));
  consts_of(q.consts, prm);
  init_consts_of(q.init_consts, prm, ip);
  q.slot.assign(n, SeqSlot());
  if ((rc = upload_slot_consts(ctx, n)) != LINS_OK) return rc;
  q.map.reset(n);
  CK(cudaMemsetAsync(q.lin.p, 0, sizeof(double) * 20 * (size_t)n, ctx->stream));
  CK(cudaMemsetAsync(q.imu_last.p, 0, sizeof(double) * 8 * (size_t)n, ctx->stream));
  CK(cudaMemsetAsync(q.pre.p, 0, sizeof(double) * 20 * (size_t)n, ctx->stream));
  CK(cudaMemsetAsync(q.icp_pose.p, 0, sizeof(double) * 20 * (size_t)n, ctx->stream));
  CK(cudaMemsetAsync(q.init_icp.p, 0, icp_state_bytes() * n, ctx->stream));
  CK(cudaMemsetAsync(q.run.results.p, 0, sizeof(lins_scan_result) * n, ctx->stream));
  CK(cudaMemsetAsync(q.run.reports.p, 0, sizeof(lins_report) * n, ctx->stream));
  CK(queue_map_state(ctx, q.map));
  rc = launch_fresh(ctx, q, n, nullptr);
  if (rc != LINS_OK) return rc;
  CK(cudaStreamSynchronize(ctx->stream));  // (the sources above are pageable host memory)
  install_run(q, n, true);
  return LINS_OK;
}

int lins_gpu_seq_restart(lins_ctx* ctx, const uint8_t* mask) {
  int rc = check_open_run(ctx, "lins_gpu_seq_restart", mask != nullptr);
  if (rc != LINS_OK) return rc;
  SeqState& q = ctx->seq;
  CK(cudaSetDevice(ctx->device));
  const int n = q.n;
  // the restarted slots' maps go: the other slots' ranges are copied into the next generation, which is swapped in
  std::vector<MapPiece> next(4 * (size_t)n);
  for (int s = 0; s < n; ++s)
    if (!mask[s]) for (int c = 0; c < 4; ++c) next[4 * (size_t)s + c] = current_piece(q.map, c, s);
  std::vector<DevCopy> copies;
  rc = build_next_maps(ctx, q.map, next, copies);
  if (rc == LINS_OK) rc = q.copies.reserve(ctx, copies.size());
  if (rc != LINS_OK) return rc;
  CK(q.status_d.reserve(3 * (size_t)n)); CK(q.h_status.reserve(3 * (size_t)n));
  // (the last step ended with a stream synchronisation: the pinned staging is free)
  // the restarted slots are new slots: unconfigured (their constants go back to the run's before the fresh state reads
  // them), untuned (the next step's tables read the context's), fresh, without YZX clouds
  bool any_configured = false;
  for (int s = 0; s < n; ++s)
    if (mask[s]) { any_configured |= q.slot[s].cfg.has_value(); q.slot[s] = SeqSlot(); }
  if (any_configured && (rc = upload_slot_consts(ctx, n)) != LINS_OK) { q.n = 0; return rc; }
  if ((rc = q.copies.stage(ctx, copies.data(), (int)copies.size(), 0)) != LINS_OK) return rc;
  for (int s = 0; s < n; ++s) q.h_status.p[s] = mask[s] ? 1 : 0;
  CK(cudaMemcpyAsync(q.status_d.p, q.h_status.p, n, cudaMemcpyHostToDevice, ctx->stream));
  rc = q.copies.launch(ctx, 0, (int)copies.size());
  if (rc == LINS_OK) rc = launch_fresh(ctx, q, n, q.status_d.p);
  if (rc != LINS_OK) { q.n = 0; return rc; }  // (some slots may have changed: the run ends, as after a failed step)
  swap_maps(q.map);
  for (int s = 0; s < n; ++s)
    if (mask[s]) { q.map.h_stale[s] = 0; q.fusion[s] = FUSION_INIT; q.status[s] = LINS_SEQ_IDLE; }
  // a new recording is a new LinsFusion with a new mapping node (and nothing fused yet)
  if (q.pub.bound) {
    for (int s = 0; s < n; ++s) if (mask[s]) q.pub.fused[s] = lins_fused_pose{};
    if ((rc = mappers_reset(ctx, ctx->mappers, mask)) != LINS_OK) return rc;
  }
  CK(queue_map_state(ctx, q.map));
  CK(cudaStreamSynchronize(ctx->stream));  // (the source above is pageable)
  return LINS_OK;
}

int lins_gpu_seq_configure(lins_ctx* ctx, const uint8_t* mask, const lins_slot_config* cfg) {
  const char* entry = "lins_gpu_seq_configure";
  int rc = check_open_run(ctx, entry, mask && cfg);
  if (rc != LINS_OK) return rc;
  SeqState& q = ctx->seq;
  const int n = q.n;
  for (int s = 0; s < n; ++s) {
    if (!mask[s]) continue;
    if ((rc = check_fresh(ctx, s, entry)) != LINS_OK) return rc;
    if (!lins_blob::config_ok(cfg[s]))
      return fail(ctx, LINS_E_INVALID, "lins_gpu_seq_configure: bad slot config (non-finite value, scan_period <= 0, or a negative noise / std)");
  }
  CK(cudaSetDevice(ctx->device));
  CK(q.status_d.reserve(3 * (size_t)n)); CK(q.h_status.reserve(3 * (size_t)n));
  // from here on the slots change: a failure ends the run, as a failed restart does
  for (int s = 0; s < n; ++s) if (mask[s]) q.slot[s].cfg = cfg[s];
  rc = upload_slot_consts(ctx, n);
  if (rc == LINS_OK) {
    for (int s = 0; s < n; ++s) q.h_status.p[s] = mask[s] ? 1 : 0;
    if (cudaMemcpyAsync(q.status_d.p, q.h_status.p, n, cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess) rc = fail(ctx, LINS_E_CUDA, "configure mask upload");
  }
  if (rc == LINS_OK) rc = launch_fresh(ctx, q, n, q.status_d.p);  // initializeCovariance with the config's stds
  if (rc == LINS_OK && cudaStreamSynchronize(ctx->stream) != cudaSuccess) rc = fail(ctx, LINS_E_CUDA, "configure");
  if (rc != LINS_OK) q.n = 0;
  return rc;
}

int lins_gpu_seq_tune(lins_ctx* ctx, const uint8_t* mask, const lins_slot_tuning* t) {
  const char* entry = "lins_gpu_seq_tune";
  int rc = check_open_run(ctx, entry, mask && t);
  if (rc != LINS_OK) return rc;
  SeqState& q = ctx->seq;
  const int n = q.n;
  for (int s = 0; s < n; ++s) {
    if (!mask[s]) continue;
    if ((rc = check_fresh(ctx, s, entry)) != LINS_OK) return rc;
    if (!lins_blob::tuning_ok(t[s]))
      return fail(ctx, LINS_E_INVALID, "lins_gpu_seq_tune: bad slot tuning (num_iter outside 0..LINS_MAX_ITER, icp_freq < 1, or a non-finite value)");
  }
  // (host state only: the step uploads the tables)
  for (int s = 0; s < n; ++s)
    if (mask[s]) {
      SeqSlot::Tuning u{t[s], {}};
      misalign_R(t[s].imu_misalign_angle, u.R);
      q.slot[s].tune = u;
    }
  return LINS_OK;
}

int lins_gpu_seq_step_ex(lins_ctx* ctx, const lins_seq_step_desc* d, const double* scan_imu) {
  int rc = check_step(ctx, d, d ? d->n_seq : 0, scan_imu);
  if (rc != LINS_OK) return rc;
  const int n = ctx->seq.n;
  const int32_t* offs[4] = {d->surf_flat_off, d->corner_sharp_off, d->surf_less_flat_off, d->corner_less_sharp_off};
  const lins_point* pts[4] = {d->surf_flat, d->corner_sharp, d->surf_less_flat, d->corner_less_sharp};
  CK(cudaSetDevice(ctx->device));
  rc = upload_clouds(ctx, ctx->seq.up, n, pts, offs, d->point_format);  // (validates the clouds; synchronises the stream first)
  if (rc != LINS_OK) return rc;
  return seq_step_run(ctx, d, offs, scan_imu);
}

int lins_gpu_seq_step(lins_ctx* ctx, const lins_seq_step_desc* d) { return lins_gpu_seq_step_ex(ctx, d, nullptr); }

int lins_gpu_seq_step_pcl(lins_ctx* ctx, const lins_seq_pcl_desc* d, const lins_feature_params* fp, const double* scan_imu) {
  int rc = check_step(ctx, d, d ? d->pcl.n_scans : 0, scan_imu);
  if (rc != LINS_OK) return rc;
  // extraction, validation of the scans and the counts' read-back: nothing of the sequences has changed yet
  std::vector<double> period(ctx->seq.n);  // (the re-stamp: each slot's period; the thresholds and extrinsic are fp's)
  for (int s = 0; s < ctx->seq.n; ++s) period[s] = slot_params(ctx, s).period;
  rc = features_run(ctx, fp, &d->pcl, period.data());
  if (rc != LINS_OK) return rc;
  return step_from_features(ctx, d->present, d->imu, d->imu_off, d->pcl.cloud_off, scan_imu);
}

int lins_gpu_seq_step_raw_mixed(lins_ctx* ctx, const lins_seq_raw_desc* d, const lins_lidar_models* t, const lins_feature_params* fp,
                                const double* scan_imu) {
  int rc = check_step(ctx, d, d ? d->raw.n_scans : 0, scan_imu);
  if (rc != LINS_OK) return rc;
  if (!fp) return fail(ctx, LINS_E_INVALID, "null feature params");
  // projection with copyPointCloud's NaN removal, then the rest of the step
  rc = projection_run(ctx, t, &d->raw, true, d->present);
  if (rc != LINS_OK) return rc;
  return step_from_projection(ctx, d->present, d->imu, d->imu_off, max_line_num(t), fp, d->raw.cloud_off, scan_imu);
}

int lins_gpu_seq_step_raw(lins_ctx* ctx, const lins_seq_raw_desc* d, const lins_lidar_model* m, const lins_feature_params* fp,
                          const double* scan_imu) {
  const lins_lidar_models t = {1, m, nullptr};
  return lins_gpu_seq_step_raw_mixed(ctx, d, &t, fp, scan_imu);
}

int lins_gpu_seq_step_cloud2_mixed(lins_ctx* ctx, const lins_seq_cloud2_desc* d, const lins_lidar_models* t, const lins_feature_params* fp,
                                   const double* scan_imu) {
  int rc = check_step(ctx, d, d ? d->cloud2.n_scans : 0, scan_imu);
  if (rc != LINS_OK) return rc;
  if (!fp) return fail(ctx, LINS_E_INVALID, "null feature params");
  const int n = ctx->seq.n;
  rc = check_models(ctx, t);
  if (rc == LINS_OK) rc = check_model_of(ctx, t, n);
  if (rc != LINS_OK) return rc;
  // the messages decoded into the projection's input (the present slots' only), then step_raw's projection and the rest
  std::vector<int32_t> off;
  rc = cloud2_run(ctx, &d->cloud2, d->present, off);
  if (rc != LINS_OK) return rc;
  rc = projection_launch(ctx, t, n, (size_t)off[n], true, d->present);
  if (rc != LINS_OK) return rc;
  return step_from_projection(ctx, d->present, d->imu, d->imu_off, max_line_num(t), fp, off.data(), scan_imu);
}

int lins_gpu_seq_step_cloud2(lins_ctx* ctx, const lins_seq_cloud2_desc* d, const lins_lidar_model* m, const lins_feature_params* fp,
                             const double* scan_imu) {
  const lins_lidar_models t = {1, m, nullptr};
  return lins_gpu_seq_step_cloud2_mixed(ctx, d, &t, fp, scan_imu);
}

int lins_gpu_seq_map_open(lins_ctx* ctx) {
  int rc = check_open_run(ctx, "lins_gpu_seq_map_open", true);
  if (rc != LINS_OK) return rc;
  SeqState& q = ctx->seq;
  if (q.has_step) return fail(ctx, LINS_E_INVALID, "lins_gpu_seq_map_open after the run's first step");
  const int n = q.n;
  SeqPubState& pb = q.pub;
  CK(cudaSetDevice(ctx->device));
  CK(pb.h_glob.reserve(20 * (size_t)n)); CK(pb.h_proj_counts.reserve(2 * (size_t)n)); CK(pb.outl.reserve(1));
  rc = mappers_open(ctx, ctx->mappers, n);
  if (rc != LINS_OK) return rc;
  const SeqSlot fresh;  // every estimator is new: no YZX clouds, globalStateYZX_ the identity
  for (SeqSlot& r : q.slot) { r.yzx = fresh.yzx; std::copy(fresh.pose, fresh.pose + 7, r.pose); }
  pb.h_outl_off.assign((size_t)n + 1, 0);
  pb.fusion_before.assign(n, FUSION_INIT);
  pb.fused.assign(n, lins_fused_pose{});
  pb.pending = false;
  pb.dev_outliers = false;
  pb.bound = true;
  return LINS_OK;
}

int lins_gpu_seq_map_step(lins_ctx* ctx, const lins_seq_map_desc* d, lins_mapper_report* reps, uint8_t* published) {
  if (!ctx) return LINS_E_INVALID;
  SeqState& q = ctx->seq;
  if (q.n == 0 || !q.pub.bound) return fail(ctx, LINS_E_NOMAP, "no sequence run bound by lins_gpu_seq_map_open");
  const int n = q.n;
  if (!d) return fail(ctx, LINS_E_INVALID, "null desc");
  if (!q.pub.pending) return fail(ctx, LINS_E_INVALID, "no sequence step since the last lins_gpu_seq_map_step");
  if (d->n_seq != n) return fail(ctx, LINS_E_INVALID, "n_seq differs from the run's");
  if (!d->time) return fail(ctx, LINS_E_INVALID, "null time");
  const bool given = d->outlier || d->outlier_off;
  if (q.pub.dev_outliers && given) return fail(ctx, LINS_E_INVALID, "outliers after a step that projected its scans on the device");
  if (!q.pub.dev_outliers) {
    if (!given) return fail(ctx, LINS_E_INVALID, "the last step's outlier clouds are required after a _ex / _pcl step");
    if (check_csr(ctx, d->outlier_off, n, d->outlier, "bad outlier offsets / cloud") != LINS_OK) return LINS_E_INVALID;
  }
  return seq_map_run(ctx, d, reps, published);
}

int lins_gpu_seq_map_published(lins_ctx* ctx, double* pose, int32_t* sizes) {
  if (!ctx) return LINS_E_INVALID;
  SeqState& q = ctx->seq;
  if (q.n == 0 || !q.pub.bound) return fail(ctx, LINS_E_NOMAP, "no sequence run bound by lins_gpu_seq_map_open");
  const SeqPubState& pb = q.pub;
  for (int s = 0; s < q.n; ++s) {
    const bool y = q.slot[s].yzx;
    if (pose) std::copy(q.slot[s].pose, q.slot[s].pose + 7, pose + 7 * (size_t)s);
    if (!sizes) continue;
    sizes[3 * s + 0] = y ? current_piece(q.map, 1, s).len : 0;
    sizes[3 * s + 1] = y ? current_piece(q.map, 0, s).len : 0;
    sizes[3 * s + 2] = y ? pb.h_outl_off[s + 1] - pb.h_outl_off[s] : 0;
  }
  return LINS_OK;
}

int lins_gpu_seq_map_fused(lins_ctx* ctx, lins_fused_pose* out) {
  if (!ctx) return LINS_E_INVALID;
  SeqState& q = ctx->seq;
  if (q.n == 0 || !q.pub.bound) return fail(ctx, LINS_E_NOMAP, "no sequence run bound by lins_gpu_seq_map_open");
  if (!out) return fail(ctx, LINS_E_INVALID, "null out");
  std::copy(q.pub.fused.begin(), q.pub.fused.end(), out);
  return LINS_OK;
}

int lins_gpu_seq_phase_ms(lins_ctx* ctx, float* ms) {
  if (!ctx || !ms) return LINS_E_INVALID;
  SeqState& q = ctx->seq;
  if (!q.ev_valid) return fail(ctx, LINS_E_INVALID, "no completed lins_gpu_seq_step");
  CK(cudaSetDevice(ctx->device));
  for (int i = 0; i < 4; ++i) CK(cudaEventElapsedTime(&ms[i], q.ev[i], q.ev[i + 1]));
  return LINS_OK;
}

int lins_gpu_seq_download(lins_ctx* ctx, double* global_state, double* filter_state, double* filter_cov, lins_scan_result* results,
                          lins_report* reports, int32_t* scan_status) {
  if (!ctx) return LINS_E_INVALID;
  SeqState& q = ctx->seq;
  if (q.n == 0) return fail(ctx, LINS_E_NOMAP, "lins_gpu_seq_begin has not been called");
  CK(cudaSetDevice(ctx->device));
  const size_t n = q.n;
  Resident& r = q.run;
  if ((results || reports) && r.results.cap < n) return fail(ctx, LINS_E_INVALID, "no step has run an IESKF yet");
  if (reports && r.reports.cap < n) return fail(ctx, LINS_E_INVALID, "no step has run an IESKF yet");
  std::vector<double> g(global_state ? n * 20 : 0), f(filter_state ? n * 20 : 0);
  if (global_state) CK(cudaMemcpyAsync(g.data(), q.glob.p, sizeof(double) * 20 * n, cudaMemcpyDeviceToHost, ctx->stream));
  if (filter_state) CK(cudaMemcpyAsync(f.data(), q.filt.p, sizeof(double) * 20 * n, cudaMemcpyDeviceToHost, ctx->stream));
  CK(d2h(ctx, filter_cov, q.cov.p, sizeof(double) * 324 * n));
  CK(d2h(ctx, results, r.results.p, sizeof(lins_scan_result) * n));
  CK(d2h(ctx, reports, r.reports.p, sizeof(lins_report) * n));
  CK(cudaStreamSynchronize(ctx->stream));
  if (global_state) strip_states(global_state, g.data(), n);
  if (filter_state) strip_states(filter_state, f.data(), n);
  if (scan_status) std::memcpy(scan_status, q.status.data(), sizeof(int32_t) * n);
  return LINS_OK;
}

int lins_gpu_seq_download_init(lins_ctx* ctx, int32_t* fusion_status, double* icp_pose, int32_t* icp_iters, int32_t* icp_converged) {
  if (!ctx) return LINS_E_INVALID;
  SeqState& q = ctx->seq;
  if (q.n == 0) return fail(ctx, LINS_E_NOMAP, "lins_gpu_seq_begin has not been called");
  const size_t n = q.n;
  if (fusion_status) std::memcpy(fusion_status, q.fusion.data(), sizeof(int32_t) * n);
  if (!icp_pose && !icp_iters && !icp_converged) return LINS_OK;
  if (icp_pose) std::memset(icp_pose, 0, sizeof(double) * 7 * n);
  if (icp_iters) std::memset(icp_iters, 0, sizeof(int32_t) * n);
  if (icp_converged) std::memset(icp_converged, 0, sizeof(int32_t) * n);
  bool any = false;
  for (size_t s = 0; s < n; ++s) any |= q.status[s] == LINS_SEQ_SECOND;
  if (!any) return LINS_OK;
  CK(cudaSetDevice(ctx->device));
  std::vector<double> pose(n * 20);
  std::vector<lins_dev::IcpState> st(n);
  CK(cudaMemcpyAsync(pose.data(), q.icp_pose.p, sizeof(double) * 20 * n, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaMemcpyAsync(st.data(), q.init_icp.p, sizeof(lins_dev::IcpState) * n, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  for (size_t s = 0; s < n; ++s) {
    if (q.status[s] != LINS_SEQ_SECOND) continue;
    if (icp_pose) state_to_pose(&pose[s * 20], icp_pose + s * 7);
    if (icp_iters) icp_iters[s] = st[s].iters;
    if (icp_converged) icp_converged[s] = st[s].converged;
  }
  return LINS_OK;
}

// ---- parity hooks: what the last step's IESKF saw and produced, and the maps the next step will use ---------------------
int lins_gpu_seq_download_ieskf(lins_ctx* ctx, double* prior_state, double* prior_cov, double* state_out, double* cov_out,
                                int32_t* query_off, int32_t* surf_ind, int32_t* corner_ind) {
  if (!ctx) return LINS_E_INVALID;
  SeqState& q = ctx->seq;
  if (q.n == 0) return fail(ctx, LINS_E_NOMAP, "lins_gpu_seq_begin has not been called");
  if (!q.has_step) return fail(ctx, LINS_E_INVALID, "no lins_gpu_seq_step since lins_gpu_seq_begin");
  CK(cudaSetDevice(ctx->device));
  const size_t n = q.n, N1 = n + 1;
  Resident& r = q.run;
  const int* ro = q.h_run_off.data();
  const bool ran = ro[N1 - 1] + ro[2 * N1 - 1] > 0;  // (else the IESKF did not run and its outputs are not this step's)
  if (!ran && (state_out || cov_out)) return fail(ctx, LINS_E_INVALID, "no sequence ran an IESKF in the last step");
  std::vector<double> a(prior_state ? n * 20 : 0), b(state_out ? n * 20 : 0);
  if (prior_state) CK(cudaMemcpyAsync(a.data(), q.prior_state.p, sizeof(double) * 20 * n, cudaMemcpyDeviceToHost, ctx->stream));
  CK(d2h(ctx, prior_cov, q.prior_cov.p, sizeof(double) * 324 * n));
  if (state_out) CK(cudaMemcpyAsync(b.data(), r.state_out.p, sizeof(double) * 20 * n, cudaMemcpyDeviceToHost, ctx->stream));
  CK(d2h(ctx, cov_out, r.cov_out.p, sizeof(double) * 324 * n));
  CK(d2h(ctx, surf_ind, r.ind_s.p, sizeof(int32_t) * 3 * ro[N1 - 1]));
  CK(d2h(ctx, corner_ind, r.ind_c.p, sizeof(int32_t) * 2 * ro[2 * N1 - 1]));
  CK(cudaStreamSynchronize(ctx->stream));
  if (prior_state) strip_states(prior_state, a.data(), n);
  if (state_out) strip_states(state_out, b.data(), n);
  if (query_off) std::memcpy(query_off, ro, sizeof(int32_t) * 2 * N1);
  return LINS_OK;
}

int lins_gpu_seq_download_maps(lins_ctx* ctx, int32_t* off, float* surf_map, float* corner_map, float* surf_tree, float* corner_tree,
                               uint8_t* stale) {
  if (!ctx) return LINS_E_INVALID;
  SeqState& q = ctx->seq;
  if (q.n == 0) return fail(ctx, LINS_E_NOMAP, "lins_gpu_seq_begin has not been called");
  CK(cudaSetDevice(ctx->device));
  const size_t N1 = q.n + 1;
  const int* mo = q.map.h_off.data();
  float* dst[4] = {surf_map, corner_map, surf_tree, corner_tree};
  for (int c = 0; c < 4; ++c) CK(d2h(ctx, dst[c], q.map.cur[c].p, sizeof(float4) * mo[c * N1 + N1 - 1]));
  CK(cudaStreamSynchronize(ctx->stream));
  if (off) std::memcpy(off, mo, sizeof(int32_t) * 4 * N1);
  if (stale) std::memcpy(stale, q.map.h_stale.data(), q.n);
  return LINS_OK;
}

}  // extern "C"
