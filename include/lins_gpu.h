/*
 * lins_gpu.h — C-ABI of the H100-native LINS iterated-ESKF update path.
 *
 * This is the drop-in boundary: every entry point replaces one seam of the reference's
 * header-only class fusion::StateEstimator (reference paths relative to /root/reference/):
 *
 *   lins_gpu_set_map        <-> kdtreeCorner_/kdtreeSurf_->setInputCloud(...)
 *                               lins/include/StateEstimator.hpp:363-364, :1156-1160
 *   lins_gpu_ieskf          <-> StateEstimator::performIESKF()            StateEstimator.hpp:465-600
 *   lins_gpu_associate      <-> findCorrespondingSurfFeatures / findCorrespondingCornerFeatures
 *                               StateEstimator.hpp:829-953, :955-1063 (+ transformToStart :1066-1080)
 *   lins_gpu_estimate_transform <-> estimateTransform / calculateTransformation
 *                               StateEstimator.hpp:1163-1196, :1198-1320 (fallback + scan-2 initialiser)
 *   lins_gpu_update_map     <-> updatePointCloud() / transformToEnd()     StateEstimator.hpp:1083-1101, :1116-1161
 *   lins_gpu_batch_*        <-> the same performIESKF, for many independent (scan pair, prior) units
 *                               resident in HBM (offline / batched odometry; SURVEY.md §8(e))
 *   lins_gpu_seq_*          <-> processImu + processScan (StateEstimator.hpp:242-270, :435-463) of many running
 *                               sequences in lockstep: IMU propagation, IESKF, ICP fallback, reset(1), roll / pitch
 *                               correction and the map refresh all on the device
 *
 * Conventions
 *   - extern "C", plain pointers and sizes; no Eigen / PCL / ROS / torch types.
 *   - every function returns 0 on success, <0 (LINS_E_*) on error; nothing throws.
 *     lins_gpu_last_error() returns a human readable message for the last failure on that ctx.
 *   - caller owns every host buffer; the library copies at call time and owns all device memory.
 *   - one ctx = one CUDA device + one CUDA stream; a ctx is not re-entrant, distinct ctxs are independent.
 *   - points are pcl::PointXYZI-layout compatible (32 B, 16-B aligned; lins/include/parameters.h:52):
 *       x@0 y@4 z@8 (pad) intensity@16 (pad..31); intensity = ring + SCAN_PERIOD*relTime
 *       (lins/src/image_projection_node.cpp:234, StateEstimator.hpp:647-650).
 *   - state vectors are 19 doubles in filter::GlobalState member order (KalmanFilter.hpp:110-115):
 *       rn[0..2] vn[3..5] qbn[6..9] (x,y,z,w — Eigen::Quaterniond::coeffs() order) ba[10..12] bw[13..15] gn[16..18]
 *   - covariances are 18x18 doubles, column-major (Eigen default), error-state order
 *       pos0 vel3 att6 acc9 gyr12 gra15 (KalmanFilter.hpp:38-45).
 */
#ifndef LINS_GPU_H_
#define LINS_GPU_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LINS_STATE_DIM 19
#define LINS_ERR_DIM 18
#define LINS_COV_SIZE 324
#define LINS_MAX_ITER 64

/* error codes */
#define LINS_OK 0
#define LINS_E_INVALID (-1)   /* bad argument */
#define LINS_E_CUDA (-2)      /* CUDA runtime failure (message in last_error) */
#define LINS_E_NOMAP (-3)     /* ieskf/associate before set_map */
#define LINS_E_TOOBIG (-4)    /* cloud larger than the ctx capacity */
#define LINS_E_NODEVICE (-5)  /* no usable CUDA device / sm_90 kernel image */

/* pcl::PointXYZI layout (parameters.h:52 `typedef pcl::PointXYZI PointType`). */
typedef struct lins_point {
  float x, y, z, pad0;
  float intensity, pad1, pad2, pad3;
} lins_point;

/* The 7 globals the hot path reads (parameters.h:104-153, exp_port.yaml:9-20) + test hooks. */
typedef struct lins_params {
  int32_t num_iter;        /* NUM_ITER, shipped 30 (exp_port.yaml:18); <= LINS_MAX_ITER */
  int32_t icp_freq;        /* ICP_FREQ, shipped 1 */
  double nearest_feature_search_sq_dist; /* NEAREST_FEATURE_SEARCH_SQ_DIST, shipped 25 */
  double lidar_std;        /* LIDAR_STD, shipped 0.01 */
  double lidar_scale;      /* LIDAR_SCALE, shipped 1 */
  double scan_period;      /* SCAN_PERIOD, shipped 0.1 */
  int32_t verbose;         /* VERBOSE (unused by the device path) */
  int32_t force_all_iters; /* test hook: 1 = ignore the ||dx||<=1e-2 exit (StateEstimator.hpp:576) so exactly
                              num_iter iterations run ("10 ESKF iters forced", BASELINE.json configs[0]) */
} lins_params;

/* What performIESKF would have logged (StateEstimator.hpp:485-496, :560, :567, :586). */
typedef struct lins_report {
  int32_t iters;      /* iterations executed (count of A2-A10 passes) */
  int32_t converged;  /* hasConverged, StateEstimator.hpp:576-578 */
  int32_t diverged;   /* hasDiverged, StateEstimator.hpp:559-570 (host must run the ICP fallback) */
  int32_t has_nan;    /* the NaN branch of the divergence test, StateEstimator.hpp:552-563 */
  int32_t m_surf[LINS_MAX_ITER];   /* accepted plane measurements per iteration */
  int32_t m_corner[LINS_MAX_ITER]; /* accepted line measurements per iteration */
  double residual_norm[LINS_MAX_ITER]; /* ||residual_|| per iteration */
  double update_norm[LINS_MAX_ITER];   /* ||updateVec_|| per iteration */
} lins_report;

/* Fixed 64-byte per-scan record of the batched mode (the unit the multi-GPU pose gather moves). */
typedef struct lins_scan_result {
  int32_t scan_id;
  uint16_t iters;
  uint16_t flags;      /* bit0 converged, bit1 diverged, bit2 has_nan */
  double pose[7];      /* rn (3) + qbn (x,y,z,w) of the updated filter state */
} lins_scan_result;

/* A batch of independent units: scan i = (new scan's query features, last scan's target features, prior).
   Clouds are concatenated; *_off has n_scans+1 entries (CSR style). */
typedef struct lins_batch_desc {
  int32_t n_scans;
  const lins_point* surf_flat;         const int32_t* surf_flat_off;         /* queries: surfPointsFlat_ */
  const lins_point* corner_sharp;      const int32_t* corner_sharp_off;      /* queries: cornerPointsSharp_ */
  const lins_point* surf_less_flat;    const int32_t* surf_less_flat_off;    /* targets: last surfPointsLessFlat_ */
  const lins_point* corner_less_sharp; const int32_t* corner_less_sharp_off; /* targets: last cornerPointsLessSharp_ */
  const double* state_in;              /* n_scans x 19 : filter_->state_ */
  const double* cov_in;                /* n_scans x 324: filter_->covariance_ */
  int32_t point_format;                /* LINS_POINTS_XYZI32 (0, default): the four clouds are pcl::PointXYZI records as typed
                                          above; LINS_POINTS_PACKED16: they are 16-byte (x, y, z, intensity) float records (cast
                                          the pointers) — what the device keeps anyway, so a caller that stores its clouds this
                                          way (and page-locks them) uploads with no host pass and half the PCIe bytes */
} lins_batch_desc;
#define LINS_POINTS_XYZI32 0
#define LINS_POINTS_PACKED16 1

typedef struct lins_ctx lins_ctx;

/* Create a context on CUDA device `device`. `stream` is a cudaStream_t passed as void* (NULL = the library
   creates its own non-blocking stream). Fails with LINS_E_NODEVICE when no CUDA device is usable: there is
   no CPU fallback. */
int lins_gpu_create(const lins_params* params, int device, void* stream, lins_ctx** out);
void lins_gpu_destroy(lins_ctx* ctx);
const char* lins_gpu_last_error(const lins_ctx* ctx);
int lins_gpu_set_params(lins_ctx* ctx, const lins_params* params);

/* ≙ kdtreeSurf_->setInputCloud(surfPointsLessFlat_), kdtreeCorner_->setInputCloud(cornerPointsLessSharp_).
   Uploads both target clouds and builds the device search index. */
int lins_gpu_set_map(lins_ctx* ctx, const lins_point* surf_less_flat, int n_surf,
                     const lins_point* corner_less_sharp, int n_corner);

/* ≙ performIESKF(): all iterations on device, no host round trip inside the loop.
   state_in/cov_in = filter_->state_/covariance_; state_out/cov_out = what filter_->update(...) would store
   when not diverged (linState_, Joseph-form Pk_). When rep->diverged is set, state_out = the prior
   (filterState) and cov_out = cov_in: the caller then runs lins_gpu_estimate_transform (the reference's
   "======Using ICP Method======" branch, StateEstimator.hpp:585-592). */
int lins_gpu_ieskf(lins_ctx* ctx, const lins_point* surf_flat, int n_surf, const lins_point* corner_sharp,
                   int n_corner, const double* state_in, const double* cov_in, double* state_out,
                   double* cov_out, lins_report* rep);

/* ≙ one call each of findCorrespondingSurfFeatures / findCorrespondingCornerFeatures at iteration `iter`
   with linState_ = lin_state (only rn/qbn are read). Dense (uncompacted) per-query outputs; any output
   pointer may be NULL. ind: -1 = none. mask = the accept test (s > 0.1 && res != 0). coeff = (s*jac, s*res).
   sel = pointSel (the de-skewed query, f32). Indices persist inside the ctx between calls like
   pointSearchSurfInd1/2/3 do, so iter % icp_freq != 0 reuses them. */
/* The correspondence IDs of the last lins_gpu_ieskf / lins_gpu_associate / lins_gpu_estimate_transform call's last search
   iteration (3 per surf query, 2 per corner query, -1 = none; either pointer may be NULL). */
int lins_gpu_download_indices(lins_ctx* ctx, int32_t* surf_ind, int32_t* corner_ind);

int lins_gpu_associate(lins_ctx* ctx, const lins_point* surf_flat, int n_surf, const lins_point* corner_sharp,
                       int n_corner, const double* lin_state, int iter, int32_t* surf_ind /*3*n_surf*/,
                       int32_t* corner_ind /*2*n_corner*/, float* surf_coeff /*4*n_surf*/,
                       float* corner_coeff /*4*n_corner*/, uint8_t* surf_mask, uint8_t* corner_mask,
                       float* surf_sel /*3*n_surf*/, float* corner_sel /*3*n_corner*/);

/* ≙ estimateTransform(scan_last_, scan_new_, t, q): 6-DoF Gauss-Newton ICP on the same association.
   pose_io = t (3) + q (x,y,z,w). iters_out/converged_out may be NULL. */
int lins_gpu_estimate_transform(lins_ctx* ctx, const lins_point* surf_flat, int n_surf,
                                const lins_point* corner_sharp, int n_corner, double* pose_io,
                                int* iters_out, int* converged_out);

/* ≙ updatePointCloud(): transformToEnd of the new scan's less-* clouds with linState_ = lin_state, written
   back in place to the host arrays (the reference overwrites scan_new_->*_ in place), and — iff
   n_corner >= 5 && n_surf >= 20 (StateEstimator.hpp:1156-1157) — installed as the new device map.
   Returns 1 in *map_replaced when the index was rebuilt. */
int lins_gpu_update_map(lins_ctx* ctx, lins_point* surf_less_flat, int n_surf, lins_point* corner_less_sharp,
                        int n_corner, const double* lin_state, int* map_replaced);

/* The same with the device-resident options: lin_state == NULL uses the posterior the last lins_gpu_ieskf left on the
   device; surf_out / corner_out receive the transformed clouds (may alias the inputs; NULL = keep them on the device only:
   no D2H, no stream synchronisation — the call returns with the refresh queued).  *map_replaced as above. */
int lins_gpu_update_map_ex(lins_ctx* ctx, const lins_point* surf_less_flat, int n_surf, const lins_point* corner_less_sharp,
                           int n_corner, const double* lin_state, lins_point* surf_out, lins_point* corner_out,
                           int* map_replaced);

/* Batched mode. upload: pack + H2D, resident afterwards. run: launch the fused kernel over the resident
   batch on the ctx stream (asynchronous). download: D2H of results + stream sync; any pointer may be NULL. */
int lins_gpu_batch_upload(lins_ctx* ctx, const lins_batch_desc* batch);
int lins_gpu_batch_run(lins_ctx* ctx);
/* cumulative number of points lins_gpu_batch_upload moved as host-packed 16-B records / as raw 32-B records (caller-pinned
   clouds are split between the pack threads and the copy engine at run time): what the PCIe byte count of a job is made of. */
int lins_gpu_batch_upload_stats(lins_ctx* ctx, int64_t* packed_points, int64_t* raw_points);
int lins_gpu_batch_download(lins_ctx* ctx, double* state_out /*n x 19*/, double* cov_out /*n x 324*/,
                            lins_scan_result* results /*n*/, lins_report* reports /*n, optional*/);
/* The correspondence IDs the resident batch holds after a run — pointSearchSurfInd1/2/3 and pointSearchCornerInd1/2
   (StateEstimator.hpp:1459-1465) of every unit's LAST search iteration, concatenated in batch order (3 per surf query,
   2 per corner query, -1 = none).  Parity hook for the batched mode; either pointer may be NULL. */
int lins_gpu_batch_download_indices(lins_ctx* ctx, int32_t* surf_ind, int32_t* corner_ind);
/* upload + run + download in one call (the end-to-end entry point). */
int lins_gpu_ieskf_batch(lins_ctx* ctx, const lins_batch_desc* batch, double* state_out, double* cov_out,
                         lins_scan_result* results);
/* device pointer of the resident lins_scan_result array (n_scans x 64 B) for a zero-copy pose gather. */
int lins_gpu_batch_results_device(lins_ctx* ctx, void** dev_ptr, int* n_scans);

/* Optional: page-lock (pin) a host buffer the caller owns — a thin wrapper over cudaHostRegister so that a caller without
   a CUDA binding of its own (the reference is plain C++ / ROS / PCL) can pin the storage of its point clouds once.
   lins_gpu_batch_upload detects pinned clouds and then DMAs the raw 32-B records straight from the caller's memory and
   packs them on the device: no host pass over the points (pageable clouds are packed by host threads into internal
   pinned staging first).  Unregister before freeing the buffer. */
int lins_gpu_host_register(void* ptr, size_t bytes);
int lins_gpu_host_unregister(void* ptr);

/* ---- sequence mode: S running sequences advanced one scan per step, all on the device -------------------------------
   Per present sequence one step runs what StateEstimator does between two scans once it is RUNNING
   (lins/src/lib/Estimator.cpp:228-252 -> StateEstimator.hpp:242-270, :435-463): the processImu calls
   (StatePredictor::predict, KalmanFilter.hpp:125-186), the processScan gate (:436-440), performIESKF (:465-600) with the
   estimateTransform fallback (:585-592, :1163-1196), filter_->update (KalmanFilter.hpp:195-200), integrateTransformation
   (:608-617), reset(1) (KalmanFilter.hpp:320-353), calculateRPfromGravity + correctRollPitch (:602-605, :427-431) and
   updatePointCloud (:1116-1161).  A run starts in one of two ways: lins_gpu_seq_begin takes S sequences the caller has
   initialised itself (each right after processSecondScan), or lins_gpu_seq_open opens S empty slots that start from their
   first scan: the step then also runs the status machine of processPCL (:294-307) — processFirstScan (:331-375), the IMU
   pre-integration and processSecondScan (:379-425) with its estimateTransform — and lins_gpu_seq_restart hands a slot to
   a new recording. */

/* the filter constants the device chain needs (exp_port.yaml:29-62) */
typedef struct lins_seq_params {
  double noise[4];         /* StatePredictor::noise_[0..3] (KalmanFilter.hpp:300-311), as kalman_filter.hpp setNoise() computes them */
  double init_pos_std[3];  /* INIT_POS_STD, m: reset(1) installs their squares (KalmanFilter.hpp:330) */
  double init_att_std[3];  /* INIT_ATT_STD, degrees (KalmanFilter.hpp:323-325) */
} lins_seq_params;

/* hand-over of S running sequences, each right after its processSecondScan (StateEstimator.hpp:379-425) */
typedef struct lins_seq_begin_desc {
  int32_t n_seq;
  const double* filter_state;  /* S x 19 : filter_->state_ */
  const double* filter_cov;    /* S x 324: filter_->covariance_ */
  const double* global_state;  /* S x 19 : globalState_ */
  const double* imu_last;      /* S x 6  : acc_last (3), gyr_last (3) of the StatePredictor */
  const lins_point* surf_map;   const int32_t* surf_map_off;    /* scan_last_->surfPointsLessFlat_ (already at scan end) */
  const lins_point* corner_map; const int32_t* corner_map_off;  /* scan_last_->cornerPointsLessSharp_ */
  int32_t point_format;        /* LINS_POINTS_XYZI32 or LINS_POINTS_PACKED16, as in lins_batch_desc */
} lins_seq_begin_desc;

/* one scan per sequence; CSR like lins_batch_desc (every *_off has n_seq + 1 entries) */
typedef struct lins_seq_step_desc {
  int32_t n_seq;                 /* == the begin call's */
  const uint8_t* present;        /* NULL = all; 0 = this sequence has no scan this step: its state is left untouched */
  const double* imu; const int32_t* imu_off;  /* k x 7 (dt, acc[3], gyr[3]): the processImu calls before the scan */
  const lins_point* surf_flat;  const int32_t* surf_flat_off;         /* queries: surfPointsFlat_ */
  const lins_point* corner_sharp; const int32_t* corner_sharp_off;    /* queries: cornerPointsSharp_ */
  const lins_point* surf_less_flat; const int32_t* surf_less_flat_off;        /* the new scan's, as extracted */
  const lins_point* corner_less_sharp; const int32_t* corner_less_sharp_off;
  int32_t point_format;
} lins_seq_step_desc;

#define LINS_SEQ_IDLE 0      /* not present this step */
#define LINS_SEQ_SKIPPED 1   /* failed the processScan gate (cornerLessSharp <= 5 || surfLessFlat <= 10): predicted state, old map */
#define LINS_SEQ_RAN 2       /* processScan ran */
#define LINS_SEQ_ICP 3       /* processScan ran and the IESKF diverged: the pose is estimateTransform's */
#define LINS_SEQ_INIT_WAIT 4 /* an initialising slot's scan failed the first / second scan gate (cornerLessSharp < 10 ||
                                surfLessFlat < 100): the slot is (back) in STATUS_INIT */
#define LINS_SEQ_FIRST 5     /* processFirstScan accepted the scan: the slot is in STATUS_FIRST_SCAN */
#define LINS_SEQ_SECOND 6    /* processSecondScan ran (with its estimateTransform): the slot is RUNNING */

/* the filter constants sequence initialisation reads (initializeCovariance, KalmanFilter.hpp:247-312; estimateInitialState,
   StateEstimator.hpp:1408-1419); INIT_POS_STD / INIT_ATT_STD are lins_seq_params' */
typedef struct lins_seq_init_params {
  double init_vel_std[3];  /* INIT_VEL_STD, m/s */
  double init_acc_std[3];  /* INIT_ACC_STD */
  double init_gyr_std[3];  /* INIT_GYR_STD */
  double init_ba[3];       /* INIT_BA: the accelerometer bias of the hand-over and the pre-integration's linearisation point */
  double init_bw[3];       /* INIT_BW: the same for the gyroscope */
} lins_seq_init_params;

/* Uploads the hand-over; replaces any running sequences of this ctx (single-scan and batched state are untouched). */
int lins_gpu_seq_begin(lins_ctx* ctx, const lins_seq_params* params, const lins_seq_begin_desc* desc);
/* Opens a run of n_seq empty slots, each what a newly constructed StateEstimator holds: STATUS_INIT, globalState_ and the
   filter state identity (gn = (0, 0, -9.81)), the covariance of initializeCovariance, no map.  Replaces any running
   sequences of this ctx, like lins_gpu_seq_begin.  LINS_E_INVALID for n_seq < 1 or a NULL argument. */
int lins_gpu_seq_open(lins_ctx* ctx, const lins_seq_params* params, const lins_seq_init_params* init, int32_t n_seq);
/* Puts every slot with mask[s] != 0 back into the fresh state of lins_gpu_seq_open (its last scan_status reads
   LINS_SEQ_IDLE); the other slots are untouched.  LINS_E_INVALID for a NULL mask or a run started by lins_gpu_seq_begin
   (it has no init params); LINS_E_NOMAP without a run. */
int lins_gpu_seq_restart(lins_ctx* ctx, const uint8_t* mask /*S*/);
/* Advances every present sequence by one scan.  Returns LINS_E_NOMAP before lins_gpu_seq_begin / lins_gpu_seq_open.  One
   stream synchronisation (the divergence check) per call; the rest is queued.  LINS_E_INVALID for a bad descriptor leaves
   the sequences as they were; any other error ends the run (the sequences are dropped, the next step returns LINS_E_NOMAP
   until a new lins_gpu_seq_begin / lins_gpu_seq_open), because the step may have advanced some of its phases already.
   A present slot runs what processImu + processPCL do in its status: in STATUS_INIT its IMU rows are ignored and the scan
   goes through processFirstScan; in STATUS_FIRST_SCAN its IMU rows are pre-integrated (IntegrationBase::propagate) and the
   scan goes through processSecondScan; RUNNING is as above. */
int lins_gpu_seq_step(lins_ctx* ctx, const lins_seq_step_desc* step);
/* The same with the IMU sample processPCL receives with each scan (acc (3), gyr (3); Estimator.cpp:238-243): S x 6, read
   for the present slots in STATUS_INIT or STATUS_FIRST_SCAN.  scan_imu may be NULL only when no present slot is
   initialising (else LINS_E_INVALID, before anything changes).  lins_gpu_seq_step(ctx, d) = lins_gpu_seq_step_ex(ctx, d, NULL). */
int lins_gpu_seq_step_ex(lins_ctx* ctx, const lins_seq_step_desc* step, const double* scan_imu /*S x 6 or NULL*/);
/* Sequence initialisation read-back (any pointer may be NULL): fusion_status[s] = the slot's StateEstimator::status_
   (0 STATUS_INIT, 1 STATUS_FIRST_SCAN, 3 STATUS_RUNNING); where the last step's scan_status is LINS_SEQ_SECOND, icp_pose
   (t (3) + q (x,y,z,w)), icp_iters and icp_converged are that scan's estimateTransform result, elsewhere zero. */
int lins_gpu_seq_download_init(lins_ctx* ctx, int32_t* fusion_status /*S*/, double* icp_pose /*S x 7*/, int32_t* icp_iters /*S*/,
                               int32_t* icp_converged /*S*/);
/* The sequences' state after the last step; any pointer may be NULL.  results / reports: the last step's performIESKF,
   valid where scan_status is LINS_SEQ_RAN or LINS_SEQ_ICP and unspecified elsewhere (zero before the first step);
   scan_status: LINS_SEQ_* of the last step. */
int lins_gpu_seq_download(lins_ctx* ctx, double* global_state /*S x 19*/, double* filter_state /*S x 19*/,
                          double* filter_cov /*S x 324*/, lins_scan_result* results /*S*/, lins_report* reports /*S*/,
                          int32_t* scan_status /*S*/);
/* CUDA-event times of the last lins_gpu_seq_step's phases, ms: ms[0] IMU propagation, ms[1] query compaction + IESKF,
   ms[2] divergence check (D2H + synchronisation) + estimateTransform fallbacks + the second scans' estimateTransform
   (one batched loop), ms[3] post kernel + sequence initialisation + map refresh. */
int lins_gpu_seq_phase_ms(lins_ctx* ctx, float* ms /*4*/);
/* Parity hooks of sequence mode (any pointer may be NULL).  download_ieskf: the last step's IESKF prior (the filter state
   and covariance after the IMU propagation, every sequence), its output (state_out / cov_out as lins_gpu_ieskf returns
   them; valid where scan_status >= LINS_SEQ_RAN), and the correspondence IDs of its last search iteration
   (pointSearchSurfInd1/2/3, pointSearchCornerInd1/2) for the sequences that ran, in sequence order: query_off holds the
   2 x (S + 1) offsets of their surf / corner queries into surf_ind (3 per query) and corner_ind (2 per query).
   download_maps: the maps the next step searches, as (x, y, z, intensity) float records, CSR with off = 4 x (S + 1)
   (surf map, corner map, surf 1-NN cloud, corner 1-NN cloud), and stale[s] = 1 where the sequence's 1-NN cloud is not its
   map (the last refresh failed the >= 5 && >= 20 guard; its 1-NN cloud is the tree range, else that range is empty). */
int lins_gpu_seq_download_ieskf(lins_ctx* ctx, double* prior_state /*S x 19*/, double* prior_cov /*S x 324*/,
                                double* state_out /*S x 19*/, double* cov_out /*S x 324*/, int32_t* query_off,
                                int32_t* surf_ind, int32_t* corner_ind);
int lins_gpu_seq_download_maps(lins_ctx* ctx, int32_t* off, float* surf_map, float* corner_map, float* surf_tree,
                               float* corner_tree, uint8_t* stale /*S*/);

/* ---- feature extraction: StateEstimator.hpp:619-827 (undistortPcl, calculateSmoothness, markOccludedPoints,
   extractFeatures with the per-ring pcl::VoxelGrid, leaf 0.2 m) on the device, from what processPCL receives: the
   segmented cloud and cloud_info of image projection (cloud_msgs/msg/cloud_info.msg).  Bit-identical to the host
   restatement csrc/host/feature_extraction.hpp except where equal curvatures decide a pick: the reference's std::sort
   leaves their order unspecified; the device keeps them in array order (DESIGN.md §4.6). */

/* n segmented scans, CSR: scan i's points are cloud[cloud_off[i] .. cloud_off[i + 1]) and its per-point cloud_info
   arrays share those offsets */
typedef struct lins_pcl_desc {
  int32_t n_scans;
  int32_t line_num;                    /* LINE_NUM, 1..128: the entries of start/end_ring_index per scan */
  const lins_point* cloud; const int32_t* cloud_off;  /* segmentedCloud; n_scans + 1 offsets */
  const uint8_t* ground_flag;          /* segmentedCloudGroundFlag */
  const uint32_t* col_ind;             /* segmentedCloudColInd */
  const float* range;                  /* segmentedCloudRange */
  const int32_t* start_ring_index;     /* n_scans x line_num: startRingIndex */
  const int32_t* end_ring_index;       /* n_scans x line_num: endRingIndex */
  const float* orientation;            /* n_scans x 3: startOrientation, endOrientation, orientationDiff */
  int32_t point_format;                /* LINS_POINTS_XYZI32 or LINS_POINTS_PACKED16, as in lins_batch_desc */
} lins_pcl_desc;

/* the extraction's constants (exp_port.yaml:7, :12-13; shipped 0.5 / 0.5 / 0); SCAN_PERIOD is lins_params.scan_period */
typedef struct lins_feature_params {
  double edge_threshold;
  double surf_threshold;
  double imu_lidar_extrinsic_angle;    /* degrees */
} lins_feature_params;

/* the largest ring span (endRingIndex - startRingIndex) of a ring with a visited sextant that the on-chip sorts take;
   a scan with a longer ring returns LINS_E_TOOBIG (VLP-16 rings hold at most 1800 points, 64 x 1024 rings 1024) */
#define LINS_FEAT_RING_CAP 2048

/* ≙ the four extraction stages of processPCL (StateEstimator.hpp:619-827) for every scan of d.  Scan i's clouds are
   written at its own input offsets (none is larger than the input): surf_flat (surfPointsFlat), corner_sharp
   (cornerPointsSharp), surf_less_flat (surfPointsLessFlat), corner_less_sharp (cornerPointsLessSharp) and, unless
   undist is NULL, the de-skewed cloud (intensity = ring + SCAN_PERIOD * relTime), all in d->point_format (XYZI32
   records carry pad0 = 1 and zero pads).  counts: n_scans x 4 in that order.  LINS_E_INVALID, before anything is
   written, for bad offsets, a NULL array, line_num outside 1..128, a non-finite point, range or orientation, or a
   visited sextant (sp < ep) outside the scan's [0, n), or rings whose visited ranges overlap or come out of order (LeGO-LOAM's
   rings are 10 points apart; abutting rings are fine); LINS_E_TOOBIG for a ring span above LINS_FEAT_RING_CAP. */
int lins_gpu_extract_features(lins_ctx* ctx, const lins_feature_params* fp, const lins_pcl_desc* d, lins_point* surf_flat,
                              lins_point* corner_sharp, lins_point* surf_less_flat, lins_point* corner_less_sharp,
                              lins_point* undist, int32_t* counts /*n_scans x 4*/);
/* CUDA-event time of the last extraction kernel (lins_gpu_extract_features, lins_gpu_seq_step_pcl or
   lins_gpu_seq_step_raw), ms */
int lins_gpu_extract_ms(lins_ctx* ctx, float* ms);

/* one processPCL-shaped scan per sequence: the IMU rows as in lins_seq_step_desc, the scans as a lins_pcl_desc with
   n_scans == n_seq (a slot that is not present should have an empty scan; its features are not used) */
typedef struct lins_seq_pcl_desc {
  int32_t n_seq;
  const uint8_t* present;              /* NULL = all */
  const double* imu; const int32_t* imu_off;
  lins_pcl_desc pcl;
} lins_seq_pcl_desc;

/* ≙ processPCL (StateEstimator.hpp:279-307) with its feature extraction (:619-827) on the device: extracts every
   slot's scan, reads the counts back (one D2H + synchronisation: the gates and the map plan are made from sizes), packs
   the features into the step's buffers and runs lins_gpu_seq_step_ex.  Bit-identical to lins_gpu_extract_features
   followed by lins_gpu_seq_step_ex with those clouds; may alternate with lins_gpu_seq_step_ex in one run.  Invalid
   input (as lins_gpu_extract_features, or as lins_gpu_seq_step_ex) returns before the sequences change. */
int lins_gpu_seq_step_pcl(lins_ctx* ctx, const lins_seq_pcl_desc* step, const lins_feature_params* fp,
                          const double* scan_imu /*S x 6 or NULL*/);

/* ---- image projection: lins/src/image_projection_node.cpp:191-415 (findStartEndAngle, projectPointCloud,
   groundRemoval, cloudSegmentation with labelComponents) on the device, from the raw sweep the LiDAR driver publishes to
   the segmented cloud, cloud_info and outlier cloud (cloudHandler :177-189 without ROS).  Bit-identical to a fresh host
   restatement csrc/host/image_projection.hpp per scan (DESIGN.md §4.7). */

/* the lidar geometry image projection reads; the reference hard-wires VLP-16 (parameters.h:82-92: N_SCAN 16, Horizon_SCAN
   1800, ang_res_x 0.2, ang_res_y 2.0, ang_bottom 15.1, groundScanInd 5) */
typedef struct lins_lidar_model {
  int32_t line_num;         /* N_SCAN: rows of the range image, 1..128 */
  int32_t scan_num;         /* Horizon_SCAN: columns, 2..LINS_FEAT_RING_CAP */
  float ang_res_x;          /* degrees per column, finite and > 0 */
  float ang_res_y;          /* degrees per row, finite and > 0 */
  float ang_bottom;         /* degrees, finite */
  int32_t ground_scan_ind;  /* groundScanInd: 0..line_num - 1 */
} lins_lidar_model;

/* n raw sweeps, CSR: sweep i's points (firing order; NaN no-returns allowed) are cloud[cloud_off[i] .. cloud_off[i + 1]).
   The points' own intensity is not read. */
typedef struct lins_raw_desc {
  int32_t n_scans;
  const lins_point* cloud; const int32_t* cloud_off;  /* n_scans + 1 offsets */
  int32_t point_format;                /* LINS_POINTS_XYZI32 or LINS_POINTS_PACKED16, as in lins_batch_desc */
} lins_raw_desc;

/* ≙ cloudHandler (image_projection_node.cpp:177-189) for every sweep of d, each on a fresh ImageProjection.  Sweep i's
   segmented cloud (seg) with its per-point cloud_info (ground_flag, col_ind, range) and its outlier cloud are written at
   its own input offsets (each pixel holds at most one point, so neither is longer than the sweep), in d->point_format
   (XYZI32 records carry pad0 = 1 and zero pads): the layout lins_pcl_desc takes.  start_ring / end_ring: n x line_num;
   ori: n x 3 (startOrientation, endOrientation, orientationDiff; NaN where the first or last point is NaN, and (0, 0, 0)
   for a sweep of fewer than 2 points, as a fresh ImageProjection holds — the host object keeps its previous scan's);
   counts: n x 2 (segmented, outlier).  LINS_E_INVALID, before anything is written, for bad offsets, a NULL array, or a
   model outside the limits of lins_lidar_model. */
int lins_gpu_project_scans(lins_ctx* ctx, const lins_lidar_model* model, const lins_raw_desc* raw, lins_point* seg,
                           uint8_t* ground_flag, uint32_t* col_ind, float* range, lins_point* outlier, int32_t* start_ring,
                           int32_t* end_ring, float* ori /*n x 3*/, int32_t* counts /*n x 2*/);
/* CUDA-event time of the last projection kernel (lins_gpu_project_scans or lins_gpu_seq_step_raw), ms */
int lins_gpu_project_ms(lins_ctx* ctx, float* ms);

/* one raw sweep per sequence: the IMU rows as in lins_seq_step_desc, the sweeps as a lins_raw_desc with n_scans == n_seq
   (a slot that is not present is neither projected nor extracted; its sweep may be empty) */
typedef struct lins_seq_raw_desc {
  int32_t n_seq;
  const uint8_t* present;              /* NULL = all */
  const double* imu; const int32_t* imu_off;
  lins_raw_desc raw;
} lins_seq_raw_desc;

/* ≙ cloudHandler (image_projection_node.cpp:177-189, including copyPointCloud's pcl::removeNaNFromPointCloud) followed
   by processPCL (StateEstimator.hpp:279-307, with the feature extraction of :619-827) for every present slot, all on the
   device: nothing goes from device to host but the feature counts (one D2H + synchronisation).  Bit-identical to: drop
   every point whose x, y or z is not finite (keeping the firing order), lins_gpu_project_scans, compact each segmented
   cloud to dense CSR, lins_gpu_seq_step_pcl.  Unlike PCL, which skips the removal when the message claims is_dense, the
   device always drops non-finite points (for an honest dense cloud the two agree).  All slots share one lidar model; a
   run that mixes sensors gives each slot its own with lins_gpu_seq_step_raw_mixed.  May alternate with
   lins_gpu_seq_step_ex and lins_gpu_seq_step_pcl in one run.  LINS_E_INVALID before anything changes for a bad
   descriptor, model (as lins_gpu_project_scans), offsets, point format, NULL array or fp, or a NULL scan_imu while a
   present slot is initialising; a segmented scan the extraction rejects (as lins_gpu_extract_features:
   LINS_E_INVALID / LINS_E_TOOBIG) returns before the sequences change; any later failure ends the run.  Afterwards
   lins_gpu_project_ms and lins_gpu_extract_ms report the step's two kernels. */
int lins_gpu_seq_step_raw(lins_ctx* ctx, const lins_seq_raw_desc* step, const lins_lidar_model* model,
                          const lins_feature_params* fp, const double* scan_imu /*S x 6 or NULL*/);

/* ---- sensor_msgs/PointCloud2 on the device: pcl::fromROSMsg<pcl::PointXYZI> of copyPointCloud
   (image_projection_node.cpp:172-177), from the message's bytes as the driver publishes them (a ROS callback's
   msg->data, or a message's data field inside a bag chunk).  Bit-identical to the host decoder
   csrc/host/rosbag_reader.hpp decode_pointcloud2 (DESIGN.md §4.8). */

/* what fromROSMsg<PointXYZI> reads of one message: its geometry and the x, y, z and intensity PointFields */
typedef struct lins_cloud2_layout {
  uint32_t height, width;       /* the message has width * height points, read row-major */
  uint32_t point_step, row_step;  /* bytes; point (r, c) starts at r * row_step + c * point_step */
  uint32_t offset[4];           /* x, y, z, intensity: byte offset inside a point */
  uint8_t datatype[4];          /* x, y, z, intensity: sensor_msgs/PointField datatype 1..8 (INT8 .. FLOAT64); intensity may
                                   be 0 = the message has no intensity field (it then reads as 0).  A field named intensity
                                   whose own datatype is 0 makes the message malformed (decode_pointcloud2 rejects it):
                                   give it a datatype outside 0..8 so that the call rejects it too (INTEGRATION.md) */
  uint8_t is_bigendian;         /* must be 0 */
  uint8_t pad_[3];
} lins_cloud2_layout;           /* 40 bytes */

/* n messages: message i's data field is data[data_off[i] .. data_off[i + 1]) (data_off non-decreasing, data_off[0] may be
   > 0), its layout layouts[i].  The blob may start at any address and the fields at any offset: nothing is assumed aligned. */
typedef struct lins_cloud2_desc {
  int32_t n_scans;
  const uint8_t* data;
  const int64_t* data_off;                /* n_scans + 1 */
  const lins_cloud2_layout* layouts;      /* n_scans */
} lins_cloud2_desc;

/* ≙ pcl::fromROSMsg<pcl::PointXYZI> of every message of d (as decode_pointcloud2 reads it: each field through
   read_scalar, then (float); a field the layout does not name is not read).  Message i's width * height records are
   written in row-major order at out + the prefix sum of the earlier messages' width * height, with pad0 = 1 and zero
   pads; counts[i] = width * height (counts may be NULL).  NaN no-returns are kept.  LINS_E_INVALID, before anything is
   uploaded or written, for a NULL array, bad data_off, a total above INT32_MAX points, or a message decode_pointcloud2
   rejects: big-endian, a datatype outside 1..8 (0 allowed for intensity only), a field with offset + size > point_step,
   or a point past its message's data ((h - 1) * row_step + (w - 1) * point_step + point_step > length, in 64-bit
   arithmetic).  The blob is uploaded as lins_gpu_batch_upload uploads clouds: through pinned staging, or in one DMA
   when the caller registered it with lins_gpu_host_register. */
int lins_gpu_decode_cloud2(lins_ctx* ctx, const lins_cloud2_desc* d, lins_point* out, int32_t* counts /*n or NULL*/);
/* CUDA-event time of the last decode kernel (lins_gpu_decode_cloud2 or lins_gpu_seq_step_cloud2), ms */
int lins_gpu_decode_ms(lins_ctx* ctx, float* ms);

/* one sensor_msgs/PointCloud2 message per sequence: the IMU rows as in lins_seq_step_desc, the messages as a
   lins_cloud2_desc with n_scans == n_seq (a slot that is not present is not decoded; its message may be empty) */
typedef struct lins_seq_cloud2_desc {
  int32_t n_seq;
  const uint8_t* present;              /* NULL = all */
  const double* imu; const int32_t* imu_off;
  lins_cloud2_desc cloud2;
} lins_seq_cloud2_desc;

/* ≙ cloudHandler from the PointCloud2 message (fromROSMsg, removeNaNFromPointCloud, image projection) followed by
   processPCL for every present slot, all on the device: lins_gpu_seq_step_raw with the decode in front.  Bit-identical to
   lins_gpu_decode_cloud2 (or the host decode_pointcloud2) followed by lins_gpu_seq_step_raw on the decoded sweeps; may
   alternate with lins_gpu_seq_step_ex / _pcl / _raw in one run.  LINS_E_INVALID before anything changes for a descriptor
   lins_gpu_decode_cloud2 rejects, and otherwise as lins_gpu_seq_step_raw.  Afterwards lins_gpu_decode_ms,
   lins_gpu_project_ms and lins_gpu_extract_ms report the step's three front-end kernels. */
int lins_gpu_seq_step_cloud2(lins_ctx* ctx, const lins_seq_cloud2_desc* step, const lins_lidar_model* model,
                             const lins_feature_params* fp, const double* scan_imu /*S x 6 or NULL*/);

/* ---- mixed sensors: one lidar model per scan, so sweeps of different sensors (a VLP-16 next to a 64-ring lidar) are
   projected in one call and their sequences run in one context (DESIGN.md §4.7). */

/* a table of lidar models and each scan's entry in it */
typedef struct lins_lidar_models {
  int32_t n_models;                /* >= 1 */
  const lins_lidar_model* models;  /* n_models, each within the limits of lins_lidar_model */
  const int32_t* model_of;         /* one entry per scan (absent slots included) in 0..n_models-1; NULL only if
                                      n_models == 1 (every scan uses models[0]) */
} lins_lidar_models;

/* lins_gpu_project_scans with scan i projected by models->models[model_of[i]]: per scan bit-identical to
   lins_gpu_project_scans with that model.  start_ring / end_ring are n x L_max, L_max the table's largest line_num: scan
   i's first line_num entries are its ring indices, the rest 0 (the padded layout lins_gpu_extract_features takes with
   line_num = L_max).  LINS_E_INVALID, before anything is uploaded or written, as lins_gpu_project_scans and for a NULL
   table or models, n_models < 1, a listed model outside its limits, a NULL model_of with n_models > 1, or a model_of
   entry outside 0..n_models-1. */
int lins_gpu_project_scans_mixed(lins_ctx* ctx, const lins_lidar_models* models, const lins_raw_desc* raw, lins_point* seg,
                                 uint8_t* ground_flag, uint32_t* col_ind, float* range, lins_point* outlier,
                                 int32_t* start_ring /*n x L_max*/, int32_t* end_ring /*n x L_max*/, float* ori /*n x 3*/,
                                 int32_t* counts /*n x 2*/);
/* lins_gpu_seq_step_raw / lins_gpu_seq_step_cloud2 with slot s's sweep projected by models->models[model_of[s]]: each
   slot bit-identical to the same slot stepped through the single-model entry with that model.  Each may alternate with
   every other step entry in one run, and a slot may change sensor when lins_gpu_seq_restart hands it a new recording.
   LINS_E_INVALID before anything changes for a table lins_gpu_project_scans_mixed rejects, and otherwise as the
   single-model entry. */
int lins_gpu_seq_step_raw_mixed(lins_ctx* ctx, const lins_seq_raw_desc* step, const lins_lidar_models* models,
                                const lins_feature_params* fp, const double* scan_imu /*S x 6 or NULL*/);
int lins_gpu_seq_step_cloud2_mixed(lins_ctx* ctx, const lins_seq_cloud2_desc* step, const lins_lidar_models* models,
                                   const lins_feature_params* fp, const double* scan_imu /*S x 6 or NULL*/);

/* Split "Jacobian kernel" (SURVEY.md §8(d) unit U1): de-skew, residual, robust weight and the factored Jacobian row
   g = [c ; p x (R^T c)], r = lidar_scale * coeff.w of every query of the resident batch, reduced per unit.  The
   linearisation point is each unit's posterior (what lins_gpu_batch_download returns as state_out, R its rotation) and the
   correspondences are the IDs of each unit's last search iteration (lins_gpu_batch_download_indices).  The rows are
   weighted iff the parameters' icp_freq == 1 (the weight of a search iteration >= 1).  Call it after lins_gpu_batch_run;
   lins_gpu_set_params in between changes the pass's scan_period, lidar_scale and weighting.
   accum_out (NULL = keep the sums on the device): n x 30 doubles, row i = unit i:
     0..20   the upper triangle of sum g g^T, row-major (g0 g0, g0 g1, .., g0 g5, g1 g1, .., g5 g5)
     21..26  sum g r
     27      sum r r
     28, 29  the accepted surf and corner rows (as doubles)
   Each sum is deterministic from run to run; it matches an exact sum of the same rows to a few f64 ulps of its
   condition scale (DESIGN.md §4.2). */
int lins_gpu_batch_jacobian_pass(lins_ctx* ctx, double* accum_out /*n x 30 or NULL*/);

/* ---- row F2 (SURVEY.md §8(f)): the mapping node's scan-to-map refinement -------------------------------------
   lins/src/lidar_mapping_node.cpp: scan2MapOptimization :1635-1652, cornerOptimization :1351-1461,
   surfOptimization :1463-1524, LMOptimization :1526-1633, pointAssociateToMap :594-608.
   All point clouds are in the mapping node's frame convention (the YZX clouds the estimator publishes);
   transform = transformTobeMapped = (rx, ry, rz, tx, ty, tz), f32 like the reference. */
#define LINS_MAP_MAX_ITER 10
typedef struct lins_map_report {
  int32_t iters;       /* LM iterations executed (<= 10) */
  int32_t converged;   /* deltaR < 0.05 deg && deltaT < 0.05 cm reached (:1628) */
  int32_t degenerate;  /* isDegenerate of iteration 0 (:1606-1617); 0 when that pass selects < 50 points and no LM step
                          runs.  matP / isDegenerate themselves persist across calls, like the reference's members */
  int32_t skipped;     /* map too small: cornerFromMapDSNum <= 10 || surfFromMapDSNum <= 100 (:1636) */
  int32_t n_sel[LINS_MAP_MAX_ITER];   /* laserCloudSelNum per iteration (< 50 => that LM step is skipped, :1535) */
  float delta_r[LINS_MAP_MAX_ITER];   /* deg */
  float delta_t[LINS_MAP_MAX_ITER];   /* cm */
} lins_map_report;

/* ≙ kdtreeCornerFromMap->setInputCloud(laserCloudCornerFromMapDS), kdtreeSurfFromMap->setInputCloud(...) (:1637-1638):
   uploads both map clouds and builds the device search structure. */
int lins_gpu_map_set(lins_ctx* ctx, const lins_point* corner_from_map, int n_corner, const lins_point* surf_from_map,
                     int n_surf);
/* ≙ the iteration loop of scan2MapOptimization (:1640-1648): up to 10 x (cornerOptimization, surfOptimization,
   LMOptimization) against the map set by lins_gpu_map_set; 5-NN search, line / plane fits, coefficients and the
   A^T A / A^T B reduction on the device, the 6x6 step on the host.  transform_io: transformTobeMapped in / out.
   (transformUpdate, :538-577, blends IMU roll / pitch afterwards and stays with the caller.) */
int lins_gpu_scan2map(lins_ctx* ctx, const lins_point* corner_last, int n_corner, const lins_point* surf_last, int n_surf,
                      float* transform_io /*6*/, lins_map_report* rep);
/* ≙ one cornerOptimization + surfOptimization pass at `transform`, dense per-point outputs (any pointer may be NULL):
   knn = pointSearchInd (5 per point, ascending distance, -1 = fewer than 5 map points), coeff = (s*la, s*lb, s*lc,
   s*ld2) resp. (s*pa, s*pb, s*pc, s*pd2), mask = the point was pushed to laserCloudOri (s > 0.1). */
int lins_gpu_map_associate(lins_ctx* ctx, const lins_point* corner_last, int n_corner, const lins_point* surf_last,
                           int n_surf, const float* transform /*6*/, int32_t* corner_knn /*5*n_corner*/,
                           int32_t* surf_knn /*5*n_surf*/, float* corner_coeff /*4*n_corner*/, float* surf_coeff /*4*n_surf*/,
                           uint8_t* corner_mask, uint8_t* surf_mask);

/* ---- the mapping node's cycle: lidar_mapping_node.cpp run() :1806-1855 behind one call per mapping cycle ------------
   One mapper per context (lins_gpu_mappers_* below run many in lockstep; the single mapper is their cycle for one slot).
   Per processed cycle: transformAssociateToMap (:411-536), extractSurroundingKeyFrames in the branch the reference
   compiles (loopClosureEnableFlag = true, parameters.h:80: the window of the 50 most recent key frames, :1204-1246),
   the local map's pcl::VoxelGrid (corner 0.2 m, surf + outlier 0.4 m, :1317-1323), downsampleCurrentScan (:1326-1349),
   scan2MapOptimization with its 10 / 100 gate and transformUpdate (:1635-1652, :538-577) and saveKeyFramesAndFactor
   (:1654-1765).  The clouds, the key-frame store, the VoxelGrids and the scan-to-map
   loop are on the device; transformAssociateToMap, transformUpdate, the key-frame test and the pose bookkeeping run on
   the host in the reference's f32 / f64 types.  Loop closure (loopClosureThread, performLoopClosure) is not performed:
   without a loop factor the iSAM2 estimate of a new key frame is the pose inserted for it up to f32 rounding (DESIGN.md §4.9), and
   correctPoses is a no-op.  The reference's constants are fixed: mappingProcessInterval 0.3 s, window 50, key-frame
   distance 0.3 m, loop search 5 m / 30 s; SCAN_PERIOD is the context's lins_params.scan_period.
   All clouds are in the mapping node's YZX frame convention, like lins_gpu_scan2map's.
   The mapper's state, its scan-to-map matP / isDegenerate included, is its own: lins_gpu_map_set, lins_gpu_scan2map,
   lins_gpu_voxel_grid and lins_gpu_mappers_* on the same context neither see nor change it, nor does it change theirs.
   The first lins_gpu_mapper_* call on a context sets it up.  One device-to-host synchronisation per processed cycle. */
#define LINS_MAPPER_WINDOW 50     /* surroundingKeyframeSearchNum (parameters.h) */
#define LINS_MAPPER_IMU_QUEUE 200 /* imuQueLength_ (:55) */
typedef struct lins_mapper_desc {
  double time;                    /* timeLaserOdometry: header stamp of the odometry and of the three clouds */
  double quat[4];                 /* odometry pose.orientation x, y, z, w; converted as laserOdometryHandler (:711-724) */
  double pos[3];                  /* odometry pose.position x, y, z */
  const lins_point* corner;       /* laserCloudCornerLast (the estimator's less-sharp corners) */
  const lins_point* surf;         /* laserCloudSurfLast (less-flat surfs) */
  const lins_point* outlier;      /* laserCloudOutlierLast */
  int32_t n_corner, n_surf, n_outlier, pad;
} lins_mapper_desc;
typedef struct lins_mapper_report {
  int32_t processed;              /* the cycle ran (timeLaserOdometry - timeLastProcessing >= 0.3, :1821) */
  int32_t skipped_interval;       /* the 0.3 s gate skipped it: nothing else changed */
  int32_t n_map_corner_ds, n_map_surf_ds;    /* laserCloudCornerFromMapDSNum / SurfFromMapDSNum (0 without key frames) */
  int32_t n_corner_ds, n_surf_ds, n_outlier_ds, n_surf_total_ds;  /* laserCloud{CornerLast,SurfLast,OutlierLast,SurfTotalLast}DSNum */
  int32_t keyframe_saved;         /* saveKeyFramesAndFactor stored a key frame */
  int32_t n_keyframes;            /* cloudKeyPoses3D->points.size() after the cycle */
  int32_t window_len;             /* recentCornerCloudKeyFrames.size() used by this cycle's local map */
  int32_t loop_candidate;         /* after a saved key frame: the key pose detectLoopClosure (:1043-1067) would pick (the
                                     nearest within 5 m whose time differs by > 30 s), else -1.  From such a cycle on the
                                     reference may close a loop this library does not */
  float transform_guess[6];       /* transformTobeMapped after transformAssociateToMap (the scan-to-map start) */
  float transform_aft_mapped[6];  /* transformAftMapped after the cycle */
  lins_map_report map;            /* the scan-to-map loop (map.skipped = 1: the 10 / 100 gate failed, :1636, and
                                     transformUpdate did not run) */
} lins_mapper_report;
/* forget every key frame, the IMU queue and the transforms: the state of a freshly constructed mapping node */
int lins_gpu_mapper_reset(lins_ctx* ctx);
/* ≙ imuHandler (:726-735) for n messages: time = header stamp, roll / pitch = what getRPY of the orientation gave
   (stored to f32 like imuRoll / imuPitch); the library keeps the 200-entry ring */
int lins_gpu_mapper_imu(lins_ctx* ctx, const double* time, const double* roll, const double* pitch, int n);
/* ≙ laserOdometryHandler (:711-724) + the cloud handlers + one pass of run() (:1806-1855).  LINS_E_TOOBIG when a
   VoxelGrid's div_x * div_y * div_z exceeds INT32_MAX (the leaf is too small for the cloud's extent); the mapper's state
   (transforms, key frames, window, IMU queue) is then unchanged, and lins_gpu_mapper_download returns no clouds until
   the next cycle completes.  rep may be NULL. */
int lins_gpu_mapper_step(lins_ctx* ctx, const lins_mapper_desc* desc, lins_mapper_report* rep);
/* the key poses (cloudKeyPoses6D: n_keyframes x 7 doubles x, y, z, roll, pitch, yaw, time; the first six are the f32
   PointTypePose fields), the window (window_len key-frame ids, oldest first, as used by the last processed cycle) and that
   cycle's clouds (x, y, z, intensity float records; sizes in its report): the local map after down-sampling, and the
   scan's corner, surf, outlier and surf-total DS clouds.  NULL skips. */
int lins_gpu_mapper_download(lins_ctx* ctx, double* key_poses, int32_t* window, float* map_corner_ds, float* map_surf_ds,
                             float* corner_ds, float* surf_ds, float* outlier_ds, float* surf_total_ds);
/* pcl::VoxelGrid<PointXYZI> on one cloud of n points (leaf > 0): the filter the mapper runs, as a call of its own.  out
   has room for n records (x, y, z, intensity floats); *n_out receives the voxel count.  LINS_E_TOOBIG as above. */
int lins_gpu_voxel_grid(lins_ctx* ctx, const lins_point* in, int n, float leaf, float* out, int* n_out);

/* ---- the mapping node's cycle for many drives in lockstep ----------------------------------------------------------
   M mapper slots on one context, each a mapping node of its own (one drive's), stepped together: one call runs the
   lins_gpu_mapper_step cycle of every present slot with one device-to-host synchronisation, whatever M is.  Per present
   slot, the report, the key poses, the window and the six clouds are bit-identical to lins_gpu_mapper_step /
   lins_gpu_mapper_download on a context of its own given the same event sequence (the interval gate, the 10 / 100 gate
   with its stale transformAftMapped, and the duplicated key frame when the window first fills included).  The slots'
   state is a member of the context of its own: lins_gpu_mapper_*, lins_gpu_map_set, lins_gpu_scan2map and
   lins_gpu_voxel_grid on the same context neither see nor change it.  Loop closure is not performed, as in the single
   mapper.  A call before lins_gpu_mappers_open returns LINS_E_NOMAP. */
/* opens M mapper slots, each a freshly constructed mapping node (as after lins_gpu_mapper_reset); replaces any open run */
int lins_gpu_mappers_open(lins_ctx* ctx, int32_t n_slots);
/* slots with mask[s] != 0 back to the fresh state (hand a slot to a new drive); others untouched */
int lins_gpu_mappers_reset(lins_ctx* ctx, const uint8_t* mask /*M*/);
/* imuHandler for every slot: slot s's rows are [off[s], off[s+1]) of time / roll / pitch (as lins_gpu_mapper_imu) */
int lins_gpu_mappers_imu(lins_ctx* ctx, const int32_t* off /*M+1*/, const double* time, const double* roll, const double* pitch);
typedef struct lins_mappers_desc {
  int32_t n_slots;                       /* == M */
  int32_t pad;
  const uint8_t* present;                /* M flags; NULL = all.  An absent slot is neither read nor changed */
  const double* time;                    /* M: timeLaserOdometry */
  const double* quat;                    /* M x 4 (x, y, z, w) */
  const double* pos;                     /* M x 3 */
  const lins_point* corner;  const int32_t* corner_off;   /* M + 1, CSR as lins_batch_desc: slot s's cloud is */
  const lins_point* surf;    const int32_t* surf_off;     /* [off[s], off[s+1]) (an absent slot's range is ignored) */
  const lins_point* outlier; const int32_t* outlier_off;
} lins_mappers_desc;
/* lins_gpu_mapper_step for every present slot; reps[s] written for present slots only (reps may be NULL).
   LINS_E_INVALID before anything changes for a bad descriptor (n_slots != M, null time / quat / pos, bad offsets, a
   NULL cloud with points).  LINS_E_TOOBIG when any slot's VoxelGrid overflows: then no slot's state changes (transforms,
   key frames, windows, IMU queues), and lins_gpu_mappers_download returns no clouds for the slots the step processed
   until their next completed cycle. */
int lins_gpu_mappers_step(lins_ctx* ctx, const lins_mappers_desc* d, lins_mapper_report* reps /*M or NULL*/);
/* lins_gpu_mapper_download of one slot */
int lins_gpu_mappers_download(lins_ctx* ctx, int32_t slot, double* key_poses, int32_t* window, float* map_corner_ds,
                              float* map_surf_ds, float* corner_ds, float* surf_ds, float* outlier_ds, float* surf_total_ds);

/* ---- sequence mode feeding its mapping nodes: LinsFusion::publishTopics (Estimator.cpp:177-202, :254-320) on the device ---
   A run opened by lins_gpu_seq_open can be bound to the context's lockstep mappers: slot s of the sequence run feeds
   mapper slot s.  After every sequence step (lins_gpu_seq_step, _ex, _pcl, _raw, _cloud2 and the _mixed forms) the run
   takes exactly one lins_gpu_seq_map_step, which publishes what each slot's estimator would and runs those slots'
   mapping cycles in one lins_gpu_mappers_step on the device clouds, with no host copy of a cloud.  A slot publishes
   after every scan of an estimator that was initialised before the scan (status_ != STATUS_INIT): its stamp,
   globalStateYZX_ and scan_last_'s YZX less-sharp, less-flat and outlier clouds, which only an accepted scan
   (LINS_SEQ_SECOND / RAN / ICP) replaces; a first scan (LINS_SEQ_FIRST) leaves them empty, a skipped scan publishes the
   previous ones again, an absent slot or an estimator still in STATUS_INIT publishes nothing.  Per slot the mapper's
   reports and downloads are bit-identical to lins_gpu_mappers_step fed the same clouds from the host.
   lins_gpu_mappers_imu, _download and _reset work on the bound run as on any lockstep run.  An unbound run is unchanged. */
typedef struct lins_seq_map_desc {
  int32_t n_seq;                 /* == S */
  int32_t pad;
  const double* time;            /* S: scan_time_ of each present slot's scan in the last step */
  const lins_point* outlier; const int32_t* outlier_off;  /* S + 1 CSR: the outlier clouds processPCL received with the
                                    last step's scans.  NULL after a _raw / _cloud2 step (the projection made them on the
                                    device), required after a lins_gpu_seq_step / _ex / _pcl step */
} lins_seq_map_desc;
/* Binds the open sequence run to the lockstep mappers, opened with M = S fresh slots (replacing any open lockstep run, as
   lins_gpu_mappers_open does).  LINS_E_NOMAP without a run; LINS_E_INVALID for a run of lins_gpu_seq_begin (a hand-over
   carries no outlier cloud and no publish state) or after the run's first step.  lins_gpu_seq_open, lins_gpu_seq_begin,
   lins_gpu_mappers_open and a step error that drops the run end the binding.  On a bound run lins_gpu_seq_restart also
   resets the restarted slots' mappers and publish state (a new recording is a new LinsFusion with a new mapping node). */
int lins_gpu_seq_map_open(lins_ctx* ctx);
/* publishTopics for every slot of the last step, then one lins_gpu_mappers_step of the slots that published: published[s]
   receives the decision, reps[s] the report of a published slot (either may be NULL).  At most one stream
   synchronisation (the mapper step's; none when no slot's cycle passes the 0.3 s gate), whatever S is.
   LINS_E_NOMAP on an unbound run.  LINS_E_INVALID before anything changes with no step since the last call, a wrong
   n_seq, a NULL time, bad outlier offsets, or outliers given after a _raw / _cloud2 step or missing after another step;
   a sequence step of a bound run whose publish is still pending returns LINS_E_INVALID before anything changes.
   LINS_E_TOOBIG as lins_gpu_mappers_step: no mapper slot changes, but the estimator side of the publish is committed
   and the next sequence step may run. */
int lins_gpu_seq_map_step(lins_ctx* ctx, const lins_seq_map_desc* d, lins_mapper_report* reps /*S or NULL*/,
                          uint8_t* published /*S or NULL*/);
/* what each slot's estimator publishes (what the last lins_gpu_seq_map_step fed a published slot's mapper): pose =
   globalStateYZX_ (S x 7: position, quaternion x y z w; the identity before the slot's first accepted scan since open /
   restart), sizes = the points of its less-sharp, less-flat and outlier YZX clouds (S x 3).  Either may be NULL.
   LINS_E_NOMAP on an unbound run. */
int lins_gpu_seq_map_published(lins_ctx* ctx, double* pose /*S x 7*/, int32_t* sizes /*S x 3*/);

/* block until everything queued on the ctx stream has finished */
int lins_gpu_sync(lins_ctx* ctx);

/* diagnostics: per-phase SM-cycle counters of the fused kernel (enable, then read after a batch_run) */
int lins_gpu_debug_phase_cycles(lins_ctx* ctx, int enable, long long* out /*64 or NULL*/);

/* kernels launched by this ctx since creation (for bench.py's gpu_launches). */
int64_t lins_gpu_launch_count(const lins_ctx* ctx);
/* library/ABI version, = 1 */
int lins_gpu_abi_version(void);

#ifdef __cplusplus
}
#endif
#endif /* LINS_GPU_H_ */
