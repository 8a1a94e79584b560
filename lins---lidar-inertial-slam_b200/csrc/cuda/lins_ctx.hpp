// lins_ctx.hpp — host state of a C-ABI context (struct lins_ctx of include/lins_gpu.h) and the helpers the translation units
// that implement the C-ABI share: lins_gpu.cu (fused kernel, single-scan and batched entry points, F1), lins_upload.cu
// (batch upload, gather lists), lins_map.cu (row F2), lins_seq.cu (sequence mode), lins_mapper.cu (the mapping node's
// host logic and VoxelGrid), lins_mappers.cu (the mapping node's cycle for one or many drives) and the front-end units.
// Host code only: a header that defines kernels cannot be included here, because every unit that includes this one
// would define them again.
#pragma once
#include <cuda_runtime.h>
#if defined(__SSE2__)
#include <emmintrin.h>
#endif

#include <algorithm>
#include <array>
#include <cstddef>
#include <cstdint>
#include <deque>
#include <optional>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

#include "../../../include/lins_gpu.h"
#include "../host/host_pool.hpp"
#include "../host/pose_graph.hpp"
#include "lins_kf_arena.hpp"
#include "lins_slot_blob.hpp"

namespace lins_dev { struct IcpState; struct BatchView; struct UnitTuning; }  // lins_kernels.cuh
namespace lins_map { struct PassConsts; struct MapLoopState; struct MapSlot; }  // lins_map.cuh

namespace lins_capi {

constexpr bool kPinned = true;

// Grow-only buffer that owns its memory: device memory, or pinned host memory when Pinned.  reserve() never shrinks; to
// grow it frees first, then allocates at least 16 elements, so the contents do not survive growth.
template <typename T, bool Pinned = false>
struct Buf {
  T* p = nullptr;
  size_t cap = 0;
  Buf() = default;
  Buf(const Buf&) = delete;
  Buf& operator=(const Buf&) = delete;
  Buf(Buf&& o) noexcept : p(o.p), cap(o.cap) { o.p = nullptr; o.cap = 0; }
  Buf& operator=(Buf&& o) noexcept { std::swap(p, o.p); std::swap(cap, o.cap); return *this; }
  ~Buf() { deallocate(); }
  cudaError_t reserve(size_t n) {
    if (n <= cap) return cudaSuccess;
    deallocate();
    const size_t want = std::max<size_t>(n, 16);
    const cudaError_t e = Pinned ? cudaMallocHost(&p, want * sizeof(T)) : cudaMalloc(&p, want * sizeof(T));
    if (e == cudaSuccess) cap = want;
    return e;
  }
  // reserve with a quarter of headroom when it has to grow: buffers whose sizes drift from call to call (a key frame's
  // clouds, the lockstep mappers' per-slot clouds) settle after a few calls instead of reallocating on most of them
  cudaError_t grow(size_t n) { return n <= cap ? cudaSuccess : reserve(n + n / 4); }

 private:
  void deallocate() {
    if (p) { if (Pinned) cudaFreeHost(p); else cudaFree(p); }
    p = nullptr; cap = 0;
  }
};

struct Resident {  // one resident batch (device) + its pinned staging (host)
  int n = 0;
  size_t nqs = 0, nqc = 0, nts = 0, ntc = 0;
  int max_q = 0;
  Buf<float4> qs, qc, ts, tc, az_s, az_c;
  Buf<float4> raw;              // raw 32-B records of clouds uploaded straight from caller-pinned memory (2 float4 per point)
  Buf<unsigned char> qscratch;  // per-CTA per-query arrays of units too large for shared memory
  Buf<int> qs_off, qc_off, ts_off, tc_off, ind_s, ind_c, counter;
  Buf<long long> timers;
  Buf<double> jac_part;         // split Jacobian kernel: per-(unit, part) sums and arrival counters
  Buf<int> jac_cnt;
  Buf<lins_dev::IcpState> icp;  // pose-update state of the ICP fallback loop (lins_gpu_estimate_transform)
  Buf<lins_dev::IcpState, kPinned> h_icp;
  Buf<double> state_in, cov_in, state_out, cov_out, accum;
  Buf<lins_scan_result> results;
  Buf<lins_report> reports;
  Buf<float> sel_s, sel_c, coeff_s, coeff_c;
  Buf<unsigned char> mask_s, mask_c;
  Buf<float4, kPinned> h_pts;   // staging for all four clouds, back to back
  Buf<int, kPinned> h_off;      // 4 x (n+1)
  Buf<double, kPinned> h_state, h_cov, h_state_out, h_cov_out, h_accum;
  Buf<lins_scan_result, kPinned> h_results;
  Buf<lins_report, kPinned> h_reports;
};

// A start / stop pair of CUDA events around device work on a stream, created on first use; valid once the stop has been
// recorded (what lins_gpu_extract_ms, lins_gpu_project_ms and lins_gpu_decode_ms read)
struct EventPair {
  cudaEvent_t ev[2] = {nullptr, nullptr};
  bool valid = false;
  EventPair() = default;
  EventPair(const EventPair&) = delete;
  EventPair& operator=(const EventPair&) = delete;
  ~EventPair() { for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e); }
  cudaError_t start(cudaStream_t s) {
    if (!ev[0])
      for (cudaEvent_t& e : ev) { const cudaError_t r = cudaEventCreate(&e); if (r != cudaSuccess) return r; }
    return cudaEventRecord(ev[0], s);
  }
  cudaError_t stop(cudaStream_t s) {
    const cudaError_t r = cudaEventRecord(ev[1], s);
    if (r == cudaSuccess) valid = true;
    return r;
  }
  cudaError_t elapsed_ms(float* ms) const { return cudaEventElapsedTime(ms, ev[0], ev[1]); }
};

// A gather list: contiguous device-to-device copies of float4 records, staged in pinned memory, copied to the device in
// one H2D and run by one launch of a block per copy (lins_upload.cu).  Each user keeps its own list: a list's staging may
// still be read by a queued H2D when another list is written.  yzx != 0: the copy writes (y, z, x, w) of each record, the
// mapping node's axis order (sequence mode's publish step); 0: the record as it is.
struct DevCopy { const float4* src; float4* dst; int n, yzx; };
struct CopyList {
  Buf<DevCopy> dev; Buf<DevCopy, kPinned> host;
  // room for n records (before any work is queued: growth frees the old buffers); records [base, base + n) from src into
  // the staging and one H2D of them (none for n = 0); one launch of the staged records [base, base + n) (none for n = 0)
  int reserve(lins_ctx* ctx, size_t n);
  int stage(lins_ctx* ctx, const DevCopy* src, int n, int base);
  int launch(lins_ctx* ctx, int base, int n);
};
// one device range of float4 records: len points at src
struct MapPiece { const float4* src = nullptr; int len = 0; };

// The map updatePointCloud keeps (StateEstimator.hpp:1116-1161) for n units: each unit's surf and corner map (the clouds
// the walks and tripods read) and, while it is stale, the surf and corner clouds its 1-NN index was last built on (after
// a refresh that failed the >= 5 && >= 20 guard; empty elsewhere).  Clouds are CSR over the units in unit order: cloud c
// (map_s, map_c, tree_s, tree_c) of unit s is [h_off[c (n + 1) + s], h_off[c (n + 1) + s + 1]) of cur[c].  nxt and h_noff
// hold the next generation while it is built.  Sequence mode keeps one for its slots, the single-scan seam one with one
// unit; n = 0: no map yet.
struct MapGen {
  int n = 0;
  Buf<float4> cur[4], nxt[4];
  std::vector<int> h_off, h_noff;
  std::vector<unsigned char> h_stale;  // 1: the unit's 1-NN clouds are tree_s / tree_c
  Buf<int> dev;                        // the device copy of h_off, then h_stale's bytes (queue_map_state)
  // n units without maps (host side only)
  void reset(int units) { n = units; h_off.assign(4 * (size_t)(n + 1), 0); h_stale.assign(n, 0); }
  const int* off() const { return dev.p; }
  const unsigned char* stale() const { return reinterpret_cast<const unsigned char*>(dev.p + 4 * (size_t)(n + 1)); }
};
// what a map refresh makes of one unit: its next four clouds and its stale flag
struct MapRefresh { MapPiece next[4]; unsigned char stale; };

// Sequence mode's publish step (lins_gpu_seq_map_*, lins_seq.cu): what LinsFusion::publishTopics hands each slot's
// mapping node (scan_last_'s YZX clouds, globalStateYZX_), kept for a run bound to the lockstep mappers (each slot's YZX
// flag and pose are in its SeqSlot).  Maps and the kept outlier clouds are in XYZ order; the mapper step's gather writes
// them YZX.
struct SeqPubState {
  bool bound = false;                  // lins_gpu_seq_map_open bound the run (ends with seq_open / seq_begin / mappers_open)
  bool pending = false;                // a step has run whose lins_gpu_seq_map_step has not
  bool dev_outliers = false;           // the last step projected its scans on the device (_raw / _cloud2): the stash holds
                                       // their outlier clouds
  std::vector<int32_t> fusion_before;  // each slot's StateEstimator::status_ before the last step
  Buf<float4> stash;                   // the last step's outlier clouds, dense in slot order at h_stash_off (n + 1)
  std::vector<int> h_stash_off;
  Buf<float4, kPinned> h_stash;        // staging of a caller's outlier clouds
  Buf<float4> outl, noutl;             // the published outlier cloud of each slot: current and next generation
  std::vector<int> h_outl_off, h_noutl_off;
  Buf<double, kPinned> h_glob;         // n x 20: the global states after the last step
  Buf<int, kPinned> h_proj_counts;     // n x 2: the last projection's counts (segmented, outlier)
  CopyList copies;                     // the outlier stash, then the next outlier generation
  std::vector<lins_fused_pose> fused;  // each slot's fused pose of the last publish step (valid = 0: none)
};

// One sequence-mode slot's setup on the host.  A slot of a new run, and a restarted one, is this record as constructed.
struct SeqSlot {
  struct Tuning {
    lins_slot_tuning t;
    double R[9];                              // its alignIMUtoVehicle rotation (row-major, built with the host's libm)
  };
  bool fresh = true;                          // not present in a step since open / restart: only a fresh slot can be
                                              // configured, tuned or loaded
  std::optional<lins_slot_config> cfg;        // lins_gpu_seq_configure
  std::optional<Tuning> tune;                 // lins_gpu_seq_tune
  bool yzx = false;                           // bound run: the slot's YZX clouds exist (false after a first scan)
  double pose[7] = {0, 0, 0, 0, 0, 0, 1};     // bound run: the slot's globalStateYZX_ (pos, quat x y z w)
};

// Sequence mode (lins_gpu_seq_*, lins_seq.cu): the running sequences' filter state and maps (a unit per sequence).
struct SeqState {
  int n = 0;                      // sequences (0 = lins_gpu_seq_begin / lins_gpu_seq_open has not run)
  double consts[10];              // lins_seq::Consts of the run's params
  // sequence initialisation (lins_gpu_seq_open runs only): init_consts = lins_seq::InitConsts, fusion = each slot's
  // StateEstimator::status_ (every slot of a lins_gpu_seq_begin run is RUNNING), pre = the pre-integration (n x 20),
  // init_icp = the second scans' estimateTransform loop state (n IcpState records), init_off = their compacted query
  // offsets (2 x (n + 1), after the IESKF's), scan_imu = the step's processPCL IMU samples (n x 6)
  bool has_init = false;
  double init_consts[24];
  std::vector<SeqSlot> slot;      // each slot's setup
  // the device tables of what each slot reads (lins_seq.cu: slot_params; every slot has an entry, so every slot takes one
  // path): its Consts / InitConsts (n x 10, n x 24; uploaded at open, configure, restart and load) and, per step, its
  // de-skew period (n), its tuning (n) and, while a slot is tuned, the alignment rows (n x 10)
  Buf<double> slot_consts, slot_init_consts, period;
  Buf<double, kPinned> h_period;
  Buf<lins_dev::UnitTuning> unit_tune; Buf<lins_dev::UnitTuning, kPinned> h_unit_tune;
  Buf<double> align; Buf<double, kPinned> h_align;
  std::vector<int32_t> fusion;
  Buf<double> pre, scan_imu;
  Buf<double, kPinned> h_scan_imu;
  Buf<unsigned char> init_icp;
  Buf<int> init_off;
  Buf<double> filt, cov, glob, lin, imu_last, icp_pose;  // n x 20, n x 324, n x 20, n x 20, n x 8, n x 20
  Buf<double> prior_state, prior_cov;                  // the last step's IESKF prior (after the IMU propagation)
  Buf<int> icp_ind_s, icp_ind_c;                       // correspondence IDs of the ICP fallback (the IESKF's stay in run)
  Buf<unsigned char> icp;                              // n IcpState records (lins_icp_step.cuh; icp_state_bytes() each)
  MapGen map;                                          // the next generation is built by the step, then swapped in
  Resident up;                                         // the step's four uploaded clouds (qs, qc, ts = new less-flat, tc = new less-sharp)
  Resident run;                                        // the IESKF batch: compacted queries of the sequences that run, outputs
  Buf<double> imu; Buf<int> imu_off;
  Buf<double, kPinned> h_imu; Buf<int, kPinned> h_imu_off;
  Buf<unsigned char> status_d;                         // 3 x n: LINS_SEQ_* of the step (read by the post kernel), the
                                                       // transformToEnd mask, the IMU rows' use (lins_seq.cu: ImuUse)
  Buf<unsigned char, kPinned> h_status;
  CopyList copies;                                     // query compaction, then the map refresh
  std::vector<int32_t> status;                         // host copy of status_d
  cudaEvent_t ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};  // phase boundaries of the last step (lins_gpu_seq_phase_ms)
  bool ev_valid = false;
  bool has_step = false;                               // a step has run since lins_gpu_seq_begin
  std::vector<int> h_run_off;                          // 2 x (n + 1): the last step's compacted query offsets (surf, corner)
  SeqPubState pub;                                     // the publish step of a run bound to the lockstep mappers
  Buf<float4> blob; Buf<float4, kPinned> h_blob;       // lins_gpu_seq_save / _load: the slot blobs on the device and
                                                       // their pinned staging (lins_checkpoint.cu)
  ~SeqState() { for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e); }
};

// One scan's feature extraction constants: cos / sin of imu_lidar_extrinsic_angle (host libm), the edge / surf thresholds
// and the re-stamp's SCAN_PERIOD
struct FeatConsts { double c, s, edge, surf, scan_period; };

// Feature extraction (lins_features.cu): the uploaded segmented scans (cloud in up.qs, CSR in up.qs_off) with their
// cloud_info, the extracted clouds at the input offsets, per-point scratch, and the counts read back (n x 5: the four
// counts in lins_seq_step_desc order, then the scan's status)
struct FeatState {
  Resident up;
  Buf<unsigned char> ground, picked, label;
  Buf<unsigned> col;
  Buf<float> range, ori;
  Buf<int> ring, counts, sind;
  Buf<double> curv;
  Buf<float4> und, out[4];
  Buf<int, kPinned> h_counts;
  Buf<FeatConsts> consts; Buf<FeatConsts, kPinned> h_consts;  // each scan's constants
  std::vector<int32_t> h_ring;
  CopyList copies;                                      // the pack into sequence mode's feature buffers
  EventPair ev;                                         // around the last extraction kernel (lins_gpu_extract_ms)
};

// One lidar model as the projection kernel reads it: the range image's rows and columns, groundScanInd, the angular
// resolutions and ang_bottom, and sinf / cosf of segmentAlphaX / Y (host libm)
struct ProjModel {
  int L, S, gsi;
  float res_x, res_y, bottom;
  float sin_x, cos_x, sin_y, cos_y;
};

// Image projection (lins_projection.cu): the uploaded raw sweeps (up.qs, CSR in up.qs_off), each resident CTA's range-image
// scratch (the largest listed model's line_num x scan_num entries: winning point, range, ground, label, out-edges, owner
// counts, owner row extents), the projected clouds and per-point cloud_info at the raw offsets, ring indices (n x 2 x the
// largest line_num: start, end),
// orientations (n x 3) and counts (n x 2: segmented, outlier); for lins_gpu_project_scans' read-back, the clouds packed
// to dense offsets (d*) and their pinned staging (h_*)
struct ProjState {
  Resident up;
  Buf<int> idx, lab, cnt, rlo, rhi;
  Buf<float> rng;
  Buf<unsigned char> gnd, edg;
  Buf<float4> seg, outl;
  Buf<unsigned char> ground;
  Buf<unsigned> col;
  Buf<float> range, ori;
  Buf<int> ring, counts;
  Buf<int, kPinned> h_counts;
  Buf<float4> dseg, doutl;
  Buf<unsigned char> dground;
  Buf<unsigned> dcol;
  Buf<float> drange;
  Buf<int> doff;
  Buf<float4, kPinned> h_seg, h_outl;
  Buf<unsigned char, kPinned> h_ground;
  Buf<unsigned, kPinned> h_col;
  Buf<float, kPinned> h_range, h_ori;
  Buf<int, kPinned> h_doff, h_ring;
  Buf<unsigned char> present;              // lins_gpu_seq_step_raw's present flags (n)
  Buf<unsigned char, kPinned> h_present;
  Buf<ProjModel> models;                   // the model table
  Buf<ProjModel, kPinned> h_models;
  Buf<int> model_of;                       // each scan's entry in the table (n; not uploaded for a one-model call)
  Buf<int, kPinned> h_model_of;
  EventPair ev;                            // around the last projection kernel (lins_gpu_project_ms)
};

// One decode record per PointCloud2 message (lins_cloud2.cu): where its data field starts in the uploaded blob, where its
// points go, and its layout
struct Cloud2Scan {
  long long base;                 // byte offset of the data field in blob
  int out;                        // first output point
  unsigned width, point_step, row_step;
  unsigned offset[4];
  unsigned char datatype[4];
};

// PointCloud2 decoding (lins_cloud2.cu): the uploaded message bytes (as 32-bit words: the decode reads aligned words), their
// pinned staging, the per-message records and, for lins_gpu_decode_cloud2's read-back, the decoded points' staging.  The
// decoded points themselves go to ctx->proj.up (qs, qs_off), where the projection reads raw sweeps.
struct Cloud2State {
  Buf<unsigned> blob;
  Buf<unsigned char, kPinned> h_blob;
  Buf<Cloud2Scan> scans; Buf<Cloud2Scan, kPinned> h_scans;
  Buf<int> prefix; Buf<int, kPinned> h_prefix;  // n + 1: the first output point of each message (what qs_off holds)
  Buf<float4, kPinned> h_out;
  EventPair ev;                            // around the last decode kernel (lins_gpu_decode_ms)
};

// The mapper (lins_mapper.cu): one VoxelGrid segment's device record — the ordered-integer encodings of the finite
// points' f32 min / max, the box, the voxel count
struct VgInfo {
  unsigned enc[6];   // min x y z, max x y z
  float base[3];     // floor(min * inv) in f32 (an integer value; |base| < 2^62 unless toobig)
  int mul[3];
  float inv;
  int any;           // at least one finite point
  int toobig;        // div_x * div_y * div_z > INT32_MAX, or a floor of min / max * inv of magnitude 2^62 or more
  int count;         // voxels
};
// PointTypePose (:57-65): the f32 pose fields and the f64 time
struct MapperKeyPose { float x, y, z, roll, pitch, yaw; double time; };
// one key frame of the device store: its corner, surf and outlier DS clouds in the map frame
struct MapperKeyFrame { Buf<float4> c[3]; int n[3] = {0, 0, 0}; };
// one key frame of a loop-closure slot's host store: its corner, surf and outlier DS clouds in the body frame, back to
// back at p in the run's pinned, mapped arena (the device reads and writes them through the same address; nullptr
// without points).  Its map-frame clouds are T(b, key pose): tf_point(tf_consts(pose), b), computed on demand.
struct HostKeyFrame { float4* p = nullptr; int n[3] = {0, 0, 0}; };
// the mapping node's scalar members the cycle reads and writes (lidar_mapping_node.cpp:198-214, :356-408): the slot
// blob's record of them, and the window
struct MapperScalars : lins_blob::MapperRec {
  std::deque<int> window;  // recent*CloudKeyFrames as key-frame ids, oldest first
  // the node's initial values: every member 0 but these two (the blob's writer memsets MapperRec, so it keeps no
  // initialisers of its own)
  MapperScalars() : MapperRec() { imuPointerLast = -1; timeLastProcessing = -1; }
};
struct MapperLast { bool valid = false; int n[6] = {0, 0, 0, 0, 0, 0}; };  // the last processed cycle's DS sizes
// a node's loop closure (lins_loops.cu): the key-pose graph (prior, chain and loop factors), isamCurrentEstimate of the
// last save, aLoopIsClosed, and what performLoopClosure reads of the node between cycles
struct MapperLoops {
  bool enabled = false;
  bool closed = false;                  // aLoopIsClosed
  bool rebuild = false;                 // correctPoses ran in this cycle: the stored clouds are re-transformed
  int n_loop = 0;                       // loop factors in the graph
  float cur[3] = {0, 0, 0};             // currentRobotPosPoint of the last processed cycle
  double time = 0;                      // timeLaserOdometry of the last odometry message
  std::vector<lins_pg::Factor> graph;
  std::vector<lins_pg::Pose3> est;      // isamCurrentEstimate of the last save
};
// a node's last global map (lins_gpu_mappers_global_map, lins_loops.cu): its report, the DS key ids and the published
// cloud in a buffer of its own (valid = false: none since open / reset)
struct MapperGlobalMap {
  bool valid = false;
  lins_global_map_report rep{};
  std::vector<int32_t> keys;
  Buf<float4> cloud;
};
// one mapping node's host state: its scalars, its key poses, the device key-frame store (the window and the newest key
// frame, each key frame's DS clouds in the map frame), on a slot with loop closure the host store of every key frame,
// and the sizes of its last processed cycle's clouds
struct MapperNode {
  MapperScalars s;
  std::vector<MapperKeyPose> poses;          // cloudKeyPoses6D
  std::vector<MapperKeyFrame> slots;         // the device key-frame store
  std::unordered_map<int, int> slot_of;      // key-frame id -> slot
  std::vector<int> free_slots;
  std::vector<HostKeyFrame> host;            // loop closure: the host store, by key-frame id (every key pose's)
  lins_arena::Holding held;                  // what the host store holds of the run's arena
  MapperLast last;
  bool stepped = false;                      // present in a step since open / reset (not fresh)
  MapperLoops loops;
  MapperGlobalMap gm;
};
// the scratch of segmented VoxelGrids (lins_mapper.cu): 32-bit keys for one segment, (segment, key) 64-bit keys for more
struct VgScratch {
  Buf<unsigned> key[2];
  Buf<unsigned long long> key64[2];
  Buf<int> idx[2], head, vid;
  Buf<unsigned char> temp;                   // CUB scratch
};
// lins_gpu_voxel_grid: its input and output cloud, the input's pinned staging, the VoxelGrid scratch and the record
// (h_info stages its initial value, then receives it back: the stream orders the two copies)
struct VoxelGridState {
  Buf<float4> in, out;
  Buf<float4, kPinned> h_in;
  VgScratch w;
  Buf<VgInfo> info; Buf<VgInfo, kPinned> h_info;
};
// The scan-to-map refinement of a table of slots (lins_map.cu): the lockstep mappers' step, the single mapper's, and the
// one slot of lins_gpu_map_set / scan2map / map_associate.  The layout is that of the table map_fill_table last filled.
struct ScanToMap {
  Buf<lins_map::MapLoopState> loop;          // per slot: the loop state (matP / isDegenerate persist)
  Buf<lins_map::MapLoopState, kPinned> h_loop;
  Buf<lins_map::PassConsts> consts;          // per slot: sin / cos + translation of the pass being run
  Buf<lins_map::PassConsts, kPinned> h_consts;
  Buf<lins_map::MapSlot> mslot;              // per slot: its maps, queries, grids and fit blocks
  Buf<lins_map::MapSlot, kPinned> h_mslot;
  Buf<int> blk_slot; Buf<int, kPinned> h_blk_slot;  // per fit block: its slot
  Buf<int> grid_start, count, cursor;        // every slot's corner and surf buckets
  Buf<float4> sorted;                        // every slot's map points, bucket-sorted
  Buf<unsigned char> scan_temp;              // CUB scratch of the buckets' scan
  Buf<float> part_d; Buf<int> part_i; Buf<double> partial;
  int n_slots = 0, buckets = 0, points = 0;  // the layout: slots, buckets, map capacity in all
  int blocks[2] = {0, 0};                    // fit blocks of the corner and the surf launch
};

// performLoopClosure of many slots in one device pass (lins_loops.cu).  Per slot with a candidate: its source (the
// latest key frame's corner + surf cloud) at src0, the running source at src, its history cloud at tin and that
// cloud's VoxelGrid at tgt (each at the slot's offsets), the 1-NN of every source point (corr, dist) and the ICP state.
struct LoopSlot { const float4* src0; float4* src; const float4* tgt; const int* n_tgt; int* corr; float* dist; int n_src, pad; };
struct LoopIcpState {
  float fin[12];          // final_transformation_ rows 0..2 (row 3 is 0 0 0 1)
  float inc[12];          // transformation_ of the last iteration
  double prev_mse, fitness;
  int iters, done, converged, n_corr0, n_src, n_fit, pad[2];
};
struct LoopPass {
  Buf<float4> src0, src, tin, tgt;
  Buf<int> corr; Buf<float> dist;
  Buf<LoopSlot> slot; Buf<LoopSlot, kPinned> h_slot;
  Buf<int2> blk; Buf<int2, kPinned> h_blk;     // per 1-NN block: (slot, first source point)
  Buf<LoopIcpState> st; Buf<LoopIcpState, kPinned> h_st;
  Buf<VgInfo> info; Buf<VgInfo, kPinned> h_info, h_init;
  Buf<int> off; Buf<int, kPinned> h_off;
  Buf<float4*> out; Buf<float4*, kPinned> h_out;
  Buf<unsigned char> jobs; Buf<unsigned char, kPinned> h_jobs;  // the gather's jobs (lins_loops.cu: GatherJob)
};

// The arena of a run's host key-frame stores: 1 MiB chunks of pinned, mapped memory, in slabs of 4 chunks first, then
// as many as the run holds, up to 64 (lins_mappers.cu: pinned_mapped_allocator)
constexpr size_t kKfChunkBytes = size_t(1) << 20;
constexpr int kKfFirstSlabChunks = 4, kKfMaxSlabChunks = 64;
lins_arena::Allocator pinned_mapped_allocator();
// A run of mapping nodes in lockstep (lins_mappers.cu): the lockstep mappers (lins_gpu_mappers_*), or the single
// mapper (lins_gpu_mapper_*) as a run of one slot.  One MapperNode per slot with its six DS clouds of the last
// processed cycle (map corner, map surf, corner, surf, outlier, surf total), and the step's shared device buffers
struct MappersState {
  int n = 0;                                 // slots (0 = not opened)
  lins_arena::Arena store{kKfChunkBytes, kKfFirstSlabChunks, kKfMaxSlabChunks, pinned_mapped_allocator()};  // the slots' host key-frame stores
  std::vector<MapperNode> node;
  std::vector<std::array<Buf<float4>, 6>> ds;
  ScanToMap stm;                             // a slot per mapping node
  Buf<float4> vin[2];                        // the VoxelGrids' inputs: round 1 (maps and scans), round 2 (surf total)
  Buf<float4, kPinned> h_in;
  VgScratch vg;
  Buf<VgInfo> vg_info; Buf<VgInfo, kPinned> h_vg_info, h_vg_init;
  Buf<int> vg_off; Buf<int, kPinned> h_vg_off;      // per round: S + 1 segment offsets
  Buf<float4*> vg_out; Buf<float4*, kPinned> h_vg_out;  // per round: S output clouds
  Buf<unsigned char> tf; Buf<unsigned char, kPinned> h_tf;  // the key frames' transform jobs
  CopyList copies;                           // the local maps' concatenation, then the surf-total one
  LoopPass lp;                               // lins_gpu_mappers_close_loops
  Buf<float4> blob; Buf<float4, kPinned> h_blob;  // lins_gpu_mapper(s)_save / _load: the slot blobs on the device and
                                                  // their pinned staging (lins_checkpoint.cu)
};

}  // namespace lins_capi

struct lins_ctx {
  template <typename T, bool Pinned = false>
  using Buf = lins_capi::Buf<T, Pinned>;
  static constexpr bool kPinned = lins_capi::kPinned;

  HostPool pool;
  int device = 0;
  cudaStream_t stream = nullptr;
  bool own_stream = false;
  lins_params prm;
  std::string err;
  int sm_count = 132;  // (replaced by the device's count in lins_gpu_create)
  int max_smem_optin = 0;
  int64_t launches = 0;
  int64_t upload_raw_points = 0, upload_packed_points = 0;  // cumulative split of lins_gpu_batch_upload (raw DMA vs host pack)
  lins_capi::Resident batch;   // lins_gpu_batch_* working set
  lins_capi::Resident single;  // lins_gpu_ieskf / associate / estimate_transform (n = 1)
  lins_capi::SeqState seq;     // lins_gpu_seq_*
  lins_capi::FeatState feat;   // lins_gpu_extract_features, lins_gpu_seq_step_pcl, lins_gpu_seq_step_raw
  lins_capi::ProjState proj;   // lins_gpu_project_scans, lins_gpu_seq_step_raw, lins_gpu_seq_step_cloud2
  lins_capi::Cloud2State c2;   // lins_gpu_decode_cloud2, lins_gpu_seq_step_cloud2
  lins_capi::MapGen map;       // the single-scan map (one unit)
  bool timers_on = false;
  bool verbose = false;  // LINS_VERBOSE: print the launch configuration
  int force_slots = 0;  // tuning knob (LINS_SLOTS): resident units per CTA
  Buf<lins_point> tmp_out;      // transformed clouds as full PointXYZI records (update_map read-back)
  cudaEvent_t tmp_ev = nullptr; // recorded after the last H2D copies that read h_tmp
  Buf<lins_point, kPinned> h_out;  // pinned staging of the update_map read-back
  Buf<double> tmp_lin;
  Buf<float4, kPinned> h_tmp;
  // row F2 (lins_gpu_map_set / scan2map / map_associate): a one-slot scan-to-map table over the map clouds (their sizes on
  // the device for MapSlot::n_map, on the host -1 before the first map_set) and the current feature clouds, and
  // map_associate's dense outputs
  struct MapState {
    Buf<float4> map_c, map_s, q_c, q_s;
    Buf<int> n_map;
    int n_map_c = -1, n_map_s = -1;
    lins_capi::ScanToMap stm;
    Buf<int32_t> knn_c, knn_s;
    Buf<float> coeff_c, coeff_s;
    Buf<uint8_t> mask_c, mask_s;
  } mp;
  lins_capi::MappersState mapper;   // lins_gpu_mapper_*: one slot, opened by the first call
  lins_capi::MappersState mappers;  // lins_gpu_mappers_*
  lins_capi::VoxelGridState vg;     // lins_gpu_voxel_grid
  double mapper_load_ms[5] = {0, 0, 0, 0, 0};  // the last mapper load's host phases (lins_gpu_mappers_load_phase_ms)
  bool mapper_load_valid = false;
};

namespace lins_capi {

inline int fail(lins_ctx* c, int code, const char* what, cudaError_t e = cudaSuccess) {
  if (c) {
    c->err = what;
    if (e != cudaSuccess) { c->err += ": "; c->err += cudaGetErrorString(e); }
  }
  return code;
}
#define CK(call)                                                                \
  do {                                                                          \
    cudaError_t _e = (call);                                                    \
    if (_e != cudaSuccess) return lins_capi::fail(ctx, LINS_E_CUDA, #call, _e); \
  } while (0)

// CSR offsets of n ranges over data: off[0] = 0, non-decreasing, data non-null when off[n] > 0 (LINS_E_INVALID: what)
inline int check_csr(lins_ctx* ctx, const int32_t* off, int n, const void* data, const char* what) {
  if (!off || off[0] != 0) return fail(ctx, LINS_E_INVALID, what);
  for (int i = 0; i < n; ++i) if (off[i + 1] < off[i]) return fail(ctx, LINS_E_INVALID, what);
  if (off[n] > 0 && !data) return fail(ctx, LINS_E_INVALID, what);
  return LINS_OK;
}
// a caller's cloud of n points: n >= 0, p non-null when n > 0 (LINS_E_INVALID: what)
inline int check_cloud(lins_ctx* ctx, const void* p, int n, const char* what) {
  return n < 0 || (n > 0 && !p) ? fail(ctx, LINS_E_INVALID, what) : LINS_OK;
}

// State rows: the C ABI passes 19 doubles per state, the device keeps 20 (the last one 0); a pose (t, q xyzw) is
// state[0..2], state[6..9].  copy_rows: n rows of src_w doubles into rows of dst_w, a wider row's tail 0.
inline void copy_rows(double* dst, size_t dst_w, const double* src, size_t src_w, size_t n) {
  for (size_t i = 0; i < n; ++i)
    for (size_t k = 0; k < dst_w; ++k) dst[i * dst_w + k] = k < src_w ? src[i * src_w + k] : 0.0;
}
inline void pad_states(double* dev, const double* abi, size_t n) { copy_rows(dev, 20, abi, 19, n); }
inline void strip_states(double* abi, const double* dev, size_t n) { copy_rows(abi, 19, dev, 20, n); }
inline void pose_to_state(const double* pose, double* state) { std::copy(pose, pose + 3, state); std::copy(pose + 3, pose + 7, state + 6); }
inline void state_to_pose(const double* state, double* pose) { std::copy(state, state + 3, pose); std::copy(state + 6, state + 10, pose + 3); }

// a D2H copy on the context's stream, skipped for a null destination or nothing to copy
inline cudaError_t d2h(lins_ctx* ctx, void* dst, const void* src, size_t bytes) {
  return dst && bytes ? cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, ctx->stream) : cudaSuccess;
}

// pcl::PointXYZI (32 B) -> (x, y, z, intensity) (16 B).  The destination is pinned staging that the copy engine
// reads next and the host never reads back: SSE2 (x86-64 baseline) with non-temporal stores.
inline void pack_into(float4* dst, const lins_point* src, int n) {
#if defined(__SSE2__)
  if ((reinterpret_cast<uintptr_t>(dst) & 15u) == 0) {
    for (int i = 0; i < n; ++i) {
      const __m128 a = _mm_loadu_ps(&src[i].x);                         // x y z pad
      const __m128 b = _mm_load_ss(&src[i].intensity);                  // i 0 0 0
      const __m128 t = _mm_shuffle_ps(a, b, _MM_SHUFFLE(0, 0, 2, 2));   // z z i i
      _mm_stream_ps(reinterpret_cast<float*>(dst + i), _mm_shuffle_ps(a, t, _MM_SHUFFLE(2, 0, 1, 0)));  // x y z i
    }
    _mm_sfence();
    return;
  }
#endif
  for (int i = 0; i < n; ++i) dst[i] = make_float4(src[i].x, src[i].y, src[i].z, src[i].intensity);
}
// (x, y, z, intensity) -> pcl::PointXYZI, the read-back of pack_into: pad0 = 1 as PCL_ADD_POINT4D sets it, the rest 0
inline lins_point unpack_point(const float4& p) {
  lins_point q;
  q.x = p.x; q.y = p.y; q.z = p.z; q.pad0 = 1.0f; q.intensity = p.w; q.pad1 = q.pad2 = q.pad3 = 0.f;
  return q;
}

// lins_gpu_extract_ms / lins_gpu_project_ms / lins_gpu_decode_ms: the CUDA-event time of e (none: the error when it has
// not run)
inline int event_ms(lins_ctx* ctx, const EventPair& e, float* ms, const char* none) {
  if (!ms) return fail(ctx, LINS_E_INVALID, "null ms");
  if (!e.valid) return fail(ctx, LINS_E_NOMAP, none);
  CK(e.elapsed_ms(ms));
  return LINS_OK;
}

// allocate the per-batch outputs / scratch for n scans with the given query totals
inline int reserve_outputs(lins_ctx* ctx, Resident& r, bool want_reports, bool want_trace) {
  CK(r.state_out.reserve((size_t)r.n * 20));
  CK(r.cov_out.reserve((size_t)r.n * 324));
  CK(r.results.reserve(r.n));
  CK(r.accum.reserve((size_t)r.n * 32));
  CK(r.az_s.reserve(r.nts + 4));
  CK(r.az_c.reserve(r.ntc + 4));
  CK(r.ind_s.reserve(3 * r.nqs + 4));
  CK(r.ind_c.reserve(2 * r.nqc + 4));
  CK(r.counter.reserve(4));
  if (want_reports) CK(r.reports.reserve(r.n));
  if (want_trace) {
    CK(r.sel_s.reserve(3 * r.nqs + 4)); CK(r.sel_c.reserve(3 * r.nqc + 4));
    CK(r.coeff_s.reserve(4 * r.nqs + 4)); CK(r.coeff_c.reserve(4 * r.nqc + 4));
    CK(r.mask_s.reserve(r.nqs + 4)); CK(r.mask_c.reserve(r.nqc + 4));
  }
  return LINS_OK;
}

// ---- two clouds through the context's pinned staging (ctx->h_tmp) ------------------------------------------------------
// h_tmp is read by asynchronous H2D copies: before it is rewritten, wait for the event recorded after the last copies that
// read it (already complete in steady state: no stream synchronisation).
inline cudaError_t tmp_staging_wait(lins_ctx* ctx) {
  if (!ctx->tmp_ev) return cudaSuccess;
  return cudaEventSynchronize(ctx->tmp_ev);
}
inline cudaError_t tmp_staging_mark(lins_ctx* ctx) {
  if (!ctx->tmp_ev) { cudaError_t e = cudaEventCreateWithFlags(&ctx->tmp_ev, cudaEventDisableTiming); if (e != cudaSuccess) return e; }
  return cudaEventRecord(ctx->tmp_ev, ctx->stream);
}

// every allocation of an upload of na + nb points into dst_a / dst_b; waits until the staging is free
inline int upload2_reserve(lins_ctx* ctx, Buf<float4>& dst_a, int na, Buf<float4>& dst_b, int nb) {
  CK(dst_a.reserve((size_t)na + 1)); CK(dst_b.reserve((size_t)nb + 1));
  if (na + nb == 0) return LINS_OK;
  CK(tmp_staging_wait(ctx));
  CK(ctx->h_tmp.reserve((size_t)na + nb + 1));
  return LINS_OK;
}
// pack a and b into the staging and queue their H2D copies into dst_a / dst_b, reserved by upload2_reserve (no stream
// synchronisation)
inline int upload2_queue(lins_ctx* ctx, Buf<float4>& dst_a, const lins_point* a, int na, Buf<float4>& dst_b, const lins_point* b, int nb) {
  if (na + nb == 0) return LINS_OK;
  pack_into(ctx->h_tmp.p, a, na);
  pack_into(ctx->h_tmp.p + na, b, nb);
  if (na) CK(cudaMemcpyAsync(dst_a.p, ctx->h_tmp.p, sizeof(float4) * (size_t)na, cudaMemcpyHostToDevice, ctx->stream));
  if (nb) CK(cudaMemcpyAsync(dst_b.p, ctx->h_tmp.p + na, sizeof(float4) * (size_t)nb, cudaMemcpyHostToDevice, ctx->stream));
  CK(tmp_staging_mark(ctx));
  return LINS_OK;
}
inline int upload2(lins_ctx* ctx, Buf<float4>& dst_a, const lins_point* a, int na, Buf<float4>& dst_b, const lins_point* b, int nb) {
  const int rc = upload2_reserve(ctx, dst_a, na, dst_b, nb);
  return rc != LINS_OK ? rc : upload2_queue(ctx, dst_a, a, na, dst_b, b, nb);
}

// lins_upload.cu: validate n units' four CSR clouds (the lins_batch_desc order: surf_flat, corner_sharp, surf_less_flat,
// corner_less_sharp) and upload them with their offsets into r (qs, qc, ts, tc); sets r.n, the totals and r.max_q
int upload_clouds(lins_ctx* ctx, Resident& r, int n, const lins_point* const pts[4], const int32_t* const offs[4], int point_format);
// lins_gpu.cu: the fused kernel's IESKF launch over bv (with r's scratch), its query tile, the estimateTransform loop of
// bv's device-resident units (pose: 20 doubles, icp: one IcpState per unit, set by the caller; n_iter launches, the largest
// NUM_ITER of the units), bv's targets pointed at the maps of g (map_targets), and transformToEnd in place on the CSR
// clouds of the units with run[u] != 0 (lin: 20 doubles per unit, period: one SCAN_PERIOD per unit, both on the device;
// a block per unit)
int fused_ieskf_launch(lins_ctx* ctx, Resident& r, const lins_dev::BatchView& bv);
int fused_qtile(int max_q);
size_t icp_state_bytes();
int icp_loop(lins_ctx* ctx, Resident& r, lins_dev::BatchView bv, double* pose, lins_dev::IcpState* icp, int n_iter);
void map_targets(lins_dev::BatchView& bv, const MapGen& g);
int transform_to_end(lins_ctx* ctx, float4* pts, const int* off, int n_units, const double* lin, const unsigned char* run,
                     const double* period);
// device-resident input of one feature extraction: n scans of line_num rings; scan i's points are pts[off[i] ..
// off[i] + count[count_stride * i]) (off[i] .. off[i + 1] when count is null), its per-point cloud_info at the same
// offsets; ring: n x 2 x line_num (start, end), ori: n x 3; total = off[n], the length of the per-point outputs
struct FeatInputs {
  int n = 0, line_num = 0, total = 0;
  const float4* pts = nullptr; const int* off = nullptr;
  const int* count = nullptr; int count_stride = 0;
  const unsigned char* ground = nullptr; const unsigned* col = nullptr; const float* range = nullptr;
  const int* ring = nullptr; const float* ori = nullptr;
};
// lins_features.cu: one scan's constants from fp and its SCAN_PERIOD
FeatConsts feat_consts(const lins_feature_params& fp, double scan_period);
// lins_features.cu: validate, upload and extract the scans of d into ctx->feat with fp and SCAN_PERIOD period[i] (host, n;
// null = the context's) for scan i; reads the counts back (one synchronisation)
int features_run(lins_ctx* ctx, const lins_feature_params* fp, const lins_pcl_desc* d, const double* period = nullptr);
// lins_features.cu: extract the scans of `in` into ctx->feat (clouds at the input offsets) with scan i's constants k[i]
// (host, in.n) and read the counts back (one D2H + synchronisation; a scan's device-side status returns LINS_E_INVALID /
// LINS_E_TOOBIG)
int features_launch(lins_ctx* ctx, const FeatConsts* k, const FeatInputs& in);
// lins_projection.cu: validate the model table and the sweeps of d, upload them and queue their projection into ctx->proj
// (no synchronisation); drop_nonfinite: copyPointCloud's NaN removal first; present (host, n; null = all): a scan whose
// flag is 0 is projected as an empty sweep.  A single-model entry passes the table {1, m, NULL}.
int projection_run(lins_ctx* ctx, const lins_lidar_models* t, const lins_raw_desc* d, bool drop_nonfinite, const uint8_t* present);
// lins_projection.cu: one model's limits; the table's (a table, n_models >= 1, every model within its limits, model_of
// given when n_models > 1); model_of's n entries within 0..n_models-1 (each LINS_E_INVALID otherwise); the table's largest
// line_num (the ring stride of the projection's output)
int check_model(lins_ctx* ctx, const lins_lidar_model* m);
int check_models(lins_ctx* ctx, const lins_lidar_models* t);
int check_model_of(lins_ctx* ctx, const lins_lidar_models* t, int n);
int max_line_num(const lins_lidar_models* t);
// lins_projection.cu: the part of projection_run after the upload: the n sweeps (total points) are in ctx->proj.up (qs,
// CSR in qs_off), the table and model_of have been checked
int projection_launch(lins_ctx* ctx, const lins_lidar_models* t, int n, size_t total, bool drop_nonfinite, const uint8_t* present);
// lins_upload.cu: n bytes from the caller's src to the device at dst, as upload_clouds moves clouds: a host thread pool copies
// 1 MiB slices into the pinned staging and queues each slice's H2D as soon as it is staged; a src in caller-pinned memory
// goes in one DMA with no host pass.  Synchronises the stream first (the staging may still be read by an earlier copy).
int upload_bytes(lins_ctx* ctx, void* dst, Buf<unsigned char, kPinned>& staging, const uint8_t* src, size_t n);
// lins_cloud2.cu: validate the messages of d (present: host, n; null = all; an absent message is neither checked nor
// decoded and has no points), upload them and queue their decode into ctx->proj.up (qs, qs_off; no synchronisation).
// off (n + 1) receives the host copy of qs_off.
int cloud2_run(lins_ctx* ctx, const lins_cloud2_desc* d, const uint8_t* present, std::vector<int32_t>& off);
// lins_map.cu: the scan-to-map refinement of a table of n_slots slots in sm.  map_fill_table: sm.h_mslot (pinned,
// n_slots) holds each slot's map and query clouds, capacities, device map counts, grid origins, start transform and run
// flag; fills the rest of the table (bucket ranges, point numbering, fit blocks, blk_slot, pass constants), reserves sm's
// buffers and queues the H2D of the table.  map_queue_grids: every slot's two grids in one bucket array (one count, one
// CUB scan, one scatter).  map_queue_loop: the start / gate kernel (a slot with run = 0 starts done), LINS_MAP_MAX_ITER
// passes of one 5-NN and one fit launch per kind over all slots and one LM launch with a warp per slot, then the loop
// states' D2H into sm.h_loop; sm.loop (n_slots) keeps each slot's matP / isDegenerate.  Nothing is synchronised.
// map_loop_report: a loop state into T and a report.
int map_fill_table(lins_ctx* ctx, ScanToMap& sm, int n_slots);
int map_queue_grids(lins_ctx* ctx, ScanToMap& sm);
int map_queue_loop(lins_ctx* ctx, ScanToMap& sm);
void map_loop_report(const lins_map::MapLoopState& st, float* T, lins_map_report* rep);
// lins_mapper.cu: queue pcl::VoxelGrid of n_seg segments of the device points `in` (segment k: [h_off[k], h_off[k + 1]),
// leaf[k]) into outputs with room for each segment's points (out for one segment; else the device table d_out, with
// d_off the device copy of h_off), the records at info (device, n_seg; their initial values staged through h_init, pinned,
// n_seg records).  The counts and flags are read back by the caller.  voxel_grid_reserve: the scratch for n points in
// n_seg segments (grow-only; call before queuing work that a growth could free under).
int voxel_grid_queue(lins_ctx* ctx, VgScratch& w, const float4* in, int n_seg, const int* h_off, const int* d_off, const float* leaf,
                     float4* out, float4* const* d_out, VgInfo* h_init, VgInfo* info);
int voxel_grid_reserve(lins_ctx* ctx, VgScratch& w, int n, int n_seg);
// lins_mapper.cu: the mapping node's host logic, which lins_mappers.cu runs for every slot.
// mapper_node_reset: a freshly constructed node (the device store's buffers are kept for reuse, the host store's arena
// holding goes back to the run's store); mapper_node_imu: imuHandler.
// mapper_cycle_begin: laserOdometryHandler into s (a copy of m.s, committed by the caller) and, unless the 0.3 s gate
// skips the cycle (false; r reports it), transformAssociateToMap and the window; window_sizes: the local map's corner and
// surf + outlier point counts.  mapper_cycle_end, after the read-back of the DS counts cnt (map corner, map surf, corner,
// surf, outlier, surf total) and of the loop state st (null: no key frames, or the 10 / 100 gate failed): transformUpdate,
// saveKeyFramesAndFactor and the loop candidate; commits s into m and fills r.  A saved key frame is left in *save for
// keyframes_queue, which transforms every listed key frame's DS clouds into its store slot in one launch.
// mapper_node_fuse: transform_fusion_node's pose for the odometry message (time, quat, pos) against the node as it
// stands, i.e. with the pair the node published after its last processed cycle (DESIGN.md §4.13).
// a key frame's clouds ds transformed by kp into kf->c; body (a host-store block, or null): also written as they are
// into body, back to back, through the mapped address
struct KfSave { MapperKeyFrame* kf; MapperKeyPose kp; const float4* ds[3]; float4* body; };
int loop_candidate(const MapperNode& m, const float cur[3], double time);
void mapper_loops_save(MapperNode& m, const MapperScalars& s, double R[3][3], double t[3]);
void mapper_correct_poses(MapperNode& m);
void mapper_node_reset(MapperNode& m, lins_arena::Arena& store);
void mapper_node_imu(MapperScalars& s, const double* time, const double* roll, const double* pitch, int n);
bool mapper_cycle_begin(const MapperNode& m, MapperScalars& s, double time, const double quat[4], const double pos[3], lins_mapper_report& r);
void mapper_window_sizes(const MapperNode& m, const MapperScalars& s, int& n_corner, int& n_surf);
void mapper_node_fuse(const MapperNode& m, double time, const double quat[4], const double pos[3], lins_fused_pose& out);
void mapper_cycle_end(MapperNode& m, MapperScalars& s, double time, double scan_period, const int cnt[6], const lins_map::MapLoopState* st,
                      lins_mapper_report& r, KfSave* save, bool* saved);
int keyframes_queue(lins_ctx* ctx, const KfSave* saves, int n, Buf<unsigned char>& dev, Buf<unsigned char, kPinned>& host);
// lins_mapper.cu: the device store's slot of key frame id (its own, a free one, or a new one), sized for n points of each
// cloud (a step's new key frame, a loaded one)
MapperKeyFrame& store_keyframe(MapperNode& m, int id, const int n[3]);
// lins_mapper.cu: a node's key poses, window and last cycle's clouds (src: its six DS clouds on the device; NULL skips)
int mapper_node_download(lins_ctx* ctx, const MapperNode& m, const float4* const src[6], double* key_poses, int32_t* window, float* const dst[6]);
// lins_mapper.cu: the non-empty copies of v through the gather list l, staged at entries base.. and run in one launch
int queue_copies(lins_ctx* ctx, CopyList& l, std::vector<DevCopy> v, int base);
// lins_mappers.cu: n_slots fresh mapping nodes in ms (replacing any open run); the slots with mask[s] != 0 back to the
// fresh state; one lockstep step of ms's present slots on a checked descriptor, from d's host clouds or, with dev
// (n_slots x 3: corner, surf, outlier), from device ranges in XYZ order that the step's gather writes YZX; period (host,
// n_slots; null = the context's): each slot's SCAN_PERIOD in transformUpdate
int mappers_open(lins_ctx* ctx, MappersState& ms, int n_slots);
int mappers_reset(lins_ctx* ctx, MappersState& ms, const uint8_t* mask);
int mappers_step(lins_ctx* ctx, MappersState& ms, const lins_mappers_desc* d, lins_mapper_report* reps, const MapPiece* dev,
                 const double* period);
int mappers_close_loops(lins_ctx* ctx, MappersState& ms, const uint8_t* mask, lins_loop_report* reps);
// lins_loops.cu: publishGlobalMap of the masked (enabled) slots into each slot's MapperGlobalMap (DESIGN.md §4.15)
int mappers_global_map(lins_ctx* ctx, MappersState& ms, const uint8_t* mask, lins_global_map_report* reps);
// lins_seq.cu: what the slot entries, a step, a restart and a load share.  check_open_run: the preamble of an entry
// (named in its messages) that needs a lins_gpu_seq_open run: LINS_E_NOMAP without a run, LINS_E_INVALID when args_ok is
// false (a null argument) or for a run of lins_gpu_seq_begin; check_fresh: LINS_E_INVALID unless slot s is fresh.
// upload_slot_consts: every slot's device constants (its config's, else the run's) for the first n slots, then a
// synchronisation
int check_open_run(lins_ctx* ctx, const char* entry, bool args_ok);
int check_fresh(lins_ctx* ctx, int s, const char* entry);
int upload_slot_consts(lins_ctx* ctx, int n);
// lins_seq.cu: a MapGen's generations.  reserve_maps: g's device state for n units and current maps of ns / nc points
// (growth loses the contents); queue_map_state: one H2D of h_off and h_stale into g.dev (a pageable source: staged before
// it returns); current_piece: cloud c of unit s in the current generation; refresh_maps: unit s's refresh by its new
// clouds (the guard rule); build_next_maps: the next generation from next[4 * s + c] (fills h_noff, reserves nxt and
// appends the copies that fill it to `copies`); swap_maps: the next generation becomes the current one
int reserve_maps(lins_ctx* ctx, MapGen& g, int n, size_t ns, size_t nc);
cudaError_t queue_map_state(lins_ctx* ctx, MapGen& g);
MapPiece current_piece(const MapGen& g, int c, int s);
MapRefresh refresh_maps(const MapGen& g, int s, MapPiece surf, MapPiece corner);
int build_next_maps(lins_ctx* ctx, MapGen& g, const std::vector<MapPiece>& next, std::vector<DevCopy>& copies);
void swap_maps(MapGen& g);

}  // namespace lins_capi
