// lins_upload.cu — lins_gpu_batch_upload: the four clouds, offsets and priors of a batch from host memory into the
// context's resident batch (lins_ctx.hpp: Resident), packing 32-B PointXYZI records into 16-B (x, y, z, intensity)
// records on host threads or, for clouds in pinned host memory, on the device.  Also the gather lists' staging and copy
// kernel (lins_ctx.hpp: CopyList).
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <thread>
#include <vector>

#include "lins_ctx.hpp"

using namespace lins_capi;

namespace {

// pcl::PointXYZI records (32 B) -> packed (x, y, z, intensity) (16 B) on the device: the upload path of clouds that
// sit in caller-pinned host memory (DMA of the raw records, no host pass over the points).
__global__ void lins_pack_points_kernel(const float4* __restrict__ raw, float4* __restrict__ out, size_t n) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float4 a = __ldcs(raw + 2 * i);       // x y z pad
    const float b = __ldcs(&raw[2 * i + 1].x);  // intensity
    out[i] = make_float4(a.x, a.y, a.z, b);
  }
}

// one block per record of a gather list (lins_ctx.hpp: CopyList); a record flagged yzx permutes each point to (y, z, x, w)
__global__ void lins_copy_kernel(const DevCopy* __restrict__ copies) {
  const DevCopy c = copies[blockIdx.x];
  if (c.yzx)
    for (int i = threadIdx.x; i < c.n; i += blockDim.x) { const float4 p = c.src[i]; c.dst[i] = make_float4(p.y, p.z, p.x, p.w); }
  else
    for (int i = threadIdx.x; i < c.n; i += blockDim.x) c.dst[i] = c.src[i];
}

}  // namespace

namespace lins_capi {

int CopyList::reserve(lins_ctx* ctx, size_t n) { CK(dev.reserve(n + 1)); CK(host.reserve(n + 1)); return LINS_OK; }

int CopyList::stage(lins_ctx* ctx, const DevCopy* src, int n, int base) {
  if (n <= 0) return LINS_OK;
  std::copy(src, src + n, host.p + base);
  CK(cudaMemcpyAsync(dev.p + base, host.p + base, sizeof(DevCopy) * n, cudaMemcpyHostToDevice, ctx->stream));
  return LINS_OK;
}

int CopyList::launch(lins_ctx* ctx, int base, int n) {
  if (n <= 0) return LINS_OK;
  lins_copy_kernel<<<n, 256, 0, ctx->stream>>>(dev.p + base);
  CK(cudaGetLastError());
  ctx->launches += 1;
  return LINS_OK;
}

int upload_clouds(lins_ctx* ctx, Resident& r, int n, const lins_point* const pts[4], const int32_t* const offs[4], int point_format) {
  CK(cudaStreamSynchronize(ctx->stream));  // the pinned staging of a previous upload may still be in flight
  if (n == 0) { r.n = 0; return LINS_OK; }
  static const char* const what[4] = {"bad surf_flat (or raw sweep) offsets / cloud", "bad corner_sharp offsets / cloud",
                                      "bad surf_less_flat offsets / cloud", "bad corner_less_sharp offsets / cloud"};
  for (int k = 0; k < 4; ++k) { const int rc = check_csr(ctx, offs[k], n, pts[k], what[k]); if (rc != LINS_OK) return rc; }
  if (point_format != LINS_POINTS_XYZI32 && point_format != LINS_POINTS_PACKED16) return fail(ctx, LINS_E_INVALID, "bad point_format");
  r.n = n;
  const bool packed16 = point_format == LINS_POINTS_PACKED16;  // the clouds are already (x, y, z, intensity) float4 records
  r.nqs = offs[0][n]; r.nqc = offs[1][n]; r.nts = offs[2][n]; r.ntc = offs[3][n];
  r.max_q = 0;
  for (int i = 0; i < n; ++i) r.max_q = std::max(r.max_q, (offs[0][i + 1] - offs[0][i]) + (offs[1][i + 1] - offs[1][i]));
  const size_t total = r.nqs + r.nqc + r.nts + r.ntc;
  CK(r.h_pts.reserve(total + 1)); CK(r.h_off.reserve(4 * (size_t)(n + 1)));
  CK(r.qs.reserve(r.nqs + 1)); CK(r.qc.reserve(r.nqc + 1)); CK(r.ts.reserve(r.nts + 1)); CK(r.tc.reserve(r.ntc + 1));
  CK(r.qs_off.reserve(n + 1)); CK(r.qc_off.reserve(n + 1)); CK(r.ts_off.reserve(n + 1)); CK(r.tc_off.reserve(n + 1));
  // pack 32-B PointXYZI -> 16-B float4 while copying into pinned staging (the copy is needed anyway: user
  // buffers are pageable), so PCIe moves half the bytes.  The pack is spread over host threads in 64 K-point
  // slices; each slice's H2D copy is queued as soon as the slice is packed, so packing and PCIe overlap.
  float4* hp = r.h_pts.p;
  size_t seg[5] = {0, r.nqs, r.nqs + r.nqc, r.nqs + r.nqc + r.nts, total};
  float4* dsts[4] = {r.qs.p, r.qc.p, r.ts.p, r.tc.p};
  int* doffs[4] = {r.qs_off.p, r.qc_off.p, r.ts_off.p, r.tc_off.p};
  // Clouds in caller-PINNED host memory (cudaHostAlloc / cudaHostRegister) can also go the other way: the copy engine reads
  // the raw 32-B records straight from the caller's buffer and a device kernel packs them — twice the PCIe bytes, but no host
  // pass over the points.  The clouds are cut into 64 K-point slices; pack threads take slices from the front of the list
  // (pack -> pinned staging -> 16-B H2D), a feeder hands slices from the back to the copy engine as raw records.
  // LINS_UPLOAD=pack: host pack only; =direct: raw DMA for every pinned cloud; =pinned: as direct, and an unpinned cloud
  // fails the call; =hybrid: both ends at once, the feeder never more than two slices ahead (kept for experiments: it did
  // not beat the better of the two pure modes).
  // pack threads: LINS_PACK_THREADS when set (a job that runs several contexts / ranks per host divides the cores
  // among them), else half the hardware threads, at most 32
  int want_threads;
  {
    unsigned hw = std::thread::hardware_concurrency();
    want_threads = (int)std::min<unsigned>(hw ? hw / 2 : 4, 32);
    if (const char* e = std::getenv("LINS_PACK_THREADS")) { const int v = std::atoi(e); if (v >= 1) want_threads = std::min(v, 64); }
  }
  const char* mode = std::getenv("LINS_UPLOAD");
  // default: host pack when this context has >= 8 pack threads to itself (measured, 2 GPUs x 3 contexts: 10 threads each
  // 6.1 M it/s per GPU; raw DMA 3.8 M whatever the threads; the two-ended split with 2-5 threads 3.3-3.6 M), raw DMA otherwise
  const bool p16 = packed16;  // (16-B records from pinned memory: always straight DMA)
  const bool mode_pack = mode ? std::strcmp(mode, "pack") == 0 : (want_threads >= 8 && !p16);
  const bool mode_direct = mode ? (std::strcmp(mode, "direct") == 0 || std::strcmp(mode, "pinned") == 0) : (want_threads < 8 || p16);
  bool pinned[4] = {false, false, false, false};
  bool any_pinned = false;
  for (int k = 0; k < 4 && !mode_pack; ++k) {
    if (seg[k + 1] == seg[k]) continue;
    cudaPointerAttributes at;
    if (cudaPointerGetAttributes(&at, pts[k]) == cudaSuccess && at.type == cudaMemoryTypeHost) { pinned[k] = true; any_pinned = true; }
    else cudaGetLastError();
    if (!pinned[k] && mode && std::strcmp(mode, "pinned") == 0) return fail(ctx, LINS_E_INVALID, "LINS_UPLOAD=pinned but a cloud is not in pinned host memory");
  }
  if (any_pinned && !packed16) CK(r.raw.reserve(2 * total + 2));
  {
    struct Slice { int k; size_t a, b; };
    std::vector<Slice> slices;  // unpinned clouds first: only the pack threads may take those
    const size_t SL = 1u << 16;
    size_t n_unpinned = 0;
    for (int pass = 0; pass < 2; ++pass)
      for (int k = 0; k < 4; ++k) {
        if ((pass == 0) == pinned[k]) continue;
        for (size_t a = 0; a < seg[k + 1] - seg[k]; a += SL) slices.push_back(Slice{k, a, std::min(a + SL, seg[k + 1] - seg[k])});
        if (pass == 0) n_unpinned = slices.size();
      }
    // one list, two ends: lo = next slice for the pack threads, hi = one past the last slice not yet taken by the DMA feeder
    std::mutex mu;
    size_t lo = 0, hi = slices.size();
    std::atomic<int> cuda_err(0);
    const int device = ctx->device;
    cudaStream_t stream = ctx->stream;
    auto take_front = [&](size_t& i) { std::lock_guard<std::mutex> g(mu); if (lo >= hi) return false; i = lo++; return true; };
    auto take_back = [&](size_t& i) { std::lock_guard<std::mutex> g(mu); if (lo >= hi || hi - 1 < n_unpinned) return false; i = --hi; return true; };
    auto worker = [&]() {
      cudaSetDevice(device);
      size_t i;
      while (take_front(i)) {
        const Slice& sl = slices[i];
        if (packed16) std::memcpy(hp + seg[sl.k] + sl.a, reinterpret_cast<const float4*>(pts[sl.k]) + sl.a, sizeof(float4) * (sl.b - sl.a));
        else pack_into(hp + seg[sl.k] + sl.a, pts[sl.k] + sl.a, (int)(sl.b - sl.a));
        cudaError_t e = cudaMemcpyAsync(dsts[sl.k] + sl.a, hp + seg[sl.k] + sl.a, sizeof(float4) * (sl.b - sl.a), cudaMemcpyHostToDevice, stream);
        if (e != cudaSuccess) cuda_err.store((int)e);
      }
    };
    const bool feed_raw = any_pinned && !mode_pack;
    int nthr = mode_direct && n_unpinned == 0 ? 0 : (int)std::min<size_t>((size_t)want_threads, std::max<size_t>(slices.size(), 1));
    // the DMA feeder (this thread): raw slices from the back, at most two in flight (all of them at once with LINS_UPLOAD=direct)
    auto feeder = [&]() {
      if (!feed_raw) return;
      cudaEvent_t ev[2] = {nullptr, nullptr};
      if (!mode_direct) for (auto& e : ev) if (cudaEventCreateWithFlags(&e, cudaEventDisableTiming) != cudaSuccess) { cuda_err.store((int)cudaGetLastError()); return; }
      size_t i;
      int turn = 0;
      while (take_back(i)) {
        const Slice& sl = slices[i];
        const size_t cnt = sl.b - sl.a;
        if (!mode_direct) cudaEventSynchronize(ev[turn]);  // (a never-recorded event is complete)
        cudaError_t e;
        if (packed16) {  // already in the device's format: one DMA, nothing else
          e = cudaMemcpyAsync(dsts[sl.k] + sl.a, reinterpret_cast<const float4*>(pts[sl.k]) + sl.a, sizeof(float4) * cnt, cudaMemcpyHostToDevice, stream);
        } else {
          float4* rawk = r.raw.p + 2 * (seg[sl.k] + sl.a);
          e = cudaMemcpyAsync(rawk, pts[sl.k] + sl.a, sizeof(lins_point) * cnt, cudaMemcpyHostToDevice, stream);
          const int blocks = (int)std::min<size_t>((cnt + 255) / 256, (size_t)ctx->sm_count * 4);
          lins_pack_points_kernel<<<blocks, 256, 0, stream>>>(rawk, dsts[sl.k] + sl.a, cnt);
          if (e == cudaSuccess) e = cudaGetLastError();
          if (e == cudaSuccess) ctx->launches += 1;
        }
        if (e != cudaSuccess) { cuda_err.store((int)e); break; }
        if (!mode_direct) { cudaEventRecord(ev[turn], stream); turn ^= 1; }
      }
      for (auto& e : ev) if (e) cudaEventDestroy(e);
    };
    if (nthr >= 1 && !slices.empty()) {
      // the pool runs the workers; the calling thread feeds the copy engine meanwhile (HostPool::run blocks, so the feeder is
      // the pool's first worker's prologue when only one thread is available)
      std::atomic<int> first(0);
      ctx->pool.run(nthr + (feed_raw ? 1 : 0), [&]() { if (feed_raw && first.fetch_add(1) == 0) { cudaSetDevice(device); feeder(); } else worker(); });
    } else {
      feeder();
    }
    if (cuda_err.load() != 0) return fail(ctx, LINS_E_CUDA, "H2D copy of a slice", (cudaError_t)cuda_err.load());
    // what went which way (lins_gpu_batch_upload_stats): slices [n_unpinned.., lo) were packed by the host, [hi, end) went raw
    size_t raw_pts = 0;
    for (size_t i = hi; i < slices.size(); ++i) raw_pts += slices[i].b - slices[i].a;
    if (packed16) raw_pts = 0;  // (16-B records either way)
    ctx->upload_raw_points += (int64_t)raw_pts;
    ctx->upload_packed_points += (int64_t)(total - raw_pts);
  }
  for (int k = 0; k < 4; ++k) std::memcpy(r.h_off.p + (size_t)k * (n + 1), offs[k], sizeof(int) * (n + 1));
  for (int k = 0; k < 4; ++k)
    CK(cudaMemcpyAsync(doffs[k], r.h_off.p + (size_t)k * (n + 1), sizeof(int) * (n + 1), cudaMemcpyHostToDevice, ctx->stream));
  return LINS_OK;
}

int upload_bytes(lins_ctx* ctx, void* dst, Buf<unsigned char, kPinned>& staging, const uint8_t* src, size_t n) {
  CK(cudaStreamSynchronize(ctx->stream));  // the pinned staging of a previous upload may still be in flight
  if (n == 0) return LINS_OK;
  cudaPointerAttributes at;
  if (cudaPointerGetAttributes(&at, src) == cudaSuccess && at.type == cudaMemoryTypeHost) {  // caller-pinned: one DMA
    CK(cudaMemcpyAsync(dst, src, n, cudaMemcpyHostToDevice, ctx->stream));
    return LINS_OK;
  }
  cudaGetLastError();
  CK(staging.reserve(n));
  // pool threads as upload_clouds counts them: LINS_PACK_THREADS, else half the hardware threads, at most 32
  int want_threads;
  {
    unsigned hw = std::thread::hardware_concurrency();
    want_threads = (int)std::min<unsigned>(hw ? hw / 2 : 4, 32);
    if (const char* e = std::getenv("LINS_PACK_THREADS")) { const int v = std::atoi(e); if (v >= 1) want_threads = std::min(v, 64); }
  }
  const size_t SL = 1u << 20, n_slices = (n + SL - 1) / SL;
  std::atomic<size_t> next(0);
  std::atomic<int> cuda_err(0);
  const int device = ctx->device;
  cudaStream_t stream = ctx->stream;
  unsigned char* hp = staging.p;
  ctx->pool.run((int)std::min<size_t>((size_t)want_threads, n_slices), [&]() {
    cudaSetDevice(device);
    for (size_t i; (i = next.fetch_add(1)) < n_slices;) {
      const size_t a = i * SL, len = std::min(SL, n - a);
      std::memcpy(hp + a, src + a, len);
      const cudaError_t e = cudaMemcpyAsync(static_cast<unsigned char*>(dst) + a, hp + a, len, cudaMemcpyHostToDevice, stream);
      if (e != cudaSuccess) cuda_err.store((int)e);
    }
  });
  if (cuda_err.load() != 0) return fail(ctx, LINS_E_CUDA, "H2D copy of a slice", (cudaError_t)cuda_err.load());
  return LINS_OK;
}

}  // namespace lins_capi

extern "C" {

int lins_gpu_batch_upload(lins_ctx* ctx, const lins_batch_desc* b) {
  if (!ctx) return LINS_E_INVALID;
  if (!b || b->n_scans < 0) return fail(ctx, LINS_E_INVALID, "bad batch");
  CK(cudaSetDevice(ctx->device));
  Resident& r = ctx->batch;
  const int n = b->n_scans;
  if (n > 0 && (!b->state_in || !b->cov_in)) return fail(ctx, LINS_E_INVALID, "null prior");
  const int32_t* offs[4] = {b->surf_flat_off, b->corner_sharp_off, b->surf_less_flat_off, b->corner_less_sharp_off};
  const lins_point* pts[4] = {b->surf_flat, b->corner_sharp, b->surf_less_flat, b->corner_less_sharp};
  int rc = upload_clouds(ctx, r, n, pts, offs, b->point_format);
  if (rc != LINS_OK || n == 0) return rc;
  CK(r.h_state.reserve((size_t)n * 20)); CK(r.h_cov.reserve((size_t)n * 324));
  CK(r.state_in.reserve((size_t)n * 20)); CK(r.cov_in.reserve((size_t)n * 324));
  pad_states(r.h_state.p, b->state_in, n);
  std::memcpy(r.h_cov.p, b->cov_in, sizeof(double) * 324 * (size_t)n);
  CK(cudaMemcpyAsync(r.state_in.p, r.h_state.p, sizeof(double) * 20 * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(r.cov_in.p, r.h_cov.p, sizeof(double) * 324 * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  return reserve_outputs(ctx, r, true, false);
}

int lins_gpu_batch_upload_stats(lins_ctx* ctx, int64_t* packed_points, int64_t* raw_points) {
  if (!ctx) return LINS_E_INVALID;
  if (packed_points) *packed_points = ctx->upload_packed_points;
  if (raw_points) *raw_points = ctx->upload_raw_points;
  return LINS_OK;
}

}  // extern "C"
