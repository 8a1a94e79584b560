// lins_cloud2.cu — sensor_msgs/PointCloud2 on the device: pcl::fromROSMsg<pcl::PointXYZI> of copyPointCloud
// (image_projection_node.cpp:172-177) for a batch of messages (lins_gpu_decode_cloud2), and sequence mode from the
// messages (lins_gpu_seq_step_cloud2, lins_seq.cu).  The contract is the host decoder csrc/host/rosbag_reader.hpp
// decode_pointcloud2, bit for bit; the per-field conversion and the layout check are lins_cloud2.cuh.  Built with
// -fmad=false like its neighbours.  DESIGN.md §4.8.
//
// The messages' data fields are uploaded as they are (one blob, lins_upload.cu: upload_bytes), then one thread per point
// writes the packed (x, y, z, intensity) float4 record lins_projection_kernel reads, in row-major order at the message's
// prefix-sum offset.  Nothing in the blob is aligned: point_step may be 22, and a data field starts wherever the message
// put it.  Every field is assembled from aligned 32-bit words with funnel shifts (the blob's device copy is word aligned
// and padded by 16 bytes, so the word after a field's last byte is always inside the allocation); no load is wider than
// its alignment.
#include <cuda_runtime.h>

#include <climits>
#include <cstring>
#include <vector>

#include "lins_cloud2.cuh"
#include "lins_ctx.hpp"

using namespace lins_capi;

namespace {

constexpr int kThreads = 256;
constexpr size_t kBlobPad = 16;  // bytes past the blob's end that the word loads may touch

// the little-endian bits of the size-byte field at byte a of the word-aligned blob w (size <= 8)
__device__ __forceinline__ uint64_t load_field(const unsigned* __restrict__ w, unsigned long long a, unsigned size) {
  const unsigned long long i = a >> 2;
  const unsigned sh = (unsigned)(a & 3u) * 8u;
  const unsigned w0 = __ldg(w + i), w1 = __ldg(w + i + 1);
  const unsigned lo = __funnelshift_r(w0, w1, sh);
  if (size <= 4) return lo;  // (to_float reads the low size bytes only)
  const unsigned hi = __funnelshift_r(w1, __ldg(w + i + 2), sh);
  return ((uint64_t)hi << 32) | lo;
}

__global__ void __launch_bounds__(kThreads) lins_cloud2_decode_kernel(const unsigned* __restrict__ blob, const Cloud2Scan* __restrict__ scans,
                                                                     const int* __restrict__ prefix, int n, int total, float4* __restrict__ out) {
  // (64-bit index: total may come within a grid stride of INT32_MAX, where an int index would wrap)
  for (long long i = (long long)blockIdx.x * kThreads + threadIdx.x; i < total; i += (long long)gridDim.x * kThreads) {
    int lo = 0, hi = n - 1;  // the message of point i: the last one whose first point is <= i (empty messages skipped)
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (__ldg(prefix + mid) <= i) lo = mid; else hi = mid - 1;
    }
    const Cloud2Scan& s = scans[lo];
    const unsigned k = (unsigned)(i - s.out), r = k / s.width, c = k - r * s.width;
    const unsigned long long p = (unsigned long long)s.base + (unsigned long long)r * s.row_step + (unsigned long long)c * s.point_step;
    float v[4];
#pragma unroll
    for (int f = 0; f < 4; ++f) {
      const unsigned dt = s.datatype[f];
      v[f] = dt ? lins_cloud2::to_float(load_field(blob, p + s.offset[f], lins_cloud2::type_size(dt)), dt) : 0.f;
    }
    out[i] = make_float4(v[0], v[1], v[2], v[3]);
  }
}

// the host validation of cloud2_run: off (n + 1) and one decode record per message, or LINS_E_INVALID
int cloud2_check(lins_ctx* ctx, const lins_cloud2_desc* d, const uint8_t* present, std::vector<int32_t>& off, std::vector<Cloud2Scan>& sc) {
  if (!d || d->n_scans < 0) return fail(ctx, LINS_E_INVALID, "bad PointCloud2 descriptor");
  const int n = d->n_scans;
  if (!d->data_off || (n > 0 && !d->layouts)) return fail(ctx, LINS_E_INVALID, "null data_off / layouts");
  for (int i = 0; i < n; ++i)
    if (d->data_off[i] < 0 || d->data_off[i + 1] < d->data_off[i]) return fail(ctx, LINS_E_INVALID, "data_off must be non-negative and non-decreasing");
  const int64_t b0 = n > 0 ? d->data_off[0] : 0, bytes = n > 0 ? d->data_off[n] - b0 : 0;
  if (bytes > 0 && !d->data) return fail(ctx, LINS_E_INVALID, "null data");
  // every message the kernel will read is checked here, in 64-bit (or wider) arithmetic, before anything is uploaded
  off.assign((size_t)n + 1, 0);
  sc.assign((size_t)std::max(n, 1), Cloud2Scan{});
  int64_t total = 0;
  for (int i = 0; i < n; ++i) {
    off[i] = (int32_t)total;
    if (present && !present[i]) continue;
    const lins_cloud2_layout& l = d->layouts[i];
    const char* why = lins_cloud2::check_layout(l, d->data_off[i + 1] - d->data_off[i]);
    if (why) return fail(ctx, LINS_E_INVALID, why);
    total += (int64_t)l.width * l.height;
    if (total > INT_MAX) return fail(ctx, LINS_E_INVALID, "more than INT32_MAX points");
    Cloud2Scan& s = sc[i];
    s.base = d->data_off[i] - b0; s.out = off[i];
    s.width = l.width; s.point_step = l.point_step; s.row_step = l.row_step;
    for (int f = 0; f < 4; ++f) { s.offset[f] = l.offset[f]; s.datatype[f] = l.datatype[f]; }
  }
  off[n] = (int32_t)total;
  return LINS_OK;
}

// upload the checked messages and queue their decode (off, sc: cloud2_check's)
int cloud2_launch(lins_ctx* ctx, const lins_cloud2_desc* d, const std::vector<int32_t>& off, const std::vector<Cloud2Scan>& sc) {
  const int n = d->n_scans;
  const int64_t b0 = n > 0 ? d->data_off[0] : 0, bytes = n > 0 ? d->data_off[n] - b0 : 0, total = off[n];
  CK(cudaSetDevice(ctx->device));
  Cloud2State& c = ctx->c2;
  Resident& up = ctx->proj.up;
  CK(c.blob.reserve(((size_t)bytes + kBlobPad) / 4 + 1));
  int rc = upload_bytes(ctx, c.blob.p, c.h_blob, d->data ? d->data + b0 : nullptr, (size_t)bytes);  // (synchronises first)
  if (rc != LINS_OK) return rc;
  up.n = n;
  CK(up.qs.reserve((size_t)total + 1)); CK(up.qs_off.reserve((size_t)n + 1));
  CK(c.scans.reserve((size_t)std::max(n, 1))); CK(c.h_scans.reserve((size_t)std::max(n, 1)));
  CK(c.prefix.reserve((size_t)n + 1)); CK(c.h_prefix.reserve((size_t)n + 1));
  std::memcpy(c.h_scans.p, sc.data(), sizeof(Cloud2Scan) * sc.size());
  std::memcpy(c.h_prefix.p, off.data(), sizeof(int32_t) * off.size());
  CK(cudaMemcpyAsync(c.scans.p, c.h_scans.p, sizeof(Cloud2Scan) * sc.size(), cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(c.prefix.p, c.h_prefix.p, sizeof(int32_t) * off.size(), cudaMemcpyHostToDevice, ctx->stream));
  CK(cudaMemcpyAsync(up.qs_off.p, c.prefix.p, sizeof(int32_t) * off.size(), cudaMemcpyDeviceToDevice, ctx->stream));
  CK(c.ev.start(ctx->stream));
  if (total > 0) {
    const int blocks = (int)std::min<int64_t>((total + kThreads - 1) / kThreads, (int64_t)ctx->sm_count * 16);
    lins_cloud2_decode_kernel<<<blocks, kThreads, 0, ctx->stream>>>(c.blob.p, c.scans.p, c.prefix.p, n, (int)total, up.qs.p);
    CK(cudaGetLastError());
    ctx->launches += 1;
  }
  CK(c.ev.stop(ctx->stream));
  return LINS_OK;
}

}  // namespace

namespace lins_capi {

int cloud2_run(lins_ctx* ctx, const lins_cloud2_desc* d, const uint8_t* present, std::vector<int32_t>& off) {
  std::vector<Cloud2Scan> sc;
  const int rc = cloud2_check(ctx, d, present, off, sc);
  return rc != LINS_OK ? rc : cloud2_launch(ctx, d, off, sc);
}

}  // namespace lins_capi

extern "C" {

int lins_gpu_decode_cloud2(lins_ctx* ctx, const lins_cloud2_desc* d, lins_point* out, int32_t* counts) {
  if (!ctx) return LINS_E_INVALID;
  std::vector<int32_t> off;
  std::vector<Cloud2Scan> sc;
  int rc = cloud2_check(ctx, d, nullptr, off, sc);
  if (rc != LINS_OK) return rc;
  const int n = d->n_scans;
  const size_t total = (size_t)off[n];
  if (total > 0 && !out) return fail(ctx, LINS_E_INVALID, "null output cloud");
  rc = cloud2_launch(ctx, d, off, sc);
  if (rc != LINS_OK) return rc;
  Cloud2State& c = ctx->c2;
  CK(c.h_out.reserve(total + 1));
  if (total) CK(cudaMemcpyAsync(c.h_out.p, ctx->proj.up.qs.p, sizeof(float4) * total, cudaMemcpyDeviceToHost, ctx->stream));
  CK(cudaStreamSynchronize(ctx->stream));
  for (size_t i = 0; i < total; ++i) out[i] = unpack_point(c.h_out.p[i]);
  if (counts) for (int i = 0; i < n; ++i) counts[i] = off[i + 1] - off[i];
  return LINS_OK;
}

int lins_gpu_decode_ms(lins_ctx* ctx, float* ms) {
  if (!ctx) return LINS_E_INVALID;
  return event_ms(ctx, ctx->c2.ev, ms, "no decode has run");
}

}  // extern "C"
