// On-device segment gather: one training batch cut out of the device-resident mel corpus (data_utils.DeviceSegments).
//
// The crop of index entry e is the seg rows corpus[starts[e] .. starts[e] + seg) of n_mels floats.  Read as a
// [T][C] matrix (T = seg / frame time steps, C = frame * n_mels channels: row tau holds frames tau*frame + j, j < frame,
// back to back) it is exactly the transpose of the sample CollateFn produces, x[b] = [C][T] (data_utils.py).  So the
// gather is a batched transpose: a CTA stages a 32 (time) x 64 (channel) tile in shared memory, reading 16-byte vectors
// along the channel axis, and writes it back as 32-float runs along time.  A plain copy: the result is exact.
#include "common.cuh"

namespace avc {

constexpr int GT_T = 32;   // time steps per tile
constexpr int GT_C = 64;   // channels per tile (16 float4 per time step)
constexpr int GT_THREADS = 256;

__global__ void __launch_bounds__(GT_THREADS) segment_gather_kernel(const avc_gather_desc d) {
  __shared__ float tile[GT_C][GT_T + 1];
  const int T = d.seg / d.frame, C = d.frame * d.n_mels;
  const int b = blockIdx.x, c0 = blockIdx.y * GT_C, t0 = blockIdx.z * GT_T;
  const int64_t start = __ldg(d.starts + __ldg(d.order + d.first + b));
  const float* src = d.corpus + start * d.n_mels;   // [T][C], row pitch C
  // load: 32 rows x 16 float4, two per thread; lanes 0-15 / 16-31 of a warp cover two consecutive rows
  const int q = threadIdx.x & 15;
#pragma unroll
  for (int r = threadIdx.x >> 4; r < GT_T; r += GT_THREADS / 16) {
    const int t = t0 + r, c = c0 + 4 * q;
    if (t < T && c < C) {
      const float4 v = ldg4(src + (int64_t)t * C + c);
      tile[4 * q + 0][r] = v.x;
      tile[4 * q + 1][r] = v.y;
      tile[4 * q + 2][r] = v.z;
      tile[4 * q + 3][r] = v.w;
    }
  }
  __syncthreads();
  // store: one warp per channel row, 32 consecutive time steps per warp instruction
  const int lane = threadIdx.x & 31, t = t0 + lane;
  float* dst = d.x + (int64_t)b * C * T;
  if (t < T) {
    for (int cc = threadIdx.x >> 5; cc < GT_C && c0 + cc < C; cc += GT_THREADS / 32)
      dst[(int64_t)(c0 + cc) * T + t] = tile[cc][lane];
  }
}

}  // namespace avc

using namespace avc;

extern "C" int avc_segment_gather(const avc_gather_desc* d, void* stream) {
  AVC_REQUIRE(d != nullptr, AVC_ERR_INVALID, "avc_segment_gather: null descriptor");
  AVC_REQUIRE(d->corpus != nullptr && d->starts != nullptr && d->order != nullptr && d->x != nullptr, AVC_ERR_INVALID,
              "avc_segment_gather: null pointer (corpus %p, starts %p, order %p, x %p)", (const void*)d->corpus,
              (const void*)d->starts, (const void*)d->order, (const void*)d->x);
  AVC_REQUIRE(d->n_mels > 0 && d->n_mels % 4 == 0, AVC_ERR_INVALID, "avc_segment_gather: n_mels must be a positive multiple of 4 (got %d)",
              d->n_mels);
  AVC_REQUIRE(d->frame > 0 && d->seg > 0 && d->seg % d->frame == 0, AVC_ERR_INVALID,
              "avc_segment_gather: seg must be a positive multiple of frame (seg %d, frame %d)", d->seg, d->frame);
  AVC_REQUIRE(d->batch >= 1, AVC_ERR_INVALID, "avc_segment_gather: batch must be >= 1 (got %d)", d->batch);
  AVC_REQUIRE(d->first >= 0, AVC_ERR_INVALID, "avc_segment_gather: first must be >= 0 (got %lld)", (long long)d->first);
  const int T = d->seg / d->frame;
  const int64_t C = (int64_t)d->frame * d->n_mels;
  AVC_REQUIRE(cdiv64(C, GT_C) <= 65535 && cdiv(T, GT_T) <= 65535, AVC_ERR_UNSUPPORTED,
              "avc_segment_gather: %lld channels x %d steps exceed the launch grid", (long long)C, T);
  const dim3 grid((unsigned)d->batch, (unsigned)cdiv64(C, GT_C), (unsigned)cdiv(T, GT_T));
  segment_gather_kernel<<<grid, GT_THREADS, 0, (cudaStream_t)stream>>>(*d);
  AVC_CHECK_LAUNCH("avc_segment_gather");
  return AVC_OK;
}
