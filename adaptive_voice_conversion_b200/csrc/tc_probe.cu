// wgmma self-test: D[128][N] = sum over `nk` K=8 steps of A_k (128x8) * B_k (Nx8)^T with tf32 inputs / fp32
// accumulation, operands given as raw shared-memory images plus the descriptor strides.  tests/test_gpu_tc.py uses it
// to pin the descriptor conventions the conv kernels rely on (no-swizzle K-major core-matrix layout, row-offset tap
// shifts).  Two warpgroups: rows 0-63 and 64-127 (the A descriptor of the second starts 8 core-matrix groups further).
#include "common.cuh"
#include "tc_common.cuh"

namespace avc {

struct ProbeArgs {
  const float* a_img;
  const float* b_img;
  int a_bytes, b_bytes;
  uint32_t a_lbo, a_sbo, b_lbo, b_sbo, a_kstep, b_kstep, a_off, b_off;
  int nk, N, reps, ld_shift;
  float* D;
  int* status;
};

template <int N>
__device__ __forceinline__ void probe_run(const ProbeArgs& a, uint32_t sa, uint32_t sb, int wg, int wt) {
  float acc[N / 2];
  tc::wgmma_fence();
  for (int r = 0; r < a.reps; ++r)
    for (int k = 0; k < a.nk; ++k) {
      const uint64_t ad = tc::make_sdesc(sa + a.a_off + k * a.a_kstep + (uint32_t)wg * 8u * a.a_sbo, a.a_lbo, a.a_sbo);
      const uint64_t bd = tc::make_sdesc(sb + a.b_off + k * a.b_kstep, a.b_lbo, a.b_sbo);
      tc::wgmma_tf32<N>(acc, ad, bd, (k > 0 || r > 0) ? 1u : 0u);
    }
  tc::wgmma_commit();
  tc::wgmma_wait<0>();
  tc::acc_fence(acc, N / 2);
  // ld_shift: columns before it stay untouched (pins that the caller's column window is honoured)
#pragma unroll
  for (int i = 0; i < N / 2; ++i) {
    const int row = 64 * wg + tc::wg_acc_row(wt, i), col = tc::wg_acc_col(wt, i);
    if (col >= a.ld_shift) a.D[(size_t)row * N + col] = acc[i];
  }
}

__global__ void __launch_bounds__(256) tc_probe_kernel(const ProbeArgs a) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const int tid = threadIdx.x, wg = tid >> 7, wt = tid & 127;
  uint8_t* sa = smem;
  uint8_t* sb = smem + ((a.a_bytes + 1023) / 1024) * 1024;
  for (int i = tid; i < a.a_bytes / 16; i += 256) reinterpret_cast<float4*>(sa)[i] = reinterpret_cast<const float4*>(a.a_img)[i];
  for (int i = tid; i < a.b_bytes / 16; i += 256) reinterpret_cast<float4*>(sb)[i] = reinterpret_cast<const float4*>(a.b_img)[i];
  tc::fence_proxy_async_smem();
  __syncthreads();
  const long long t0 = clock64();
  switch (a.N) {
#define PROBE_CASE(n) \
  case n: probe_run<n>(a, tc::smem_u32(sa), tc::smem_u32(sb), wg, wt); break;
    PROBE_CASE(16) PROBE_CASE(32) PROBE_CASE(48) PROBE_CASE(64) PROBE_CASE(80) PROBE_CASE(96) PROBE_CASE(112) PROBE_CASE(128)
    PROBE_CASE(144) PROBE_CASE(160) PROBE_CASE(176) PROBE_CASE(192) PROBE_CASE(208) PROBE_CASE(224) PROBE_CASE(240) PROBE_CASE(256)
#undef PROBE_CASE
  }
  if (tid == 0) {
    a.status[0] = 0;
    a.status[1] = (int)(clock64() - t0);  // cycles: issue of the first MMA -> all complete (warpgroup 0)
  }
}

}  // namespace avc

using namespace avc;

static int g_probe_ld_shift = 0;
extern "C" void avc_tc_probe_set_ld_shift(int shift) { g_probe_ld_shift = shift < 0 ? 0 : shift; }

extern "C" int avc_tc_probe_gemm(const float* a_img, int a_bytes, const float* b_img, int b_bytes, const uint32_t* strides /*[10]*/,
                                 int nk, int N, int a_mn, int b_mn, int reps, float* D, int* status, void* stream) {
  AVC_REQUIRE(a_img && b_img && strides && D && status, AVC_ERR_INVALID, "avc_tc_probe_gemm: null argument");
  AVC_REQUIRE(a_bytes % 16 == 0 && b_bytes % 16 == 0 && N % 16 == 0 && N >= 16 && N <= 256 && nk >= 1, AVC_ERR_INVALID,
              "avc_tc_probe_gemm: bad sizes");
  // tf32 wgmma reads K-major operands only, and the kernels use the no-swizzle layout
  AVC_REQUIRE(a_mn == 0 && b_mn == 0 && strides[8] == 0 && strides[9] == 0, AVC_ERR_UNSUPPORTED,
              "avc_tc_probe_gemm: tf32 operands must be K-major without swizzle");
  ProbeArgs a;
  a.a_img = a_img; a.b_img = b_img; a.a_bytes = a_bytes; a.b_bytes = b_bytes;
  a.a_lbo = strides[0]; a.a_sbo = strides[1]; a.b_lbo = strides[2]; a.b_sbo = strides[3];
  a.a_kstep = strides[4]; a.b_kstep = strides[5]; a.a_off = strides[6]; a.b_off = strides[7];
  a.nk = nk; a.N = N; a.reps = reps < 1 ? 1 : reps; a.ld_shift = g_probe_ld_shift; a.D = D; a.status = status;
  const int smem = ((a_bytes + 1023) / 1024) * 1024 + b_bytes + 1024;
  AVC_REQUIRE(smem <= 200 * 1024, AVC_ERR_INVALID, "avc_tc_probe_gemm: images too large");
  cudaError_t e = cudaFuncSetAttribute(tc_probe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
  if (e != cudaSuccess) { set_error("avc_tc_probe_gemm: %s", cudaGetErrorString(e)); return AVC_ERR_CUDA; }
  tc_probe_kernel<<<1, 256, smem, (cudaStream_t)stream>>>(a);
  AVC_CHECK_LAUNCH("tc_probe");
  return AVC_OK;
}
