// Conv weight gradient on the tensor cores (mma.sync m16n8k8, TF32 in, fp32 accumulate in registers):
//   dW[co][ci][j] += sum_{b,t} dc[b][co][t] * xpad[b][ci][t + j]        (stride 1)
// (autograd of pad_layer + nn.Conv1d w.r.t. the weight, model.py:21-32 under solver.py:90).
//
// GEMM view: M = co (128 per CTA), N = taps x ci (WT_NT ci per CTA), reduction K = time rows of a batch
// slice.  The A4 activation layout [c/4][t][4] keeps 4 channels of one time step in a 16-byte unit,
// so staging is a plain cp.async of units into an XOR-swizzled MN-major tile:
//     byte(c, row) = (c/32)*LBO + row*128 + ((((c%32)/8) ^ (row%4)) * 32) + (c%8)*4
// (conflict-free 16-byte stores).  tf32 wgmma reads K-major operands only, so the MMAs are warp-level:
// every warp owns 16 co rows and loads its fragments from the staged tile with 32-bit shared loads.
// The K taps are row shifts into ONE staged input tile whose reflect padding is resolved while staging.
// Each CTA owns (co tile, ci tile, batch slice); partial sums go to a scratch buffer
// [slice][tap][ci/4][co][4] and are reduced into the canonical nn.Conv1d gradient layout by
// wgrad_tc_reduce_kernel (deterministic, no atomics), or added in place (ATOMIC, see below).
#include "common.cuh"
#include "tc_common.cuh"

namespace avc {

constexpr int WT_NT = 32;  // ci columns per CTA (K x 32 accumulator columns: <= 128 registers per thread)

struct WgTcArgs {
  avc_wgrad_desc d;
  float* scratch;
  int nslices, tiles_per_slice, G, RA, RX, ntpad, coutp, TX, H;  // H: rows of one parity block (stride 2)
  uint32_t buf_bytes, x_off;
  int* status;
};

__device__ __forceinline__ float rtf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}
__device__ __forceinline__ float4 rtf32_4(float4 v) { return make_float4(rtf32(v.x), rtf32(v.y), rtf32(v.z), rtf32(v.w)); }

// 16-byte async global->shared copy; !valid writes zeros (src-size 0, nothing is read)
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc, bool valid) {
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(tc::smem_u32(smem_dst)), "l"(gsrc), "r"(sz) : "memory");
}

// byte offset of the 16-byte unit (channel chunk q = c/4, row) inside an operand buffer
__device__ __forceinline__ uint32_t mn_unit_off(int q, int row, uint32_t atom_bytes) {
  return (uint32_t)(q >> 3) * atom_bytes + (uint32_t)row * 128u + (uint32_t)((((q & 7) >> 1) ^ (row & 3)) << 5) + (uint32_t)((q & 1) << 4);
}

// one m16n8k8 TF32 tensor-core MMA (operands are fp32 bit patterns; the tensor core reads their TF32 part)
__device__ __forceinline__ void mma_tf32_16x8x8(float* c, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0, %1, %2, %3}, {%4, %5, %6, %7}, {%8, %9}, {%0, %1, %2, %3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t lds_u32(const uint8_t* p) { return *reinterpret_cast<const uint32_t*>(p); }

// Accumulator of one warp: co rows 16 warp + lane / 4 (+ 8) of the 128-row tile, n8 tile nt = 4 tap + (ci / 8) of the
// WT_NT = 32 ci columns; acc[4 nt + {0, 1}] = columns 8 (nt % 4) + 2 (lane % 4) + {0, 1}, acc[4 nt + {2, 3}] the row + 8.
constexpr int WG_NT_MAX = 4 * 8;   // n8 tiles for K <= 8

// All MMAs of one staged tile (nsamp samples, reduction over their time rows) for the warp's 16 co rows.
__device__ __forceinline__ void wgrad_mma_tile(const WgTcArgs& a, const uint8_t* sA, const uint8_t* sX, int nsamp, float* acc, int warp,
                                               int lane) {
  const int K = a.d.K, T = a.d.Tout, S = a.d.stride, H = a.H, TX = a.TX;
  const uint32_t atomA = (uint32_t)a.RA * 128u, atomX = (uint32_t)a.RX * 128u;
  const int gid = lane >> 2, tig = lane & 3;
  const int m0 = warp * 16 + gid, m1 = m0 + 8;
  const uint8_t* pA0 = sA + ((m0 & 3) << 2);
  const uint8_t* pA1 = sA + ((m1 & 3) << 2);
  for (int g = 0; g < nsamp; ++g) {
    for (int ks = 0; ks < T / 8; ++ks) {
      const int r0 = g * T + 8 * ks + tig;
      const uint32_t a0 = lds_u32(pA0 + mn_unit_off(m0 >> 2, r0, atomA)), a1 = lds_u32(pA1 + mn_unit_off(m1 >> 2, r0, atomA));
      const uint32_t a2 = lds_u32(pA0 + mn_unit_off(m0 >> 2, r0 + 4, atomA)), a3 = lds_u32(pA1 + mn_unit_off(m1 >> 2, r0 + 4, atomA));
#pragma unroll
      for (int nt = 0; nt < WG_NT_MAX; ++nt) {
        if (nt < 4 * K) {
          const int j = nt >> 2, n = (nt & 3) * 8 + gid;
          // tap j reads padded input position t + j (stride 1), or parity block j & 1, row t + j / 2 (stride 2)
          const int xr = (S == 1 ? g * TX + j : g * 2 * H + (j & 1) * H + (j >> 1)) + 8 * ks + tig;
          const uint8_t* pX = sX + ((n & 3) << 2);
          const uint32_t b0 = lds_u32(pX + mn_unit_off(n >> 2, xr, atomX)), b1 = lds_u32(pX + mn_unit_off(n >> 2, xr + 4, atomX));
          mma_tf32_16x8x8(acc + 4 * nt, a0, a1, a2, a3, b0, b1);
        }
      }
    }
  }
}

// partial dW of this CTA: scratch[sl][tap][ci/4][co][4] (ATOMIC: added into the layer's accumulation buffer)
template <bool ATOMIC>
__device__ __forceinline__ void wgrad_store(const WgTcArgs& a, const float* acc, int warp, int lane) {
  const avc_wgrad_desc& d = a.d;
  const int ci0 = blockIdx.x * WT_NT, co0 = blockIdx.y * 128, sl = blockIdx.z;
  const int gid = lane >> 2, tig = lane & 3;
#pragma unroll
  for (int nt = 0; nt < WG_NT_MAX; ++nt) {
    if (nt < 4 * d.K) {
      const int j = nt >> 2, ci = ci0 + (nt & 3) * 8 + 2 * tig;
      if (ci < d.Cin) {
        float* sbase = a.scratch + (((size_t)(ATOMIC ? 0 : sl) * d.K + j) * (size_t)(d.Cin >> 2)) * (size_t)a.coutp * 4;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const int co = co0 + warp * 16 + gid + 8 * h;
          float* p = sbase + ((size_t)(ci >> 2) * a.coutp + co) * 4 + (ci & 3);
          const float v0 = acc[4 * nt + 2 * h], v1 = acc[4 * nt + 2 * h + 1];
          if constexpr (ATOMIC)
            asm volatile("red.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(v0), "f"(v1) : "memory");
          else
            *reinterpret_cast<float2*>(p) = make_float2(v0, v1);
        }
      }
    }
  }
}

constexpr int WG_THREADS = 256;   // 8 warps: staging, then 16 co rows of MMAs each

// Stage one tile of operands with cp.async: dc as [4 atoms of 32 co][G*T rows][128 B], x with the reflect padding resolved
// as [ntpad/32 atoms][G*(T+K-1) rows][128 B] (stride 2: even and odd padded positions in separate row blocks, so tap j
// addresses rows (j&1)*H + t + (j>>1) -- contiguous in t).  A warp writes 4 rows x the 8 units of one 128-byte atom row
// (four whole bank sweeps); each thread walks its rows with (g, t) kept incrementally.
__device__ __forceinline__ void wgrad_stage(const WgTcArgs& a, uint8_t* sA, uint8_t* sX, int b0, int nsamp, int tid) {
  const avc_wgrad_desc& d = a.d;
  const int ci0 = blockIdx.x * WT_NT, co0 = blockIdx.y * 128;
  const int T = d.Tout, TX = a.TX, S = d.stride, H = a.H;
  const uint32_t atomA = (uint32_t)a.RA * 128u, atomX = (uint32_t)a.RX * 128u;
  {
    const int q = ((tid >> 5) & 3) * 8 + (tid & 7), r_lo = ((tid >> 7) << 2) + ((tid >> 3) & 3);
    const int co = co0 + 4 * q;
    const bool cv = co < d.Cout;
    const float* colsrc = d.dc + (size_t)((cv ? co : 0) >> 2) * T * 4;
    int g = r_lo / T, t = r_lo - g * T;
    for (int r = r_lo; r < nsamp * T; r += 8) {
      cp_async16(sA + mn_unit_off(q, r, atomA), colsrc + (size_t)(b0 + g) * d.dc_bstride + (size_t)t * 4, cv);
      t += 8;
      while (t >= T) { t -= T; ++g; }
    }
  }
  {
    const int nq_x = a.ntpad >> 2;
    const int natom = nq_x >> 3, wpa = 8 / natom;             // warps per atom
    const int w = tid >> 5, atom = w % natom, rg = w / natom;  // row group of this warp
    const int q = atom * 8 + (tid & 7), r_lo = (rg << 2) + ((tid >> 3) & 3), rstep = wpa << 2;
    const int ci = ci0 + 4 * q;
    const bool civ = ci < d.Cin;
    const float* colsrc = d.x + (size_t)((civ ? ci : 0) >> 2) * d.Tin * 4;
    int g = r_lo / TX, u = r_lo - g * TX;
    for (int r0 = r_lo; r0 < nsamp * TX; r0 += rstep) {
      const int r = S == 1 ? r0 : g * 2 * H + (u & 1) * H + (u >> 1);
      const int p = src_pos(u - d.pad_left, d.Tin, AVC_PAD_REFLECT, 1);
      const bool v = civ && p >= 0;
      cp_async16(sX + mn_unit_off(q, r, atomX), colsrc + (size_t)(b0 + g) * d.x_bstride + (size_t)(p >= 0 ? p : 0) * 4, v);
      u += rstep;
      while (u >= TX) { u -= TX; ++g; }
    }
  }
  asm volatile("cp.async.commit_group;" ::: "memory");
}

// Weight gradient of one (ci tile, co tile, batch slice): the copies of tile i+1 are in flight (cp.async, second
// buffer) while the MMAs of tile i run.
template <bool ATOMIC>
__global__ void __launch_bounds__(WG_THREADS, 1) conv_wgrad_split_kernel(const WgTcArgs a) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int tile0 = blockIdx.z * a.tiles_per_slice;
  const int tile1 = min(cdiv(a.d.B, a.G), tile0 + a.tiles_per_slice);
  float acc[4 * WG_NT_MAX];
#pragma unroll
  for (int i = 0; i < 4 * WG_NT_MAX; ++i) acc[i] = 0.f;
  if (tile1 > tile0) wgrad_stage(a, smem, smem + a.x_off, tile0 * a.G, min(a.G, a.d.B - tile0 * a.G), tid);
  for (int tile = tile0; tile < tile1; ++tile) {
    const int it = tile - tile0;
    uint8_t* sA = smem + (size_t)(it & 1) * a.buf_bytes;
    if (tile + 1 < tile1) {
      uint8_t* sN = smem + (size_t)((it + 1) & 1) * a.buf_bytes;
      wgrad_stage(a, sN, sN + a.x_off, (tile + 1) * a.G, min(a.G, a.d.B - (tile + 1) * a.G), tid);
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    wgrad_mma_tile(a, sA, sA + a.x_off, min(a.G, a.d.B - tile * a.G), acc, warp, lane);
    __syncthreads();   // the buffer is restaged two tiles later
  }
  if (tile1 > tile0) wgrad_store<ATOMIC>(a, acc, warp, lane);
}

// dW[co][ci][j] += sum over slices of scratch[sl][j][ci/4][co][ci%4]
// block (32, 8): x = output float4 (coalesced 512 B per warp), y = slice group; four independent 16-byte loads in
// flight per thread (the partials sit in L2)
__global__ void __launch_bounds__(256) wgrad_tc_reduce_kernel(const float* __restrict__ scratch, float* __restrict__ dw, int Cout, int Cin,
                                                              int K, int coutp, int nslices) {
  __shared__ float4 part[8][32];
  const int64_t n = (int64_t)K * (Cin >> 2) * coutp;
  const int64_t slice_stride = n * 4;
  const int64_t i = (int64_t)blockIdx.x * 32 + threadIdx.x;
  float4 s = zero4();
  if (i < n) {
    int sl = threadIdx.y;
    float4 s1 = zero4();
    const float* p = scratch + i * 4;
    for (; sl + 24 < nslices; sl += 32) {
      const float4 v0 = ldg4(p + (sl + 0) * slice_stride), v1 = ldg4(p + (sl + 8) * slice_stride);
      const float4 v2 = ldg4(p + (sl + 16) * slice_stride), v3 = ldg4(p + (sl + 24) * slice_stride);
      s.x += v0.x + v2.x; s.y += v0.y + v2.y; s.z += v0.z + v2.z; s.w += v0.w + v2.w;
      s1.x += v1.x + v3.x; s1.y += v1.y + v3.y; s1.z += v1.z + v3.z; s1.w += v1.w + v3.w;
    }
    s.x += s1.x; s.y += s1.y; s.z += s1.z; s.w += s1.w;
    for (; sl < nslices; sl += 8) {
      const float4 v = ldg4(scratch + sl * slice_stride + i * 4);
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
  }
  part[threadIdx.y][threadIdx.x] = s;
  __syncthreads();
  if (threadIdx.y == 0 && i < n) {
#pragma unroll
    for (int y = 1; y < 8; ++y) { const float4 v = part[y][threadIdx.x]; s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w; }
    const int co = (int)(i % coutp);
    if (co < Cout) {
      const int64_t r = i / coutp;
      const int c4 = (int)(r % (Cin >> 2)), j = (int)(r / (Cin >> 2));
      float* o = dw + ((int64_t)co * Cin + c4 * 4) * K + j;
      o[0] += s.x; o[K] += s.y; o[2 * K] += s.z; o[3 * K] += s.w;
    }
  }
}

// dW[co][ci][j] += acc[j][ci/4][co][ci%4]; acc = 0.   grid.y = layer (device item table), grid.x covers the largest
// layer (surplus blocks exit).  A block moves a 32 co x 32 ci x K tile through shared memory so that BOTH sides are
// coalesced: 512-byte runs of the accumulation buffer in, (32 ci x K)-float runs of the nn.Conv1d gradient out.  (Round
// 1 wrote the gradient with a 4-byte scatter at stride K: 209 us per step, now the kernel is copy-bound.)
__global__ void __launch_bounds__(256) wgrad_acc_flush_kernel(const avc_wgrad_acc_item* __restrict__ items) {
  __shared__ float tile[32][32 * 8 + 1];
  const avc_wgrad_acc_item it = items[blockIdx.y];
  const int K = it.K, C4 = it.Cin >> 2;
  const int coutp = cdiv(it.Cout, 128) * 128;
  const int ncg = cdiv(C4, 8);                      // groups of 8 four-channel chunks (32 input channels)
  const int nblk = (coutp >> 5) * ncg;
  if ((int)blockIdx.x >= nblk) return;
  const int cot = blockIdx.x / ncg, cg = blockIdx.x - cot * ncg;
  const int co0 = cot << 5, c40 = cg << 3;
  const int tid = threadIdx.x, col = tid & 31, c4l = tid >> 5;
  if (c40 + c4l < C4) {
    for (int j = 0; j < K; ++j) {
      float4* a4 = reinterpret_cast<float4*>(it.acc) + ((size_t)j * C4 + c40 + c4l) * coutp + co0 + col;
      const float4 s = *a4;
      *a4 = zero4();
      float* t = &tile[col][(c4l * 4) * K + j];
      t[0] = s.x; t[K] = s.y; t[2 * K] = s.z; t[3 * K] = s.w;
    }
  }
  __syncthreads();
  const int nci = min(32, it.Cin - c40 * 4);         // input channels of this tile
  const int run = nci * K;                            // contiguous floats of one output-channel row
  for (int r = tid >> 5; r < 32; r += 8) {
    const int co = co0 + r;
    if (co >= it.Cout) break;
    float* o = it.dw + ((size_t)co * it.Cin + c40 * 4) * K;
    for (int e = tid & 31; e < run; e += 32) o[e] += tile[r][e];
  }
}

static int wgrad_tc_plan(const avc_wgrad_desc* d, WgTcArgs& a) {
  const int T = d->Tout, K = d->K;
  a.d = *d;
  a.G = T >= 128 ? 1 : 128 / T;
  if (d->stride == 2) a.G = T >= 64 ? 1 : 64 / T;  // the parity-split input tile is twice as tall
  a.RA = a.G * T;
  // padded input positions one sample contributes: stride 1: T+K-1; stride 2: 2(T-1)+K
  a.TX = d->stride == 1 ? T + K - 1 : 2 * (T - 1) + K;
  a.H = ((a.TX + 1) / 2 + 3) / 4 * 4;
  // atom stride must keep every atom base 512 B aligned: the swizzle XOR is keyed on absolute
  // shared-memory address bits [7,9)
  // (and 1024 B aligned for the tensor-map copies of the TMA-staged kernel: a swizzled destination must sit on the
  // swizzle pattern's 8-row period)
  a.RX = d->stride == 1 ? (a.G * a.TX + 7) / 8 * 8 : a.G * 2 * a.H;
  a.ntpad = WT_NT;
  a.coutp = cdiv(d->Cout, 128) * 128;
  a.x_off = (uint32_t)(4 * a.RA * 128 + 1023) / 1024 * 1024;
  a.buf_bytes = (a.x_off + (uint32_t)((a.ntpad / 32) * a.RX * 128) + 1023) / 1024 * 1024;
  const int ntiles = cdiv(d->B, a.G);
  const int cta_per_slice = cdiv(d->Cin, WT_NT) * cdiv(d->Cout, 128);
  int nsl = 132 / cta_per_slice;
  if (nsl < 1) nsl = 1;
  if (nsl > ntiles) nsl = ntiles;
  a.tiles_per_slice = cdiv(ntiles, nsl);
  a.nslices = cdiv(ntiles, a.tiles_per_slice);
  return AVC_OK;
}

static bool wgrad_tc_supported(const avc_wgrad_desc* d) {
  return (d->stride == 1 || d->stride == 2) && d->Tout % 8 == 0 && d->Tout <= 128 && d->K >= 1 && d->K <= 8 && d->Cin % 4 == 0 &&
         d->Cout % 4 == 0 && d->Tin + d->K - 1 >= (d->Tout - 1) * d->stride + 1 && (d->stride == 1 || d->Tout <= 64);
}

int wgrad_reduce(const float* scratch, float* dw, int Cout, int Cin, int K, int coutp, int nslices, cudaStream_t stream) {
  const int64_t n = (int64_t)K * (Cin / 4) * coutp;
  AVC_LAUNCH(wgrad_tc_reduce_kernel, (int)cdiv64(n, 32), dim3(32, 8), 0, stream, scratch, dw, Cout, Cin, K, coutp, nslices);
  AVC_CHECK_LAUNCH("wgrad_tc_reduce");
  return AVC_OK;
}

}  // namespace avc

using namespace avc;

extern "C" int64_t avc_wgrad_tc_scratch_floats(const avc_wgrad_desc* d) {
  if (!d || !wgrad_tc_supported(d)) return -1;
  WgTcArgs a;
  wgrad_tc_plan(d, a);
  return (int64_t)a.nslices * d->K * d->Cin * a.coutp;
}

static int wgrad_tc_launch(const avc_wgrad_desc* d, float* scratch, int* status, void* stream, bool accumulate, const char* who) {
  AVC_REQUIRE(d && d->x && d->dc && scratch && status && (accumulate || d->dw), AVC_ERR_INVALID, "%s: null argument", who);
  AVC_REQUIRE(d->B > 0 && d->Cin > 0 && d->Cout > 0 && d->Tin > 0 && d->Tout > 0, AVC_ERR_INVALID, "%s: bad shape", who);
  AVC_REQUIRE(wgrad_tc_supported(d), AVC_ERR_UNSUPPORTED, "%s: needs stride 1 (Tout <= 128) or 2 (Tout <= 64), Tout %% 8 == 0, K <= 8", who);
  WgTcArgs a;
  wgrad_tc_plan(d, a);
  a.scratch = scratch;
  a.status = status;
  const int smem = 2 * (int)a.buf_bytes;
  AVC_REQUIRE(smem <= 224 * 1024, AVC_ERR_UNSUPPORTED, "%s: tile does not fit shared memory", who);
  static bool attr_done = false;
  if (!attr_done) {
    cudaError_t e = cudaFuncSetAttribute(conv_wgrad_split_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(conv_wgrad_split_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 224 * 1024);
    if (e != cudaSuccess) {
      set_error("%s: cudaFuncSetAttribute: %s", who, cudaGetErrorString(e));
      return AVC_ERR_CUDA;
    }
    attr_done = true;
  }
  dim3 grid(cdiv(d->Cin, WT_NT), cdiv(d->Cout, 128), a.nslices);
  if (accumulate) AVC_LAUNCH(conv_wgrad_split_kernel<true>, grid, WG_THREADS, smem, (cudaStream_t)stream, a);
  else AVC_LAUNCH(conv_wgrad_split_kernel<false>, grid, WG_THREADS, smem, (cudaStream_t)stream, a);
  AVC_CHECK_LAUNCH(who);
  if (accumulate) return AVC_OK;
  return wgrad_reduce(scratch, d->dw, d->Cout, d->Cin, d->K, a.coutp, a.nslices, (cudaStream_t)stream);
}

extern "C" int avc_conv_wgrad_tc(const avc_wgrad_desc* d, float* scratch, int* status, void* stream) {
  return wgrad_tc_launch(d, scratch, status, stream, false, "avc_conv_wgrad_tc");
}

// ---- accumulate-in-place variant: every layer owns a zeroed [K][Cin/4][coutp][4] accumulation
// buffer; avc_conv_wgrad_tc_acc adds into it (vector atomics), avc_wgrad_acc_flush folds every
// layer's buffer into its nn.Conv1d gradient and zeroes it again -- ONE launch per backward pass.
extern "C" int64_t avc_wgrad_acc_floats(int Cout, int Cin, int K) {
  if (Cout <= 0 || Cin <= 0 || K <= 0 || Cin % 4 != 0) return -1;
  return (int64_t)K * Cin * (cdiv(Cout, 128) * 128);
}
extern "C" int avc_conv_wgrad_tc_acc(const avc_wgrad_desc* d, float* acc, int* status, void* stream) {
  return wgrad_tc_launch(d, acc, status, stream, true, "avc_conv_wgrad_tc_acc");
}
extern "C" int avc_wgrad_acc_flush(const avc_wgrad_acc_item* items_dev, int n_items, int64_t max_units, void* stream) {
  AVC_REQUIRE(items_dev && n_items > 0 && max_units > 0, AVC_ERR_INVALID, "avc_wgrad_acc_flush: bad argument");
  // a layer needs (coutp / 32) * ceil(Cin / 32) blocks <= units / (256 K) + coutp / 32: max_units / 256 plus a margin
  // covers every layer (surplus blocks exit at once)
  dim3 grid((unsigned)cdiv64(max_units, 256) + 64u, (unsigned)n_items);
  AVC_LAUNCH(wgrad_acc_flush_kernel, grid, 256, 0, (cudaStream_t)stream, items_dev);
  AVC_CHECK_LAUNCH("wgrad_acc_flush");
  return AVC_OK;
}
