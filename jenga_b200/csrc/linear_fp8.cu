// Opt-in W8A8 FP8 Linear (SURVEY §8 f-1: after carving, the block Linears are the largest remaining
// term).  Two entry points:
//   jenga_quantize_rows_fp8  a_scale[m] = amax(row m) / 448 (1 for an all-zero row),
//                            out[m, :] = e4m3_rn_satfinite(x[m, :] / a_scale[m])
//   jenga_linear_fp8         Y[M, N] = bf16( (A8 . W8^T)[m, n] * a_scale[m] * w_scale[n] + bias[n] )
// The GEMM is a persistent sm_90a kernel over 128 x 128 output tiles: a producer warp streams 128-byte
// K slices of A8 and W8 by TMA (128-byte swizzle) into a kStages mbarrier ring, and two consumer
// warpgroups (64 rows each) run shared x shared e4m3 wgmma on them.  Hopper's FP8 wgmma does not keep a
// full fp32 accumulator, so each 128-wide K slice is accumulated in wgmma registers of its own and then
// added to a separate fp32 accumulator; the wgmma of slice k + 1 runs while slice k is added.
#include <cuda_bf16.h>

#include "jenga_internal.h"
#include "sm90_ptx.cuh"

namespace jenga {
namespace {

// ------------------------------------------------------------------------------------------
// Row quantisation: one CTA per row (grid-stride), two passes over the row (the second hits L1/L2)
// ------------------------------------------------------------------------------------------
constexpr int kQThreads = 256;

__global__ void __launch_bounds__(kQThreads)
quantize_rows_fp8_kernel(const uint16_t* __restrict__ x, long long x_stride, long long rows, int cols,
                         uint8_t* __restrict__ out, long long out_stride, float* __restrict__ scale) {
  __shared__ float s_max[kQThreads / 32];
  const int nvec = cols / 8;
  for (long long row = blockIdx.x; row < rows; row += gridDim.x) {
    const uint4* src = reinterpret_cast<const uint4*>(x + row * x_stride);
    float m = 0.f;
    for (int v = threadIdx.x; v < nvec; v += kQThreads) {
      const uint4 w = __ldg(src + v);
      const uint32_t u[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
        m = fmaxf(m, fmaxf(fabsf(__uint_as_float(u[i] << 16)), fabsf(__uint_as_float(u[i] & 0xffff0000u))));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) s_max[threadIdx.x >> 5] = m;
    __syncthreads();
#pragma unroll
    for (int w = 0; w < kQThreads / 32; ++w) m = fmaxf(m, s_max[w]);
    __syncthreads();   // s_max is rewritten by the next row
    const float s = m > 0.f ? __fdiv_rn(m, 448.0f) : 1.0f;
    if (threadIdx.x == 0) scale[row] = s;
    uint2* dst = reinterpret_cast<uint2*>(out + row * out_stride);
    for (int v = threadIdx.x; v < nvec; v += kQThreads) {
      const uint4 w = __ldg(src + v);
      const uint32_t u[4] = {w.x, w.y, w.z, w.w};
      float f[8];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        f[2 * i] = __fdiv_rn(__uint_as_float(u[i] << 16), s);
        f[2 * i + 1] = __fdiv_rn(__uint_as_float(u[i] & 0xffff0000u), s);
      }
      dst[v] = make_uint2(pack4_e4m3(f[0], f[1], f[2], f[3]), pack4_e4m3(f[4], f[5], f[6], f[7]));
    }
  }
}

// ------------------------------------------------------------------------------------------
// GEMM
// ------------------------------------------------------------------------------------------
constexpr int kBM = 128, kBN = 128, kBK = 128;        // tile rows, tile columns, K bytes per stage
constexpr int kStages = 6;
constexpr int kTileA = kBM * kBK;                     // 16 KB
constexpr int kStageBytes = kTileA + kBN * kBK;       // + 16 KB of W
constexpr int kOffBars = kStages * kStageBytes;
constexpr int kSmemBytes = kOffBars + 2 * kStages * 8 + 1024;   // + slack for the 1024-B alignment
constexpr int kThreads = 384;                         // consumer warpgroups 0, 1; producer warpgroup 2
constexpr int kGroupM = 8;                            // M tiles per group of the tile order

struct GemmParams {
  long long m;
  int n, k;
  int tiles_m, tiles_n;
  const float* a_scale;
  const float* w_scale;
  int w_scale_stride;   // 1: per output channel, 0: one per-tensor value
  const void* bias;     // may be null
  int bias_f32;
  uint16_t* out;
  long long out_stride;
};

// Tile t -> (tm, tn).  Groups of kGroupM M tiles are walked column by column, M fastest, so the CTAs
// that run at the same time read a few A row panels and a few W column panels, which stay in L2.
__device__ __forceinline__ void tile_coords(int t, const GemmParams& p, int& tm, int& tn) {
  const int per_group = kGroupM * p.tiles_n;
  const int g = t / per_group;
  const int first = g * kGroupM;
  const int gm = min(kGroupM, p.tiles_m - first);
  const int r = t - g * per_group;
  tm = first + r % gm;
  tn = r / gm;
}

__device__ __forceinline__ void issue_slice(float (&d)[64], uint8_t* smem, uint64_t* full, uint32_t it, int wg) {
  const int s = static_cast<int>(it % kStages);
  mbar_wait(&full[s], (it / kStages) & 1u, nullptr);
  const uint32_t a_addr = smem_u32(smem + s * kStageBytes) + wg * 64 * kBK;   // this warpgroup's 64 rows
  const uint32_t w_addr = smem_u32(smem + s * kStageBytes + kTileA);
  wgmma_fence();
#pragma unroll
  for (int kc = 0; kc < kBK / 32; ++kc)
    wgmma_128_ss_e4m3(d, gmma_desc_sw128(a_addr + kc * 32, 16, 1024), gmma_desc_sw128(w_addr + kc * 32, 16, 1024),
                      kc > 0 ? 1u : 0u);
  wgmma_commit();
}

// the slice in `d` has retired: free its stage and promote it into the fp32 accumulator
__device__ __forceinline__ void retire_slice(float (&acc)[64], float (&d)[64], uint64_t* empty, uint32_t it,
                                             int lane) {
  fence_regs(d);
  __syncwarp();
  if (lane == 0) mbar_arrive(&empty[it % kStages]);
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] += d[i];
}

__global__ void __launch_bounds__(kThreads, 1)
linear_fp8_kernel(const __grid_constant__ CUtensorMap tm_a, const __grid_constant__ CUtensorMap tm_w,
                  const GemmParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw_addr + 1023u) & ~1023u) - raw_addr);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + kOffBars);
  uint64_t* empty = full + kStages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n_tiles = p.tiles_m * p.tiles_n;
  const int nk = (p.k + kBK - 1) / kBK;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_a);
    tma_prefetch_desc(&tm_w);
#pragma unroll
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&full[s], 1u);
      mbar_init(&empty[s], 8u);   // one arrival per consumer warp
    }
    fence_mbar_init();
  }
  __syncthreads();

  if (warp >= 8) {
    // =============================== producer warpgroup ===============================
    setmaxnreg_dec<40>();
    if (warp == 8 && lane == 0) {
      uint32_t it = 0;
      for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
        int tm, tn;
        tile_coords(t, p, tm, tn);
        for (int kb = 0; kb < nk; ++kb, ++it) {
          const int s = static_cast<int>(it % kStages);
          if (it >= kStages) mbar_wait(&empty[s], ((it / kStages) & 1u) ^ 1u, nullptr);
          uint8_t* dst = smem + s * kStageBytes;
          // rows past M / N and columns past K are zero-filled, and still counted in the bytes
          mbar_arrive_expect_tx(&full[s], kStageBytes);
          tma_load_2d(dst, &tm_a, &full[s], kb * kBK, tm * kBM);
          tma_load_2d(dst + kTileA, &tm_w, &full[s], kb * kBK, tn * kBN);
        }
      }
    }
    return;
  }

  // =============================== consumers ===============================
  setmaxnreg_inc<232>();
  const int wg = warp >> 2;
  const int row_in = wg * 64 + (warp & 3) * 16 + (lane >> 2);   // accumulator rows row_in, row_in + 8
  float acc[64], d0[64], d1[64];
  uint32_t it = 0;
  for (int t = blockIdx.x; t < n_tiles; t += gridDim.x) {
    int tm, tn;
    tile_coords(t, p, tm, tn);
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    // two slices in flight per warpgroup: d0 holds the even slices, d1 the odd ones
    issue_slice(d0, smem, full, it, wg);
    for (int kb = 0; kb < nk; kb += 2) {
      if (kb + 1 < nk) {
        issue_slice(d1, smem, full, it + kb + 1, wg);
        wgmma_wait<1>();
      } else {
        wgmma_wait<0>();
      }
      retire_slice(acc, d0, empty, it + kb, lane);
      if (kb + 1 >= nk) break;
      if (kb + 2 < nk) {
        issue_slice(d0, smem, full, it + kb + 2, wg);
        wgmma_wait<1>();
      } else {
        wgmma_wait<0>();
      }
      retire_slice(acc, d1, empty, it + kb + 1, lane);
    }
    it += nk;

    // epilogue: scale, bias, bf16; rows past M and columns past N are not stored
    const long long r0 = static_cast<long long>(tm) * kBM + row_in;
    const bool live0 = r0 < p.m, live1 = r0 + 8 < p.m;
    const float as0 = live0 ? __ldg(p.a_scale + r0) : 0.f;
    const float as1 = live1 ? __ldg(p.a_scale + r0 + 8) : 0.f;
    uint16_t* o0 = p.out + r0 * p.out_stride;
    uint16_t* o1 = o0 + 8 * p.out_stride;
#pragma unroll
    for (int j = 0; j < kBN / 8; ++j) {
      const int c = tn * kBN + j * 8 + (lane & 3) * 2;
      if (c < p.n) {   // N % 8 == 0: c < N implies c + 1 < N
        const float ws0 = __ldg(p.w_scale + static_cast<long long>(c) * p.w_scale_stride);
        const float ws1 = __ldg(p.w_scale + static_cast<long long>(c + 1) * p.w_scale_stride);
        float b0 = 0.f, b1 = 0.f;
        if (p.bias) {
          if (p.bias_f32) {
            b0 = __ldg(static_cast<const float*>(p.bias) + c);
            b1 = __ldg(static_cast<const float*>(p.bias) + c + 1);
          } else {
            const uint32_t bw = __ldg(reinterpret_cast<const uint32_t*>(static_cast<const uint16_t*>(p.bias) + c));
            b0 = __uint_as_float(bw << 16);
            b1 = __uint_as_float(bw & 0xffff0000u);
          }
        }
        if (live0)
          *reinterpret_cast<uint32_t*>(o0 + c) =
              pack2<true>(__fadd_rn(__fmul_rn(__fmul_rn(acc[4 * j], as0), ws0), b0),
                          __fadd_rn(__fmul_rn(__fmul_rn(acc[4 * j + 1], as0), ws1), b1));
        if (live1)
          *reinterpret_cast<uint32_t*>(o1 + c) =
              pack2<true>(__fadd_rn(__fmul_rn(__fmul_rn(acc[4 * j + 2], as1), ws0), b0),
                          __fadd_rn(__fmul_rn(__fmul_rn(acc[4 * j + 3], as1), ws1), b1));
      }
    }
  }
}

// 2-D e4m3 operand [rows, k] with a row pitch of `stride` bytes; box {128 bytes of K, 128 rows}
int make_operand_map(CUtensorMap* map, const void* base, long long rows, int k, long long stride) {
  const cuuint64_t dims[2] = {static_cast<cuuint64_t>(k), static_cast<cuuint64_t>(rows)};
  const cuuint64_t strides[1] = {static_cast<cuuint64_t>(stride)};
  const cuuint32_t box[2] = {static_cast<cuuint32_t>(kBK), static_cast<cuuint32_t>(kBM)};
  const cuuint32_t elem_strides[2] = {1, 1};
  return encode_tensor_map(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(base), dims, strides, box,
                           elem_strides, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                           CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

bool aligned(const void* p, uintptr_t n) { return reinterpret_cast<uintptr_t>(p) % n == 0; }

}  // namespace
}  // namespace jenga

using namespace jenga;

extern "C" int jenga_quantize_rows_fp8(const void* x, int64_t x_stride, int64_t rows, int32_t cols, void* out,
                                       int64_t out_stride, float* scale, void* stream) {
  if (!x || !out || !scale) return set_error(JENGA_E_INVALID, "quantize_rows_fp8: null pointer");
  if (rows <= 0 || cols <= 0 || x_stride < cols || out_stride < cols)
    return set_error(JENGA_E_INVALID, "quantize_rows_fp8: bad shape");
  if (cols % 16) return set_error(JENGA_E_UNSUPPORTED, "quantize_rows_fp8: cols %d is not a multiple of 16", cols);
  if (x_stride % 8 || out_stride % 16 || !aligned(x, 16) || !aligned(out, 16) || !aligned(scale, 4))
    return set_error(JENGA_E_INVALID, "quantize_rows_fp8: rows must be 16-byte aligned (strides, pointers)");
  const long long g = rows < kNumSMs * 16LL ? rows : kNumSMs * 16LL;
  quantize_rows_fp8_kernel<<<static_cast<unsigned>(g), kQThreads, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint16_t*>(x), x_stride, rows, cols, static_cast<uint8_t*>(out), out_stride, scale);
  const cudaError_t ce = cudaGetLastError();
  return ce == cudaSuccess ? JENGA_OK : set_cuda_error(ce, "quantize_rows_fp8 launch");
}

extern "C" int jenga_linear_fp8(const JengaLinearFp8Args* a, void* stream) {
  if (!a || !a->a || !a->a_scale || !a->w || !a->w_scale || !a->out)
    return set_error(JENGA_E_INVALID, "linear_fp8: null pointer");
  if (a->m <= 0 || a->n <= 0 || a->k <= 0 || a->a_stride < a->k || a->out_stride < a->n)
    return set_error(JENGA_E_INVALID, "linear_fp8: bad shape");
  if (a->k % 16 || a->n % 8)
    return set_error(JENGA_E_UNSUPPORTED, "linear_fp8: K %d must be a multiple of 16 and N %d of 8", a->k, a->n);
  if (a->w_scale_stride != 0 && a->w_scale_stride != 1)
    return set_error(JENGA_E_INVALID, "linear_fp8: w_scale_stride must be 0 (per tensor) or 1 (per channel)");
  if (a->bias && a->bias_dtype != JENGA_BF16 && a->bias_dtype != JENGA_F32)
    return set_error(JENGA_E_INVALID, "linear_fp8: bias dtype must be bf16 or f32");
  if (a->a_stride % 16 || a->out_stride % 8 || !aligned(a->a, 16) || !aligned(a->w, 16) || !aligned(a->out, 16) ||
      !aligned(a->a_scale, 4) || !aligned(a->w_scale, 4) || (a->bias && !aligned(a->bias, 8)))
    return set_error(JENGA_E_INVALID, "linear_fp8: pointers and strides must be 16-byte aligned");
  const long long tiles_m = (a->m + kBM - 1) / kBM;
  const long long tiles_n = (a->n + kBN - 1) / kBN;
  if (tiles_m * tiles_n > 0x7fffffffLL) return set_error(JENGA_E_UNSUPPORTED, "linear_fp8: too many tiles");
  CUtensorMap tm_a, tm_w;
  int rc;
  if ((rc = make_operand_map(&tm_a, a->a, a->m, a->k, a->a_stride)) != JENGA_OK ||
      (rc = make_operand_map(&tm_w, a->w, a->n, a->k, a->k)) != JENGA_OK)
    return rc;
  GemmParams p{};
  p.m = a->m;
  p.n = a->n;
  p.k = a->k;
  p.tiles_m = static_cast<int>(tiles_m);
  p.tiles_n = static_cast<int>(tiles_n);
  p.a_scale = a->a_scale;
  p.w_scale = a->w_scale;
  p.w_scale_stride = a->w_scale_stride;
  p.bias = a->bias;
  p.bias_f32 = a->bias_dtype == JENGA_F32;
  p.out = static_cast<uint16_t*>(a->out);
  p.out_stride = a->out_stride;
  cudaError_t ce = cudaFuncSetAttribute(linear_fp8_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);
  if (ce != cudaSuccess) return set_cuda_error(ce, "cudaFuncSetAttribute(linear_fp8)");
  const long long n_tiles = tiles_m * tiles_n;
  const unsigned grid = static_cast<unsigned>(n_tiles < kNumSMs ? n_tiles : kNumSMs);
  linear_fp8_kernel<<<grid, kThreads, kSmemBytes, static_cast<cudaStream_t>(stream)>>>(tm_a, tm_w, p);
  ce = cudaGetLastError();
  return ce == cudaSuccess ? JENGA_OK : set_cuda_error(ce, "linear_fp8 launch");
}
