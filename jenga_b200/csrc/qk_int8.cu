// INT8 quantisation of Q and K for the opt-in INT8 Q.K^T variant of the carved attention (SURVEY §8
// f-3; SageAttention's recipe).  Per (batch, head) and per group of `group_rows` rows:
//   scale = max|x - mean| / 127,  out = clamp(rint((x - mean) / scale), -127, 127)
// with mean = the per-(batch, head) channel mean of x ("smoothing", K only) or 0 (Q).  Subtracting
// the same vector from every key adds a constant to each score row, which the softmax ignores, but
// it removes the common channel bias that would otherwise set the K scales.
// Padding rows [rows, out_rows) are quantised as x = 0, i.e. as (0 - mean): the dense rows attend
// the zero padding of a ragged sequence, so their keys must be the smoothed zero, not a zero code.
// Up to three HBM-bound passes: partial column sums per 128-row block (into `out`, used as scratch),
// their reduction to the mean in a fixed order (deterministic), and one quantising pass per group.
// For the LSE of the INT8 path the Q pass can also write each row's shift Q'_i . mean(K): every score
// of row i is short by that much after K smoothing.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "jenga_internal.h"

namespace jenga {
namespace {

constexpr int kD = 128;
constexpr int kThreads = 256;   // 16 threads per row (8 channels each), 16 rows per pass

template <bool kBF16>
__device__ __forceinline__ void load8(const uint16_t* p, float (&f)[8]) {
  const uint4 x = __ldg(reinterpret_cast<const uint4*>(p));
  const uint32_t w[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if constexpr (kBF16) {
      f[2 * k] = __uint_as_float(w[k] << 16);
      f[2 * k + 1] = __uint_as_float(w[k] & 0xffff0000u);
    } else {
      f[2 * k] = __half2float(__ushort_as_half(static_cast<uint16_t>(w[k] & 0xffffu)));
      f[2 * k + 1] = __half2float(__ushort_as_half(static_cast<uint16_t>(w[k] >> 16)));
    }
  }
}

// part[(bh * nblk + blk) * 128 + c] = sum of x[b, 128 blk .. 128 blk + 127, h, c] (rows < `rows`)
template <bool kBF16>
__global__ void __launch_bounds__(kThreads)
colsum_kernel(const uint16_t* __restrict__ x, long long sb, long long ss, long long sh, long long rows, int heads,
              long long items, long long nblk, float* __restrict__ part) {
  __shared__ float red[16][kD];
  const int cc = threadIdx.x & 15, r0 = threadIdx.x >> 4;
  for (long long it = blockIdx.x; it < items; it += gridDim.x) {
    const long long bh = it / nblk, blk = it - bh * nblk;
    const int b = static_cast<int>(bh / heads), h = static_cast<int>(bh - static_cast<long long>(b) * heads);
    const uint16_t* base = x + b * sb + h * sh + cc * 8;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const long long row = blk * 128 + r0 + 16 * i;
      if (row < rows) {
        float f[8];
        load8<kBF16>(base + row * ss, f);
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] += f[k];
      }
    }
#pragma unroll
    for (int k = 0; k < 8; ++k) red[r0][cc * 8 + k] = acc[k];
    __syncthreads();
    if (threadIdx.x < kD) {
      float s = 0.f;
#pragma unroll
      for (int r = 0; r < 16; ++r) s += red[r][threadIdx.x];
      part[it * kD + threadIdx.x] = s;
    }
    __syncthreads();
  }
}

// mean[bh * 128 + c] = (sum over blk of part[bh][blk][c], in block order) / rows
__global__ void __launch_bounds__(kD)
mean_kernel(const float* __restrict__ part, long long nblk, long long rows, float* __restrict__ mean) {
  const long long bh = blockIdx.x;
  float s = 0.f;
  for (long long blk = 0; blk < nblk; ++blk) s += part[(bh * nblk + blk) * kD + threadIdx.x];
  mean[bh * kD + threadIdx.x] = s / static_cast<float>(rows);
}

template <bool kBF16, int kGroup>
__global__ void __launch_bounds__(kThreads)
quantize_kernel(const uint16_t* __restrict__ x, long long sb, long long ss, long long sh, long long rows, int heads,
                const float* __restrict__ mean, long long out_rows, int8_t* __restrict__ out,
                float* __restrict__ scale, const float* __restrict__ shift_mean, float* __restrict__ shift) {
  constexpr int kPer = kGroup / 16;   // rows per thread
  __shared__ float wmax[kThreads / 32];
  const int cc = threadIdx.x & 15, r0 = threadIdx.x >> 4;
  const long long ngroups = out_rows / kGroup;
  const long long bh = blockIdx.y;   // gridDim.y == batch * heads
  const int b = static_cast<int>(bh / heads), h = static_cast<int>(bh - static_cast<long long>(b) * heads);
  for (long long g = blockIdx.x; g < ngroups; g += gridDim.x) {
    float mu[8];
#pragma unroll
    for (int k = 0; k < 8; ++k) mu[k] = mean ? mean[bh * kD + cc * 8 + k] : 0.f;
    float y[kPer][8];
    float m = 0.f;
#pragma unroll
    for (int i = 0; i < kPer; ++i) {
      const long long row = g * kGroup + r0 + 16 * i;
      float f[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
      if (row < rows) load8<kBF16>(x + b * sb + row * ss + h * sh + cc * 8, f);
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        y[i][k] = f[k] - mu[k];
        m = fmaxf(m, fabsf(y[i][k]));
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) wmax[threadIdx.x >> 5] = m;
    __syncthreads();
#pragma unroll
    for (int w = 0; w < kThreads / 32; ++w) m = fmaxf(m, wmax[w]);
    __syncthreads();   // wmax is rewritten by the next group
    const float sc = __fdiv_rn(m, 127.0f);
    if (threadIdx.x == 0) scale[bh * ngroups + g] = sc;
#pragma unroll
    for (int i = 0; i < kPer; ++i) {
      const long long row = g * kGroup + r0 + 16 * i;
      uint32_t w[2] = {0u, 0u};
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const float qv = sc > 0.f ? fminf(fmaxf(rintf(__fdiv_rn(y[i][k], sc)), -127.f), 127.f) : 0.f;
        w[k >> 2] |= (static_cast<uint32_t>(static_cast<int>(qv)) & 0xffu) << (8 * (k & 3));
        y[i][k] = qv;   // the code, for the shift below
      }
      *reinterpret_cast<uint2*>(out + ((static_cast<long long>(b) * out_rows + row) * heads + h) * kD + cc * 8) =
          make_uint2(w[0], w[1]);
    }
    if (shift) {   // shift[bh][row] = sc * sum_c code[row][c] * shift_mean[bh][c]; a row is 16 lanes of a half-warp
      float km[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) km[k] = shift_mean[bh * kD + cc * 8 + k];
#pragma unroll
      for (int i = 0; i < kPer; ++i) {
        float d = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k) d = fmaf(y[i][k], km[k], d);
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
        if (cc == 0) shift[bh * out_rows + g * kGroup + r0 + 16 * i] = d * sc;
      }
    }
  }
}

template <bool kBF16>
int launch_all(const uint16_t* x, long long sb, long long ss, long long sh, int batch, long long rows, int heads,
               int group_rows, int smooth, float* mean, int8_t* out, long long out_rows, float* scale,
               const float* shift_mean, float* shift, cudaStream_t s) {
  const long long bhs = static_cast<long long>(batch) * heads;
  if (smooth) {
    const long long nblk = (rows + 127) / 128;
    float* part = reinterpret_cast<float*>(out);   // bhs * nblk * 512 B <= bhs * out_rows * 128 B
    long long blocks = bhs * nblk;
    if (blocks > static_cast<long long>(kNumSMs) * 8) blocks = static_cast<long long>(kNumSMs) * 8;
    colsum_kernel<kBF16><<<static_cast<unsigned>(blocks), kThreads, 0, s>>>(x, sb, ss, sh, rows, heads, bhs * nblk,
                                                                            nblk, part);
    cudaError_t ce = cudaGetLastError();
    if (ce != cudaSuccess) return set_cuda_error(ce, "quantize_int8 colsum launch");
    mean_kernel<<<static_cast<unsigned>(bhs), kD, 0, s>>>(part, nblk, rows, mean);
    ce = cudaGetLastError();
    if (ce != cudaSuccess) return set_cuda_error(ce, "quantize_int8 mean launch");
  }
  const long long ngroups = out_rows / group_rows;
  long long per_bh = (static_cast<long long>(kNumSMs) * 8 + bhs - 1) / bhs;
  if (per_bh > ngroups) per_bh = ngroups;
  const dim3 grid(static_cast<unsigned>(per_bh), static_cast<unsigned>(bhs));
  const float* mu = smooth ? mean : nullptr;
  if (group_rows == 64)
    quantize_kernel<kBF16, 64><<<grid, kThreads, 0, s>>>(x, sb, ss, sh, rows, heads, mu, out_rows, out, scale,
                                                         shift_mean, shift);
  else
    quantize_kernel<kBF16, 128><<<grid, kThreads, 0, s>>>(x, sb, ss, sh, rows, heads, mu, out_rows, out, scale,
                                                          shift_mean, shift);
  const cudaError_t ce = cudaGetLastError();
  return ce == cudaSuccess ? JENGA_OK : set_cuda_error(ce, "quantize_int8 launch");
}

}  // namespace
}  // namespace jenga

using namespace jenga;

// The checks of jenga_quantize_int8, shared with jenga_quantize_q_int8_lse_shift; then the launch.
static int quantize_checked(const void* x, int32_t dtype, int32_t batch, int64_t rows, int32_t heads, int64_t stride_b,
                            int64_t stride_s, int64_t stride_h, int32_t group_rows, int32_t smooth, float* mean,
                            int8_t* out, int64_t out_rows, float* scale, const float* shift_mean, float* shift,
                            void* stream) {
  if (!x || !out || !scale || (smooth && !mean)) return set_error(JENGA_E_INVALID, "quantize_int8: null pointer");
  if (dtype != JENGA_BF16 && dtype != JENGA_F16) return set_error(JENGA_E_INVALID, "quantize_int8: dtype must be bf16/f16");
  if (group_rows != 64 && group_rows != 128)
    return set_error(JENGA_E_UNSUPPORTED, "quantize_int8: group_rows %d (64 or 128 are built)", group_rows);
  if (batch <= 0 || rows <= 0 || heads <= 0 || heads > 65535 || static_cast<long long>(batch) * heads > 65535)
    return set_error(JENGA_E_INVALID, "quantize_int8: bad shape");
  if (out_rows % 128 || out_rows < (rows + 127) / 128 * 128)
    return set_error(JENGA_E_INVALID, "quantize_int8: out_rows %lld must be a multiple of 128 and >= round_up(rows, 128)",
                     static_cast<long long>(out_rows));
  if (stride_b <= 0 || stride_s <= 0 || stride_h <= 0 || stride_b % 8 || stride_s % 8 || stride_h % 8 ||
      reinterpret_cast<uintptr_t>(x) % 16 || reinterpret_cast<uintptr_t>(out) % 16 ||
      reinterpret_cast<uintptr_t>(scale) % 4 || reinterpret_cast<uintptr_t>(mean) % 4 ||
      reinterpret_cast<uintptr_t>(shift_mean) % 4 || reinterpret_cast<uintptr_t>(shift) % 4)
    return set_error(JENGA_E_INVALID, "quantize_int8: bad strides / alignment");
  const uint16_t* xp = static_cast<const uint16_t*>(x);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  return dtype == JENGA_BF16
             ? launch_all<true>(xp, stride_b, stride_s, stride_h, batch, rows, heads, group_rows, smooth, mean, out,
                                out_rows, scale, shift_mean, shift, s)
             : launch_all<false>(xp, stride_b, stride_s, stride_h, batch, rows, heads, group_rows, smooth, mean, out,
                                 out_rows, scale, shift_mean, shift, s);
}

extern "C" int jenga_quantize_int8(const void* x, int32_t dtype, int32_t batch, int64_t rows, int32_t heads,
                                   int64_t stride_b, int64_t stride_s, int64_t stride_h, int32_t group_rows,
                                   int32_t smooth, float* mean, int8_t* out, int64_t out_rows, float* scale,
                                   void* stream) {
  return quantize_checked(x, dtype, batch, rows, heads, stride_b, stride_s, stride_h, group_rows, smooth, mean, out,
                          out_rows, scale, nullptr, nullptr, stream);
}

extern "C" int jenga_quantize_q_int8_lse_shift(const void* q, int32_t dtype, int32_t batch, int64_t rows,
                                               int32_t heads, int64_t stride_b, int64_t stride_s, int64_t stride_h,
                                               const float* k_mean, int8_t* out, int64_t out_rows, float* scale,
                                               float* shift, void* stream) {
  if (!k_mean || !shift) return set_error(JENGA_E_INVALID, "quantize_q_int8_lse_shift: null k_mean / shift pointer");
  return quantize_checked(q, dtype, batch, rows, heads, stride_b, stride_s, stride_h, 64, 0, nullptr, out, out_rows,
                          scale, k_mean, shift, stream);
}
