// FP8 (e4m3) quantisation of V for the opt-in FP8 P.V variant of the carved attention (SURVEY §8
// f-3; the reference lists "Quantization (sage-attention)" on its own roadmap, README.md:36-39).
// Per (batch, head): amax = max |v| over all tokens and channels, v8 = e4m3(v * 448 / amax).
// Two HBM-bound passes over V (read 2 x S*H*D*2 B, write S*H*D B); the maximum is exact and
// order-independent (atomicMax on the bit pattern of non-negative floats).
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>

#include "jenga_internal.h"

namespace jenga {
namespace {

template <bool kBF16>
__device__ __forceinline__ float ld16(uint16_t v) {
  if constexpr (kBF16) return __uint_as_float(static_cast<uint32_t>(v) << 16);
  else return __half2float(__ushort_as_half(v));
}

template <bool kBF16>
__global__ void __launch_bounds__(256)
v_absmax_kernel(const uint16_t* __restrict__ v, long long sb, long long ss, long long sh, long long rows, int heads,
                float* __restrict__ amax) {
  const int h = blockIdx.y, b = blockIdx.z;
  const uint16_t* base = v + b * sb + h * sh;
  const long long nvec = rows * 16;   // 16 uint4 per 128-channel row
  float m = 0.f;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nvec;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i >> 4;
    const int c = static_cast<int>(i & 15);
    const uint4 x = __ldg(reinterpret_cast<const uint4*>(base + r * ss) + c);
    const uint32_t w[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      m = fmaxf(m, fabsf(ld16<kBF16>(static_cast<uint16_t>(w[k] & 0xffffu))));
      m = fmaxf(m, fabsf(ld16<kBF16>(static_cast<uint16_t>(w[k] >> 16))));
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<int*>(amax + b * heads + h), __float_as_int(m));
}

template <bool kBF16>
__global__ void __launch_bounds__(256)
v_quantize_kernel(const uint16_t* __restrict__ v, long long sb, long long ss, long long sh, long long rows, int heads,
                  const float* __restrict__ amax, uint8_t* __restrict__ out) {
  const int h = blockIdx.y, b = blockIdx.z;
  const uint16_t* base = v + b * sb + h * sh;
  const float a = amax[b * heads + h];
  const float inv = a > 0.f ? 448.0f / a : 1.0f;
  const long long nvec = rows * 16;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < nvec;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i >> 4;
    const int c = static_cast<int>(i & 15);
    const uint4 x = __ldg(reinterpret_cast<const uint4*>(base + r * ss) + c);
    const uint32_t w[4] = {x.x, x.y, x.z, x.w};
    uint32_t o[2];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float2 f = make_float2(ld16<kBF16>(static_cast<uint16_t>(w[k] & 0xffffu)) * inv,
                                   ld16<kBF16>(static_cast<uint16_t>(w[k] >> 16)) * inv);
      const uint32_t p2 = __nv_cvt_float2_to_fp8x2(f, __NV_SATFINITE, __NV_E4M3);   // low byte = f.x
      if (k & 1) o[k >> 1] |= p2 << 16; else o[k >> 1] = p2;
    }
    *reinterpret_cast<uint2*>(out + ((static_cast<long long>(b) * rows + r) * heads + h) * 128 + c * 8) =
        make_uint2(o[0], o[1]);
  }
}

}  // namespace
}  // namespace jenga

using namespace jenga;

extern "C" int jenga_quantize_v_fp8(const void* v, int32_t dtype, int32_t batch, int64_t rows, int32_t heads,
                                    int64_t stride_b, int64_t stride_s, int64_t stride_h, void* out_fp8, float* amax,
                                    void* stream) {
  if (!v || !out_fp8 || !amax) return set_error(JENGA_E_INVALID, "quantize_v_fp8: null pointer");
  if (dtype != JENGA_BF16 && dtype != JENGA_F16) return set_error(JENGA_E_INVALID, "quantize_v_fp8: dtype must be bf16/f16");
  if (batch <= 0 || rows <= 0 || heads <= 0 || stride_s % 8 || stride_h % 8 || stride_b % 8 ||
      reinterpret_cast<uintptr_t>(v) % 16 || reinterpret_cast<uintptr_t>(out_fp8) % 8)
    return set_error(JENGA_E_INVALID, "quantize_v_fp8: bad shape / alignment");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  cudaError_t ce = cudaMemsetAsync(amax, 0, sizeof(float) * batch * heads, s);
  if (ce != cudaSuccess) return set_cuda_error(ce, "quantize_v_fp8 memset");
  long long per_head = (rows * 16 + 255) / 256;
  const long long cap = (static_cast<long long>(kNumSMs) * 8 + heads * batch - 1) / (heads * batch);
  if (per_head > cap) per_head = cap > 0 ? cap : 1;
  dim3 grid(static_cast<unsigned>(per_head), heads, batch);
  const uint16_t* vp = static_cast<const uint16_t*>(v);
  if (dtype == JENGA_BF16) {
    v_absmax_kernel<true><<<grid, 256, 0, s>>>(vp, stride_b, stride_s, stride_h, rows, heads, amax);
    v_quantize_kernel<true><<<grid, 256, 0, s>>>(vp, stride_b, stride_s, stride_h, rows, heads, amax, static_cast<uint8_t*>(out_fp8));
  } else {
    v_absmax_kernel<false><<<grid, 256, 0, s>>>(vp, stride_b, stride_s, stride_h, rows, heads, amax);
    v_quantize_kernel<false><<<grid, 256, 0, s>>>(vp, stride_b, stride_s, stride_h, rows, heads, amax, static_cast<uint8_t*>(out_fp8));
  }
  ce = cudaGetLastError();
  return ce == cudaSuccess ? JENGA_OK : set_cuda_error(ce, "quantize_v_fp8 launch");
}
