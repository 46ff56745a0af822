// Step-skip residual cache and TeaCache gate (SURVEY §8 a-13) as device ops.
//
// The reference decides per denoising step whether the block loop — and with it the whole hot
// path — runs, and otherwise replays the previous step's residual:
//   HunyuanVideo  jenga_hyvideo.py:128-179   fixed list of computed steps; skipped step:
//                 `img += self.previous_residual`; computed step: `ori_img = img.clone()` …
//                 `self.previous_residual = img - ori_img`
//   Wan2.1        jenga_wan.py:595-648       TeaCache: accumulated, polynomial-rescaled relative
//                 L1 change of the modulated timestep embedding against a threshold, separately
//                 for the conditional (even) and unconditional (odd) forward
// Here: two HBM-bound elementwise kernels (16-byte vectors, grid sized to the SM count) and one
// single-CTA gate kernel that also performs the `.clone()` of the embedding, keeps its
// accumulator on the device and writes the decision flag to device or mapped host memory.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "jenga_internal.h"

namespace jenga {
namespace {

template <int kDtype>
__device__ __forceinline__ float ld16(uint16_t v) {
  if constexpr (kDtype == JENGA_BF16) return __uint_as_float(static_cast<uint32_t>(v) << 16);
  else return __half2float(__ushort_as_half(v));
}
template <int kDtype>
__device__ __forceinline__ uint16_t st16(float x) {
  if constexpr (kDtype == JENGA_BF16) return __bfloat16_as_ushort(__float2bfloat16_rn(x));
  else return __half_as_ushort(__float2half_rn(x));
}

// out = a (+|-) b, elementwise, fp32 arithmetic rounded once to the 16-bit type — what ATen's
// add/sub kernels do for bf16/fp16 operands.  kSub: out = a - b.  out may alias a.
template <int kDtype, bool kSub>
__global__ void __launch_bounds__(256)
residual_kernel(const uint4* __restrict__ a, const uint4* __restrict__ b, uint4* out, long long n_vec,
                const uint16_t* a_tail, const uint16_t* b_tail, uint16_t* out_tail, int n_tail) {
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n_vec; i += stride) {
    const uint4 x = a[i];
    const uint4 y = __ldg(b + i);
    const uint32_t xs[4] = {x.x, x.y, x.z, x.w}, ys[4] = {y.x, y.y, y.z, y.w};
    uint32_t r[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float x0 = ld16<kDtype>(xs[j] & 0xffffu), x1 = ld16<kDtype>(xs[j] >> 16);
      const float y0 = ld16<kDtype>(ys[j] & 0xffffu), y1 = ld16<kDtype>(ys[j] >> 16);
      const float r0 = kSub ? x0 - y0 : x0 + y0, r1 = kSub ? x1 - y1 : x1 + y1;
      r[j] = st16<kDtype>(r0) | (static_cast<uint32_t>(st16<kDtype>(r1)) << 16);
    }
    out[i] = make_uint4(r[0], r[1], r[2], r[3]);
  }
  if (blockIdx.x == 0 && threadIdx.x < n_tail) {
    const float x = ld16<kDtype>(a_tail[threadIdx.x]), y = ld16<kDtype>(b_tail[threadIdx.x]);
    out_tail[threadIdx.x] = st16<kDtype>(kSub ? x - y : x + y);
  }
}

__global__ void __launch_bounds__(256)
residual_f32_kernel(const float* a, const float* __restrict__ b, float* out, long long n, int sub) {
  const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n; i += stride)
    out[i] = sub ? a[i] - b[i] : a[i] + b[i];
}

int launch_residual(const void* a, const void* b, void* out, long long n, int dtype, bool sub, cudaStream_t s) {
  if (!a || !b || !out || n < 0) return set_error(JENGA_E_INVALID, "residual: null pointer / negative size");
  if (n == 0) return JENGA_OK;
  const int grid = kNumSMs * 8;
  if (dtype == JENGA_F32) {
    residual_f32_kernel<<<grid, 256, 0, s>>>(static_cast<const float*>(a), static_cast<const float*>(b),
                                             static_cast<float*>(out), n, sub ? 1 : 0);
  } else if (dtype == JENGA_BF16 || dtype == JENGA_F16) {
    if (reinterpret_cast<uintptr_t>(a) % 16 || reinterpret_cast<uintptr_t>(b) % 16 ||
        reinterpret_cast<uintptr_t>(out) % 16)
      return set_error(JENGA_E_INVALID, "residual: pointers must be 16-byte aligned");
    const long long n_vec = n / 8;
    const int n_tail = static_cast<int>(n - n_vec * 8);
    const uint16_t* at = static_cast<const uint16_t*>(a) + n_vec * 8;
    const uint16_t* bt = static_cast<const uint16_t*>(b) + n_vec * 8;
    uint16_t* ot = static_cast<uint16_t*>(out) + n_vec * 8;
#define JENGA_RES(DT, SUB)                                                                              \
  residual_kernel<DT, SUB><<<grid, 256, 0, s>>>(static_cast<const uint4*>(a), static_cast<const uint4*>(b), \
                                                static_cast<uint4*>(out), n_vec, at, bt, ot, n_tail)
    if (dtype == JENGA_BF16) { if (sub) JENGA_RES(JENGA_BF16, true); else JENGA_RES(JENGA_BF16, false); }
    else { if (sub) JENGA_RES(JENGA_F16, true); else JENGA_RES(JENGA_F16, false); }
#undef JENGA_RES
  } else {
    return set_error(JENGA_E_INVALID, "residual: dtype must be bf16, f16 or f32");
  }
  const cudaError_t ce = cudaGetLastError();
  return ce == cudaSuccess ? JENGA_OK : set_cuda_error(ce, "residual launch");
}

// ------------------------------------------------------------------------------------------
// TeaCache gate (jenga_wan.py:597-626).  One CTA: fixed-order two-level sums (thread-strided
// partials in fp32 pairs promoted to double, then a shared-memory tree) -> deterministic.
//   rel   = mean|cur - prev| / mean|prev|            (means over the same n: ratio of sums)
//   accum += polyval(coeff, rel)                     (numpy poly1d: coeff[0] is the highest power)
//   calc  = force || accum >= thresh;  if (calc) accum = 0
//   prev  = cur                                      (the reference's modulated_inp.clone())
// state[0] = accum (double, device).  flag: int32, device or mapped host memory.
// ------------------------------------------------------------------------------------------
template <typename T>
__device__ __forceinline__ float to_f(T v);
template <> __device__ __forceinline__ float to_f<float>(float v) { return v; }

template <typename T>
__global__ void __launch_bounds__(1024)
teacache_gate_kernel(const T* __restrict__ cur, T* prev, long long n, JengaTeaCacheArgs a) {
  __shared__ double s_num[1024], s_den[1024];
  double num = 0.0, den = 0.0;
  for (long long i = threadIdx.x; i < n; i += blockDim.x) {
    const float c = to_f<T>(cur[i]);
    if (!a.force) {
      const float p = to_f<T>(prev[i]);
      num += static_cast<double>(fabsf(c - p));
      den += static_cast<double>(fabsf(p));
    }
    if (a.update_prev) prev[i] = cur[i];
  }
  s_num[threadIdx.x] = num;
  s_den[threadIdx.x] = den;
  __syncthreads();
  for (int off = blockDim.x / 2; off > 0; off >>= 1) {
    if (threadIdx.x < off) {
      s_num[threadIdx.x] += s_num[threadIdx.x + off];
      s_den[threadIdx.x] += s_den[threadIdx.x + off];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    double accum = a.state[0];
    int calc;
    if (a.force) {
      calc = 1;
      accum = 0.0;
    } else {
      // the reference divides two fp32 means and hands the fp32 quotient to numpy (float64)
      const float rel32 = static_cast<float>(s_num[0] / static_cast<double>(n)) /
                          static_cast<float>(s_den[0] / static_cast<double>(n));
      const double rel = static_cast<double>(rel32);
      double y = 0.0;
      for (int k = 0; k < a.n_coeff; ++k) y = y * rel + a.coeff[k];
      accum += y;
      calc = accum < a.thresh ? 0 : 1;
      if (calc) accum = 0.0;
    }
    a.state[0] = accum;
    if (a.rel_out) a.rel_out[0] = a.force ? 0.0 : static_cast<double>(
        static_cast<float>(s_num[0] / static_cast<double>(n)) / static_cast<float>(s_den[0] / static_cast<double>(n)));
    *a.flag = calc;
    __threadfence_system();
  }
}

}  // namespace
}  // namespace jenga

extern "C" int jenga_residual_apply(void* x, const void* residual, int64_t n, int32_t dtype, void* stream) {
  return jenga::launch_residual(x, residual, x, n, dtype, false, static_cast<cudaStream_t>(stream));
}

extern "C" int jenga_residual_store(const void* x_new, const void* x_old, void* residual, int64_t n,
                                    int32_t dtype, void* stream) {
  return jenga::launch_residual(x_new, x_old, residual, n, dtype, true, static_cast<cudaStream_t>(stream));
}

extern "C" int jenga_teacache_gate(const JengaTeaCacheArgs* a, void* stream) {
  using namespace jenga;
  if (!a || !a->cur || !a->prev || !a->state || !a->flag)
    return set_error(JENGA_E_INVALID, "teacache_gate: null pointer");
  if (a->n <= 0 || a->n_coeff < 1 || a->n_coeff > 8)
    return set_error(JENGA_E_INVALID, "teacache_gate: bad sizes");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  // the reference asserts fp32 embeddings (wan/modules/model_mul.py: `assert e.dtype == torch.float32
  // and e0.dtype == torch.float32`); 16-bit inputs would take ATen's 16-bit mean/divide roundings,
  // which this kernel does not restate
  if (a->dtype != JENGA_F32) return set_error(JENGA_E_UNSUPPORTED, "teacache_gate: embeddings must be f32");
  teacache_gate_kernel<float><<<1, 1024, 0, s>>>(static_cast<const float*>(a->cur), static_cast<float*>(a->prev),
                                                 a->n, *a);
  const cudaError_t ce = cudaGetLastError();
  return ce == cudaSuccess ? JENGA_OK : set_cuda_error(ce, "teacache_gate launch");
}

// ------------------------------------------------------------------------------------------
// ProRes stage switch (SURVEY §8 f-2): at the step where Jenga's progressive-resolution schedule
// moves to the next (larger) latent grid the reference runs, on the whole latent,
//   x0      = latents.float() + noise_pred.float() * (sigmas[-1] - sigmas[i])        scheduling_flow_match_discrete.py:258-282
//   x0_up   = F.interpolate(x0, size=(T, H2, W2), mode="trilinear")                   pipeline_hunyuan_video_prores.py:729
//   latents = x0_up * (1 - sigma_next) + noise.float() * sigma_next                   scheduling_flow_match_discrete.py:284-299
// as ~8 ATen kernels.  Here it is one gather kernel over the OUTPUT grid (one thread per output
// voxel and channel): the 8 source taps are read from latents and noise_pred directly, so x0 is
// never materialised.  Interpolation follows ATen's upsample_trilinear3d (align_corners=False):
// src = max(0, scale*(dst+0.5)-0.5) with scale = in/out, taps (i0, min(i0+1, in-1)), weights
// (1-lambda, lambda), nested as t(h(w)).
// ------------------------------------------------------------------------------------------
namespace jenga {
namespace {

__device__ __forceinline__ void src_index(float scale, int dst, int in_size, int& i0, int& ip, float& l0, float& l1) {
  const float s = fmaxf(scale * (static_cast<float>(dst) + 0.5f) - 0.5f, 0.f);
  i0 = static_cast<int>(s);
  if (i0 > in_size - 1) i0 = in_size - 1;
  ip = (i0 < in_size - 1) ? 1 : 0;
  l1 = s - static_cast<float>(i0);
  l0 = 1.f - l1;
}

__global__ void __launch_bounds__(256)
prores_switch_kernel(const float* __restrict__ lat, const float* __restrict__ pred, const float* __restrict__ noise,
                     float* __restrict__ out, int NC, int it, int ih, int iw, int ot, int oh, int ow,
                     float d_sigma, float sigma_next) {
  const long long total = static_cast<long long>(NC) * ot * oh * ow;
  const float st = static_cast<float>(it) / static_cast<float>(ot);
  const float sh = static_cast<float>(ih) / static_cast<float>(oh);
  const float sw = static_cast<float>(iw) / static_cast<float>(ow);
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(i % ow);
    const int y = static_cast<int>((i / ow) % oh);
    const int z = static_cast<int>((i / (static_cast<long long>(ow) * oh)) % ot);
    const long long nc = i / (static_cast<long long>(ow) * oh * ot);
    int t0, tp, h0, hp, w0, wp;
    float t0l, t1l, h0l, h1l, w0l, w1l;
    src_index(st, z, it, t0, tp, t0l, t1l);
    src_index(sh, y, ih, h0, hp, h0l, h1l);
    src_index(sw, x, iw, w0, wp, w0l, w1l);
    const long long base = nc * it * ih * iw;
    auto x0 = [&](int tt, int hh, int ww) {
      const long long o = base + (static_cast<long long>(tt) * ih + hh) * iw + ww;
      return __fadd_rn(__ldg(lat + o), __fmul_rn(__ldg(pred + o), d_sigma));
    };
    const float v =
        t0l * (h0l * (w0l * x0(t0, h0, w0) + w1l * x0(t0, h0, w0 + wp)) +
               h1l * (w0l * x0(t0, h0 + hp, w0) + w1l * x0(t0, h0 + hp, w0 + wp))) +
        t1l * (h0l * (w0l * x0(t0 + tp, h0, w0) + w1l * x0(t0 + tp, h0, w0 + wp)) +
               h1l * (w0l * x0(t0 + tp, h0 + hp, w0) + w1l * x0(t0 + tp, h0 + hp, w0 + wp)));
    out[i] = __fadd_rn(__fmul_rn(v, 1.0f - sigma_next), __fmul_rn(__ldg(noise + i), sigma_next));
  }
}

}  // namespace
}  // namespace jenga

extern "C" int jenga_prores_switch(const float* latents, const float* noise_pred, const float* noise, float* out,
                                   int32_t batch_channels, int32_t in_t, int32_t in_h, int32_t in_w,
                                   int32_t out_t, int32_t out_h, int32_t out_w, float d_sigma, float sigma_next,
                                   void* stream) {
  using namespace jenga;
  if (!latents || !noise_pred || !noise || !out) return set_error(JENGA_E_INVALID, "prores_switch: null pointer");
  if (batch_channels <= 0 || in_t <= 0 || in_h <= 0 || in_w <= 0 || out_t <= 0 || out_h <= 0 || out_w <= 0)
    return set_error(JENGA_E_INVALID, "prores_switch: bad shape");
  const long long total = static_cast<long long>(batch_channels) * out_t * out_h * out_w;
  long long blocks = (total + 255) / 256;
  if (blocks > static_cast<long long>(kNumSMs) * 16) blocks = static_cast<long long>(kNumSMs) * 16;
  prores_switch_kernel<<<static_cast<unsigned>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      latents, noise_pred, noise, out, batch_channels, in_t, in_h, in_w, out_t, out_h, out_w, d_sigma, sigma_next);
  const cudaError_t ce = cudaGetLastError();
  return ce == cudaSuccess ? JENGA_OK : set_cuda_error(ce, "prores_switch launch");
}
