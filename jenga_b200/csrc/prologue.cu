// Attention prologue for the HunyuanVideo DiT blocks: per-head RMSNorm(q,k) + RoPE(q,k on
// image tokens) + img||txt concatenation + block mean-pool of q and k, in ONE pass over qkv.
//
// Replaces (hyvideo/modules/models_mul_block_gc_ha_multigpu.py:200-241, single-stream
// :417-435) the chain  rearrange -> RMSNorm.forward (norm_layers.py:32-59) x4 ->
// apply_rotary_emb (posemb_layers.py:181-229) -> torch.cat x3  (~16 elementwise kernels and
// three 680 MB concatenation copies) and the two pooling reductions of the mask builder
// (attention_block_triton_diffres.py:216-217).
//
// Rounding points reproduced exactly (SURVEY Appendix A-10):
//   n  = bf16( x_f32 * rsqrt(mean(x_f32^2) + eps) )          norm_layers.py:56  .type_as(x)
//   y  = bf16( n * w )                                        :58  (bf16 x bf16 product)
//   r  = bf16( y_f32*cos + rotate_half(y_f32)*sin )           posemb_layers.py:211-212
//        with separate fp32 multiplies and add (no FMA contraction), interleaved pairs
//        rotate_half(y)[2i] = -y[2i+1], [2i+1] = y[2i]        :133-137
// Text tokens get the norm but no RoPE (:226-227).  v is copied unchanged.
//
// HBM-bound: reads qkv once (3*S*H*D*2 B) + cos/sin (2*L*D*4 B, L1/L2-shared by all heads),
// writes q,k,v once.  One CTA per 128-token block; a half-warp owns one (token, head) row
// (8 channels per lane), so the norm reduction is 4 shuffles and each lane keeps the pooling
// partial sums of its own 8 channels across the 128 tokens of the block.
#include <cstdlib>

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "sm90_ptx.cuh"
#include "jenga_internal.h"

namespace jenga {

namespace {

constexpr int kBlock = 128;

template <bool kBF16>
__device__ __forceinline__ float rnd(float x) {
  if constexpr (kBF16) {
    return __bfloat162float(__float2bfloat16_rn(x));
  } else {
    return __half2float(__float2half_rn(x));
  }
}

struct PrologueParams {
  // image and text qkv: [B, L, 3, H, D] views; element strides for (batch, token, which, head)
  const uint16_t* img;
  const uint16_t* txt;
  long long img_sb, img_ss, img_sw, img_sh;
  long long txt_sb, txt_ss, txt_sw, txt_sh;
  int L, T, H;                  // image tokens, text tokens, heads (D == 128)
  const uint16_t* w_img_q;      // [D] norm weights (may be null == ones)
  const uint16_t* w_img_k;
  const uint16_t* w_txt_q;
  const uint16_t* w_txt_k;
  const float* cos_t;           // [L or table rows, D] fp32
  const float* sin_t;
  const long long* rope_index;  // optional [L]: row of the table for token i (hilbert_order)
  float eps;
  uint16_t* q;                  // [B, S, H, D] contiguous, S = L + T
  uint16_t* k;
  uint16_t* v;
  uint16_t* q_pool;             // [B, H, nb, D] or null
  uint16_t* k_pool;
  int nb;                       // ceil(S / 128)
};

template <bool kBF16>
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint4 v;
  v.x = pack2<kBF16>(f[0], f[1]);
  v.y = pack2<kBF16>(f[2], f[3]);
  v.z = pack2<kBF16>(f[4], f[5]);
  v.w = pack2<kBF16>(f[6], f[7]);
  return v;
}

// x (8 channels of one head row, spread over 16 lanes) -> normed, weighted, optionally rotated;
// values are left rounded to the 16-bit dtype (as floats).  c/s: this thread's 8 cos/sin values.
template <bool kBF16>
__device__ __forceinline__ void norm_rope8(float (&x)[8], const float (&w)[8], bool has_w, float eps,
                                           bool rotate, const float4 (&cs)[2], const float4 (&sn)[2],
                                           unsigned half_mask) {
  float ss = 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) ss = fmaf(x[i], x[i], ss);
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) ss += __shfl_xor_sync(half_mask, ss, o);
  const float r = rsqrtf(ss * (1.0f / 128.0f) + eps);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    float n = rnd<kBF16>(__fmul_rn(x[i], r));
    if (has_w) n = rnd<kBF16>(__fmul_rn(n, w[i]));
    x[i] = n;
  }
  if (rotate) {
    const float c[8] = {cs[0].x, cs[0].y, cs[0].z, cs[0].w, cs[1].x, cs[1].y, cs[1].z, cs[1].w};
    const float s[8] = {sn[0].x, sn[0].y, sn[0].z, sn[0].w, sn[1].x, sn[1].y, sn[1].z, sn[1].w};
    float y[8];
#pragma unroll
    for (int i = 0; i < 8; i += 2) {
      y[i] = rnd<kBF16>(__fadd_rn(__fmul_rn(x[i], c[i]), __fmul_rn(-x[i + 1], s[i])));
      y[i + 1] = rnd<kBF16>(__fadd_rn(__fmul_rn(x[i + 1], c[i + 1]), __fmul_rn(x[i], s[i + 1])));
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) x[i] = y[i];
  }
}

template <bool kBF16>
__device__ __forceinline__ void unpack8(const uint4& v, float (&f)[8]) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = unpack2<kBF16>(w[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}

template <bool kBF16>
__global__ void __launch_bounds__(384, 2)
hy_prologue_kernel(const PrologueParams p) {
  __shared__ float s_w[4][128];  // img_q, img_k, txt_q, txt_k norm weights
  const int blk = blockIdx.x;
  const int b = blockIdx.y;
  const int S = p.L + p.T;
  const int lane16 = threadIdx.x & 15;  // 8-channel chunk inside the head row
  const int d0 = lane16 * 8;
  const int rows_per_iter = blockDim.x >> 4;  // (token, head) rows handled per pass
  const long long tok0 = static_cast<long long>(blk) * kBlock;
  const int n_tok = static_cast<int>(max(0ll, min(static_cast<long long>(kBlock), S - tok0)));
  const bool has_w = p.w_img_q != nullptr;
  if (has_w) {
    for (int i = threadIdx.x; i < 4 * 128; i += blockDim.x) {
      const uint16_t* src = (i < 128) ? p.w_img_q : (i < 256) ? p.w_img_k : (i < 384) ? p.w_txt_q : p.w_txt_k;
      const uint16_t raw = src[i & 127];
      s_w[i >> 7][i & 127] = kBF16 ? __uint_as_float(static_cast<uint32_t>(raw) << 16)
                                   : __half2float(__ushort_as_half(raw));
    }
  }
  __syncthreads();

  // A thread always serves the same head set {h : (h - hslot) % rows_per_iter == 0} so its
  // pooling accumulators are per (head, chunk).  With H <= rows_per_iter (24 <= 24) that is
  // exactly one head per half-warp and the CTA's tokens are walked sequentially.
  const int hslot = threadIdx.x >> 4;
  // the two half-warps of a warp may serve different head counts: shuffle inside the half only
  const unsigned half_mask = (threadIdx.x & 16) ? 0xffff0000u : 0x0000ffffu;
  for (int h = hslot; h < p.H; h += rows_per_iter) {
    float qsum[8], ksum[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) qsum[i] = ksum[i] = 0.f;
    for (int t = 0; t < n_tok; ++t) {
      const long long tok = tok0 + t;
      const bool is_img = tok < p.L;
      const uint16_t* src = is_img ? p.img + b * p.img_sb + tok * p.img_ss + h * p.img_sh + d0
                                   : p.txt + b * p.txt_sb + (tok - p.L) * p.txt_ss + h * p.txt_sh + d0;
      const long long sw = is_img ? p.img_sw : p.txt_sw;
      const uint4 rq = __ldg(reinterpret_cast<const uint4*>(src));
      const uint4 rk = __ldg(reinterpret_cast<const uint4*>(src + sw));
      const uint4 rv = __ldg(reinterpret_cast<const uint4*>(src + 2 * sw));
      float4 rc[2], rs[2];
      if (is_img && p.cos_t) {
        const long long row = p.rope_index ? __ldg(p.rope_index + tok) : tok;
        const float4* cp = reinterpret_cast<const float4*>(p.cos_t + row * 128 + d0);
        const float4* sp = reinterpret_cast<const float4*>(p.sin_t + row * 128 + d0);
        rc[0] = __ldg(cp);
        rc[1] = __ldg(cp + 1);
        rs[0] = __ldg(sp);
        rs[1] = __ldg(sp + 1);
      }
      float q[8], k[8], wq[8], wk[8];
      unpack8<kBF16>(rq, q);
      unpack8<kBF16>(rk, k);
      if (has_w) {
        const float* wqs = s_w[is_img ? 0 : 2] + d0;
        const float* wks = s_w[is_img ? 1 : 3] + d0;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          wq[i] = wqs[i];
          wk[i] = wks[i];
        }
      }
      // tested again rather than reusing is_img: with is_img kept live across the loads, the f16
      // instantiation spills 8 more bytes per thread
      const bool rotate = tok < p.L && p.cos_t != nullptr;
      norm_rope8<kBF16>(q, wq, has_w, p.eps, rotate, rc, rs, half_mask);
      norm_rope8<kBF16>(k, wk, has_w, p.eps, rotate, rc, rs, half_mask);
      const long long o = ((static_cast<long long>(b) * S + tok) * p.H + h) * 128 + d0;
      *reinterpret_cast<uint4*>(p.q + o) = pack8<kBF16>(q);
      *reinterpret_cast<uint4*>(p.k + o) = pack8<kBF16>(k);
      *reinterpret_cast<uint4*>(p.v + o) = rv;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        qsum[i] += q[i];
        ksum[i] += k[i];
      }
    }
    if (p.q_pool) {
      float qm[8], km[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        qm[i] = qsum[i] * (1.0f / kBlock);  // missing tail rows count as zeros (padding)
        km[i] = ksum[i] * (1.0f / kBlock);
      }
      const long long o = ((static_cast<long long>(b) * p.H + h) * p.nb + blk) * 128 + d0;
      *reinterpret_cast<uint4*>(p.q_pool + o) = pack8<kBF16>(qm);
      *reinterpret_cast<uint4*>(p.k_pool + o) = pack8<kBF16>(km);
    }
  }
}

}  // namespace

int hy_prologue_impl(const JengaHyPrologueArgs* a, cudaStream_t stream) {
  if (!a || !a->img_qkv || !a->q || !a->k || !a->v)
    return set_error(JENGA_E_INVALID, "hy_prologue: null pointer");
  if (a->dtype != JENGA_BF16 && a->dtype != JENGA_F16)
    return set_error(JENGA_E_INVALID, "hy_prologue: dtype must be bf16/f16");
  if (a->head_dim != 128) return set_error(JENGA_E_UNSUPPORTED, "hy_prologue: head_dim must be 128");
  if (a->batch <= 0 || a->heads <= 0 || a->img_tokens <= 0 || a->txt_tokens < 0)
    return set_error(JENGA_E_INVALID, "hy_prologue: bad shape");
  if (a->txt_tokens > 0 && !a->txt_qkv) return set_error(JENGA_E_INVALID, "hy_prologue: txt_qkv missing");
  const bool any_w = a->w_img_q || a->w_img_k || a->w_txt_q || a->w_txt_k;
  const bool all_w = a->w_img_q && a->w_img_k && (a->txt_tokens == 0 || (a->w_txt_q && a->w_txt_k));
  if (any_w && !all_w) return set_error(JENGA_E_INVALID, "hy_prologue: give all norm weights or none");
  if ((a->rope_cos == nullptr) != (a->rope_sin == nullptr))
    return set_error(JENGA_E_INVALID, "hy_prologue: cos and sin go together");
  if ((a->q_pool == nullptr) != (a->k_pool == nullptr))
    return set_error(JENGA_E_INVALID, "hy_prologue: q_pool and k_pool go together");
  const long long st[] = {a->img_stride_b, a->img_stride_s, a->img_stride_w, a->img_stride_h,
                          a->txt_stride_b, a->txt_stride_s, a->txt_stride_w, a->txt_stride_h};
  for (long long s : st)
    if (s % 8) return set_error(JENGA_E_INVALID, "hy_prologue: strides must be multiples of 8 elements");
  PrologueParams p{};
  p.img = static_cast<const uint16_t*>(a->img_qkv);
  p.txt = static_cast<const uint16_t*>(a->txt_qkv);
  p.img_sb = a->img_stride_b; p.img_ss = a->img_stride_s; p.img_sw = a->img_stride_w; p.img_sh = a->img_stride_h;
  p.txt_sb = a->txt_stride_b; p.txt_ss = a->txt_stride_s; p.txt_sw = a->txt_stride_w; p.txt_sh = a->txt_stride_h;
  p.L = static_cast<int>(a->img_tokens);
  p.T = static_cast<int>(a->txt_tokens);
  p.H = a->heads;
  p.w_img_q = static_cast<const uint16_t*>(a->w_img_q);
  p.w_img_k = static_cast<const uint16_t*>(a->w_img_k);
  p.w_txt_q = static_cast<const uint16_t*>(a->w_txt_q ? a->w_txt_q : a->w_img_q);
  p.w_txt_k = static_cast<const uint16_t*>(a->w_txt_k ? a->w_txt_k : a->w_img_k);
  p.cos_t = a->rope_cos;
  p.sin_t = a->rope_sin;
  p.rope_index = reinterpret_cast<const long long*>(a->rope_index);
  p.eps = a->eps;
  p.q = static_cast<uint16_t*>(a->q);
  p.k = static_cast<uint16_t*>(a->k);
  p.v = static_cast<uint16_t*>(a->v);
  p.q_pool = static_cast<uint16_t*>(a->q_pool);
  p.k_pool = static_cast<uint16_t*>(a->k_pool);
  const long long S = a->img_tokens + a->txt_tokens;
  p.nb = static_cast<int>((S + kBlock - 1) / kBlock);
  int threads = a->heads * 16;
  if (threads > 384) threads = 384;
  threads = ((threads + 31) / 32) * 32;
  // Default: the bulk-async (cp.async.bulk) persistent form in prologue_bulk.cu, q/k/v bit-identical
  // to this file's kernel.  It returns a positive value for
  // layouts it does not take (head stride != 128, > 24 heads, misaligned rows, first use on a stream
  // that is being captured into a graph) and then the register-staged kernel below runs instead.
  // JENGA_PROLOGUE=classic forces the kernel below (read per call: tests switch it in-process).
  const char* mode = std::getenv("JENGA_PROLOGUE");
  const bool classic = mode && mode[0] == 'c';
  if (!classic) {
    const int r = hy_prologue_bulk_try(a, stream);
    if (r <= 0) return r;
  }
  dim3 grid(p.nb, a->batch);
  if (a->dtype == JENGA_BF16)
    hy_prologue_kernel<true><<<grid, threads, 0, stream>>>(p);
  else
    hy_prologue_kernel<false><<<grid, threads, 0, stream>>>(p);
  cudaError_t ce = cudaGetLastError();
  return ce == cudaSuccess ? JENGA_OK : set_cuda_error(ce, "hy_prologue launch");
}

}  // namespace jenga

// =============================================================================================
// Wan2.1 self-attention prologue: full-width RMSNorm (WanRMSNorm, wan/modules/model_mul.py:74-90)
// + 3-axis complex RoPE in fp64 (rope_apply :40-71, with the freq_remap gather :63-65), output
// rounded fp64 -> fp32 (`.float()` :71) -> bf16 (the operator's cast, wan/...diffres.py:456-463).
// One warp per token; two passes over the token's C = H*D channels (second pass hits L1/L2).
// =============================================================================================
namespace jenga {
namespace {

struct WanPrologueParams {
  const void* x;        // [B, L, C] projection output (bf16 or f32)
  const void* w;        // [C] norm weight (bf16 or f32)
  int x_f32, w_f32;
  long long sb, ss;     // element strides of x (batch, token)
  int L, C, H;          // tokens, channels, heads (D = C / H = 128)
  float eps;
  const double* freqs;  // [rows, 64, 2] (re, im) — torch.view_as_real of the complex128 table
  int freq_rows;
  int gf, gh, gw;       // latent grid (F, H, W); tokens >= F*H*W get no rotation (:66)
  const long long* remap;  // optional [F*H*W]: position of token i (hilbert_order)
  uint16_t* out;        // [B, L, H, 128] bf16, contiguous
};

__device__ __forceinline__ float bf16_round(float v) { return __bfloat162float(__float2bfloat16_rn(v)); }

__global__ void __launch_bounds__(256)
wan_prologue_kernel(const WanPrologueParams p) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.y;
  if (warp >= p.L) return;
  const long long tok = warp;
  const char* xrow = static_cast<const char*>(p.x) + (b * p.sb + tok * p.ss) * (p.x_f32 ? 4 : 2);
  auto load_x = [&](int c) -> float {
    return p.x_f32 ? reinterpret_cast<const float*>(xrow)[c]
                   : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(xrow)[c]);
  };
  // pass 1: mean of squares in fp32 (x.float().pow(2).mean(-1))
  float ss = 0.f;
  for (int c = lane * 2; c < p.C; c += 64) {
    const float a = load_x(c), bb = load_x(c + 1);
    ss = fmaf(a, a, ss);
    ss = fmaf(bb, bb, ss);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const float r = rsqrtf(ss / static_cast<float>(p.C) + p.eps);
  // rotation source position
  const long long n_grid = static_cast<long long>(p.gf) * p.gh * p.gw;
  const bool rotate = tok < n_grid && p.freqs != nullptr;
  int fi = 0, hi = 0, wi = 0;
  if (rotate) {
    const long long pos = p.remap ? __ldg(p.remap + tok) : tok;
    fi = static_cast<int>(pos / (static_cast<long long>(p.gh) * p.gw));
    const int rem = static_cast<int>(pos - static_cast<long long>(fi) * p.gh * p.gw);
    hi = rem / p.gw;
    wi = rem - hi * p.gw;
  }
  const int c3 = 64 / 3;              // 21
  const int s0 = 64 - 2 * c3;         // 22: split sizes [22, 21, 21] (:44)
  // pass 2: one complex pair (2 channels) per lane step
  for (int c = lane * 2; c < p.C; c += 64) {
    float y[2];
#pragma unroll
    for (int t = 0; t < 2; ++t) {
      float v = __fmul_rn(load_x(c + t), r);          // _norm in fp32
      if (!p.x_f32) v = bf16_round(v);                // .type_as(x)
      float wv = p.w ? (p.w_f32 ? reinterpret_cast<const float*>(p.w)[c + t]
                                : __bfloat162float(reinterpret_cast<const __nv_bfloat16*>(p.w)[c + t]))
                     : 1.0f;
      v = __fmul_rn(v, wv);                            // * self.weight (promotes to fp32 unless both bf16)
      if (!p.x_f32 && !p.w_f32) v = bf16_round(v);
      y[t] = v;
    }
    float o0 = y[0], o1 = y[1];
    if (rotate) {
      const int j = (c & 127) >> 1;  // complex index inside the head
      const int row = j < s0 ? fi : (j < s0 + c3 ? hi : wi);
      const double2 f = __ldg(reinterpret_cast<const double2*>(p.freqs) + static_cast<long long>(row) * 64 + j);
      const double a = static_cast<double>(y[0]), bb = static_cast<double>(y[1]);
      // complex128 product (a + bi)(c + di), then .float()
      o0 = static_cast<float>(a * f.x - bb * f.y);
      o1 = static_cast<float>(a * f.y + bb * f.x);
    }
    const uint32_t packed = pack2<true>(o0, o1);
    reinterpret_cast<uint32_t*>(p.out + (static_cast<long long>(b) * p.L + tok) * p.C)[c >> 1] = packed;
  }
}

}  // namespace

int wan_prologue_impl(const JengaWanPrologueArgs* a, cudaStream_t stream) {
  if (!a || !a->x || !a->out) return set_error(JENGA_E_INVALID, "wan_prologue: null pointer");
  if (a->head_dim != 128) return set_error(JENGA_E_UNSUPPORTED, "wan_prologue: head_dim must be 128");
  if (a->batch <= 0 || a->tokens <= 0 || a->heads <= 0) return set_error(JENGA_E_INVALID, "wan_prologue: bad shape");
  if ((a->x_dtype != JENGA_BF16 && a->x_dtype != JENGA_F32) || (a->w && a->w_dtype != JENGA_BF16 && a->w_dtype != JENGA_F32))
    return set_error(JENGA_E_INVALID, "wan_prologue: dtypes must be bf16 or f32");
  if (a->freqs && (a->grid_f <= 0 || a->grid_h <= 0 || a->grid_w <= 0 || a->grid_f > a->freq_rows ||
                   a->grid_h > a->freq_rows || a->grid_w > a->freq_rows))
    return set_error(JENGA_E_INVALID, "wan_prologue: grid exceeds the frequency table");
  WanPrologueParams p{};
  p.x = a->x; p.w = a->w;
  p.x_f32 = a->x_dtype == JENGA_F32; p.w_f32 = a->w_dtype == JENGA_F32;
  p.sb = a->stride_b; p.ss = a->stride_s;
  p.L = static_cast<int>(a->tokens); p.H = a->heads; p.C = a->heads * 128;
  p.eps = a->eps;
  p.freqs = a->freqs; p.freq_rows = a->freq_rows;
  p.gf = a->grid_f; p.gh = a->grid_h; p.gw = a->grid_w;
  p.remap = reinterpret_cast<const long long*>(a->freq_remap);
  p.out = static_cast<uint16_t*>(a->out);
  dim3 grid(static_cast<unsigned>((a->tokens + 7) / 8), static_cast<unsigned>(a->batch));
  wan_prologue_kernel<<<grid, 256, 0, stream>>>(p);
  cudaError_t ce = cudaGetLastError();
  return ce == cudaSuccess ? JENGA_OK : set_cuda_error(ce, "wan_prologue launch");
}

}  // namespace jenga
