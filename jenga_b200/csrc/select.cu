// Block scoring and selection — the device-side replacement of the reference's
// _build_block_index_with_importance_optimized
//   (hyvideo/modules/attention_block_triton_diffres.py:198-295, wan twin :306-411).
//
// The reference strings ~25 ATen kernels together (mean, bmm, softmax, sort, cumsum, four
// boolean-mask gathers that each synchronise with the host, index_put, OR) and materialises a
// [B,H,nq,nb] bool tensor.  Here it is two kernels, no host sync, and the result is the packed
// bit rows the attention kernel consumes:
//   block_pool_kernel   : HBM-bound mean over each 128-token block (one read of q and k)
//   select_blocks_kernel: per (head, 8 query blocks): pooled scores -> fp32 softmax -> full
//                         descending sort (ties: lower index first, like CUDA torch.sort) ->
//                         cumulative-probability cut -> max(count, top_k) -> union with
//                         neighbour / first-frame / text columns -> bit row
// Rounding points follow the reference under torch.autocast(bf16) (SURVEY Appendix A-5):
// pooled means, the pooled dot products and their product with D^-1/2 are each rounded to the
// input dtype; softmax and the cumulative sum are fp32.
#include <cstdlib>
#include <cstring>

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "sm90_ptx.cuh"
#include "jenga_internal.h"

namespace jenga {

namespace {

constexpr int kBlock = 128;

template <int kDtype>
__device__ __forceinline__ float round_to(float x) {
  if constexpr (kDtype == JENGA_BF16) {
    return __bfloat162float(__float2bfloat16_rn(x));
  } else {
    return __half2float(__float2half_rn(x));
  }
}
template <int kDtype>
__device__ __forceinline__ uint16_t to_bits16(float x) {
  if constexpr (kDtype == JENGA_BF16) {
    return __bfloat16_as_ushort(__float2bfloat16_rn(x));
  } else {
    return __half_as_ushort(__float2half_rn(x));
  }
}
template <int kDtype>
__device__ __forceinline__ float from_bits16(uint16_t v) {
  if constexpr (kDtype == JENGA_BF16) {
    return __uint_as_float(static_cast<uint32_t>(v) << 16);
  } else {
    return __half2float(__ushort_as_half(v));
  }
}

// ------------------------------------------------------------------------------------------
// block_pool: pooled[b,h,blk,:] = round(mean over the 128 rows of the block), rows >= S count
// as zeros (the Wan / I2V variants zero-pad before pooling, wan/…:448-451).
// ref :216-217.  kIn: element type of x (bf16, f16 or f32).  With f32 input every element is
// first rounded to bf16 (wan/…:456-463 casts before the builder runs) and, if cast_out is
// given, the rounded copy is written contiguously as [B,S,H,D] bf16.
// grid: (block, batch); thread -> 8 consecutive channels of one head.
// ------------------------------------------------------------------------------------------
template <int kIn, int kOut>
__global__ void __launch_bounds__(256)
block_pool_kernel(const void* __restrict__ x, uint16_t* __restrict__ pooled,
                  uint16_t* __restrict__ cast_out, int heads, int head_dim, long long rows,
                  long long sb, long long ss, long long sh, int n_blocks) {
  const int blk = blockIdx.x;
  const int b = blockIdx.y;
  const int vec_per_head = head_dim / 8;
  const int vecs = heads * vec_per_head;
  const long long row0 = static_cast<long long>(blk) * kBlock;
  const int n_rows = static_cast<int>(min(static_cast<long long>(kBlock), rows - row0));
  for (int vidx = threadIdx.x; vidx < vecs; vidx += blockDim.x) {
    const int h = vidx / vec_per_head;
    const int d0 = (vidx - h * vec_per_head) * 8;
    float acc[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) acc[i] = 0.f;
    if constexpr (kIn == JENGA_F32) {
      const float* base = static_cast<const float*>(x) + b * sb + h * sh + d0;
#pragma unroll 4
      for (int r = 0; r < n_rows; ++r) {
        const float4* p = reinterpret_cast<const float4*>(base + (row0 + r) * ss);
        const float4 lo = __ldg(p), hi = __ldg(p + 1);
        const float f[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
        uint16_t o16[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          o16[i] = to_bits16<kOut>(f[i]);
          acc[i] += from_bits16<kOut>(o16[i]);
        }
        if (cast_out) {
          uint4 v;
          v.x = o16[0] | (static_cast<uint32_t>(o16[1]) << 16);
          v.y = o16[2] | (static_cast<uint32_t>(o16[3]) << 16);
          v.z = o16[4] | (static_cast<uint32_t>(o16[5]) << 16);
          v.w = o16[6] | (static_cast<uint32_t>(o16[7]) << 16);
          *reinterpret_cast<uint4*>(cast_out + ((static_cast<long long>(b) * rows + row0 + r) * heads + h) *
                                                   head_dim + d0) = v;
        }
      }
    } else {
      const uint16_t* base = static_cast<const uint16_t*>(x) + b * sb + h * sh + d0;
#pragma unroll 8
      for (int r = 0; r < n_rows; ++r) {
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(base + (row0 + r) * ss));
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          acc[2 * i] += from_bits16<kIn>(static_cast<uint16_t>(w[i] & 0xffffu));
          acc[2 * i + 1] += from_bits16<kIn>(static_cast<uint16_t>(w[i] >> 16));
        }
      }
    }
    uint16_t o16[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) o16[i] = to_bits16<kOut>(acc[i] * (1.0f / kBlock));
    uint4 v;
    v.x = o16[0] | (static_cast<uint32_t>(o16[1]) << 16);
    v.y = o16[2] | (static_cast<uint32_t>(o16[3]) << 16);
    v.z = o16[4] | (static_cast<uint32_t>(o16[5]) << 16);
    v.w = o16[6] | (static_cast<uint32_t>(o16[7]) << 16);
    *reinterpret_cast<uint4*>(pooled + ((static_cast<long long>(b) * heads + h) * n_blocks + blk) * head_dim +
                              d0) = v;
  }
}

// ------------------------------------------------------------------------------------------
// select_blocks
// ------------------------------------------------------------------------------------------
struct SelectParams {
  const uint16_t* q_pool;  // [BH, nq, D]
  const uint16_t* k_pool;  // [BH, nk_pool, D]  (first n_img rows are used)
  int nk_pool;
  int head_dim;
  int nq;           // query blocks (image rows)
  int n_img;        // ranked key blocks == text_start_block
  int nb;           // all key blocks (bit row covers these)
  int words;        // bit-row pitch
  int top_k;
  float p_threshold;
  int text_blocks;
  int first_frame_blocks;
  const uint32_t* nbr_bits;  // [nbr_rows, nbr_words] or null
  int nbr_rows, nbr_words;
  uint32_t* out_bits;  // [BH, nq, words]
  int32_t* out_counts;  // [BH, nq] importance count n (before unions), may be null
  int rows_per_cta;          // fused kernel: rows handled by one CTA
  long long total_rows;      // two-kernel path: batch_heads * nq
  int npow2;  // sort width
};

// Warp-cooperative bitonic sort, descending, of n2 (power of two) 64-bit keys in shared memory.
// Each lane owns n2/64 compare-exchange PAIRS per pass (no idle half), indexed so that the two
// elements of a pair are (i, i|j) with bit j of i clear.
__device__ void warp_bitonic_desc(unsigned long long* keys, int n2, int lane) {
  const int npairs = n2 >> 1;
  for (int k = 2; k <= n2; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
#pragma unroll 4
      for (int t = lane; t < npairs; t += 32) {
        const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
        const int ixj = i | j;
        const unsigned long long a = keys[i], b = keys[ixj];
        const bool desc_seg = (i & k) == 0;
        if (desc_seg ? (a < b) : (a > b)) {
          keys[i] = b;
          keys[ixj] = a;
        }
      }
      __syncwarp();
    }
  }
}

// Register-resident variant for <= 1024 keys: lane L owns sorted positions [32L, 32L+32).
// Compare-exchange partners at distance < 32 live in the same lane (pure register moves);
// distance >= 32 is one 64-bit shuffle.  ~3x fewer instructions than the shared-memory version
// and no shared-memory traffic.
__device__ __forceinline__ void warp_bitonic_desc_regs(unsigned long long (&key)[32], int lane) {
#pragma unroll
  for (int k = 2; k <= 1024; k <<= 1) {
#pragma unroll
    for (int j = k >> 1; j > 0; j >>= 1) {
      if (j >= 32) {
        const int lj = j >> 5;
        const bool lower = (lane & lj) == 0;
        const bool desc = ((lane << 5) & k) == 0;
        const bool keep_max = lower == desc;
#pragma unroll
        for (int r = 0; r < 32; ++r) {
          const unsigned long long other = __shfl_xor_sync(0xffffffffu, key[r], lj);
          const bool take = keep_max ? (other > key[r]) : (other < key[r]);
          key[r] = take ? other : key[r];
        }
      } else {
#pragma unroll
        for (int r = 0; r < 32; ++r) {
          if ((r & j) == 0) {
            const int r2 = r | j;
            // k < 32: direction is a compile-time function of r; k >= 32: of the lane
            const bool desc = (k < 32) ? ((r & k) == 0) : (((lane << 5) & k) == 0);
            const unsigned long long a = key[r], b = key[r2];
            const bool swap = desc ? (a < b) : (a > b);
            key[r] = swap ? b : a;
            key[r2] = swap ? a : b;
          }
        }
      }
    }
  }
}

template <int kDtype, bool kRegSort>
__global__ void __launch_bounds__(256)
select_blocks_kernel(const SelectParams p) {
  extern __shared__ uint8_t smem_sel[];
  const int R = p.rows_per_cta;
  const int D = p.head_dim;
  // carve: q rows fp32 [R][D] | scores fp32 [R][n_img] | keys u64 [R][npow2] | bits [R][words]
  float* s_q = reinterpret_cast<float*>(smem_sel);
  float* s_sc = s_q + R * D;
  unsigned long long* s_keys =
      reinterpret_cast<unsigned long long*>(s_sc + ((R * p.n_img + 1) & ~1));
  uint32_t* s_bits = reinterpret_cast<uint32_t*>(s_keys + (kRegSort ? 0 : static_cast<size_t>(R) * p.npow2));

  const int groups = (p.nq + R - 1) / R;
  const int bh = blockIdx.x / groups;
  const int m0 = (blockIdx.x - bh * groups) * R;
  const int nrows = min(R, p.nq - m0);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nwarps = blockDim.x >> 5;

  // ---- pooled q rows -> fp32 shared
  for (int i = threadIdx.x; i < nrows * D; i += blockDim.x) {
    const int r = i / D, d = i - r * D;
    s_q[i] = from_bits16<kDtype>(p.q_pool[(static_cast<size_t>(bh) * p.nq + m0 + r) * D + d]);
  }
  for (int i = threadIdx.x; i < R * p.words; i += blockDim.x) s_bits[i] = 0;
  __syncthreads();

  // ---- scores: s[r][j] = round(round(q_r . k_j) * D^-1/2)     (ref :227)
  const float inv_sqrt_d = static_cast<float>(1.0 / sqrt(static_cast<double>(D)));
  for (int j = threadIdx.x; j < p.n_img; j += blockDim.x) {
    const uint4* krow =
        reinterpret_cast<const uint4*>(p.k_pool + (static_cast<size_t>(bh) * p.nk_pool + j) * D);
    float acc[8];
#pragma unroll
    for (int r = 0; r < 8; ++r) acc[r] = 0.f;
    for (int d8 = 0; d8 < D / 8; ++d8) {
      const uint4 v = __ldg(krow + d8);
      const uint32_t w[4] = {v.x, v.y, v.z, v.w};
      float kf[8];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        kf[2 * i] = from_bits16<kDtype>(static_cast<uint16_t>(w[i] & 0xffffu));
        kf[2 * i + 1] = from_bits16<kDtype>(static_cast<uint16_t>(w[i] >> 16));
      }
#pragma unroll
      for (int r = 0; r < 8; ++r) {
        if (r < nrows) {
          const float* qr = s_q + r * D + d8 * 8;
#pragma unroll
          for (int i = 0; i < 8; ++i) acc[r] = fmaf(qr[i], kf[i], acc[r]);
        }
      }
    }
#pragma unroll
    for (int r = 0; r < 8; ++r)
      if (r < nrows) s_sc[r * p.n_img + j] = round_to<kDtype>(round_to<kDtype>(acc[r]) * inv_sqrt_d);
  }
  __syncthreads();

  // ---- one warp per row: softmax, sort, cut, unions
  for (int r = warp; r < nrows; r += nwarps) {
    const int m = m0 + r;
    float* sc = s_sc + r * p.n_img;
    unsigned long long* keys = s_keys + static_cast<size_t>(r) * p.npow2;
    uint32_t* bits = s_bits + r * p.words;
    // softmax in fp32 (ref :238; autocast promotes softmax to fp32)
    float mx = -INFINITY;
    for (int j = lane; j < p.n_img; j += 32) mx = fmaxf(mx, sc[j]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
    for (int j = lane; j < p.n_img; j += 32) {
      const float e = expf(sc[j] - mx);
      sc[j] = e;
      sum += e;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    int n;
    if constexpr (kRegSort) {
      // keys: (prob bits, ~index): a descending sort puts equal probs in index order
      const float inv = 1.0f;  // probabilities are normalised below with a true division
      (void)inv;
      unsigned long long key[32];
#pragma unroll
      for (int q = 0; q < 32; ++q) {
        const int j = lane * 32 + q;
        unsigned long long kk = 0ull;
        if (j < p.n_img) {
          const float pr = sc[j] / sum;
          kk = (static_cast<unsigned long long>(__float_as_uint(pr)) << 32) |
               static_cast<unsigned long long>(0xffffffffu - static_cast<uint32_t>(j));
        }
        key[q] = kk;
      }
      warp_bitonic_desc_regs(key, lane);
      // cumulative probability in sorted order (ref :242-246): lane chunks in rank order
      float part = 0.f;
#pragma unroll
      for (int q = 0; q < 32; ++q) part += __uint_as_float(static_cast<uint32_t>(key[q] >> 32));
      float prefix = part;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const float t = __shfl_up_sync(0xffffffffu, prefix, o);
        if (lane >= o) prefix += t;
      }
      float run = prefix - part;
      int local = 0;
#pragma unroll
      for (int q = 0; q < 32; ++q) {
        run += __uint_as_float(static_cast<uint32_t>(key[q] >> 32));
        if (lane * 32 + q < p.n_img && run <= p.p_threshold) ++local;
      }
      int tot = local;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, o);
      n = min(max(tot + 1, p.top_k), p.n_img);  // ref :247-250
#pragma unroll
      for (int q = 0; q < 32; ++q) {
        if (lane * 32 + q < n) {
          const uint32_t idx = 0xffffffffu - static_cast<uint32_t>(key[q] & 0xffffffffull);
          atomicOr(&bits[idx >> 5], 1u << (idx & 31));
        }
      }
    } else {
    // keys: (prob bits, ~index) so that a descending sort puts equal probs in index order
    for (int j = lane; j < p.npow2; j += 32) {
      unsigned long long key = 0ull;
      if (j < p.n_img) {
        const float pr = sc[j] / sum;
        sc[j] = pr;
        key = (static_cast<unsigned long long>(__float_as_uint(pr)) << 32) |
              static_cast<unsigned long long>(0xffffffffu - static_cast<uint32_t>(j));
      }
      keys[j] = key;  // padding keys are 0 -> sort to the end
    }
    __syncwarp();
    warp_bitonic_desc(keys, p.npow2, lane);
    // cumulative probability in sorted order (ref :242-246): count = #(cumsum <= p) + 1.
    // cumsum of non-negative terms is monotone, so this is the first index that exceeds p.
    // Warp-parallel: each lane sums a contiguous chunk, chunks are combined in order.
    int count;
    {
      const int per = (p.n_img + 31) / 32;
      const int lo = lane * per, hi = min(p.n_img, lo + per);
      float part = 0.f;
      for (int i = lo; i < hi; ++i) part += __uint_as_float(static_cast<uint32_t>(keys[i] >> 32));
      float prefix = part;  // inclusive scan over lanes
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const float t = __shfl_up_sync(0xffffffffu, prefix, o);
        if (lane >= o) prefix += t;
      }
      float run = prefix - part;  // exclusive prefix of this lane's chunk
      int local = 0;              // #elements in my chunk with cumsum <= p
      for (int i = lo; i < hi; ++i) {
        run += __uint_as_float(static_cast<uint32_t>(keys[i] >> 32));
        if (run <= p.p_threshold) ++local;
      }
      int tot = local;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, o);
      count = tot + 1;
    }
    n = min(max(count, p.top_k), p.n_img);  // ref :247-250
    for (int i = lane; i < n; i += 32) {
      const uint32_t idx = 0xffffffffu - static_cast<uint32_t>(keys[i] & 0xffffffffull);
      atomicOr(&bits[idx >> 5], 1u << (idx & 31));
    }
    }
    __syncwarp();
    // unions (ref :280-293, wan :400-406); all restricted to the columns they address
    for (int w = lane; w < p.words; w += 32) {
      uint32_t v = bits[w];
      const int lo = w * 32;
      auto range_bits = [&](int a, int b) -> uint32_t {  // bits of [a,b) that fall in word w
        const int s = max(a, lo), e = min(b, lo + 32);
        if (e <= s) return 0u;
        const uint32_t hi_mask = (e - lo) >= 32 ? 0xffffffffu : ((1u << (e - lo)) - 1u);
        return hi_mask & ~((s - lo) > 0 ? ((1u << (s - lo)) - 1u) : 0u);
      };
      if (p.nbr_bits && m < p.nbr_rows && w < p.nbr_words)
        v |= p.nbr_bits[static_cast<size_t>(m) * p.nbr_words + w] & range_bits(0, p.n_img);
      if (m < p.first_frame_blocks) v |= range_bits(0, min(p.first_frame_blocks, p.nb));
      if (p.text_blocks > 0) v |= range_bits(p.n_img, min(p.n_img + p.text_blocks, p.nb));
      p.out_bits[(static_cast<size_t>(bh) * p.nq + m) * p.words + w] = v;
    }
    if (p.out_counts && lane == 0) p.out_counts[static_cast<size_t>(bh) * p.nq + m] = n;
  }
}

// ------------------------------------------------------------------------------------------
// Two-kernel fast path (n_img <= 1024, caller-provided score workspace):
//   pooled_scores_kernel : smem-tiled fp32 GEMM  scores = round(round(qp kp^T) * D^-1/2)
//   select_rows_kernel   : one warp per row — softmax, 32-bit register bitonic sort of the
//                          probabilities, cut, then selection by threshold with ties taken in
//                          index order (== a stable descending sort of (prob, index)).
// Same arithmetic, in the same order, as select_blocks_kernel: the dot products accumulate
// over d ascending with fmaf, so both paths produce identical bit rows.
// ------------------------------------------------------------------------------------------
template <int kDtype>
__global__ void __launch_bounds__(256)
pooled_scores_kernel(const uint16_t* __restrict__ q_pool, const uint16_t* __restrict__ k_pool,
                     float* __restrict__ scores, int nq, int nk_pool, int n_img, int D) {
  // 64 x 64 output tile per CTA, K = D = 128 resident in shared memory, 4 x 4 outputs per thread
  extern __shared__ float sm_sc[];
  float* As = sm_sc;                // [128][64 + 4]
  float* Bs = sm_sc + 128 * 68;     // [128][64 + 4]
  const int bh = blockIdx.z;
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  const int t = threadIdx.x;
  for (int i = t; i < 64 * 16; i += 256) {
    const int row = i >> 4, chunk = i & 15;
    uint4 va = make_uint4(0, 0, 0, 0), vb = make_uint4(0, 0, 0, 0);
    if (m0 + row < nq) va = __ldg(reinterpret_cast<const uint4*>(q_pool + (static_cast<size_t>(bh) * nq + m0 + row) * D) + chunk);
    if (n0 + row < n_img) vb = __ldg(reinterpret_cast<const uint4*>(k_pool + (static_cast<size_t>(bh) * nk_pool + n0 + row) * D) + chunk);
    const uint32_t wa[4] = {va.x, va.y, va.z, va.w}, wb[4] = {vb.x, vb.y, vb.z, vb.w};
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      As[(chunk * 8 + 2 * e) * 68 + row] = from_bits16<kDtype>(static_cast<uint16_t>(wa[e] & 0xffffu));
      As[(chunk * 8 + 2 * e + 1) * 68 + row] = from_bits16<kDtype>(static_cast<uint16_t>(wa[e] >> 16));
      Bs[(chunk * 8 + 2 * e) * 68 + row] = from_bits16<kDtype>(static_cast<uint16_t>(wb[e] & 0xffffu));
      Bs[(chunk * 8 + 2 * e + 1) * 68 + row] = from_bits16<kDtype>(static_cast<uint16_t>(wb[e] >> 16));
    }
  }
  __syncthreads();
  const int ty = t >> 4, tx = t & 15;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
#pragma unroll 8
  for (int k = 0; k < 128; ++k) {
    const float4 a = *reinterpret_cast<const float4*>(As + k * 68 + ty * 4);
    const float4 b = *reinterpret_cast<const float4*>(Bs + k * 68 + tx * 4);
    const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
  }
  const float inv_sqrt_d = static_cast<float>(1.0 / sqrt(static_cast<double>(D)));
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= nq) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n < n_img)
        scores[(static_cast<size_t>(bh) * nq + m) * n_img + n] =
            round_to<kDtype>(round_to<kDtype>(acc[i][j]) * inv_sqrt_d);  // ref :227
    }
  }
}

// Tensor-core form of the pooled-score GEMM (the reference does this step with a bf16 cuBLAS
// bmm, …triton_diffres.py:227): mma.sync m16n8k16, 16-bit operands, fp32 accumulate, same two
// rounding points on the way out.  Legacy warp-level MMA on purpose: the whole problem is
// 5 GFLOP (24 heads x 900 x 900 x 128) — a wgmma pipeline would cost more to set up than
// the math takes.  64x64 outputs per CTA, 4 warps of 32x32.
template <int kDtype>
__device__ __forceinline__ void mma_16816(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  if constexpr (kDtype == JENGA_BF16) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  } else {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  }
}

template <int kDtype>
__global__ void __launch_bounds__(128)
pooled_scores_mma_kernel(const uint16_t* __restrict__ q_pool, const uint16_t* __restrict__ k_pool,
                         float* __restrict__ scores, int nq, int nk_pool, int n_img) {
  constexpr int D = 128, LD = D + 8;             // +8 halves: ldmatrix rows land in distinct banks
  __shared__ __align__(16) uint16_t As[64 * LD];
  __shared__ __align__(16) uint16_t Bs[64 * LD];
  const int bh = blockIdx.z;
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  for (int i = t; i < 64 * 16; i += 128) {
    const int row = i >> 4, chunk = i & 15;
    uint4 va = make_uint4(0, 0, 0, 0), vb = make_uint4(0, 0, 0, 0);
    if (m0 + row < nq) va = __ldg(reinterpret_cast<const uint4*>(q_pool + (static_cast<size_t>(bh) * nq + m0 + row) * D) + chunk);
    if (n0 + row < n_img) vb = __ldg(reinterpret_cast<const uint4*>(k_pool + (static_cast<size_t>(bh) * nk_pool + n0 + row) * D) + chunk);
    *reinterpret_cast<uint4*>(As + row * LD + chunk * 8) = va;
    *reinterpret_cast<uint4*>(Bs + row * LD + chunk * 8) = vb;
  }
  __syncthreads();
  const int wm = warp >> 1, wn = warp & 1;
  float acc[2][4][4];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc[i][j][e] = 0.f;
  const int mat = lane >> 3, r8 = lane & 7;
#pragma unroll
  for (int ks = 0; ks < D / 16; ++ks) {
    const int k0 = ks * 16;
    uint32_t a[2][4], b[2][4];
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
      ldmatrix_x4(a[mi], As + (wm * 32 + mi * 16 + r8 + (mat & 1) * 8) * LD + k0 + (mat >> 1) * 8);
#pragma unroll
    for (int nj = 0; nj < 2; ++nj)
      ldmatrix_x4(b[nj], Bs + (wn * 32 + nj * 16 + r8 + (mat >> 1) * 8) * LD + k0 + (mat & 1) * 8);
#pragma unroll
    for (int mi = 0; mi < 2; ++mi)
#pragma unroll
      for (int n8 = 0; n8 < 4; ++n8)
        mma_16816<kDtype>(acc[mi][n8], a[mi], b[n8 >> 1][(n8 & 1) * 2], b[n8 >> 1][(n8 & 1) * 2 + 1]);
  }
  const float inv_sqrt_d = 0.08838834764831845f;  // 128^-1/2
#pragma unroll
  for (int mi = 0; mi < 2; ++mi)
#pragma unroll
    for (int n8 = 0; n8 < 4; ++n8)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int m = m0 + wm * 32 + mi * 16 + (lane >> 2) + (e >> 1) * 8;
        const int n = n0 + wn * 32 + n8 * 8 + (lane & 3) * 2 + (e & 1);
        if (m < nq && n < n_img)
          scores[(static_cast<size_t>(bh) * nq + m) * n_img + n] =
              round_to<kDtype>(round_to<kDtype>(acc[mi][n8][e]) * inv_sqrt_d);  // ref :227
      }
}

// 32-bit descending bitonic sort, lane L owns sorted positions [32L, 32L+32)
__device__ __forceinline__ void warp_bitonic_desc_u32(uint32_t (&key)[32], int lane) {
#pragma unroll
  for (int k = 2; k <= 1024; k <<= 1) {
#pragma unroll
    for (int j = k >> 1; j > 0; j >>= 1) {
      if (j >= 32) {
        const int lj = j >> 5;
        const bool keep_max = ((lane & lj) == 0) == (((lane << 5) & k) == 0);
#pragma unroll
        for (int r = 0; r < 32; ++r) {
          const uint32_t other = __shfl_xor_sync(0xffffffffu, key[r], lj);
          key[r] = keep_max ? max(key[r], other) : min(key[r], other);
        }
      } else {
#pragma unroll
        for (int r = 0; r < 32; ++r) {
          if ((r & j) == 0) {
            const int r2 = r | j;
            const bool desc = (k < 32) ? ((r & k) == 0) : (((lane << 5) & k) == 0);
            const uint32_t a = key[r], b = key[r2];
            const uint32_t hi = max(a, b), lo = min(a, b);
            key[r] = desc ? hi : lo;
            key[r2] = desc ? lo : hi;
          }
        }
      }
    }
  }
}

__global__ void __launch_bounds__(128)
select_rows_kernel(const float* __restrict__ scores, const SelectParams p) {
  __shared__ uint32_t s_bits_all[4][64];  // up to 2048 key blocks per row
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long rowid = static_cast<long long>(blockIdx.x) * 4 + warp;  // (bh, m) flattened
  if (rowid >= p.total_rows) return;
  const int bh = static_cast<int>(rowid / p.nq);
  const int m = static_cast<int>(rowid - static_cast<long long>(bh) * p.nq);
  uint32_t* bits = s_bits_all[warp];
  for (int w = lane; w < p.words; w += 32) bits[w] = 0;
  __syncwarp();
  const float* sc = scores + rowid * p.n_img;
  // softmax in fp32 over the ranked blocks (ref :238), element j = q*32 + lane
  float v[32];
  float mx = -INFINITY;
#pragma unroll
  for (int q = 0; q < 32; ++q) {
    const int j = q * 32 + lane;
    v[q] = j < p.n_img ? __ldg(sc + j) : -INFINITY;
    mx = fmaxf(mx, v[q]);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  float sum = 0.f;
#pragma unroll
  for (int q = 0; q < 32; ++q) {
    const int j = q * 32 + lane;
    v[q] = j < p.n_img ? expf(v[q] - mx) : 0.f;
    sum += v[q];
  }
  // same summation tree as select_blocks_kernel: per-lane strided partials, then butterfly
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  uint32_t key[32];
#pragma unroll
  for (int q = 0; q < 32; ++q) {
    const int j = q * 32 + lane;
    v[q] = j < p.n_img ? v[q] / sum : 0.f;          // probabilities (>= 0: bit order == value order)
    key[q] = j < p.n_img ? __float_as_uint(v[q]) : 0u;
  }
  warp_bitonic_desc_u32(key, lane);
  // cumulative probability in sorted order (ref :242-246), lane chunks in rank order
  float part = 0.f;
#pragma unroll
  for (int q = 0; q < 32; ++q) part += __uint_as_float(key[q]);
  float prefix = part;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const float t = __shfl_up_sync(0xffffffffu, prefix, o);
    if (lane >= o) prefix += t;
  }
  float run = prefix - part;
  int local = 0;
#pragma unroll
  for (int q = 0; q < 32; ++q) {
    run += __uint_as_float(key[q]);
    if (lane * 32 + q < p.n_img && run <= p.p_threshold) ++local;
  }
  int tot = local;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) tot += __shfl_xor_sync(0xffffffffu, tot, o);
  const int n = min(max(tot + 1, p.top_k), p.n_img);  // ref :247-250
  // threshold = n-th largest probability; how many strictly larger
  uint32_t tau_local = 0;
  int gt_local = 0;
#pragma unroll
  for (int q = 0; q < 32; ++q)
    if (lane * 32 + q == n - 1) tau_local = key[q];
  const uint32_t tau = __shfl_sync(0xffffffffu, tau_local, (n - 1) >> 5);
#pragma unroll
  for (int q = 0; q < 32; ++q)
    if (lane * 32 + q < n && key[q] > tau) ++gt_local;
  int gt = gt_local;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) gt += __shfl_xor_sync(0xffffffffu, gt, o);
  const int need_ties = n - gt;  // members of the tie group at the cut, taken in index order
  int taken = 0;
#pragma unroll
  for (int q = 0; q < 32; ++q) {
    const int j = q * 32 + lane;
    const uint32_t pb = __float_as_uint(v[q]);
    const bool valid = j < p.n_img;
    const bool is_tie = valid && pb == tau;
    const uint32_t tm = __ballot_sync(0xffffffffu, is_tie);
    const int rank = taken + __popc(tm & ((1u << lane) - 1u));
    const bool sel = valid && (pb > tau || (is_tie && rank < need_ties));
    const uint32_t sm = __ballot_sync(0xffffffffu, sel);
    if (lane == 0 && q < p.words) bits[q] = sm;  // word q covers blocks [32q, 32q+32)
    taken += __popc(tm);
  }
  __syncwarp();
  for (int w = lane; w < p.words; w += 32) {
    uint32_t val = bits[w];
    const int lo = w * 32;
    auto range_bits = [&](int a, int b) -> uint32_t {
      const int s0 = max(a, lo), e0 = min(b, lo + 32);
      if (e0 <= s0) return 0u;
      const uint32_t hi_mask = (e0 - lo) >= 32 ? 0xffffffffu : ((1u << (e0 - lo)) - 1u);
      return hi_mask & ~((s0 - lo) > 0 ? ((1u << (s0 - lo)) - 1u) : 0u);
    };
    if (p.nbr_bits && m < p.nbr_rows && w < p.nbr_words)
      val |= p.nbr_bits[static_cast<size_t>(m) * p.nbr_words + w] & range_bits(0, p.n_img);
    if (m < p.first_frame_blocks) val |= range_bits(0, min(p.first_frame_blocks, p.nb));
    if (p.text_blocks > 0) val |= range_bits(p.n_img, min(p.n_img + p.text_blocks, p.nb));
    p.out_bits[rowid * p.words + w] = val;
  }
  if (p.out_counts && lane == 0) p.out_counts[rowid] = n;
}

}  // namespace

int block_pool_impl(const void* x, void* pooled, void* cast_out, int in_dtype, int out_dtype,
                    int batch, int heads, int head_dim, long long rows, long long sb, long long ss,
                    long long sh, int n_blocks, cudaStream_t stream) {
  if (!x || !pooled) return set_error(JENGA_E_INVALID, "block_pool: null pointer");
  if (batch <= 0 || heads <= 0 || head_dim <= 0 || head_dim % 8 || rows <= 0 || n_blocks <= 0)
    return set_error(JENGA_E_INVALID, "block_pool: bad shape");
  if (static_cast<long long>(n_blocks - 1) * kBlock >= rows)
    return set_error(JENGA_E_INVALID, "block_pool: n_blocks beyond the rows");
  const int esz = in_dtype == JENGA_F32 ? 4 : 2;
  if ((sb * esz) % 16 || (ss * esz) % 16 || (sh * esz) % 16 || reinterpret_cast<uintptr_t>(x) % 16 ||
      reinterpret_cast<uintptr_t>(pooled) % 16)
    return set_error(JENGA_E_INVALID, "block_pool: 16-byte alignment required");
  if (out_dtype != JENGA_BF16 && out_dtype != JENGA_F16)
    return set_error(JENGA_E_INVALID, "block_pool: pooled dtype must be bf16/f16");
  if (in_dtype != JENGA_F32 && in_dtype != out_dtype)
    return set_error(JENGA_E_INVALID, "block_pool: 16-bit input must match the pooled dtype");
  if (in_dtype == JENGA_F32 && out_dtype != JENGA_BF16)
    return set_error(JENGA_E_UNSUPPORTED, "block_pool: f32 input is rounded to bf16 only");
  dim3 grid(n_blocks, batch);
  const int vecs = heads * head_dim / 8;
  // Threads per CTA: the largest multiple of 32 up to 192 that divides the CTA's 16-byte vectors, so every
  // pass over a row is fully populated (at H=24, 256 threads would be one full pass + one half-empty pass).
  int threads = vecs >= 256 ? 256 : ((vecs + 31) / 32) * 32;
  for (int t = 192; t >= 64; t -= 32)
    if (vecs % t == 0) {
      threads = t;
      break;
    }
  uint16_t* po = static_cast<uint16_t*>(pooled);
  uint16_t* co = static_cast<uint16_t*>(cast_out);
  if (in_dtype == JENGA_F32)
    block_pool_kernel<JENGA_F32, JENGA_BF16><<<grid, threads, 0, stream>>>(x, po, co, heads, head_dim, rows, sb, ss, sh, n_blocks);
  else if (in_dtype == JENGA_BF16)
    block_pool_kernel<JENGA_BF16, JENGA_BF16><<<grid, threads, 0, stream>>>(x, po, nullptr, heads, head_dim, rows, sb, ss, sh, n_blocks);
  else
    block_pool_kernel<JENGA_F16, JENGA_F16><<<grid, threads, 0, stream>>>(x, po, nullptr, heads, head_dim, rows, sb, ss, sh, n_blocks);
  cudaError_t ce = cudaGetLastError();
  return ce == cudaSuccess ? JENGA_OK : set_cuda_error(ce, "block_pool launch");
}

int select_blocks_impl(const JengaSelectArgs* a, cudaStream_t stream) {
  if (!a || !a->q_pool || !a->k_pool || !a->out_bits)
    return set_error(JENGA_E_INVALID, "select_blocks: null pointer");
  if (a->dtype != JENGA_BF16 && a->dtype != JENGA_F16)
    return set_error(JENGA_E_INVALID, "select_blocks: dtype must be bf16/f16");
  if (a->batch_heads <= 0 || a->nq <= 0 || a->n_img <= 0 || a->nb < a->n_img ||
      a->nk_pool < a->n_img || a->head_dim <= 0 || a->head_dim % 8)
    return set_error(JENGA_E_INVALID, "select_blocks: bad shape");
  if (a->mask_words * 32 < a->nb) return set_error(JENGA_E_INVALID, "select_blocks: mask_words too small");
  if (a->top_k < 0 || a->text_blocks < 0 || a->first_frame_blocks < 0)
    return set_error(JENGA_E_INVALID, "select_blocks: negative count");
  if (a->workspace && a->n_img <= 1024 && a->mask_words <= 64 && a->head_dim == 128) {
    const size_t need = static_cast<size_t>(a->batch_heads) * a->nq * a->n_img * sizeof(float);
    if (static_cast<size_t>(a->workspace_bytes) < need)
      return set_error(JENGA_E_WORKSPACE, "select_blocks: workspace %lld < %zu bytes", (long long)a->workspace_bytes, need);
    float* scores = static_cast<float*>(a->workspace);
    dim3 g1((a->n_img + 63) / 64, (a->nq + 63) / 64, a->batch_heads);
    // JENGA_SELECT_GEMM=simt selects the fp32 SIMT GEMM whose summation order equals the fused
    // single-kernel path bit for bit (tests); the default is the tensor-core form.
    static const bool simt = [] { const char* e = std::getenv("JENGA_SELECT_GEMM"); return e && std::strcmp(e, "simt") == 0; }();
    cudaError_t ce;
    if (simt) {
      const int smem1 = 2 * 128 * 68 * 4;
      auto k1 = a->dtype == JENGA_BF16 ? pooled_scores_kernel<JENGA_BF16> : pooled_scores_kernel<JENGA_F16>;
      ce = cudaFuncSetAttribute(k1, cudaFuncAttributeMaxDynamicSharedMemorySize, smem1);
      if (ce != cudaSuccess) return set_cuda_error(ce, "cudaFuncSetAttribute(pooled_scores)");
      k1<<<g1, 256, smem1, stream>>>(static_cast<const uint16_t*>(a->q_pool), static_cast<const uint16_t*>(a->k_pool),
                                     scores, a->nq, a->nk_pool, a->n_img, a->head_dim);
    } else {
      auto k1 = a->dtype == JENGA_BF16 ? pooled_scores_mma_kernel<JENGA_BF16> : pooled_scores_mma_kernel<JENGA_F16>;
      k1<<<g1, 128, 0, stream>>>(static_cast<const uint16_t*>(a->q_pool), static_cast<const uint16_t*>(a->k_pool),
                                 scores, a->nq, a->nk_pool, a->n_img);
    }
    SelectParams p{};
    p.nq = a->nq; p.n_img = a->n_img; p.nb = a->nb; p.words = a->mask_words; p.top_k = a->top_k;
    p.p_threshold = a->p_threshold; p.text_blocks = a->text_blocks; p.first_frame_blocks = a->first_frame_blocks;
    p.nbr_bits = a->nbr_bits; p.nbr_rows = a->nbr_rows; p.nbr_words = a->nbr_words;
    p.out_bits = a->out_bits; p.out_counts = a->out_counts;
    const long long rows = static_cast<long long>(a->batch_heads) * a->nq;
    if (rows > 0x7fffffffll) return set_error(JENGA_E_UNSUPPORTED, "select_blocks: too many rows");
    p.total_rows = rows;
    select_rows_kernel<<<static_cast<unsigned>((rows + 3) / 4), 128, 0, stream>>>(scores, p);
    ce = cudaGetLastError();
    return ce == cudaSuccess ? JENGA_OK : set_cuda_error(ce, "select_blocks (2-kernel) launch");
  }
  int npow2 = 32;
  while (npow2 < a->n_img) npow2 <<= 1;
  const bool reg_sort = a->n_img <= 1024;  // register-resident 1024-wide sort
  auto smem_for = [&](int R) -> size_t {
    return static_cast<size_t>(R) * a->head_dim * 4 + static_cast<size_t>((R * a->n_img + 1) & ~1) * 4 +
           (reg_sort ? 0 : static_cast<size_t>(R) * npow2 * 8) + static_cast<size_t>(R) * a->mask_words * 4;
  };
  int R = 8;
  while (R > 1 && smem_for(R) > 200 * 1024) R >>= 1;
  if (smem_for(R) > 220 * 1024)
    return set_error(JENGA_E_UNSUPPORTED, "select_blocks: %d key blocks exceed the shared-memory sort", a->n_img);
  SelectParams p{};
  p.q_pool = static_cast<const uint16_t*>(a->q_pool);
  p.k_pool = static_cast<const uint16_t*>(a->k_pool);
  p.nk_pool = a->nk_pool;
  p.head_dim = a->head_dim;
  p.nq = a->nq;
  p.n_img = a->n_img;
  p.nb = a->nb;
  p.words = a->mask_words;
  p.top_k = a->top_k;
  p.p_threshold = a->p_threshold;
  p.text_blocks = a->text_blocks;
  p.first_frame_blocks = a->first_frame_blocks;
  p.nbr_bits = a->nbr_bits;
  p.nbr_rows = a->nbr_rows;
  p.nbr_words = a->nbr_words;
  p.out_bits = a->out_bits;
  p.out_counts = a->out_counts;
  p.rows_per_cta = R;
  p.npow2 = npow2;
  const size_t smem = smem_for(R);
  const long long groups = (a->nq + R - 1) / R;
  const long long grid = groups * a->batch_heads;
  auto kern = a->dtype == JENGA_BF16
                  ? (reg_sort ? select_blocks_kernel<JENGA_BF16, true> : select_blocks_kernel<JENGA_BF16, false>)
                  : (reg_sort ? select_blocks_kernel<JENGA_F16, true> : select_blocks_kernel<JENGA_F16, false>);
  cudaError_t ce = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  if (ce != cudaSuccess) return set_cuda_error(ce, "cudaFuncSetAttribute(select_blocks)");
  kern<<<static_cast<unsigned>(grid), 256, smem, stream>>>(p);
  ce = cudaGetLastError();
  return ce == cudaSuccess ? JENGA_OK : set_cuda_error(ce, "select_blocks launch");
}

}  // namespace jenga
