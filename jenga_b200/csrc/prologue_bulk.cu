// HunyuanVideo attention prologue, bulk-async form (same results as prologue.cu's hy_prologue_kernel;
// see that file for the reference lines and the rounding chain).
//
// Why a second form.  The classic kernel keeps a token's q/k/v in registers between an LDG and an
// STG: 24 warps per SM, ~340 instructions per warp and token, one global round trip per token —
// ncu: IPC 0.37 per scheduler, long-scoreboard bound, 0.58 of the HBM peak, and 902 uniform CTAs on
// 296 slots leave a nearly empty fourth wave.  Here every byte moves by bulk-async copies
// (cp.async.bulk, the non-tensor TMA path), so bytes in flight cost no registers or issue slots:
//
//   producer thread: global -> shared, one token per ring stage: the token's q, k, v rows (H*256 B
//                   each, contiguous in the qkv projection output) + its cos/sin rows (512 B each,
//                   gathered through rope_index), completion on the stage's `full` mbarrier
//   24 compute warps (two groups of 12 = even / odd tokens; a half-warp per head as before):
//                   LDS -> RMSNorm -> weight (packed 16-bit multiply: the bf16 x bf16 product
//                   rounded once, exactly what the fp32 multiply + rounding did) -> RoPE -> STS in
//                   place + pooling partial sums in registers; v is never touched by a thread
//   store thread  : shared -> global bulk stores of the q, k, v rows; a stage returns to the
//                   producer once its stores have read it (cp.async.bulk.wait_group.read)
//
// One persistent CTA per SM.  Work items are whole 128-token blocks in contiguous chunks per CTA;
// the (number of blocks) mod (number of CTAs) left-over blocks are cut into P <= 8 token ranges
// spread over all CTAs so that the tail costs 1/P of a block instead of a whole one.  Their pooled
// means are combined deterministically: every part writes fp32 partial sums to a scratch buffer and
// takes a ticket; the last one adds the P parts in part order.
#include <cstdlib>
#include <map>
#include <mutex>
#include <utility>

#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include "sm90_ptx.cuh"
#include "jenga_internal.h"

namespace jenga {

namespace {

constexpr int kBlock = 128;
constexpr int kStages = 10;
constexpr int kStoreLag = 3;   // bulk-store groups whose shared-memory reads may still be pending
constexpr int kGroupThreads = 384;                 // 24 heads x 16 lanes
constexpr int kComputeThreads = 2 * kGroupThreads; // even / odd tokens
constexpr int kThreads = kComputeThreads + 64;     // + producer warp + store warp (one thread each)
constexpr int kMaxHeads = 24;

struct BulkParams {
  const uint16_t* img;
  const uint16_t* txt;
  long long img_sb, img_ss, img_sw;   // element strides (batch, token, which); head stride == 128
  long long txt_sb, txt_ss, txt_sw;
  int L, T, H, B;
  const uint16_t* w_img_q;            // null == ones
  const uint16_t* w_img_k;
  const uint16_t* w_txt_q;
  const uint16_t* w_txt_k;
  const float* cos_t;
  const float* sin_t;
  const long long* rope_index;
  float eps;
  uint16_t* q;
  uint16_t* k;
  uint16_t* v;
  uint16_t* q_pool;
  uint16_t* k_pool;
  int nb;          // blocks per batch element
  int n_full;      // whole blocks per CTA (contiguous chunk)
  int rem_begin;   // first left-over block (global block index)
  int R, P;        // left-over blocks, parts per left-over block
  float* scratch;  // [R*P][H][2][128] fp32 partial sums
  int* tickets;    // [R], zero between launches
};

struct Item {
  int b, blk;        // batch element, block inside it
  long long tok0;    // first token (inside the batch element)
  int nt;            // tokens
  int rem, part;     // left-over block number (-1: whole block) and part
};

__device__ __forceinline__ bool get_item(const BulkParams& p, int i, Item& it) {
  const int c = blockIdx.x;
  const int S = p.L + p.T;
  int g;
  if (i < p.n_full) {
    g = c * p.n_full + i;
    it.rem = -1;
    it.part = 0;
  } else if (i == p.n_full && c < p.R * p.P) {
    it.rem = c / p.P;
    it.part = c - it.rem * p.P;
    g = p.rem_begin + it.rem;
  } else {
    return false;
  }
  it.b = g / p.nb;
  it.blk = g - it.b * p.nb;
  const int per = it.rem < 0 ? kBlock : kBlock / p.P;
  it.tok0 = static_cast<long long>(it.blk) * kBlock + it.part * per;
  const long long left = S - it.tok0;
  it.nt = static_cast<int>(left < 0 ? 0 : (left < per ? left : per));
  return true;
}

__device__ __forceinline__ void bulk_load(uint32_t smem_dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_dst),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void bulk_store(void* dst, uint32_t smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst), "r"(smem_src), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int kPending>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(kPending) : "memory");
}
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ uint2 lds64(uint32_t addr) {
  uint2 v;
  asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(addr));
  return v;
}
__device__ __forceinline__ float4 lds128f(uint32_t addr) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(addr));
  return v;
}
__device__ __forceinline__ void sts128(uint32_t addr, uint4 v) {
  asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// packed 16-bit pair product with one rounding per lane == round16(float(a) * float(b)): the fp32
// product of two bf16 (8-bit significands) or two fp16 (11-bit) values is exact
template <bool kBF16>
__device__ __forceinline__ uint32_t mul16x2(uint32_t a, uint32_t b) {
  uint32_t r;
  if constexpr (kBF16) {
    asm("mul.rn.bf16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
  } else {
    asm("mul.rn.f16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
  }
  return r;
}

// 1/rms of a head row: 8 channels in a lane (4 packed words), the row over 16 lanes.  Same
// summation order as prologue.cu's norm_rope8 (x0..x7 fma chain, then xor-shuffles 8,4,2,1).
template <bool kBF16>
__device__ __forceinline__ float row_rnorm(const uint32_t (&w)[4], const float eps) {
  float ss = 0.f;
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float2 t = unpack2<kBF16>(w[j]);
    ss = fmaf(t.x, t.x, ss);
    ss = fmaf(t.y, t.y, ss);
  }
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  return rsqrtf(ss * (1.0f / 128.0f) + eps);
}

// One packed pair (channels 2i, 2i+1): norm -> weight -> RoPE with the rounding points of
// prologue.cu's norm_rope8; returns the packed result and adds it to the pooling sums.
template <bool kBF16, bool kW, bool kRot>
__device__ __forceinline__ uint32_t finish_pair(const uint32_t raw, const float inv, const uint32_t w, const float c0,
                                                const float c1, const float s0, const float s1, float& sum0, float& sum1) {
  const float2 x = unpack2<kBF16>(raw);
  uint32_t pk = pack2<kBF16>(__fmul_rn(x.x, inv), __fmul_rn(x.y, inv));
  if constexpr (kW) pk = mul16x2<kBF16>(pk, w);
  float2 y = unpack2<kBF16>(pk);
  if constexpr (kRot) {
    const float a0 = __fadd_rn(__fmul_rn(y.x, c0), __fmul_rn(-y.y, s0));
    const float a1 = __fadd_rn(__fmul_rn(y.y, c1), __fmul_rn(y.x, s1));
    pk = pack2<kBF16>(a0, a1);
    y = unpack2<kBF16>(pk);
  }
  sum0 += y.x;
  sum1 += y.y;
  return pk;
}

// A token's q and k rows of one lane (8 channels each), in place in the ring stage.  Two halves of the
// 8 channels: each half's cos/sin chunk and weight pair is loaded once and serves q and k.
template <bool kBF16, bool kW, bool kRot>
__device__ __forceinline__ void token_rows(const uint32_t q_addr, const uint32_t k_addr, const uint32_t cs_addr,
                                           const uint32_t w_addr, const float eps, const bool active, float (&qsum)[8],
                                           float (&ksum)[8]) {
  const uint4 q4 = lds128(q_addr);
  const uint4 k4 = lds128(k_addr);
  uint32_t rq[4] = {q4.x, q4.y, q4.z, q4.w}, rk[4] = {k4.x, k4.y, k4.z, k4.w};
  const float inv_q = row_rnorm<kBF16>(rq, eps), inv_k = row_rnorm<kBF16>(rk, eps);
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    float4 c4 = make_float4(0.f, 0.f, 0.f, 0.f), s4 = c4;
    if constexpr (kRot) {
      c4 = lds128f(cs_addr + 16u * half);
      s4 = lds128f(cs_addr + 512u + 16u * half);
    }
    uint2 wq = make_uint2(0u, 0u), wk = wq;
    if constexpr (kW) {
      wq = lds64(w_addr + 8u * half);
      wk = lds64(w_addr + 256u + 8u * half);
    }
    rq[2 * half] = finish_pair<kBF16, kW, kRot>(rq[2 * half], inv_q, wq.x, c4.x, c4.y, s4.x, s4.y, qsum[4 * half], qsum[4 * half + 1]);
    rq[2 * half + 1] = finish_pair<kBF16, kW, kRot>(rq[2 * half + 1], inv_q, wq.y, c4.z, c4.w, s4.z, s4.w, qsum[4 * half + 2], qsum[4 * half + 3]);
    rk[2 * half] = finish_pair<kBF16, kW, kRot>(rk[2 * half], inv_k, wk.x, c4.x, c4.y, s4.x, s4.y, ksum[4 * half], ksum[4 * half + 1]);
    rk[2 * half + 1] = finish_pair<kBF16, kW, kRot>(rk[2 * half + 1], inv_k, wk.y, c4.z, c4.w, s4.z, s4.w, ksum[4 * half + 2], ksum[4 * half + 3]);
  }
  if (active) {
    sts128(q_addr, make_uint4(rq[0], rq[1], rq[2], rq[3]));
    sts128(k_addr, make_uint4(rk[0], rk[1], rk[2], rk[3]));
  }
}

template <bool kBF16>
__device__ __forceinline__ uint4 pack_mean(const float (&sum)[8]) {
  uint4 v;
  v.x = pack2<kBF16>(sum[0] * (1.0f / kBlock), sum[1] * (1.0f / kBlock));
  v.y = pack2<kBF16>(sum[2] * (1.0f / kBlock), sum[3] * (1.0f / kBlock));
  v.z = pack2<kBF16>(sum[4] * (1.0f / kBlock), sum[5] * (1.0f / kBlock));
  v.w = pack2<kBF16>(sum[6] * (1.0f / kBlock), sum[7] * (1.0f / kBlock));
  return v;
}

template <bool kBF16>
__global__ void __launch_bounds__(kThreads, 1)
hy_prologue_bulk_kernel(const BulkParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t row_bytes = static_cast<uint32_t>(p.H) * 256u;
  const uint32_t stage_bytes = 3u * row_bytes + 1024u;
  // [stages][pool exchange: H x 2 x 128 f32][weights: 4 x 128 x 16-bit][barriers][flag]
  uint8_t* s_pool_raw = smem + kStages * stage_bytes;
  float* s_pool = reinterpret_cast<float*>(s_pool_raw);
  uint16_t* s_w = reinterpret_cast<uint16_t*>(s_pool_raw + static_cast<size_t>(p.H) * 1024);
  uint64_t* bar_full = reinterpret_cast<uint64_t*>(reinterpret_cast<uint8_t*>(s_w) + 1024);
  uint64_t* bar_done = bar_full + kStages;    // a stage's rows have been rewritten in place
  uint64_t* bar_empty = bar_done + kStages;
  int* s_flag = reinterpret_cast<int*>(bar_empty + kStages);
  const uint32_t stage0 = smem_u32(smem);
  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const bool has_w = p.w_img_q != nullptr;
  const int S = p.L + p.T;

  if (tid == 0) {
    for (int s = 0; s < kStages; ++s) {
      mbar_init(&bar_full[s], 1);
      mbar_init(&bar_done[s], kGroupThreads / 32);
      mbar_init(&bar_empty[s], 1);
    }
    fence_mbar_init();
  }
  if (has_w) {
    for (int i = tid; i < 4 * 128; i += kThreads) {
      const uint16_t* src = (i < 128) ? p.w_img_q : (i < 256) ? p.w_img_k : (i < 384) ? p.w_txt_q : p.w_txt_k;
      s_w[i] = src[i & 127];
    }
  }
  __syncthreads();

  if (warp >= kComputeThreads / 32) {
    const int lane = tid & 31;
    if (warp == kComputeThreads / 32 && lane == 0) {
      // ---------------------------------------------------------------- producer (one thread)
      uint32_t n = 0;
      Item it;
      for (int i = 0; get_item(p, i, it); ++i) {
        // table rows of the next 8 tokens are fetched while the current 8 are issued
        constexpr int kAhead = 8;
        long long cur[kAhead], nxt[kAhead];
        auto fetch = [&](int t0, long long (&dst)[kAhead]) {
#pragma unroll
          for (int j = 0; j < kAhead; ++j) {
            const long long tok = it.tok0 + t0 + j;
            dst[j] = tok;
            if (p.cos_t && p.rope_index && t0 + j < it.nt && tok < p.L) dst[j] = __ldg(p.rope_index + tok);
          }
        };
        fetch(0, cur);
        for (int t0 = 0; t0 < it.nt; t0 += kAhead) {
          fetch(t0 + kAhead, nxt);
#pragma unroll
          for (int j = 0; j < kAhead; ++j) {
            const int t = t0 + j;
            if (t < it.nt) {
              const uint32_t s = n % kStages;
              if (n >= kStages) mbar_wait(&bar_empty[s], ((n / kStages) - 1) & 1, nullptr);
              const long long tok = it.tok0 + t;
              const bool is_img = tok < p.L;
              const bool rotate = is_img && p.cos_t != nullptr;
              const uint16_t* src = is_img ? p.img + it.b * p.img_sb + tok * p.img_ss
                                           : p.txt + it.b * p.txt_sb + (tok - p.L) * p.txt_ss;
              const long long sw = is_img ? p.img_sw : p.txt_sw;
              const uint32_t dst = stage0 + s * stage_bytes;
              mbar_arrive_expect_tx(&bar_full[s], 3u * row_bytes + (rotate ? 1024u : 0u));
              bulk_load(dst, src, row_bytes, &bar_full[s]);
              bulk_load(dst + row_bytes, src + sw, row_bytes, &bar_full[s]);
              bulk_load(dst + 2u * row_bytes, src + 2 * sw, row_bytes, &bar_full[s]);
              if (rotate) {
                bulk_load(dst + 3u * row_bytes, p.cos_t + cur[j] * 128, 512u, &bar_full[s]);
                bulk_load(dst + 3u * row_bytes + 512u, p.sin_t + cur[j] * 128, 512u, &bar_full[s]);
              }
              ++n;
            }
          }
#pragma unroll
          for (int j = 0; j < kAhead; ++j) cur[j] = nxt[j];
        }
      }
    } else if (warp == kComputeThreads / 32 + 1 && lane == 0) {
      // ---------------------------------------------------------------- store thread
      uint32_t n = 0;
      Item it;
      for (int i = 0; get_item(p, i, it); ++i) {
        for (int t = 0; t < it.nt; ++t, ++n) {
          const uint32_t s = n % kStages;
          mbar_wait(&bar_done[s], (n / kStages) & 1, nullptr);
          const long long o = ((static_cast<long long>(it.b) * S + it.tok0 + t) * p.H) * 128;
          const uint32_t src = stage0 + s * stage_bytes;
          bulk_store(p.q + o, src, row_bytes);
          bulk_store(p.k + o, src + row_bytes, row_bytes);
          bulk_store(p.v + o, src + 2u * row_bytes, row_bytes);
          bulk_commit();
          if (n >= kStoreLag) {
            bulk_wait_read<kStoreLag>();   // the stores of token n - kStoreLag have read their stage
            mbar_arrive(&bar_empty[(n - kStoreLag) % kStages]);
          }
        }
      }
      // tokens n - kStoreLag .. n - 1 still own their stages; nobody waits for those, but the stores
      // must have left shared memory before the CTA exits
      bulk_wait_all();
    }
  } else {
    // ------------------------------------------------------------------ compute warps
    const int g = tid / kGroupThreads;           // token parity this group serves
    const int lt = tid - g * kGroupThreads;
    const int hslot = lt >> 4;
    const bool active = hslot < p.H;
    const int h = active ? hslot : p.H - 1;      // idle half-warps shadow the last head, store nothing
    const int lane16 = lt & 15;
    const int d0 = lane16 * 8;
    const uint32_t my_off = static_cast<uint32_t>(h) * 256u + static_cast<uint32_t>(lane16) * 16u;
    const uint32_t w_base = smem_u32(s_w) + static_cast<uint32_t>(lane16) * 16u;
    static_assert(kStages % 2 == 0, "a group's tokens advance two ring stages at a time");
    uint32_t s = static_cast<uint32_t>(g), ph = 0;   // ring stage and phase of this group's next token
    uint32_t nbase = 0;                              // tokens of the items before this one
    const uint32_t bar_full0 = smem_u32(bar_full), bar_done0 = smem_u32(bar_done);
    const uint32_t cs_off = 3u * row_bytes + static_cast<uint32_t>(lane16) * 32u;
    Item it;
    for (int i = 0; get_item(p, i, it); ++i) {
      float qsum[8], ksum[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) qsum[e] = ksum[e] = 0.f;
      const long long img_left = p.L - it.tok0;
      const int n_img = img_left <= 0 ? 0 : (img_left < it.nt ? static_cast<int>(img_left) : it.nt);
      for (int t = static_cast<int>((static_cast<uint32_t>(g) - nbase) & 1u); t < it.nt; t += 2) {
        mbar_wait(reinterpret_cast<uint64_t*>(__cvta_shared_to_generic(bar_full0 + 8u * s)), ph, nullptr);
        const bool is_img = t < n_img;
        const bool rotate = is_img && p.cos_t != nullptr;
        const uint32_t st = stage0 + s * stage_bytes;
        const uint32_t qa = st + my_off, ka = qa + row_bytes, ca = st + cs_off;
        const uint32_t wa = w_base + (is_img ? 0u : 512u);   // this token's packed norm weights (q; k at +256)
        if (has_w) {
          if (rotate) token_rows<kBF16, true, true>(qa, ka, ca, wa, p.eps, active, qsum, ksum);
          else token_rows<kBF16, true, false>(qa, ka, ca, wa, p.eps, active, qsum, ksum);
        } else {
          if (rotate) token_rows<kBF16, false, true>(qa, ka, ca, wa, p.eps, active, qsum, ksum);
          else token_rows<kBF16, false, false>(qa, ka, ca, wa, p.eps, active, qsum, ksum);
        }
        fence_proxy_async_smem();   // the bulk store reads these rows through the async proxy
        __syncwarp();
        if ((tid & 31) == 0) mbar_arrive(reinterpret_cast<uint64_t*>(__cvta_shared_to_generic(bar_done0 + 8u * s)));
        s += 2;
        if (s >= kStages) {
          s -= kStages;
          ph ^= 1u;
        }
      }
      nbase += static_cast<uint32_t>(it.nt);
      if (p.q_pool) {
        // group 1 (odd tokens) hands its sums to group 0 through shared memory
        float* mine = s_pool + (h * 2) * 128 + d0;
        if (g == 1 && active) {
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            mine[e] = qsum[e];
            mine[128 + e] = ksum[e];
          }
        }
        named_bar_sync(1, kComputeThreads);
        if (g == 0) {
          if (active) {
#pragma unroll
            for (int e = 0; e < 8; ++e) {
              qsum[e] += mine[e];
              ksum[e] += mine[128 + e];
            }
          }
          if (it.rem < 0 || p.P == 1) {
            if (active) {
              const long long o = ((static_cast<long long>(it.b) * p.H + h) * p.nb + it.blk) * 128 + d0;
              *reinterpret_cast<uint4*>(p.q_pool + o) = pack_mean<kBF16>(qsum);
              *reinterpret_cast<uint4*>(p.k_pool + o) = pack_mean<kBF16>(ksum);
            }
          } else {
            float* part = p.scratch + ((static_cast<long long>(it.rem) * p.P + it.part) * p.H + h) * 256 + d0;
            if (active) {
              *reinterpret_cast<float4*>(part) = make_float4(qsum[0], qsum[1], qsum[2], qsum[3]);
              *reinterpret_cast<float4*>(part + 4) = make_float4(qsum[4], qsum[5], qsum[6], qsum[7]);
              *reinterpret_cast<float4*>(part + 128) = make_float4(ksum[0], ksum[1], ksum[2], ksum[3]);
              *reinterpret_cast<float4*>(part + 132) = make_float4(ksum[4], ksum[5], ksum[6], ksum[7]);
            }
            __threadfence();
            named_bar_sync(2, kGroupThreads);
            if (lt == 0) *s_flag = atomicAdd(p.tickets + it.rem, 1);
            named_bar_sync(2, kGroupThreads);
            if (*s_flag == p.P - 1) {   // every other part of this block is in the scratch buffer
              __threadfence();
              if (active) {
                float qa[8], ka[8];
                for (int pp = 0; pp < p.P; ++pp) {
                  const float* src = p.scratch + ((static_cast<long long>(it.rem) * p.P + pp) * p.H + h) * 256 + d0;
                  const float4 a0 = __ldcg(reinterpret_cast<const float4*>(src));
                  const float4 a1 = __ldcg(reinterpret_cast<const float4*>(src + 4));
                  const float4 b0 = __ldcg(reinterpret_cast<const float4*>(src + 128));
                  const float4 b1 = __ldcg(reinterpret_cast<const float4*>(src + 132));
                  const float qv[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
                  const float kv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
                  for (int e = 0; e < 8; ++e) {
                    qa[e] = pp == 0 ? qv[e] : qa[e] + qv[e];
                    ka[e] = pp == 0 ? kv[e] : ka[e] + kv[e];
                  }
                }
                const long long o = ((static_cast<long long>(it.b) * p.H + h) * p.nb + it.blk) * 128 + d0;
                *reinterpret_cast<uint4*>(p.q_pool + o) = pack_mean<kBF16>(qa);
                *reinterpret_cast<uint4*>(p.k_pool + o) = pack_mean<kBF16>(ka);
              }
              if (lt == 0) p.tickets[it.rem] = 0;   // ready for the next launch on this stream
            }
          }
        }
        named_bar_sync(1, kComputeThreads);   // s_pool may be overwritten by the next item
      }
    }
  }
}

// scratch for the left-over blocks' partial sums: one per (device, stream), so launches that could
// overlap (different streams) never share it and launches on one stream are ordered anyway
struct Scratch {
  float* partial = nullptr;
  int* tickets = nullptr;
};
std::mutex g_mu;
std::map<std::pair<int, cudaStream_t>, Scratch> g_scratch;
constexpr int kMaxCtas = 256;

bool get_scratch(cudaStream_t stream, Scratch* out) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return false;
  std::lock_guard<std::mutex> lock(g_mu);
  auto key = std::make_pair(dev, stream);
  auto itr = g_scratch.find(key);
  if (itr != g_scratch.end()) {
    *out = itr->second;
    return true;
  }
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(stream, &cs) != cudaSuccess || cs != cudaStreamCaptureStatusNone) {
    (void)cudaGetLastError();
    return false;   // no allocation while a graph is being captured: the caller takes the classic kernel
  }
  Scratch s;
  const size_t bytes = static_cast<size_t>(kMaxCtas) * kMaxHeads * 256 * sizeof(float);
  if (cudaMalloc(&s.partial, bytes) != cudaSuccess) { (void)cudaGetLastError(); return false; }
  if (cudaMalloc(&s.tickets, kMaxCtas * sizeof(int)) != cudaSuccess) {
    (void)cudaGetLastError();
    cudaFree(s.partial);
    return false;
  }
  if (cudaMemset(s.tickets, 0, kMaxCtas * sizeof(int)) != cudaSuccess) { (void)cudaGetLastError(); return false; }
  g_scratch[key] = s;
  *out = s;
  return true;
}

}  // namespace

// Returns JENGA_OK when the bulk-async kernel was launched, a positive value when the arguments are
// outside what it handles (the caller then launches the classic kernel), or an error code.
int hy_prologue_bulk_try(const JengaHyPrologueArgs* a, cudaStream_t stream) {
  constexpr int kNotApplicable = 1;
  if (a->heads > kMaxHeads || a->head_dim != 128) return kNotApplicable;
  if (a->img_stride_h != 128 || (a->txt_tokens > 0 && a->txt_stride_h != 128)) return kNotApplicable;
  const void* ptrs[] = {a->img_qkv, a->txt_qkv, a->q, a->k, a->v, a->rope_cos, a->rope_sin};
  for (const void* ptr : ptrs)
    if (reinterpret_cast<uintptr_t>(ptr) % 16) return kNotApplicable;
  int dev = 0, sms = 0, smem_max = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
      cudaDeviceGetAttribute(&smem_max, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess)
    return set_cuda_error(cudaGetLastError(), "hy_prologue(bulk): device query");
  const size_t row_bytes = static_cast<size_t>(a->heads) * 256;
  const size_t smem = kStages * (3 * row_bytes + 1024) + static_cast<size_t>(a->heads) * 1024 + 1024 +
                      3 * kStages * sizeof(uint64_t) + 16;
  if (smem > static_cast<size_t>(smem_max)) return kNotApplicable;

  BulkParams p{};
  p.img = static_cast<const uint16_t*>(a->img_qkv);
  p.txt = static_cast<const uint16_t*>(a->txt_qkv);
  p.img_sb = a->img_stride_b; p.img_ss = a->img_stride_s; p.img_sw = a->img_stride_w;
  p.txt_sb = a->txt_stride_b; p.txt_ss = a->txt_stride_s; p.txt_sw = a->txt_stride_w;
  p.L = static_cast<int>(a->img_tokens);
  p.T = static_cast<int>(a->txt_tokens);
  p.H = a->heads;
  p.B = a->batch;
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
  const long long nbk = static_cast<long long>(p.nb) * a->batch;
  // JENGA_PROLOGUE_CTAS: grid override for tests (exercises whole-block chunks on small inputs)
  const char* ce_env = std::getenv("JENGA_PROLOGUE_CTAS");
  const int ctas_env = ce_env ? std::atoi(ce_env) : 0;
  int ctas = ctas_env > 0 ? ctas_env : sms;
  if (ctas > kMaxCtas) ctas = kMaxCtas;
  p.n_full = static_cast<int>(nbk / ctas);
  p.R = static_cast<int>(nbk - static_cast<long long>(p.n_full) * ctas);
  p.rem_begin = p.n_full * ctas;
  p.P = 1;
  if (p.R > 0)
    while (p.P < 8 && p.R * p.P * 2 <= ctas) p.P *= 2;
  const int grid = p.n_full > 0 ? ctas : p.R * p.P;
  if (p.R > 0 && p.P > 1 && p.q_pool) {
    Scratch sc;
    if (!get_scratch(stream, &sc)) return kNotApplicable;
    p.scratch = sc.partial;
    p.tickets = sc.tickets;
  }
  auto kern = a->dtype == JENGA_BF16 ? hy_prologue_bulk_kernel<true> : hy_prologue_bulk_kernel<false>;
  cudaError_t ce = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
  if (ce != cudaSuccess) return set_cuda_error(ce, "cudaFuncSetAttribute(hy_prologue bulk)");
  kern<<<grid, kThreads, smem, stream>>>(p);
  ce = cudaGetLastError();
  return ce == cudaSuccess ? JENGA_OK : set_cuda_error(ce, "hy_prologue(bulk) launch");
}

}  // namespace jenga
