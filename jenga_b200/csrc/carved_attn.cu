// Carved (block-sparse) flash-attention forward for sm_90a.
//
// Replaces the reference's Triton one-hot kernel
//   hyvideo/modules/attention_block_triton_diffres.py:38-136 (+ launcher :139-196)
// and its text-row flash_attn_func call (:371-380) with ONE launch.
//
// Work decomposition: one CTA per (batch*head, 128-row query block); 288 threads:
//   warps 0..7  two consumer warpgroups of 64 query rows each: S = Q~ K^T by wgmma (Q and K from
//               shared memory, S in registers), online softmax in base 2 on the registers, then
//               O += P V by wgmma with P as the register A operand; final O / l -> global
//   warp 8      TMA producer: Q once, then one K tile and one V tile per live key block into a
//               two-stage ring (K and V slots are released separately, so the next K tile lands
//               while the P.V product of the current one runs)
// S and O are fp32 register accumulators (64 + 64 registers per thread); one CTA per SM with
// ~164 KB of shared memory, two warpgroups whose softmax and MMA phases interleave on the SM.
//
// HBM/L2 layout: q,k,v stay in the caller's [B,S,H,D] layout; TMA boxes are {64 d, 128 rows}
// with 128-byte swizzle.  K boxes are K-major wgmma operands, V boxes MN-major (no transpose).
// CTAs are numbered head-major so that all CTAs in flight read the same head's K/V out of L2.
#include "carved_attn_common.cuh"

namespace jenga {

namespace {

using attn::BlockWalker;
using attn::KernelParams;

constexpr int kBlock = 128;           // rows per q block == keys per kv block
constexpr int kHeadDim = 128;
constexpr int kConsumerThreads = 256;
constexpr int kThreads = kConsumerThreads + 32;
constexpr int kStages = 2;                       // K/V ring depth
constexpr int kBoxBytes = kBlock * 64 * 2;       // 16 KB: 128 rows x 64 d (one TMA box)
constexpr int kTileBytes = 2 * kBoxBytes;        // 32 KB: 128 rows x 128 d (two d halves)
constexpr int kMaxMaskWords = 256;               // up to 8192 key blocks (1M tokens)

// shared-memory carve-up (offsets from the 1024-aligned base)
constexpr int kOffQ = 0;
constexpr int kOffK = kOffQ + kTileBytes;
constexpr int kOffV = kOffK + kStages * kTileBytes;
constexpr int kOffBars = kOffV + kStages * kTileBytes;
constexpr int kOffMask = kOffBars + 128;
constexpr int kSmemBytes = 1024 /*align slack*/ + kOffMask + kMaxMaskWords * 4;

enum BarId {
  Q_FULL = 0,
  K_FULL = 1, V_FULL = K_FULL + kStages,
  K_EMPTY = V_FULL + kStages, V_EMPTY = K_EMPTY + kStages,   // one arrival per consumer warp
  NUM_BARS = V_EMPTY + kStages
};
static_assert(NUM_BARS * 8 <= 128, "barrier block overflow");

// byte offset of (row, col) inside a 128-byte-swizzled tile of 128-byte rows (1024-B aligned)
__device__ __forceinline__ uint32_t sw128(uint32_t row, uint32_t col) {
  return row * 128u + ((((col >> 4) ^ row) & 7u) << 4) + (col & 15u);
}

// kPvFp8 (opt-in): P and V enter the P.V product as FP8 e4m3 — V quantised per head by
// jenga_quantize_v_fp8 (scale = absmax/448), P converted with cvt.rn.satfinite.e4m3x2 (p <= 2^8 by
// the lazy-rescale bound, e4m3 max 448) — through wgmma m64n128k32 e4m3 (half the P.V tensor cycles).
// 8-bit wgmma operands must be K-major, so the consumers transpose each V tile in shared memory
// into V^T with the keys of every 32-key group permuted to match the order in which the S
// accumulator fragment already holds P: no shuffles of P.  Q.K^T, the softmax and l are unchanged.
template <bool kBF16, bool kPvFp8 = false>
__global__ void __launch_bounds__(kThreads, 1)
carved_attn_fwd_kernel(const __grid_constant__ CUtensorMap tm_q,
                       const __grid_constant__ CUtensorMap tm_k,
                       const __grid_constant__ CUtensorMap tm_v, const KernelParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw_addr + 1023u) & ~1023u) - raw_addr);
  uint8_t* sQ = smem + kOffQ;
  uint8_t* sK = smem + kOffK;  // + stage * kTileBytes
  uint8_t* sV = smem + kOffV;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kOffBars);
  uint32_t* s_mask = reinterpret_cast<uint32_t*>(smem + kOffMask);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  // ---- which tile is this CTA?  head-major; within a head the (long) dense blocks first ----
  const int per_bh = p.nq_sparse + p.nq_dense;
  const int bh = blockIdx.x / per_bh;
  const int local = blockIdx.x - bh * per_bh;
  const bool dense = local < p.nq_dense;
  const int qb = dense ? p.nq_sparse + local : local - p.nq_dense;
  const int b = bh / p.heads;
  const int h = bh - b * p.heads;
  const long long q_row0 = static_cast<long long>(qb) * kBlock;
  // ref :58 — seqlen is read from device memory (cu_seqlens_q[1]); no host round trip
  const long long seqlen_over = p.seqlen_dev ? static_cast<long long>(__ldg(p.seqlen_dev)) : -1;
  const long long q_limit_sparse = seqlen_over >= 0 ? seqlen_over : p.q_limit_sparse;
  const long long kv_limit =
      dense ? p.kv_limit_dense : (seqlen_over >= 0 ? seqlen_over : p.kv_limit_sparse);
  // ref :59-61 — a sparse q block entirely past seqlen is skipped (its rows stay zero)
  const bool skip_all = (!dense && q_row0 >= q_limit_sparse);

  // ---- stage the row mask in shared memory ----
  const int nwords = p.mask_words;
  for (int w = threadIdx.x; w < nwords; w += kThreads) {
    uint32_t bits;
    if (skip_all) {
      bits = 0;
    } else if (dense) {
      const int rem = p.nb_kv - w * 32;
      bits = rem >= 32 ? 0xffffffffu : (rem > 0 ? ((1u << rem) - 1u) : 0u);
    } else {
      bits = p.mask_bits[(static_cast<size_t>(bh) * p.nq_sparse + qb) * nwords + w];
      const int rem = p.nb_kv - w * 32;  // never walk past the key blocks that exist
      if (rem < 32) bits &= rem > 0 ? ((1u << rem) - 1u) : 0u;
    }
    s_mask[w] = bits;
  }

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_q);
    tma_prefetch_desc(&tm_k);
    tma_prefetch_desc(&tm_v);
#pragma unroll
    for (int i = 0; i < NUM_BARS; ++i) mbar_init(&bars[i], i >= K_EMPTY ? 8u : 1u);
    fence_mbar_init();
  }
  __syncthreads();

  int n_tiles = 0;
  for (int w = 0; w < nwords; ++w) n_tiles += __popc(s_mask[w]);

  if (warp == kConsumerThreads / 32) {
    // =============================== TMA producer ===============================
    if (n_tiles > 0 && lane == 0) {
      mbar_arrive_expect_tx(&bars[Q_FULL], kTileBytes);
      tma_load_4d(sQ, &tm_q, &bars[Q_FULL], 0, static_cast<int>(q_row0), h, b);
      tma_load_4d(sQ + kBoxBytes, &tm_q, &bars[Q_FULL], 64, static_cast<int>(q_row0), h, b);
      BlockWalker it(s_mask, nwords);
      int j = 0;
      for (int blk = it.next(); blk >= 0; blk = it.next(), ++j) {
        const int s = j % kStages;
        const uint32_t par = ((j / kStages) & 1) ^ 1;   // slot-free parity (a fresh barrier passes)
        const int row0 = blk * kBlock;
        uint8_t* k_dst = sK + s * kTileBytes;
        uint8_t* v_dst = sV + s * kTileBytes;
        mbar_wait(&bars[K_EMPTY + s], par, p.err_flag);
        mbar_arrive_expect_tx(&bars[K_FULL + s], kTileBytes);
        tma_load_4d(k_dst, &tm_k, &bars[K_FULL + s], 0, row0, h, b);
        tma_load_4d(k_dst + kBoxBytes, &tm_k, &bars[K_FULL + s], 64, row0, h, b);
        mbar_wait(&bars[V_EMPTY + s], par, p.err_flag);
        if constexpr (kPvFp8) {   // 128 keys x 128 one-byte channels = one 16 KB box
          mbar_arrive_expect_tx(&bars[V_FULL + s], kBoxBytes);
          tma_load_4d(v_dst, &tm_v, &bars[V_FULL + s], 0, row0, h, b);
        } else {
          mbar_arrive_expect_tx(&bars[V_FULL + s], kTileBytes);
          tma_load_4d(v_dst, &tm_v, &bars[V_FULL + s], 0, row0, h, b);
          tma_load_4d(v_dst + kBoxBytes, &tm_v, &bars[V_FULL + s], 64, row0, h, b);
        }
      }
    }
    return;
  }

  // =============================== consumers ===============================
  const int wg = warp >> 2;                       // warpgroup: query rows [64 wg, 64 wg + 64)
  const int g = lane >> 2, qd = lane & 3;
  // accumulator fragment: element i of a thread is row g + 8 ((i >> 1) & 1) of the warp's 16 rows,
  // column 8 (i >> 2) + 2 qd + (i & 1)
  const int row_lo = wg * 64 + (warp & 3) * 16 + g;
  float m_used[2] = {-INFINITY, -INFINITY};  // running (possibly stale) max, in scaled log2 units
  float l_sum[2] = {0.f, 0.f};               // this thread's partial sums (its 32 columns)
  float o[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  // sparse class: Q~ = round(Q * qk_scale) and raw S is already in log2 units (c = 1)
  // dense class : raw S, scaled inside the exponent (c = qk_scale), like FlashAttention
  const float c = dense ? p.qk_scale : 1.0f;

  if (n_tiles > 0) {
    mbar_wait(&bars[Q_FULL], 0, p.err_flag);
    if (!dense) {
      // ref :87-88  q = (q * qk_scale).to(dtype) — elementwise, so swizzle-agnostic
      uint4* q4 = reinterpret_cast<uint4*>(sQ);
#pragma unroll 4
      for (int i = 0; i < kTileBytes / 16 / kConsumerThreads; ++i) {
        uint4 v = q4[threadIdx.x + i * kConsumerThreads];
        uint32_t* e = reinterpret_cast<uint32_t*>(&v);
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const float2 f = unpack2<kBF16>(e[t]);
          e[t] = pack2<kBF16>(f.x * p.qk_scale, f.y * p.qk_scale);
        }
        q4[threadIdx.x + i * kConsumerThreads] = v;
      }
      fence_proxy_async_smem();  // generic-proxy writes -> visible to the tensor core proxy
      named_bar_sync(1, kConsumerThreads);
    }
    const uint32_t q_addr = smem_u32(sQ) + wg * 64 * 128;   // this warpgroup's 64 rows of each d half

    BlockWalker it(s_mask, nwords);
    int j = 0;
    for (int blk = it.next(); blk >= 0; blk = it.next(), ++j) {
      const int s = j % kStages;
      const uint32_t par = (j / kStages) & 1;
      // ref :113-114 — text_amp is a constant added to every score of a text key block, in
      // log2 units (sparse class only, where c == 1): fold it into the exponent offset.
      const float amp = (!dense && blk >= p.text_block_start) ? p.text_amp : 0.f;

      // ---- S = Q~ K^T (64 x 128 per warpgroup, K = 128 in 8 steps) ----
      float sc[64];
      mbar_wait(&bars[K_FULL + s], par, p.err_flag);
      {
        const uint32_t k_addr = smem_u32(sK + s * kTileBytes);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < kHeadDim / 16; ++kk) {
          const uint32_t off = (kk & 3) * 32 + (kk >> 2) * kBoxBytes;
          wgmma_128_ss<kBF16>(sc, gmma_desc_sw128(q_addr + off, 16, 1024),
                              gmma_desc_sw128(k_addr + off, 16, 1024), kk > 0 ? 1u : 0u);
        }
        wgmma_commit();
        wgmma_wait<0>();
        fence_regs(sc);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars[K_EMPTY + s]);

      // ---- online softmax on the registers ----
      const long long col0 = static_cast<long long>(blk) * kBlock;
      if (col0 + kBlock > kv_limit) {  // rare: only the tile that straddles seqlen
#pragma unroll
        for (int i = 0; i < 64; ++i)
          if (col0 + (i >> 2) * 8 + qd * 2 + (i & 1) >= kv_limit) sc[i] = -INFINITY;  // ref :117-118
      }
      float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
      for (int i = 0; i < 64; i += 4) {
        mx[0] = fmaxf(mx[0], fmaxf(sc[i], sc[i + 1]));
        mx[1] = fmaxf(mx[1], fmaxf(sc[i + 2], sc[i + 3]));
      }
      float m_cand[2];
      bool need = false;
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
        mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
        m_cand[r] = fmaxf(m_used[r], fmaf(mx[r], c, amp));
        // Lazy rescale: the reference rescales acc by exp2(m_old - m_new) every tile
        // (:121-132).  O/l is invariant to the reference point, so it only moves when the
        // max grew by more than 2^8 — the final O/l is the same up to fp32 rounding.
        need = need || (m_cand[r] - m_used[r]) > 8.0f;   // false for NaN (-inf - -inf)
      }
      if (__any_sync(0xffffffffu, need)) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const float alpha = (m_cand[r] == -INFINITY) ? 1.0f : fast_exp2(m_used[r] - m_cand[r]);
          l_sum[r] *= alpha;
#pragma unroll
          for (int i = 2 * r; i < 64; i += 4) {
            o[i] *= alpha;
            o[i + 1] *= alpha;
          }
          m_used[r] = m_cand[r];
        }
      }
      // p = exp2(s*c + off); l accumulates the unrounded p (ref :131), P is rounded to the
      // input dtype for the PV product (ref :128)
      float off[2];
#pragma unroll
      for (int r = 0; r < 2; ++r) off[r] = amp - ((m_used[r] == -INFINITY) ? 0.f : m_used[r]);
#pragma unroll
      for (int i = 0; i < 64; ++i) {
        const int r = (i >> 1) & 1;
        sc[i] = fast_exp2(fmaf(sc[i], c, off[r]));
        l_sum[r] += sc[i];
      }

      // ---- O += P V ----
      mbar_wait(&bars[V_FULL + s], par, p.err_flag);
      uint8_t* vs = sV + s * kTileBytes;
      if constexpr (kPvFp8) {
        // V^T[d][32 g + L] = V[32 g + perm(L)][d], perm(4 t + u) = {2t, 2t+1, 2t+8, 2t+9}[u] (+16 for
        // t >= 4): the k-order of the e4m3 A fragment (4 consecutive k per byte quad) read off the
        // f32 accumulator fragment (pairs of adjacent columns, 8 apart)
        uint8_t* vt = vs + kBoxBytes;
#pragma unroll
        for (int it4 = 0; it4 < 4; ++it4) {
          const int u = threadIdx.x + it4 * kConsumerThreads;
          const int dc = u & 31, lc = u >> 5;
          const int t = lc & 7;
          const int k0 = (lc >> 3) * 32 + (t >= 4 ? 16 : 0) + 2 * (t & 3);
          const uint32_t r0 = *reinterpret_cast<const uint32_t*>(vs + sw128(k0, 4 * dc));
          const uint32_t r1 = *reinterpret_cast<const uint32_t*>(vs + sw128(k0 + 1, 4 * dc));
          const uint32_t r2 = *reinterpret_cast<const uint32_t*>(vs + sw128(k0 + 8, 4 * dc));
          const uint32_t r3 = *reinterpret_cast<const uint32_t*>(vs + sw128(k0 + 9, 4 * dc));
          const uint32_t lo01 = __byte_perm(r0, r1, 0x5140), hi01 = __byte_perm(r0, r1, 0x7362);
          const uint32_t lo23 = __byte_perm(r2, r3, 0x5140), hi23 = __byte_perm(r2, r3, 0x7362);
          *reinterpret_cast<uint32_t*>(vt + sw128(4 * dc + 0, 4 * lc)) = __byte_perm(lo01, lo23, 0x5410);
          *reinterpret_cast<uint32_t*>(vt + sw128(4 * dc + 1, 4 * lc)) = __byte_perm(lo01, lo23, 0x7632);
          *reinterpret_cast<uint32_t*>(vt + sw128(4 * dc + 2, 4 * lc)) = __byte_perm(hi01, hi23, 0x5410);
          *reinterpret_cast<uint32_t*>(vt + sw128(4 * dc + 3, 4 * lc)) = __byte_perm(hi01, hi23, 0x7632);
        }
        fence_proxy_async_smem();
        named_bar_sync(2, kConsumerThreads);
        uint32_t a[4][4];
#pragma unroll
        for (int kc = 0; kc < 4; ++kc) {
          const float* x = sc + 16 * kc;
          a[kc][0] = pack4_e4m3(x[0], x[1], x[4], x[5]);
          a[kc][1] = pack4_e4m3(x[2], x[3], x[6], x[7]);
          a[kc][2] = pack4_e4m3(x[8], x[9], x[12], x[13]);
          a[kc][3] = pack4_e4m3(x[10], x[11], x[14], x[15]);
        }
        const uint32_t vt_addr = smem_u32(vt);
        fence_regs(o);
        wgmma_fence();
#pragma unroll
        for (int kc = 0; kc < 4; ++kc)
          wgmma_128_rs_e4m3(o, a[kc], gmma_desc_sw128(vt_addr + kc * 32, 16, 1024), 1u);
      } else {
        uint32_t a[8][4];
#pragma unroll
        for (int kk = 0; kk < 8; ++kk)
#pragma unroll
          for (int t = 0; t < 4; ++t) a[kk][t] = pack2<kBF16>(sc[8 * kk + 2 * t], sc[8 * kk + 2 * t + 1]);
        const uint32_t v_addr = smem_u32(vs);
        fence_regs(o);
        wgmma_fence();
#pragma unroll
        for (int kk = 0; kk < 8; ++kk)   // 16 keys = 16 rows x 128 B inside each V box
          wgmma_128_rs_bmn<kBF16>(o, a[kk], gmma_desc_sw128(v_addr + kk * 16 * 128, kBoxBytes, 1024), 1u);
      }
      wgmma_commit();
      wgmma_wait<0>();
      fence_regs(o);
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars[V_EMPTY + s]);
    }
  }

  // ---- epilogue: O / l -> global (ref :135-136); rows past the limit are zeros (:156) ----
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l_sum[r] += __shfl_xor_sync(0xffffffffu, l_sum[r], 1);
    l_sum[r] += __shfl_xor_sync(0xffffffffu, l_sum[r], 2);
  }
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const long long q_row = q_row0 + row_lo + 8 * r;
    const bool in_tensor = q_row < p.q_rows;
    const bool zero_row = (n_tiles == 0) || (!dense && q_row >= q_limit_sparse);
    float inv_l = zero_row ? 0.f : 1.0f / l_sum[r];
    if constexpr (kPvFp8) inv_l *= __ldg(p.v_fp8_amax + b * p.heads + h) * (1.0f / 448.0f);   // undo the V scale
    if (p.lse_out && dense && in_tensor && qd == 0) {
      // softmax_lse of flash_attn (natural log): ln sum_j exp(s_j * sm_scale) = (m + log2 l) * ln 2
      p.lse_out[(static_cast<long long>(b) * p.heads + h) * p.q_rows + q_row] =
          zero_row ? -INFINITY : (m_used[r] + log2f(l_sum[r])) * 0.6931471805599453f;
    }
    if (!in_tensor) continue;
    // destination(s) of this row
    long long o_off = b * p.o_stride_b + q_row * p.o_stride_s + static_cast<long long>(h) * p.o_stride_h;
    uint16_t* obase = reinterpret_cast<uint16_t*>(p.out);
    int n_dst = 1;  // > 1 only for replicated (text) rows under Ulysses
    if (p.sp_world > 0) {
      // Fused Ulysses exchange (ref xdit_ring_atten.py:206-219 does this with two all-to-alls
      // after the kernel): image row t belongs to rank t / sp_rows; text rows go to every rank.
      const long long n_img = p.sp_rows * p.sp_world;
      const int gh = p.sp_head_base + h;
      if (q_row < n_img) {
        const int owner = static_cast<int>(q_row / p.sp_rows);
        obase = reinterpret_cast<uint16_t*>(p.peer_out[owner]);
        o_off = ((q_row - owner * p.sp_rows) * p.sp_heads_total + gh) * kHeadDim;
      } else {
        n_dst = p.sp_world;
        o_off = ((p.sp_rows + (q_row - n_img)) * p.sp_heads_total + gh) * kHeadDim;
      }
    }
#pragma unroll
    for (int n8 = 0; n8 < 16; ++n8) {
      const int i = 4 * n8 + 2 * r;
      const int col = 8 * n8 + 2 * qd;
      const uint32_t v = pack2<kBF16>(zero_row ? 0.f : o[i] * inv_l, zero_row ? 0.f : o[i + 1] * inv_l);
      if (n_dst > 1) {
        for (int rr = 0; rr < n_dst; ++rr)
          *reinterpret_cast<uint32_t*>(reinterpret_cast<uint16_t*>(p.peer_out[rr]) + o_off + col) = v;
      } else if (!p.out_f32) {
        *reinterpret_cast<uint32_t*>(obase + o_off + col) = v;
      } else {  // wan/…:530-532: the 16-bit result is widened back to the query dtype
        *reinterpret_cast<float2*>(reinterpret_cast<float*>(p.out) + o_off + col) = unpack2<kBF16>(v);
      }
    }
  }
}

}  // namespace

// ------------------------------------------------------------------------------------------
// Host side
// ------------------------------------------------------------------------------------------
static int make_tile_map(CUtensorMap* map, const void* base, int dtype, long long rows, int heads,
                         int batch, long long stride_b, long long stride_s, long long stride_h,
                         int box_rows) {
  // dims (fastest first): d, row, head, batch.  Box {64, box_rows, 1, 1}, 128-B swizzle.
  const cuuint64_t dims[4] = {static_cast<cuuint64_t>(kHeadDim), static_cast<cuuint64_t>(rows),
                              static_cast<cuuint64_t>(heads), static_cast<cuuint64_t>(batch)};
  const cuuint64_t strides[3] = {static_cast<cuuint64_t>(stride_s) * 2,
                                 static_cast<cuuint64_t>(stride_h) * 2,
                                 static_cast<cuuint64_t>(stride_b) * 2};
  const cuuint32_t box[4] = {64, static_cast<cuuint32_t>(box_rows), 1, 1};
  const cuuint32_t elem_strides[4] = {1, 1, 1, 1};
  const CUtensorMapDataType dt =
      dtype == JENGA_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  return encode_tensor_map(map, dt, 4, const_cast<void*>(base), dims, strides, box, elem_strides,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                           CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

// V as FP8: contiguous [B, S, H, 128] bytes; box {128 channels, 128 keys}
static int make_v8_map(CUtensorMap* map, const void* base, long long rows, int heads, int batch) {
  const cuuint64_t dims[4] = {static_cast<cuuint64_t>(kHeadDim), static_cast<cuuint64_t>(rows),
                              static_cast<cuuint64_t>(heads), static_cast<cuuint64_t>(batch)};
  const cuuint64_t strides[3] = {static_cast<cuuint64_t>(heads) * kHeadDim, static_cast<cuuint64_t>(kHeadDim),
                                 static_cast<cuuint64_t>(rows) * heads * kHeadDim};
  const cuuint32_t box[4] = {128, static_cast<cuuint32_t>(kBlock), 1, 1};
  const cuuint32_t elem_strides[4] = {1, 1, 1, 1};
  return encode_tensor_map(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 4, const_cast<void*>(base), dims, strides, box,
                           elem_strides, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                           CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

static bool stride_ok(long long s) { return s > 0 && (s * 2) % 16 == 0; }

int carved_attn_fwd_impl(const JengaAttnArgs* a, cudaStream_t stream) {
  if (!a || !a->q || !a->k || !a->v || (!a->out && a->sp_world <= 0)) return set_error(JENGA_E_INVALID, "null pointer");
  if (a->dtype != JENGA_BF16 && a->dtype != JENGA_F16)
    return set_error(JENGA_E_INVALID, "dtype must be bf16 or f16");
  if (a->head_dim != kHeadDim)
    return set_error(JENGA_E_UNSUPPORTED, "head_dim %d: only 128 is built", a->head_dim);
  if (a->batch <= 0 || a->heads <= 0 || a->q_rows <= 0 || a->kv_rows <= 0)
    return set_error(JENGA_E_INVALID, "empty shape");
  if (a->nq_sparse < 0 || a->nq_dense < 0 || a->nq_sparse + a->nq_dense == 0)
    return set_error(JENGA_E_INVALID, "no query blocks");
  if (static_cast<long long>(a->nq_sparse + a->nq_dense - 1) * kBlock >= a->q_rows)
    return set_error(JENGA_E_INVALID, "query blocks exceed q_rows");
  const long long nb_kv = (a->kv_rows + kBlock - 1) / kBlock;
  const int need_words = static_cast<int>((nb_kv + 31) / 32);
  if (a->nq_sparse > 0 && (!a->mask_bits || a->mask_words < need_words))
    return set_error(JENGA_E_INVALID, "mask_bits missing or mask_words %d < %d", a->mask_words,
                     need_words);
  const int words = a->nq_sparse > 0 ? a->mask_words : need_words;
  if (words > kMaxMaskWords)
    return set_error(JENGA_E_UNSUPPORTED, "more than %d key blocks", kMaxMaskWords * 32);
  const long long strides[] = {a->q_stride_b, a->q_stride_s, a->q_stride_h, a->k_stride_b,
                               a->k_stride_s, a->k_stride_h, a->v_stride_b, a->v_stride_s,
                               a->v_stride_h, a->o_stride_b, a->o_stride_s, a->o_stride_h};
  for (int i = 0; i < 12; ++i)
    if (!stride_ok(strides[i]) && !(i >= 9 && a->sp_world > 0))
      return set_error(JENGA_E_INVALID, "strides must be positive multiples of 8");
  if (a->out_dtype != a->dtype && a->out_dtype != JENGA_F32)
    return set_error(JENGA_E_INVALID, "out_dtype must equal dtype or be f32");
  const uintptr_t ptrs[] = {(uintptr_t)a->q, (uintptr_t)a->k, (uintptr_t)a->v, (uintptr_t)a->out};
  for (uintptr_t q : ptrs)
    if (q % 16) return set_error(JENGA_E_INVALID, "pointers must be 16-byte aligned");
  if (!(a->sm_scale > 0.f)) return set_error(JENGA_E_INVALID, "sm_scale must be positive");
  if (a->sp_world != 0 &&
      (a->sp_world < 0 || a->sp_world > 8 || a->sp_rank < 0 || a->sp_rank >= a->sp_world || !a->out_peers_host ||
       a->sp_rows <= 0 || a->batch != 1 || a->out_dtype != a->dtype))
    return set_error(JENGA_E_INVALID, "bad Ulysses epilogue arguments");
  const int sp_head_base = a->sp_head_base_valid ? a->sp_head_base : a->sp_rank * a->heads;
  if (a->sp_world != 0 &&
      ((!a->sp_head_base_valid && a->sp_heads_total != a->heads * a->sp_world) || sp_head_base < 0 ||
       sp_head_base + a->heads > a->sp_heads_total))
    return set_error(JENGA_E_INVALID, "bad Ulysses head range");

  const bool pv_fp8 = a->v_fp8 != nullptr;
  if (pv_fp8) {
    if (!a->v_fp8_amax || a->dtype != JENGA_BF16)
      return set_error(JENGA_E_UNSUPPORTED, "fp8 P.V: needs v_fp8_amax and bf16 q/k");
    if (reinterpret_cast<uintptr_t>(a->v_fp8) % 16) return set_error(JENGA_E_INVALID, "v_fp8 must be 16-byte aligned");
  }
  CUtensorMap tm_q, tm_k, tm_v;
  int rc;
  if ((rc = make_tile_map(&tm_q, a->q, a->dtype, a->q_rows, a->heads, a->batch, a->q_stride_b,
                          a->q_stride_s, a->q_stride_h, kBlock)))
    return rc;
  if ((rc = make_tile_map(&tm_k, a->k, a->dtype, a->kv_rows, a->heads, a->batch, a->k_stride_b,
                          a->k_stride_s, a->k_stride_h, kBlock)))
    return rc;
  if (pv_fp8) {
    if ((rc = make_v8_map(&tm_v, a->v_fp8, a->kv_rows, a->heads, a->batch))) return rc;
  } else if ((rc = make_tile_map(&tm_v, a->v, a->dtype, a->kv_rows, a->heads, a->batch, a->v_stride_b,
                                 a->v_stride_s, a->v_stride_h, kBlock)))
    return rc;

  KernelParams p{};
  p.heads = a->heads;
  p.nq_sparse = a->nq_sparse;
  p.nq_dense = a->nq_dense;
  p.nb_kv = static_cast<int>(nb_kv);
  p.mask_words = words;
  p.text_block_start = a->text_block_start;
  p.q_rows = a->q_rows;
  p.q_limit_sparse = a->q_limit_sparse;
  p.kv_limit_sparse = a->kv_limit_sparse;
  p.kv_limit_dense = a->kv_limit_dense;
  p.qk_scale = static_cast<float>(static_cast<double>(a->sm_scale) * 1.44269504);  // ref :172
  p.text_amp = a->text_amp;
  p.mask_bits = a->mask_bits;
  if (a->sp_world > 0) {
    p.sp_world = a->sp_world;
    p.sp_rank = a->sp_rank;
    p.sp_heads_total = a->sp_heads_total;
    p.sp_head_base = sp_head_base;
    p.sp_rows = a->sp_rows;
    for (int r = 0; r < a->sp_world; ++r) p.peer_out[r] = a->out_peers_host[r];
  }
  p.seqlen_dev = a->seqlen_dev;
  p.out_f32 = a->out_dtype == JENGA_F32 ? 1 : 0;
  p.out = a->out;
  p.o_stride_b = a->o_stride_b;
  p.o_stride_s = a->o_stride_s;
  p.o_stride_h = a->o_stride_h;
  p.err_flag = a->err_flag;
  p.lse_out = a->lse_out;
  p.v_fp8_amax = a->v_fp8_amax;

  const long long grid = static_cast<long long>(a->batch) * a->heads * (a->nq_sparse + a->nq_dense);
  if (grid > 0x7fffffffll) return set_error(JENGA_E_UNSUPPORTED, "grid too large");
  auto kern = pv_fp8 ? carved_attn_fwd_kernel<true, true>
                     : (a->dtype == JENGA_BF16 ? carved_attn_fwd_kernel<true> : carved_attn_fwd_kernel<false>);
  cudaError_t ce = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);
  if (ce != cudaSuccess) return set_cuda_error(ce, "cudaFuncSetAttribute(carved_attn)");
  kern<<<static_cast<unsigned>(grid), kThreads, kSmemBytes, stream>>>(tm_q, tm_k, tm_v, p);
  ce = cudaGetLastError();
  if (ce != cudaSuccess) return set_cuda_error(ce, "carved_attn launch");
  return JENGA_OK;
}

}  // namespace jenga
