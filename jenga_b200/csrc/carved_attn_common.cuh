// Parameters and mask walker of the carved-attention kernel (carved_attn.cu), and the warp-specialised
// pipeline it shares with the Wan I2V cross-attention kernel (wan_cross_attn.cu): tile geometry and
// shared-memory carve-up, the producer's TMA ring, and the consumer warpgroups' Q.K^T / online softmax /
// P.V loop.
#pragma once
#include "sm90_ptx.cuh"
#include "jenga_internal.h"

namespace jenga {
namespace attn {

struct KernelParams {
  int heads;
  int nq_sparse, nq_dense;
  int nb_kv;
  int mask_words;
  int text_block_start;
  long long q_rows;           // rows present in q / out
  long long q_limit_sparse;   // sparse rows >= this produce zeros
  long long kv_limit_sparse;  // key columns >= this are masked for sparse q blocks
  long long kv_limit_dense;   // ... for dense q blocks
  float qk_scale;             // sm_scale * log2(e)
  float text_amp;
  const uint32_t* mask_bits;
  const int* seqlen_dev;      // optional: overrides q_limit_sparse / kv_limit_sparse
  void* out;
  long long o_stride_b, o_stride_s, o_stride_h;  // elements
  int out_f32;                // 1: write fp32 (values still rounded through the MMA dtype)
  // Ulysses fused epilogue (sp_world > 0): O rows are stored straight into the token owner's
  // buffer over NVLink instead of `out`.  peer_out[r] = base of rank r's [batch, sp_rows + dense rows,
  // sp_heads_total, D] buffer; this rank's heads are [sp_rank*heads, (sp_rank+1)*heads).
  int sp_world, sp_rank, sp_heads_total;
  int sp_head_base;           // global head index of local head 0 (default sp_rank*heads)
  long long sp_rows;          // image rows owned per rank
  unsigned long long peer_out[8];
  float* lse_out;             // optional [B, H, q_rows] natural-log LSE of the dense rows
  const float* v_fp8_amax;    // fp8 P.V variant: per (batch, head) absmax of V (scale = amax / 448)
  // INT8 Q.K^T variant: per-(b*H+h) rows of scales, 64-row groups of Q and 128-key blocks of K
  const float* q_scale;
  const float* k_scale;
  long long q_groups, k_groups;   // scales per (batch, head): q_rows_padded / 64, kv_rows_padded / 128
  // INT8 Q.K^T with lse_out: [B*H, q_rows_padded] shift c_i = Q'_i . mean(K) that K smoothing took
  // off every score of row i (jenga_quantize_q_int8_lse_shift); the LSE adds sm_scale * c_i back
  const float* q_lse_shift;
  int* err_flag;
  // optional [grid] item of each CTA (carved_attn_order_kernel); NULL: CTA i runs item i
  const int* order;
};

// Walks the set bits of the row mask in ascending key-block order.
struct BlockWalker {
  const uint32_t* words;
  int nwords;
  int w;
  uint32_t bits;
  __device__ BlockWalker(const uint32_t* m, int n) : words(m), nwords(n), w(0), bits(n ? m[0] : 0) {}
  __device__ int next() {  // -1 when exhausted
    while (bits == 0) {
      if (++w >= nwords) return -1;
      bits = words[w];
    }
    const int j = __ffs(bits) - 1;
    bits &= bits - 1;
    return w * 32 + j;
  }
};

// ------------------------------------------------------------------------------------------
// Pipeline.  One CTA per 128-row query block, 384 threads in three warpgroups:
//   warpgroups 0, 1  consumers, 64 query rows each (Consumer below)
//   warpgroup 2      producer: warp 8 issues TMA (produce below); the other warps are the kernel's
// setmaxnreg moves registers from the producer to the consumers: Q~, S, O and the packed P of the
// previous tile are all live in a consumer at once.
// ------------------------------------------------------------------------------------------
constexpr int kBlock = 128;           // rows per q block == keys per kv block
constexpr int kHeadDim = 128;
constexpr int kConsumerThreads = 256;
constexpr int kThreads = kConsumerThreads + 128;  // + the producer warpgroup
constexpr int kStages = 2;                       // K/V ring depth
constexpr int kBoxBytes = kBlock * 64 * 2;       // 16 KB: 128 rows x 64 d (one TMA box)
constexpr int kTileBytes = 2 * kBoxBytes;        // 32 KB: 128 rows x 128 d (two d halves)
constexpr uint32_t kBarTurn = 3;                 // named barriers 3, 4: consumer warpgroup 0's, 1's turn

// shared-memory carve-up (offsets from the 1024-aligned base); a kernel's own data start at kOffEnd
constexpr int kOffQ = 0;
constexpr int kOffK = kOffQ + kTileBytes;
constexpr int kOffV = kOffK + kStages * kTileBytes;
constexpr int kOffBars = kOffV + kStages * kTileBytes;
constexpr int kOffEnd = kOffBars + 128;

enum BarId {
  Q_FULL = 0,
  K_FULL = 1, V_FULL = K_FULL + kStages,
  K_EMPTY = V_FULL + kStages, V_EMPTY = K_EMPTY + kStages,   // one arrival per consumer warp
  VT_FULL = V_EMPTY + kStages,                                // FP8 P.V: one arrival per transpose warp
  NUM_BARS = VT_FULL + kStages
};
static_assert(NUM_BARS * 8 <= kOffEnd - kOffBars, "barrier block overflow");

// byte offset of (row, col) inside a 128-byte-swizzled tile of 128-byte rows (1024-B aligned)
__device__ __forceinline__ uint32_t sw128(uint32_t row, uint32_t col) {
  return row * 128u + ((((col >> 4) ^ row) & 7u) << 4) + (col & 15u);
}

// sum over the four threads that hold one accumulator row
__device__ __forceinline__ float row_sum(float x) {
  x += __shfl_xor_sync(0xffffffffu, x, 1);
  return x + __shfl_xor_sync(0xffffffffu, x, 2);
}

// The tensor maps key tile j of the producer's walk is read through.
struct KvMaps {
  const CUtensorMap* k;
  const CUtensorMap* v;
};

// One 128-row tile by TMA, completing on `bar`: a one-byte operand (INT8 Q / K, FP8 V) is a single
// 128-channel box, a 16-bit one two 64-d halves.
template <bool kOneByte>
__device__ __forceinline__ void load_tile(uint8_t* dst, const CUtensorMap* map, uint64_t* bar, int row0, int h,
                                          int b) {
  mbar_arrive_expect_tx(bar, kOneByte ? kBoxBytes : kTileBytes);
  tma_load_4d(dst, map, bar, 0, row0, h, b);
  if constexpr (!kOneByte) tma_load_4d(dst + kBoxBytes, map, bar, 64, row0, h, b);
}

// Producer (one thread): Q once, then the K and V tiles of every key tile into the kStages ring; K
// and V slots are released separately.  next_kv(j, maps) returns the first key row of tile j and sets
// its maps, or returns a negative row past the last tile.  Keep the loop running on that row: the
// other loop shapes tried made ptxas move the consumers' descriptor arithmetic off the uniform
// datapath, which cost the carved kernel 8% on an H100.
template <bool kPvFp8, bool kQkInt8, class NextKv>
__device__ __forceinline__ void produce(uint8_t* smem, uint64_t* bars, int* err_flag, const CUtensorMap* tm_q,
                                        int q_row0, int h, int b, NextKv next_kv) {
  load_tile<kQkInt8>(smem + kOffQ, tm_q, &bars[Q_FULL], q_row0, h, b);
  KvMaps m;
  int j = 0;
  for (int row0 = next_kv(0, m); row0 >= 0; row0 = next_kv(++j, m)) {
    const int s = j % kStages;
    const uint32_t par = ((j / kStages) & 1) ^ 1;   // slot-free parity (a fresh barrier passes)
    mbar_wait(&bars[K_EMPTY + s], par, err_flag);
    load_tile<kQkInt8>(smem + kOffK + s * kTileBytes, m.k, &bars[K_FULL + s], row0, h, b);
    mbar_wait(&bars[V_EMPTY + s], par, err_flag);
    load_tile<kPvFp8>(smem + kOffV + s * kTileBytes, m.v, &bars[V_FULL + s], row0, h, b);
  }
}

// What the softmax of one key tile needs to know about it.
struct Tile {
  long long col0;       // key column of the tile's first row
  long long kv_limit;   // key columns >= this are masked
  float ct;             // exponent factor: p = exp2(s * ct + amp - m)
  float amp;            // constant added to every score of the tile, in log2 units
  bool restart;         // the tile opens a new segment (see Consumer::run)
};

// One consumer warpgroup: S = Q~ K^T by wgmma (16-bit Q~ in registers, loaded once with ldmatrix; K
// from shared memory; S in registers), online softmax in base 2 on the registers, then O += P V by
// wgmma with P as the register A operand.  S and O are fp32 register accumulators (64 + 64 registers
// per thread).  Accumulator fragment: element i of a thread is row g + 8 ((i >> 1) & 1) of the warp's
// 16 rows, column 8 (i >> 2) + 2 qd + (i & 1), with g = lane / 4 and qd = lane % 4.
template <bool kBF16, bool kPvFp8 = false, bool kQkInt8 = false>
struct Consumer {
  uint8_t* smem;
  uint64_t* bars;
  int* err_flag;
  int wg;                         // warpgroup: query rows [64 wg, 64 wg + 64)
  int lane, qd;
  int row_lo;                     // row of the accumulator elements i with (i & 2) == 0
  float m_used[2] = {-INFINITY, -INFINITY};   // running (possibly stale) max, in scaled log2 units
  float l_sum[2] = {0.f, 0.f};                 // this thread's partial sums (its 32 columns)
  float o[64];
  uint32_t qa[kQkInt8 ? 1 : 8][4];   // 16-bit Q: A operand of every Q.K^T wgmma
  float sc[64];                      // S_j, then P_j in fp32
  int32_t si[kQkInt8 ? 64 : 1];      // kQkInt8: integer S_j while its wgmma runs
  uint32_t pa[kPvFp8 ? 4 : 8][4];    // P_{j-1}: A operand of the P.V wgmma; untouched while it runs
  float alpha[2];

  __device__ __forceinline__ Consumer(uint8_t* smem_, uint64_t* bars_, int* err_flag_)
      : smem(smem_), bars(bars_), err_flag(err_flag_), wg(threadIdx.x >> 7), lane(threadIdx.x & 31), qd(lane & 3),
        row_lo(wg * 64 + ((threadIdx.x >> 5) & 3) * 16 + (lane >> 2)) {
#pragma unroll
    for (int i = 0; i < 64; ++i) o[i] = 0.f;
  }

  // Waits for Q.  16-bit Q: the warpgroup's 64 rows go to registers as the A operand of all its Q.K^T
  // wgmmas (16 k per step: matrices {rows 0-7, 8-15} x {k 0-7, 8-15} of the warp's 16 rows).
  // kQkInt8 leaves Q in shared memory: the s32 accumulator already takes the registers Q would need.
  __device__ __forceinline__ void load_q() {
    mbar_wait(&bars[Q_FULL], 0, err_flag);
    if constexpr (!kQkInt8) {
      const int warp = threadIdx.x >> 5;
      const int q_row = wg * 64 + (warp & 3) * 16 + (lane & 7) + 8 * ((lane >> 3) & 1);
#pragma unroll
      for (int kk = 0; kk < kHeadDim / 16; ++kk)
        ldmatrix_x4(qa[kk], smem + kOffQ + (kk >> 2) * kBoxBytes + sw128(q_row, (kk & 3) * 32 + (lane >> 4) * 16));
    }
  }

  // Turns: a warpgroup waits on its own barrier before it issues GEMMs and arrives on the other's
  // once they are issued, so one warpgroup's softmax runs while the other's GEMMs occupy the tensor
  // cores.  Warpgroup 1 arrives ahead for warpgroup 0's first turn and skips the hand-over after its
  // own last turn: both take the same number of turns, so every barrier sees as many arrivals as waits.
  __device__ __forceinline__ void turn_begin() { named_bar_sync(kBarTurn + wg, kConsumerThreads); }
  __device__ __forceinline__ void turn_end(bool last) {
    if (!(last && wg == 1)) named_bar_arrive(kBarTurn + (wg ^ 1), kConsumerThreads);
  }
  __device__ __forceinline__ void release(int bar) {
    __syncwarp();
    if (lane == 0) mbar_arrive(&bars[bar]);
  }

  // ---- S = Q~ K^T (64 x 128 per warpgroup, K = 128 in 8 steps) ----
  __device__ __forceinline__ void issue_qk(int s) {
    const uint32_t k_addr = smem_u32(smem + kOffK + s * kTileBytes);
    if constexpr (kQkInt8) {   // K = 128 in 4 steps of 32 one-byte channels inside the swizzled row
      const uint32_t q_addr = smem_u32(smem + kOffQ) + wg * 64 * 128;   // this warpgroup's 64 rows
#pragma unroll
      for (int kc = 0; kc < kHeadDim / 32; ++kc)
        wgmma_128_ss_s8(si, gmma_desc_sw128(q_addr + kc * 32, 16, 1024),
                        gmma_desc_sw128(k_addr + kc * 32, 16, 1024), kc > 0 ? 1u : 0u);
    } else {
#pragma unroll
      for (int kk = 0; kk < kHeadDim / 16; ++kk) {
        const uint32_t off = (kk & 3) * 32 + (kk >> 2) * kBoxBytes;
        wgmma_128_rs<kBF16>(sc, qa[kk], gmma_desc_sw128(k_addr + off, 16, 1024), kk > 0 ? 1u : 0u);
      }
    }
    wgmma_commit();
  }
  // S_j has retired: make it visible (and, for kQkInt8, exact fp32: |S| <= 128 * 127^2 < 2^22, so
  // the s32 value lands in the mantissa of 1.5 * 2^23 — two ALU ops, no 16/clk I2F)
  __device__ __forceinline__ void scores_ready() {
    if constexpr (kQkInt8) {
      fence_regs(si);
#pragma unroll
      for (int i = 0; i < 64; ++i) sc[i] = __int_as_float(si[i] + 0x4B400000) - 12582912.f;
    } else {
      fence_regs(sc);
    }
  }
  // ---- O += P V ----
  __device__ __forceinline__ void issue_pv(int s) {
    if constexpr (kPvFp8) {   // V^T in the upper half of the V slot
      const uint32_t vt_addr = smem_u32(smem + kOffV + s * kTileBytes + kBoxBytes);
#pragma unroll
      for (int kc = 0; kc < 4; ++kc)
        wgmma_128_rs_e4m3(o, pa[kc], gmma_desc_sw128(vt_addr + kc * 32, 16, 1024), 1u);
    } else {
      const uint32_t v_addr = smem_u32(smem + kOffV + s * kTileBytes);
#pragma unroll
      for (int kk = 0; kk < 8; ++kk)   // 16 keys = 16 rows x 128 B inside each V box
        wgmma_128_rs_bmn<kBF16>(o, pa[kk], gmma_desc_sw128(v_addr + kk * 16 * 128, kBoxBytes, 1024), 1u);
    }
    wgmma_commit();
  }
  // ---- online softmax of the key tile whose columns start at col0, on sc; true when O must be
  // rescaled by alpha.  ct scales the scores inside the exponent; amp is added to every score of the
  // tile in log2 units (ref :113-114), so it folds into the exponent offset ----
  __device__ __forceinline__ bool softmax(long long col0, long long kv_limit, float ct, float amp) {
    if (col0 + kBlock > kv_limit) {  // rare: only the tile that straddles the key limit
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
      m_cand[r] = fmaxf(m_used[r], fmaf(mx[r], ct, amp));
      // Lazy rescale: the reference rescales acc by exp2(m_old - m_new) every tile
      // (:121-132).  O/l is invariant to the reference point, so it only moves when the
      // max grew by more than 2^8 — the final O/l is the same up to fp32 rounding.
      need = need || (m_cand[r] - m_used[r]) > 8.0f;   // false for NaN (-inf - -inf)
    }
    const bool rescale = __any_sync(0xffffffffu, need);
    if (rescale) {
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        alpha[r] = (m_cand[r] == -INFINITY) ? 1.0f : fast_exp2(m_used[r] - m_cand[r]);
        l_sum[r] *= alpha[r];
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
      sc[i] = fast_exp2(fmaf(sc[i], ct, off[r]));
      l_sum[r] += sc[i];
    }
    return rescale;
  }
  __device__ __forceinline__ void rescale_o() {
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
      for (int i = 2 * r; i < 64; i += 4) {
        o[i] *= alpha[r];
        o[i + 1] *= alpha[r];
      }
  }
  // P_j -> the A operand of its P.V.  FP8: the keys of each 32-key group in the order of the V^T
  // transpose (carved_attn.cu), which is the order the accumulator fragment already holds them in.
  __device__ __forceinline__ void pack_p() {
    if constexpr (kPvFp8) {
#pragma unroll
      for (int kc = 0; kc < 4; ++kc) {
        const float* x = sc + 16 * kc;
        pa[kc][0] = pack4_e4m3(x[0], x[1], x[4], x[5]);
        pa[kc][1] = pack4_e4m3(x[2], x[3], x[6], x[7]);
        pa[kc][2] = pack4_e4m3(x[8], x[9], x[12], x[13]);
        pa[kc][3] = pack4_e4m3(x[10], x[11], x[14], x[15]);
      }
    } else {
#pragma unroll
      for (int kk = 0; kk < 8; ++kk)
#pragma unroll
        for (int t = 0; t < 4; ++t) pa[kk][t] = pack2<kBF16>(sc[8 * kk + 2 * t], sc[8 * kk + 2 * t + 1]);
    }
  }

  // The tile loop, FlashAttention-3's schedule.  In-warpgroup pipelining: iteration j issues
  // S_j = Q~ K_j^T, then O += P_{j-1} V_{j-1}; it waits for S_j alone, runs softmax_j while
  // P_{j-1} V_{j-1} is still on the tensor cores, then waits for that and applies the lazy rescale
  // O *= alpha_j.  The prologue computes S_0 and its softmax, the epilogue issues the last P V.  O and
  // l see the same operations in the same order as a plain S, softmax, P V loop, so the result is the
  // same bit for bit.  Ping-pong: the two warpgroups take turns to issue their GEMMs (turn_begin),
  // warpgroup 0 first.
  //
  // next_tile(j, t) fills key tile j of the n_tiles >= 1 tiles (the same walk as the producer's); it
  // runs before the tile's waits, so what it reads from global memory never stalls the softmax.  The
  // last tile's slot comes from n_tiles rather than from the loop's exit index, which lets ptxas keep
  // the shared-memory descriptor arithmetic on the uniform datapath.
  //
  // A tile with t.restart opens a new segment, which is computed as a fresh launch over its tiles
  // would compute it: m and l restart after S_j retires; after P_{j-1} V_{j-1} retires,
  // segment_end(l) gets the finished segment's l (O is still in o), and O restarts from zero, which
  // is what a fresh launch's first rescale makes of its zero O.
  template <class NextTile, class SegmentEnd>
  __device__ __forceinline__ void run(int n_tiles, NextTile next_tile, SegmentEnd segment_end) {
    constexpr int kVReady = kPvFp8 ? VT_FULL : V_FULL;
    if (wg == 1) named_bar_arrive(kBarTurn, kConsumerThreads);
    // prologue: S_0 and its softmax
    Tile t;
    next_tile(0, t);
    mbar_wait(&bars[K_FULL], 0, err_flag);
    turn_begin();
    wgmma_fence();
    issue_qk(0);
    turn_end(false);
    wgmma_wait<0>();
    scores_ready();
    release(K_EMPTY);
    if (softmax(t.col0, t.kv_limit, t.ct, t.amp)) rescale_o();
    pack_p();
    for (int j = 1; j < n_tiles; ++j) {   // S_j and P_{j-1} V_{j-1}
      next_tile(j, t);
      const int s = j % kStages, sv = (j - 1) % kStages;
      mbar_wait(&bars[kVReady + sv], ((j - 1) / kStages) & 1, err_flag);
      mbar_wait(&bars[K_FULL + s], (j / kStages) & 1, err_flag);
      turn_begin();
      fence_regs(o);
      wgmma_fence();
      issue_qk(s);
      issue_pv(sv);
      turn_end(false);
      wgmma_wait<1>();
      scores_ready();
      release(K_EMPTY + s);
      float l_done[2];
      if (t.restart) {
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          l_done[r] = l_sum[r];
          l_sum[r] = 0.f;
          m_used[r] = -INFINITY;
        }
      }
      const bool rescale = softmax(t.col0, t.kv_limit, t.ct, t.amp);
      wgmma_wait<0>();
      fence_regs(o);
      release(V_EMPTY + sv);
      if (t.restart) {
        segment_end(l_done);
#pragma unroll
        for (int i = 0; i < 64; ++i) o[i] = 0.f;
      } else if (rescale) {
        rescale_o();
      }
      pack_p();
    }
    // epilogue: P V of the last tile
    const int sv = (n_tiles - 1) % kStages;
    mbar_wait(&bars[kVReady + sv], ((n_tiles - 1) / kStages) & 1, err_flag);
    turn_begin();
    fence_regs(o);
    wgmma_fence();
    issue_pv(sv);
    turn_end(true);
    wgmma_wait<0>();
    fence_regs(o);
    release(V_EMPTY + sv);
  }
};

}  // namespace attn

// ------------------------------------------------------------------------------------------
// Host side
// ------------------------------------------------------------------------------------------
// 16-bit [B, S, H, 128] operand: dims (fastest first) d, row, head, batch; box {64 d, 128 rows},
// 128-B swizzle, rows past `rows` zero-filled.
static inline int make_tile_map(CUtensorMap* map, const void* base, int dtype, long long rows, int heads,
                                int batch, long long stride_b, long long stride_s, long long stride_h) {
  const cuuint64_t dims[4] = {static_cast<cuuint64_t>(attn::kHeadDim), static_cast<cuuint64_t>(rows),
                              static_cast<cuuint64_t>(heads), static_cast<cuuint64_t>(batch)};
  const cuuint64_t strides[3] = {static_cast<cuuint64_t>(stride_s) * 2,
                                 static_cast<cuuint64_t>(stride_h) * 2,
                                 static_cast<cuuint64_t>(stride_b) * 2};
  const cuuint32_t box[4] = {64, static_cast<cuuint32_t>(attn::kBlock), 1, 1};
  const cuuint32_t elem_strides[4] = {1, 1, 1, 1};
  const CUtensorMapDataType dt =
      dtype == JENGA_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
  return encode_tensor_map(map, dt, 4, const_cast<void*>(base), dims, strides, box, elem_strides,
                           CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                           CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

// element stride of a 16-bit operand: TMA needs positive multiples of 16 bytes
static inline bool stride_ok(long long s) { return s > 0 && (s * 2) % 16 == 0; }

}  // namespace jenga
