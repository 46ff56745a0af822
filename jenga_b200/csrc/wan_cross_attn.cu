// Wan2.1-I2V cross-attention for sm_90a: the image and the text attention of one query block in one
// launch, summed as the reference sums them.
//
// Replaces WanI2VCrossAttention.forward's attention part (wan/modules/model_mul.py:240-247): two
// flash_attention calls over the 257 CLIP keys and the text keys, each returned as fp32
// (wan/modules/attention.py:130), added in fp32 and cast to bf16 by self.o under autocast:
//   out[r,h,:] = bf16( f32(A_img[r,h,:]) + f32(A_txt[r,h,:]) ),  A_seg = bf16(softmax(q K_seg^T D^-1/2) V_seg)
//
// Each segment is computed with the dense-class arithmetic of the carved-attention kernel
// (carved_attn.cu): wgmma S = Q K^T with Q in registers, fp32 scores scaled inside exp2 by
// sm_scale * log2 e, the same lazy-rescale rule, P rounded to bf16 for P V, fp32 O and l, O * (1 / l)
// rounded to bf16.  So A_img and A_txt are bit for bit what one dense launch over that segment
// returns.  At the segment boundary A_img is normalised, rounded and parked in the shared-memory Q
// tile (Q lives in registers by then; each warp overwrites only its own 16 Q rows), and m / l / O
// start afresh for the text tiles.
//
// Layout: one CTA per (batch*head, 128 query rows), head-major, 384 threads as in carved_attn.cu —
// two consumer warpgroups (64 query rows each, the ping-pong / in-warpgroup pipelined schedule) and a
// producer warpgroup whose warp 8 issues TMA: Q once, then the image K/V tiles and the text K/V tiles
// (each pair through its own tensor maps) into a two-stage ring.  Rows past a tensor's extent are
// zero-filled by TMA and masked by the segment's column limit, so no padding copies are needed.
#include <cfloat>

#include "sm90_ptx.cuh"
#include "jenga_internal.h"

namespace jenga {

namespace {

constexpr int kBlock = 128;
constexpr int kHeadDim = 128;
constexpr int kConsumerThreads = 256;
constexpr int kThreads = kConsumerThreads + 128;
constexpr int kStages = 2;
constexpr int kBoxBytes = kBlock * 64 * 2;       // 16 KB: 128 rows x 64 d
constexpr int kTileBytes = 2 * kBoxBytes;        // 32 KB: 128 rows x 128 d
constexpr uint32_t kBarTurn = 3;                 // named barriers 3, 4: consumer warpgroup 0's, 1's turn

constexpr int kOffQ = 0;
constexpr int kOffK = kOffQ + kTileBytes;
constexpr int kOffV = kOffK + kStages * kTileBytes;
constexpr int kOffBars = kOffV + kStages * kTileBytes;
constexpr int kSmemBytes = 1024 /*align slack*/ + kOffBars + 128;

enum BarId {
  Q_FULL = 0,
  K_FULL = 1, V_FULL = K_FULL + kStages,
  K_EMPTY = V_FULL + kStages, V_EMPTY = K_EMPTY + kStages,   // one arrival per consumer warp
  NUM_BARS = V_EMPTY + kStages
};
static_assert(NUM_BARS * 8 <= 128, "barrier block overflow");

struct CrossParams {
  int heads;
  int nq;                         // query blocks per (batch, head)
  int n_img, n_txt;               // key tiles of each segment
  long long q_rows, img_rows, txt_rows;
  float qk_scale;                 // sm_scale * log2(e)
  uint16_t* out;
  long long o_stride_b, o_stride_s, o_stride_h;
  int* err_flag;
};

__device__ __forceinline__ uint32_t sw128(uint32_t row, uint32_t col) {
  return row * 128u + ((((col >> 4) ^ row) & 7u) << 4) + (col & 15u);
}

__global__ void __launch_bounds__(kThreads, 1)
wan_i2v_cross_attn_kernel(const __grid_constant__ CUtensorMap tm_q,
                          const __grid_constant__ CUtensorMap tm_ki, const __grid_constant__ CUtensorMap tm_vi,
                          const __grid_constant__ CUtensorMap tm_kt, const __grid_constant__ CUtensorMap tm_vt,
                          const CrossParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw_addr + 1023u) & ~1023u) - raw_addr);
  uint8_t* sQ = smem + kOffQ;
  uint8_t* sK = smem + kOffK;
  uint8_t* sV = smem + kOffV;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kOffBars);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int bh = blockIdx.x / p.nq;
  const int qb = blockIdx.x - bh * p.nq;
  const int b = bh / p.heads;
  const int h = bh - b * p.heads;
  const long long q_row0 = static_cast<long long>(qb) * kBlock;
  const int n_tiles = p.n_img + p.n_txt;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tm_q);
    tma_prefetch_desc(&tm_ki);
    tma_prefetch_desc(&tm_vi);
    tma_prefetch_desc(&tm_kt);
    tma_prefetch_desc(&tm_vt);
#pragma unroll
    for (int i = 0; i < NUM_BARS; ++i) mbar_init(&bars[i], i >= K_EMPTY ? 8u : 1u);
    fence_mbar_init();
  }
  __syncthreads();

  if (warp >= kConsumerThreads / 32) {
    // =============================== producer warpgroup ===============================
    setmaxnreg_dec<24>();
    if (warp == kConsumerThreads / 32 && lane == 0) {
      mbar_arrive_expect_tx(&bars[Q_FULL], kTileBytes);
      tma_load_4d(sQ, &tm_q, &bars[Q_FULL], 0, static_cast<int>(q_row0), h, b);
      tma_load_4d(sQ + kBoxBytes, &tm_q, &bars[Q_FULL], 64, static_cast<int>(q_row0), h, b);
      for (int j = 0; j < n_tiles; ++j) {
        const int s = j % kStages;
        const uint32_t par = ((j / kStages) & 1) ^ 1;   // slot-free parity (a fresh barrier passes)
        const bool img = j < p.n_img;
        const CUtensorMap* tk = img ? &tm_ki : &tm_kt;
        const CUtensorMap* tv = img ? &tm_vi : &tm_vt;
        const int row0 = (img ? j : j - p.n_img) * kBlock;
        uint8_t* k_dst = sK + s * kTileBytes;
        uint8_t* v_dst = sV + s * kTileBytes;
        mbar_wait(&bars[K_EMPTY + s], par, p.err_flag);
        mbar_arrive_expect_tx(&bars[K_FULL + s], kTileBytes);
        tma_load_4d(k_dst, tk, &bars[K_FULL + s], 0, row0, h, b);
        tma_load_4d(k_dst + kBoxBytes, tk, &bars[K_FULL + s], 64, row0, h, b);
        mbar_wait(&bars[V_EMPTY + s], par, p.err_flag);
        mbar_arrive_expect_tx(&bars[V_FULL + s], kTileBytes);
        tma_load_4d(v_dst, tv, &bars[V_FULL + s], 0, row0, h, b);
        tma_load_4d(v_dst + kBoxBytes, tv, &bars[V_FULL + s], 64, row0, h, b);
      }
    }
    return;
  }

  // =============================== consumers ===============================
  setmaxnreg_inc<240>();
  const int wg = warp >> 2;                       // warpgroup: query rows [64 wg, 64 wg + 64)
  const int g = lane >> 2, qd = lane & 3;
  // accumulator fragment: element i of a thread is row g + 8 ((i >> 1) & 1) of the warp's 16 rows,
  // column 8 (i >> 2) + 2 qd + (i & 1)
  const int row_lo = wg * 64 + (warp & 3) * 16 + g;
  float m_used[2] = {-INFINITY, -INFINITY};
  float l_sum[2] = {0.f, 0.f};
  float l_img[2];
  float o[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) o[i] = 0.f;
  const float c = p.qk_scale;
  // the parked bf16 A_img of this warp: its own 16 Q rows of the two Q boxes (2 x 2 KB), word k of a
  // lane at (k & 15) * 32 + lane of box k >> 4 — conflict-free, and no other warp reads it
  uint32_t* park = reinterpret_cast<uint32_t*>(sQ + warp * 2048) + lane;
  auto park_at = [&](int k) -> uint32_t* { return park + (k >> 4) * (kBoxBytes / 4) + (k & 15) * 32; };

  mbar_wait(&bars[Q_FULL], 0, p.err_flag);
  uint32_t qa[8][4];
  {
    const int q_row = wg * 64 + (warp & 3) * 16 + (lane & 7) + 8 * ((lane >> 3) & 1);
#pragma unroll
    for (int kk = 0; kk < kHeadDim / 16; ++kk)
      ldmatrix_x4(qa[kk], sQ + (kk >> 2) * kBoxBytes + sw128(q_row, (kk & 3) * 32 + (lane >> 4) * 16));
  }

  float sc[64];
  uint32_t pa[8][4];
  float alpha[2];

  auto turn_begin = [&] { named_bar_sync(kBarTurn + wg, kConsumerThreads); };
  auto turn_end = [&](bool last) {
    if (!(last && wg == 1)) named_bar_arrive(kBarTurn + (wg ^ 1), kConsumerThreads);
  };
  auto release = [&](int bar) {
    __syncwarp();
    if (lane == 0) mbar_arrive(&bars[bar]);
  };
  auto issue_qk = [&](int s) {
    const uint32_t k_addr = smem_u32(sK + s * kTileBytes);
#pragma unroll
    for (int kk = 0; kk < kHeadDim / 16; ++kk) {
      const uint32_t off = (kk & 3) * 32 + (kk >> 2) * kBoxBytes;
      wgmma_128_rs<true>(sc, qa[kk], gmma_desc_sw128(k_addr + off, 16, 1024), kk > 0 ? 1u : 0u);
    }
    wgmma_commit();
  };
  auto issue_pv = [&](int s) {
    const uint32_t v_addr = smem_u32(sV + s * kTileBytes);
#pragma unroll
    for (int kk = 0; kk < 8; ++kk)
      wgmma_128_rs_bmn<true>(o, pa[kk], gmma_desc_sw128(v_addr + kk * 16 * 128, kBoxBytes, 1024), 1u);
    wgmma_commit();
  };
  // online softmax of key tile j on sc (the dense class of carved_attn.cu: no text_amp, c = qk_scale);
  // true when O must be rescaled by alpha
  auto softmax = [&](int j) -> bool {
    const float amp = 0.f;
    const bool img = j < p.n_img;
    const long long col0 = static_cast<long long>(img ? j : j - p.n_img) * kBlock;
    const long long kv_limit = img ? p.img_rows : p.txt_rows;
    if (col0 + kBlock > kv_limit) {  // the last tile of a segment
#pragma unroll
      for (int i = 0; i < 64; ++i)
        if (col0 + (i >> 2) * 8 + qd * 2 + (i & 1) >= kv_limit) sc[i] = -INFINITY;
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
      need = need || (m_cand[r] - m_used[r]) > 8.0f;   // lazy rescale; false for NaN (-inf - -inf)
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
    float off[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) off[r] = amp - ((m_used[r] == -INFINITY) ? 0.f : m_used[r]);
#pragma unroll
    for (int i = 0; i < 64; ++i) {
      const int r = (i >> 1) & 1;
      sc[i] = fast_exp2(fmaf(sc[i], c, off[r]));
      l_sum[r] += sc[i];
    }
    return rescale;
  };
  auto rescale_o = [&] {
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
      for (int i = 2 * r; i < 64; i += 4) {
        o[i] *= alpha[r];
        o[i + 1] *= alpha[r];
      }
  };
  auto pack_p = [&] {
#pragma unroll
    for (int kk = 0; kk < 8; ++kk)
#pragma unroll
      for (int t = 0; t < 4; ++t) pa[kk][t] = pack2<true>(sc[8 * kk + 2 * t], sc[8 * kk + 2 * t + 1]);
  };
  // 1 / l of the finished segment, l summed over the four threads of each row
  auto inv_rows = [&](const float (&l)[2], float (&inv)[2]) {
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      float t = l[r];
      t += __shfl_xor_sync(0xffffffffu, t, 1);
      t += __shfl_xor_sync(0xffffffffu, t, 2);
      inv[r] = 1.0f / t;
    }
  };

  if (wg == 1) named_bar_arrive(kBarTurn, kConsumerThreads);
  // prologue: S_0 and its softmax
  mbar_wait(&bars[K_FULL], 0, p.err_flag);
  turn_begin();
  wgmma_fence();
  issue_qk(0);
  turn_end(false);
  wgmma_wait<0>();
  fence_regs(sc);
  release(K_EMPTY);
  if (softmax(0)) rescale_o();
  pack_p();
  for (int j = 1; j < n_tiles; ++j) {   // S_j and P_{j-1} V_{j-1}
    const int s = j % kStages, sv = (j - 1) % kStages;
    const bool boundary = j == p.n_img;   // S_j is the first text tile, P_{j-1} the last image tile
    mbar_wait(&bars[V_FULL + sv], ((j - 1) / kStages) & 1, p.err_flag);
    mbar_wait(&bars[K_FULL + s], (j / kStages) & 1, p.err_flag);
    turn_begin();
    fence_regs(o);
    wgmma_fence();
    issue_qk(s);
    issue_pv(sv);
    turn_end(false);
    wgmma_wait<1>();
    fence_regs(sc);
    release(K_EMPTY + s);
    if (boundary) {   // the image l is complete; the text softmax starts as a fresh launch would
#pragma unroll
      for (int r = 0; r < 2; ++r) {
        l_img[r] = l_sum[r];
        l_sum[r] = 0.f;
        m_used[r] = -INFINITY;
      }
    }
    const bool rescale = softmax(j);
    wgmma_wait<0>();
    fence_regs(o);
    release(V_EMPTY + sv);
    if (boundary) {
      // A_img = bf16(O / l) as the dense epilogue rounds it, parked; O restarts from zero (what a
      // fresh launch's first rescale makes of its zero O)
      float inv[2];
      inv_rows(l_img, inv);
      __syncwarp();
#pragma unroll
      for (int k = 0; k < 32; ++k) *park_at(k) = pack2<true>(o[2 * k] * inv[k & 1], o[2 * k + 1] * inv[k & 1]);
#pragma unroll
      for (int i = 0; i < 64; ++i) o[i] = 0.f;
    } else if (rescale) {
      rescale_o();
    }
    pack_p();
  }
  // epilogue: P V of the last text tile
  {
    const int sv = (n_tiles - 1) % kStages;
    mbar_wait(&bars[V_FULL + sv], ((n_tiles - 1) / kStages) & 1, p.err_flag);
    turn_begin();
    fence_regs(o);
    wgmma_fence();
    issue_pv(sv);
    turn_end(true);
    wgmma_wait<0>();
    fence_regs(o);
    release(V_EMPTY + sv);
  }

  // ---- out = bf16(f32(A_img) + f32(A_txt)); rows past q_rows are not stored ----
  float inv[2];
  inv_rows(l_sum, inv);
#pragma unroll
  for (int k = 0; k < 32; ++k) {
    const int r = k & 1;
    const long long q_row = q_row0 + row_lo + 8 * r;
    if (q_row >= p.q_rows) continue;
    const float2 ft = unpack2<true>(pack2<true>(o[2 * k] * inv[r], o[2 * k + 1] * inv[r]));
    const float2 fi = unpack2<true>(*park_at(k));
    const long long o_off = b * p.o_stride_b + q_row * p.o_stride_s + static_cast<long long>(h) * p.o_stride_h +
                            8 * (k >> 1) + 2 * qd;
    *reinterpret_cast<uint32_t*>(p.out + o_off) = pack2<true>(ft.x + fi.x, ft.y + fi.y);
  }
}

// dims (fastest first): d, row, head, batch.  Box {64, 128, 1, 1}, 128-B swizzle, zero fill past `rows`.
int make_bf16_map(CUtensorMap* map, const void* base, long long rows, int heads, int batch, long long stride_b,
                  long long stride_s, long long stride_h) {
  const cuuint64_t dims[4] = {static_cast<cuuint64_t>(kHeadDim), static_cast<cuuint64_t>(rows),
                              static_cast<cuuint64_t>(heads), static_cast<cuuint64_t>(batch)};
  const cuuint64_t strides[3] = {static_cast<cuuint64_t>(stride_s) * 2, static_cast<cuuint64_t>(stride_h) * 2,
                                 static_cast<cuuint64_t>(stride_b) * 2};
  const cuuint32_t box[4] = {64, static_cast<cuuint32_t>(kBlock), 1, 1};
  const cuuint32_t elem_strides[4] = {1, 1, 1, 1};
  return encode_tensor_map(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 4, const_cast<void*>(base), dims, strides, box,
                           elem_strides, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                           CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
}

bool stride_ok(long long s) { return s > 0 && (s * 2) % 16 == 0; }

int wan_i2v_cross_attn_impl(const JengaWanCrossArgs* a, cudaStream_t stream) {
  if (!a) return set_error(JENGA_E_INVALID, "wan_i2v_cross_attn: null pointer");
  if (!a->q || !a->k_img || !a->v_img || !a->k_txt || !a->v_txt || !a->out)
    return set_error(JENGA_E_INVALID, "wan_i2v_cross_attn: null pointer");
  if (a->dtype != JENGA_BF16) return set_error(JENGA_E_INVALID, "wan_i2v_cross_attn: dtype must be bf16");
  if (a->head_dim != kHeadDim)
    return set_error(JENGA_E_INVALID, "wan_i2v_cross_attn: head_dim %d, only 128 is built", a->head_dim);
  if (a->batch <= 0 || a->heads <= 0 || a->q_rows <= 0)
    return set_error(JENGA_E_INVALID, "wan_i2v_cross_attn: empty shape");
  if (a->img_rows <= 0 || a->txt_rows <= 0)
    return set_error(JENGA_E_INVALID, "wan_i2v_cross_attn: img_rows and txt_rows must be >= 1");
  const long long strides[] = {a->q_stride_b,  a->q_stride_s,  a->q_stride_h,  a->ki_stride_b, a->ki_stride_s,
                               a->ki_stride_h, a->vi_stride_b, a->vi_stride_s, a->vi_stride_h, a->kt_stride_b,
                               a->kt_stride_s, a->kt_stride_h, a->vt_stride_b, a->vt_stride_s, a->vt_stride_h,
                               a->o_stride_b,  a->o_stride_s,  a->o_stride_h};
  for (long long s : strides)
    if (!stride_ok(s))
      return set_error(JENGA_E_INVALID, "wan_i2v_cross_attn: strides must be positive multiples of 8 elements (16 bytes)");
  const uintptr_t ptrs[] = {(uintptr_t)a->q, (uintptr_t)a->k_img, (uintptr_t)a->v_img,
                            (uintptr_t)a->k_txt, (uintptr_t)a->v_txt, (uintptr_t)a->out};
  for (uintptr_t q : ptrs)
    if (q % 16) return set_error(JENGA_E_INVALID, "wan_i2v_cross_attn: pointers must be 16-byte aligned");
  if (!(a->sm_scale > 0.f)) return set_error(JENGA_E_INVALID, "wan_i2v_cross_attn: sm_scale must be positive");
  if (a->q_rows > 0x7fffffffll || a->img_rows > 0x7fffffffll || a->txt_rows > 0x7fffffffll)
    return set_error(JENGA_E_UNSUPPORTED, "wan_i2v_cross_attn: more than 2^31 rows");
  const long long nq = (a->q_rows + kBlock - 1) / kBlock;
  const long long grid = static_cast<long long>(a->batch) * a->heads * nq;
  if (grid > 0x7fffffffll) return set_error(JENGA_E_UNSUPPORTED, "wan_i2v_cross_attn: grid too large");

  CUtensorMap tm_q, tm_ki, tm_vi, tm_kt, tm_vt;
  int rc;
  if ((rc = make_bf16_map(&tm_q, a->q, a->q_rows, a->heads, a->batch, a->q_stride_b, a->q_stride_s, a->q_stride_h)) ||
      (rc = make_bf16_map(&tm_ki, a->k_img, a->img_rows, a->heads, a->batch, a->ki_stride_b, a->ki_stride_s,
                          a->ki_stride_h)) ||
      (rc = make_bf16_map(&tm_vi, a->v_img, a->img_rows, a->heads, a->batch, a->vi_stride_b, a->vi_stride_s,
                          a->vi_stride_h)) ||
      (rc = make_bf16_map(&tm_kt, a->k_txt, a->txt_rows, a->heads, a->batch, a->kt_stride_b, a->kt_stride_s,
                          a->kt_stride_h)) ||
      (rc = make_bf16_map(&tm_vt, a->v_txt, a->txt_rows, a->heads, a->batch, a->vt_stride_b, a->vt_stride_s,
                          a->vt_stride_h)))
    return rc;

  CrossParams p{};
  p.heads = a->heads;
  p.nq = static_cast<int>(nq);
  p.n_img = static_cast<int>((a->img_rows + kBlock - 1) / kBlock);
  p.n_txt = static_cast<int>((a->txt_rows + kBlock - 1) / kBlock);
  p.q_rows = a->q_rows;
  p.img_rows = a->img_rows;
  p.txt_rows = a->txt_rows;
  p.qk_scale = static_cast<float>(static_cast<double>(a->sm_scale) * 1.44269504);   // as carved_attn.cu
  p.out = static_cast<uint16_t*>(a->out);
  p.o_stride_b = a->o_stride_b;
  p.o_stride_s = a->o_stride_s;
  p.o_stride_h = a->o_stride_h;
  p.err_flag = a->err_flag;

  cudaError_t ce = cudaFuncSetAttribute(wan_i2v_cross_attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        kSmemBytes);
  if (ce != cudaSuccess) return set_cuda_error(ce, "cudaFuncSetAttribute(wan_i2v_cross_attn)");
  wan_i2v_cross_attn_kernel<<<static_cast<unsigned>(grid), kThreads, kSmemBytes, stream>>>(tm_q, tm_ki, tm_vi, tm_kt,
                                                                                           tm_vt, p);
  ce = cudaGetLastError();
  if (ce != cudaSuccess) return set_cuda_error(ce, "wan_i2v_cross_attn launch");
  return JENGA_OK;
}

}  // namespace

}  // namespace jenga

extern "C" int jenga_wan_i2v_cross_attn(const JengaWanCrossArgs* args, void* stream) {
  return jenga::wan_i2v_cross_attn_impl(args, static_cast<cudaStream_t>(stream));
}
