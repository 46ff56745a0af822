// Carved (block-sparse) flash-attention forward for sm_90a.
//
// Replaces the reference's Triton one-hot kernel
//   hyvideo/modules/attention_block_triton_diffres.py:38-136 (+ launcher :139-196)
// and its text-row flash_attn_func call (:371-380) with ONE launch.
//
// Work decomposition: one CTA per (batch*head, 128-row query block), running the pipeline of
// carved_attn_common.cuh over the live key blocks of its row; final O / l -> global.  With FP8 P.V,
// producer warps 9..11 also transpose each V tile (see kPvFp8), so setmaxnreg leaves the producer 40
// registers instead of 24 and gives the consumers 232 instead of 240.  Keeping Q~ in registers takes a
// third of the shared-memory reads off Q.K^T: only K is read per tile.  One CTA per SM, ~164 KB of
// shared memory.
//
// HBM/L2 layout: q,k,v stay in the caller's [B,S,H,D] layout; TMA boxes are {64 d, 128 rows}
// with 128-byte swizzle.  K boxes are K-major wgmma operands, V boxes MN-major (no transpose).
// CTAs are numbered head-major so that all CTAs in flight read the same head's K/V out of L2.
// With a schedule (jenga_carved_attn_fwd_sched) a small pass first orders the work: every dense
// block first (the longest), then each head's sparse blocks by live-tile count, longest first.  The
// CTAs that run side by side then walk rows of nearly equal length, finish together and start the
// next rows together, so they sweep the keys in step and share each K/V tile through L2.
#include <cfloat>

#include "carved_attn_common.cuh"

namespace jenga {

namespace {

using namespace attn;

constexpr int kTransposeWarps = 3;               // producer warps 9..11 (FP8 P.V only)
constexpr int kMaxMaskWords = 256;               // up to 8192 key blocks (1M tokens)
constexpr int kSmemBytes = 1024 /*align slack*/ + kOffEnd + kMaxMaskWords * 4;   // + the row mask

// kPvFp8 (opt-in): P and V enter the P.V product as FP8 e4m3 — V quantised per head by
// jenga_quantize_v_fp8 (scale = absmax/448), P converted with cvt.rn.satfinite.e4m3x2 (p <= 2^8 by
// the lazy-rescale bound, e4m3 max 448) — through wgmma m64n128k32 e4m3 (half the P.V tensor cycles).
// 8-bit wgmma operands must be K-major, so three producer warps transpose each V tile in shared
// memory into V^T (the upper half of the V slot) with the keys of every 32-key group permuted to
// match the order in which the S accumulator fragment already holds P: no shuffles of P.  The
// consumers wait for V^T on VT_FULL instead of V_FULL and otherwise run the same schedule.
// Q.K^T, the softmax and l are unchanged.
//
// kQkInt8 (opt-in, SageAttention's recipe): Q and K enter Q.K^T as int8 made by jenga_quantize_int8 —
// Q per 64-row group (one scale per consumer warpgroup), K per 128-key block after subtracting its
// per-head channel mean (a constant per score row: every softmax is unchanged) — through wgmma
// m64n128k32 s8 x s8 -> s32 (half the Q.K^T tensor cycles).  Q and K tiles are one 16 KB box each;
// Q stays in shared memory (the s32 accumulator already takes the registers Q would need).
// The s32 scores become fp32 exactly (|S| < 2^22) and both classes scale them inside the exponent by
// c = q_scale * k_scale[blk] * qk_scale, so the sparse class skips its Q~ pre-scaling.  text_amp,
// the masks, the lazy rescale and P.V (bf16/f16, or e4m3 with kPvFp8) are unchanged.
template <bool kBF16, bool kPvFp8 = false, bool kQkInt8 = false>
__global__ void __launch_bounds__(kThreads, 1)
carved_attn_fwd_kernel(const __grid_constant__ CUtensorMap tm_q,
                       const __grid_constant__ CUtensorMap tm_k,
                       const __grid_constant__ CUtensorMap tm_v, const KernelParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw_addr + 1023u) & ~1023u) - raw_addr);
  uint8_t* sV = smem + kOffV;  // + stage * kTileBytes
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + kOffBars);
  uint32_t* s_mask = reinterpret_cast<uint32_t*>(smem + kOffEnd);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  // ---- which tile is this CTA?  Items are numbered head-major, within a head the dense blocks
  // first; p.order (when given) says which item each CTA runs ----
  const int item = p.order ? __ldg(p.order + blockIdx.x) : static_cast<int>(blockIdx.x);
  const int per_bh = p.nq_sparse + p.nq_dense;
  const int bh = item / per_bh;
  const int local = item - bh * per_bh;
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
    for (int i = 0; i < NUM_BARS; ++i)
      mbar_init(&bars[i], i >= VT_FULL ? kTransposeWarps : (i >= K_EMPTY ? 8u : 1u));
    fence_mbar_init();
  }
  __syncthreads();

  int n_tiles = 0;
  for (int w = 0; w < nwords; ++w) n_tiles += __popc(s_mask[w]);

  if (warp >= kConsumerThreads / 32) {
    // =============================== producer warpgroup ===============================
    setmaxnreg_dec<kPvFp8 ? 40 : 24>();
    if (warp == kConsumerThreads / 32) {
      if (n_tiles > 0 && lane == 0) {   // TMA: the live key blocks in mask order
        BlockWalker it(s_mask, nwords);
        produce<kPvFp8, kQkInt8>(smem, bars, p.err_flag, &tm_q, static_cast<int>(q_row0), h, b,
                                 [&](int, KvMaps& m) {
                                   m = {&tm_k, &tm_v};
                                   return it.next() * kBlock;   // < 0 past the last live block
                                 });
      }
    } else if constexpr (kPvFp8) {
      // V^T[d][32 g + L] = V[32 g + perm(L)][d], perm(4 t + u) = {2t, 2t+1, 2t+8, 2t+9}[u] (+16 for
      // t >= 4): the k-order of the e4m3 A fragment (4 consecutive k per byte quad) read off the
      // f32 accumulator fragment (pairs of adjacent columns, 8 apart).  V^T is written into the
      // unused upper half of the slot, which the consumers free together with V (V_EMPTY).
      const int t0 = threadIdx.x - kConsumerThreads - 32;
      for (int j = 0; j < n_tiles; ++j) {
        const int s = j % kStages;
        mbar_wait(&bars[V_FULL + s], (j / kStages) & 1, p.err_flag);
        const uint8_t* vs = sV + s * kTileBytes;
        uint8_t* vt = sV + s * kTileBytes + kBoxBytes;
        for (int u = t0; u < kBlock * kHeadDim / 16; u += kTransposeWarps * 32) {
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
        fence_proxy_async_smem();  // generic-proxy writes -> visible to the tensor core proxy
        __syncwarp();
        if (lane == 0) mbar_arrive(&bars[VT_FULL + s]);
      }
    }
    return;
  }

  // =============================== consumers ===============================
  setmaxnreg_inc<kPvFp8 ? 232 : 240>();
  Consumer<kBF16, kPvFp8, kQkInt8> cons(smem, bars, p.err_flag);
  // sparse class: Q~ = round(Q * qk_scale) and raw S is already in log2 units (c = 1)
  // dense class : raw S, scaled inside the exponent (c = qk_scale), like FlashAttention
  // kQkInt8     : integer S, scaled inside the exponent by c = q_scale * k_scale[blk] * qk_scale
  const float c = dense ? p.qk_scale : 1.0f;
  const float qs = kQkInt8 && n_tiles > 0 ? __ldg(p.q_scale + bh * p.q_groups + 2 * qb + cons.wg) * p.qk_scale : 0.f;

  if (n_tiles > 0) {
    cons.load_q();
    if constexpr (!kQkInt8) {
      if (!dense) {   // ref :87-88  q = (q * qk_scale).to(dtype)
#pragma unroll
        for (int kk = 0; kk < kHeadDim / 16; ++kk)
#pragma unroll
          for (int t = 0; t < 4; ++t) {
            const float2 f = unpack2<kBF16>(cons.qa[kk][t]);
            cons.qa[kk][t] = pack2<kBF16>(f.x * p.qk_scale, f.y * p.qk_scale);
          }
      }
    }
    BlockWalker it(s_mask, nwords);
    cons.run(
        n_tiles,
        [&](int, Tile& t) {
          const int blk = it.next();
          // exponent factor: kQkInt8's is never 0, which would turn the -inf of masked columns into
          // NaN.  ref :113-114 — text_amp is a constant added to every score of a text key block, in
          // log2 units (sparse class only, where c == 1)
          t = {static_cast<long long>(blk) * kBlock, kv_limit,
               kQkInt8 ? fmaxf(qs * __ldg(p.k_scale + bh * p.k_groups + blk), FLT_MIN) : c,
               (!dense && blk >= p.text_block_start) ? p.text_amp : 0.f, false};
        },
        [](const float (&)[2]) {});   // one segment
  }

  // ---- epilogue: O / l -> global (ref :135-136); rows past the limit are zeros (:156) ----
#pragma unroll
  for (int r = 0; r < 2; ++r) cons.l_sum[r] = row_sum(cons.l_sum[r]);
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const long long q_row = q_row0 + cons.row_lo + 8 * r;
    const bool in_tensor = q_row < p.q_rows;
    const bool zero_row = (n_tiles == 0) || (!dense && q_row >= q_limit_sparse);
    float inv_l = zero_row ? 0.f : 1.0f / cons.l_sum[r];
    if constexpr (kPvFp8) inv_l *= __ldg(p.v_fp8_amax + b * p.heads + h) * (1.0f / 448.0f);   // undo the V scale
    if (p.lse_out && dense && in_tensor && cons.qd == 0) {
      // softmax_lse of flash_attn (natural log): ln sum_j exp(s_j * sm_scale) = (m + log2 l) * ln 2.
      // kQkInt8 scored Q'.(K - mean): every score of the row is short by sm_scale * c_i, in log2
      // units qk_scale * c_i
      float lse2 = cons.m_used[r] + log2f(cons.l_sum[r]);
      if constexpr (kQkInt8) lse2 += p.qk_scale * __ldg(p.q_lse_shift + bh * p.q_groups * 64 + q_row);
      p.lse_out[(static_cast<long long>(b) * p.heads + h) * p.q_rows + q_row] =
          zero_row ? -INFINITY : lse2 * 0.6931471805599453f;
    }
    if (!in_tensor) continue;
    // destination(s) of this row
    long long o_off = b * p.o_stride_b + q_row * p.o_stride_s + static_cast<long long>(h) * p.o_stride_h;
    uint16_t* obase = reinterpret_cast<uint16_t*>(p.out);
    int n_dst = 1;  // > 1 only for replicated (text) rows under Ulysses
    if (p.sp_world > 0) {
      // Fused Ulysses exchange (ref xdit_ring_atten.py:206-219 does this with two all-to-alls
      // after the kernel): image row t belongs to rank t / sp_rows; text rows go to every rank.
      // Every owner's buffer is [batch, sp_rows + T, sp_heads_total, D]: sample b's rows sit in slab b.
      const long long n_img = p.sp_rows * p.sp_world;
      const long long slab_rows = p.sp_rows + (p.q_rows > n_img ? p.q_rows - n_img : 0);
      const int gh = p.sp_head_base + h;
      if (q_row < n_img) {
        const int owner = static_cast<int>(q_row / p.sp_rows);
        obase = reinterpret_cast<uint16_t*>(p.peer_out[owner]);
        o_off = ((b * slab_rows + q_row - owner * p.sp_rows) * p.sp_heads_total + gh) * kHeadDim;
      } else {
        // every rank's buffer; with one rank that is peer_out[0] through the single-store path
        obase = reinterpret_cast<uint16_t*>(p.peer_out[0]);
        n_dst = p.sp_world;
        o_off = ((b * slab_rows + p.sp_rows + (q_row - n_img)) * p.sp_heads_total + gh) * kHeadDim;
      }
    }
#pragma unroll
    for (int n8 = 0; n8 < 16; ++n8) {
      const int i = 4 * n8 + 2 * r;
      const int col = 8 * n8 + 2 * cons.qd;
      const uint32_t v = pack2<kBF16>(zero_row ? 0.f : cons.o[i] * inv_l, zero_row ? 0.f : cons.o[i + 1] * inv_l);
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

// live tiles of sparse row r of head bh: what the attention kernel's mask staging keeps
__device__ int sparse_row_tiles(const KernelParams& p, int bh, int r, long long q_limit) {
  if (static_cast<long long>(r) * kBlock >= q_limit) return 0;
  const uint32_t* m = p.mask_bits + (static_cast<size_t>(bh) * p.nq_sparse + r) * p.mask_words;
  int n = 0;
  for (int w = 0; w < p.mask_words; ++w) {
    uint32_t bits = __ldg(m + w);
    const int rem = p.nb_kv - w * 32;
    if (rem < 32) bits &= rem > 0 ? ((1u << rem) - 1u) : 0u;
    n += __popc(bits);
  }
  return n;
}

constexpr int kOrderThreads = 256;

// One CTA per batch*head.  order[0, B*H*nq_dense) = the dense items (head-major); then, head after
// head, the head's sparse items by live-tile count, longest first, ties in row order (a stable
// counting sort: the schedule is deterministic).  Items are numbered as the attention kernel decodes
// them.  Dynamic shared memory: (nb_kv + 1 + kOrderThreads) ints.
__global__ void __launch_bounds__(kOrderThreads) carved_attn_order_kernel(const KernelParams p, int* order) {
  extern __shared__ int s_order[];
  int* start = s_order;                   // [nb_kv + 1]: count histogram, then first slot per count
  int* chunk = s_order + p.nb_kv + 1;     // [kOrderThreads]: counts of the current chunk of rows
  const int bh = blockIdx.x;
  const int per_bh = p.nq_sparse + p.nq_dense;
  for (int i = threadIdx.x; i < p.nq_dense; i += kOrderThreads) order[bh * p.nq_dense + i] = bh * per_bh + i;
  if (p.nq_sparse == 0) return;
  const long long seqlen_over = p.seqlen_dev ? static_cast<long long>(__ldg(p.seqlen_dev)) : -1;
  const long long q_limit = seqlen_over >= 0 ? seqlen_over : p.q_limit_sparse;
  for (int c = threadIdx.x; c <= p.nb_kv; c += kOrderThreads) start[c] = 0;
  __syncthreads();
  for (int r = threadIdx.x; r < p.nq_sparse; r += kOrderThreads) atomicAdd(&start[sparse_row_tiles(p, bh, r, q_limit)], 1);
  __syncthreads();
  if (threadIdx.x == 0) {   // descending exclusive scan; O(nb_kv) against the kernel's O(nq * nb_kv)
    int run = 0;
    for (int c = p.nb_kv; c >= 0; --c) {
      const int t = start[c];
      start[c] = run;
      run += t;
    }
  }
  __syncthreads();
  int* dst = order + static_cast<size_t>(gridDim.x) * p.nq_dense + static_cast<size_t>(bh) * p.nq_sparse;
  for (int base = 0; base < p.nq_sparse; base += kOrderThreads) {
    const int r = base + threadIdx.x;
    const int c = r < p.nq_sparse ? sparse_row_tiles(p, bh, r, q_limit) : -1;
    chunk[threadIdx.x] = c;
    __syncthreads();
    if (c >= 0) {
      int rank = 0;   // rows of this chunk before r with the same count
      for (int t = 0; t < static_cast<int>(threadIdx.x); ++t) rank += chunk[t] == c;
      dst[start[c] + rank] = bh * per_bh + p.nq_dense + r;
    }
    __syncthreads();
    if (c >= 0) atomicAdd(&start[c], 1);
    __syncthreads();
  }
}

}  // namespace

// ------------------------------------------------------------------------------------------
// Host side
// ------------------------------------------------------------------------------------------
// one-byte operands (FP8 V, int8 Q / K): contiguous [B, S, H, 128] bytes; box {128 channels, 128 rows}
static int make_bytes_map(CUtensorMap* map, const void* base, long long rows, int heads, int batch) {
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

int64_t carved_attn_sched_workspace_bytes(long long batch, long long heads, long long nq_sparse, long long nq_dense) {
  if (batch <= 0 || heads <= 0 || nq_sparse < 0 || nq_dense < 0) return 0;
  return batch * heads * (nq_sparse + nq_dense) * static_cast<int64_t>(sizeof(int));
}

int carved_attn_fwd_impl(const JengaAttnArgs* a, cudaStream_t stream, const JengaQkInt8Args* qk,
                         const JengaAttnSched* sched, bool qk_ex, const float* q_lse_shift) {
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
  if (qk) {
    if (!qk->q_i8 || !qk->q_scale || !qk->k_i8 || !qk->k_scale)
      return set_error(JENGA_E_INVALID, "qk_int8: null int8 operand or scale pointer");
    // jenga_carved_attn_fwd_qk_int8 / _sched refuse both; jenga_carved_attn_fwd_qk_int8_ex (qk_ex) builds
    // the Ulysses epilogue, and the LSE when it is given the per-row shift that undoes K smoothing
    if (a->lse_out && (!qk_ex || !q_lse_shift))
      return set_error(JENGA_E_UNSUPPORTED, "qk_int8: lse_out needs q_lse_shift (K smoothing shifts the LSE by q.mean)");
    if (a->sp_world > 0 && !qk_ex)
      return set_error(JENGA_E_UNSUPPORTED, "qk_int8: the Ulysses epilogue is built only in jenga_carved_attn_fwd_qk_int8_ex");
    const long long q_need = (a->q_rows + kBlock - 1) / kBlock * kBlock;
    const long long kv_need = (a->kv_rows + kBlock - 1) / kBlock * kBlock;
    if (qk->q_rows_padded < q_need || qk->kv_rows_padded < kv_need || qk->q_rows_padded % kBlock ||
        qk->kv_rows_padded % kBlock)
      return set_error(JENGA_E_INVALID, "qk_int8: padded rows (%lld, %lld) must be multiples of 128 >= (%lld, %lld)",
                       static_cast<long long>(qk->q_rows_padded), static_cast<long long>(qk->kv_rows_padded),
                       q_need, kv_need);
    if (reinterpret_cast<uintptr_t>(qk->q_i8) % 16 || reinterpret_cast<uintptr_t>(qk->k_i8) % 16 ||
        reinterpret_cast<uintptr_t>(qk->q_scale) % 4 || reinterpret_cast<uintptr_t>(qk->k_scale) % 4 ||
        reinterpret_cast<uintptr_t>(q_lse_shift) % 4)
      return set_error(JENGA_E_INVALID, "qk_int8: int8 operands must be 16-byte and scales 4-byte aligned");
  }
  if (a->sp_world != 0 &&
      (a->sp_world < 0 || a->sp_world > 8 || a->sp_rank < 0 || a->sp_rank >= a->sp_world || !a->out_peers_host ||
       a->sp_rows <= 0 || a->out_dtype != a->dtype))
    return set_error(JENGA_E_INVALID, "bad Ulysses epilogue arguments");
  const int sp_head_base = a->sp_head_base_valid ? a->sp_head_base : a->sp_rank * a->heads;
  if (a->sp_world != 0 &&
      ((!a->sp_head_base_valid && a->sp_heads_total != a->heads * a->sp_world) || sp_head_base < 0 ||
       sp_head_base + a->heads > a->sp_heads_total))
    return set_error(JENGA_E_INVALID, "bad Ulysses head range");
  for (int r = 0; r < a->sp_world; ++r)
    if (!a->out_peers_host[r] || a->out_peers_host[r] % 16)
      return set_error(JENGA_E_INVALID, "Ulysses out_peers_host[%d] is null or not 16-byte aligned", r);

  const bool pv_fp8 = a->v_fp8 != nullptr;
  if (pv_fp8) {
    if (!a->v_fp8_amax || a->dtype != JENGA_BF16)
      return set_error(JENGA_E_UNSUPPORTED, "fp8 P.V: needs v_fp8_amax and bf16 q/k");
    if (reinterpret_cast<uintptr_t>(a->v_fp8) % 16) return set_error(JENGA_E_INVALID, "v_fp8 must be 16-byte aligned");
  }
  const long long grid = static_cast<long long>(a->batch) * a->heads * (a->nq_sparse + a->nq_dense);
  if (grid > 0x7fffffffll) return set_error(JENGA_E_UNSUPPORTED, "grid too large");
  if (sched) {
    const int64_t need = carved_attn_sched_workspace_bytes(a->batch, a->heads, a->nq_sparse, a->nq_dense);
    if (!sched->workspace) return set_error(JENGA_E_INVALID, "sched: null workspace");
    if (reinterpret_cast<uintptr_t>(sched->workspace) % alignof(int))
      return set_error(JENGA_E_INVALID, "sched: workspace must be 4-byte aligned");
    if (sched->workspace_bytes < need)
      return set_error(JENGA_E_WORKSPACE, "sched: workspace %lld < %lld bytes",
                       static_cast<long long>(sched->workspace_bytes), static_cast<long long>(need));
  }
  CUtensorMap tm_q, tm_k, tm_v;
  int rc;
  if (qk) {
    if ((rc = make_bytes_map(&tm_q, qk->q_i8, qk->q_rows_padded, a->heads, a->batch))) return rc;
    if ((rc = make_bytes_map(&tm_k, qk->k_i8, qk->kv_rows_padded, a->heads, a->batch))) return rc;
  } else {
    if ((rc = make_tile_map(&tm_q, a->q, a->dtype, a->q_rows, a->heads, a->batch, a->q_stride_b,
                            a->q_stride_s, a->q_stride_h)))
      return rc;
    if ((rc = make_tile_map(&tm_k, a->k, a->dtype, a->kv_rows, a->heads, a->batch, a->k_stride_b,
                            a->k_stride_s, a->k_stride_h)))
      return rc;
  }
  if (pv_fp8) {
    if ((rc = make_bytes_map(&tm_v, a->v_fp8, a->kv_rows, a->heads, a->batch))) return rc;
  } else if ((rc = make_tile_map(&tm_v, a->v, a->dtype, a->kv_rows, a->heads, a->batch, a->v_stride_b,
                                 a->v_stride_s, a->v_stride_h)))
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
  if (qk) {
    p.q_scale = qk->q_scale;
    p.k_scale = qk->k_scale;
    p.q_groups = qk->q_rows_padded / 64;
    p.k_groups = qk->kv_rows_padded / kBlock;
    p.q_lse_shift = q_lse_shift;
  }

  cudaError_t ce;
  if (sched) {
    p.order = static_cast<const int*>(sched->workspace);
    const int bhs = a->batch * a->heads;
    carved_attn_order_kernel<<<bhs, kOrderThreads, (p.nb_kv + 1 + kOrderThreads) * sizeof(int), stream>>>(
        p, static_cast<int*>(sched->workspace));
    ce = cudaGetLastError();
    if (ce != cudaSuccess) return set_cuda_error(ce, "carved_attn order launch");
  }
  const bool bf16 = a->dtype == JENGA_BF16;
  auto kern = qk ? (pv_fp8 ? carved_attn_fwd_kernel<true, true, true>
                           : (bf16 ? carved_attn_fwd_kernel<true, false, true> : carved_attn_fwd_kernel<false, false, true>))
                 : (pv_fp8 ? carved_attn_fwd_kernel<true, true>
                           : (bf16 ? carved_attn_fwd_kernel<true> : carved_attn_fwd_kernel<false>));
  ce = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmemBytes);
  if (ce != cudaSuccess) return set_cuda_error(ce, "cudaFuncSetAttribute(carved_attn)");
  kern<<<static_cast<unsigned>(grid), kThreads, kSmemBytes, stream>>>(tm_q, tm_k, tm_v, p);
  ce = cudaGetLastError();
  if (ce != cudaSuccess) return set_cuda_error(ce, "carved_attn launch");
  return JENGA_OK;
}

}  // namespace jenga
