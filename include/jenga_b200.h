/*
 * jenga_b200 — C ABI of the H100-native AttenCarve hot path.
 *
 * Drop-in boundary for the AttenCarve path of dvlab-research/Jenga:
 * gilbert token reordering, block scoring/selection and the 128x128 block-sparse
 * self-attention (RMSNorm + RoPE prologue), as hand-written sm_90a CUDA.
 *
 * Conventions (every entry point):
 *   - plain pointers and sizes only; device pointers unless the name says "host";
 *   - returns 0 on success, a negative JENGA_E_* code otherwise; never throws;
 *   - never allocates device memory (callers pass workspaces sized by the *_bytes queries);
 *   - never synchronises: work is enqueued on `stream` (a cudaStream_t passed as void*);
 *   - there is NO CPU fallback: without a CUDA device every compute call returns
 *     JENGA_E_CUDA.
 *
 * "ref:" comments cite the reference interface each entry point replaces
 * (paths relative to the Jenga repository root).
 */
#ifndef JENGA_B200_H_
#define JENGA_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* The version changes when an existing struct layout or signature changes; entry points that are only
 * added (the FP8 Linear ones below, jenga_wan_i2v_cross_attn, the INT8 _ex / _lse_shift ones) keep it,
 * so older callers stay valid. */
#define JENGA_B200_ABI_VERSION 3

enum {
  JENGA_OK = 0,
  JENGA_E_INVALID = -1,     /* bad argument (shape, stride, alignment, dtype)        */
  JENGA_E_UNSUPPORTED = -2, /* valid in the reference but not built here (e.g. D!=128) */
  JENGA_E_CUDA = -3,        /* CUDA runtime / driver error; see jenga_last_error()   */
  JENGA_E_WORKSPACE = -4    /* workspace too small                                   */
};

enum { JENGA_BF16 = 0, JENGA_F16 = 1, JENGA_F32 = 2 };

int jenga_abi_version(void);
/* Thread-local, human-readable description of the last non-zero return. */
const char* jenga_last_error(void);

/* ------------------------------------------------------------------------------------------
 * (a-1..a-3) gilbert curve permutations and block adjacency — host, once per resolution.
 * ref: gilbert.py:442 gilbert_mapping, :332 sliced_gilbert_mapping,
 *      :597 gilbert_block_neighbor_mapping, :679 sliced_gilbert_block_neighbor_mapping.
 * linear index = z*h*w + y*w + x over a (t,h,w) latent grid.  Outputs are host arrays of
 * t*h*w int64 (permutations) and nb*nb bytes (0/1), nb = ceil(t*h*w / block).
 * sliced != 0 selects the per-frame ("sliced") curve used by Wan2.1.
 * ---------------------------------------------------------------------------------------- */
int jenga_gilbert_mapping_host(int t, int h, int w, int sliced, int64_t* linear_to_hilbert,
                               int64_t* hilbert_to_linear);
int jenga_gilbert_block_neighbors_host(int t, int h, int w, int block, int sliced,
                                       uint8_t* neighbors /* [nb*nb] */);
/* Adjacency of the blocks of ANY voxel->curve-index table (e.g. a transposed curve,
 * gilbert.py:274 transpose_gilbert_mapping, which the sliced adjacency builder accepts at :704). */
int jenga_block_neighbors_from_mapping_host(int t, int h, int w, int block,
                                            const int64_t* linear_to_hilbert,
                                            uint8_t* neighbors /* [nb*nb] */);
/* The same adjacency as CSR (SURVEY §8 f-4): row_ptr[nb+1], col_idx[nnz] ascending per row.
 * Call with col_idx == NULL to size (nnz_out), then with capacity >= nnz. */
int jenga_gilbert_block_neighbors_csr_host(int t, int h, int w, int block, int sliced,
                                           int32_t* row_ptr, int32_t* col_idx,
                                           int64_t col_capacity, int64_t* nnz_out);
/* Scalar curve index of one voxel.  ref: gilbert.py:12 gilbert_xyz2d.  The table of the last
 * queried box is cached per thread, so a loop over a box costs one walk. */
int64_t jenga_gilbert_xyz2d(int x, int y, int z, int width, int height, int depth);

/* ------------------------------------------------------------------------------------------
 * (a-4) token gather / scatter along the curve.
 * ref: jenga_hyvideo.py:116-118,226; jenga_wan.py:559,655 (x[:, hilbert_order], x[:, l2h]).
 * dst[b, i, :] = src[b, index[i], :] for i < n_index; rows are `row_bytes` contiguous bytes
 * (multiple of 16), batch strides in bytes.  index is int64 on the device.
 * ---------------------------------------------------------------------------------------- */
int jenga_gather_rows(const void* src, void* dst, const int64_t* index, int64_t n_index,
                      int64_t n_src_rows, int64_t row_bytes, int batch, int64_t src_batch_stride,
                      int64_t dst_batch_stride, void* stream);

/* ------------------------------------------------------------------------------------------
 * (a-9, a-10) carved attention forward.
 * ref: hyvideo/modules/attention_block_triton_diffres.py:38-136 (kernel), :139-196 (launcher),
 *      :371-380 (text rows through flash_attn_func); wan/... and hyvideo_i2v/... twins.
 *
 * q,k,v,out are [B, S, H, D] with D contiguous (element strides given for b, s, h).
 * Query blocks of 128 rows come in two classes, both written to `out` by one launch:
 *   sparse  : q-blocks [0, nq_sparse)  — key blocks from `mask_bits` (ref one-hot kernel);
 *   dense   : q-blocks [nq_sparse, nq_sparse + nq_dense) — every key block (ref text rows).
 * mask_bits: [B*H, nq_sparse, mask_words] uint32, bit j of word w set <=> key block 32*w+j
 * is attended (ascending order, like the reference loop over the one-hot row).
 * ---------------------------------------------------------------------------------------- */
typedef struct JengaAttnArgs {
  const void* q;
  const void* k;
  const void* v;
  void* out;
  int32_t dtype; /* JENGA_BF16 | JENGA_F16 */
  int32_t batch, heads, head_dim;
  int64_t q_rows, kv_rows;                           /* S of q/out and of k/v            */
  int64_t q_stride_b, q_stride_s, q_stride_h;        /* element strides                 */
  int64_t k_stride_b, k_stride_s, k_stride_h;
  int64_t v_stride_b, v_stride_s, v_stride_h;
  int64_t o_stride_b, o_stride_s, o_stride_h;
  int32_t nq_sparse, nq_dense;
  const uint32_t* mask_bits;
  int32_t mask_words;
  /* sparse class (ref Triton kernel): Q is pre-scaled by sm_scale*log2(e) and re-rounded to
   * the input dtype (:87-88), text_amp is added in log2 units to key blocks >=
   * text_block_start (:113-114), key columns >= kv_limit_sparse are masked (:117-118),
   * query rows >= q_limit_sparse produce zeros (:136 + zeros_like :156). */
  float sm_scale;
  float text_amp;
  int32_t text_block_start;
  int64_t kv_limit_sparse;
  int64_t q_limit_sparse;
  /* dense class (ref flash_attn_func on the text rows): plain softmax(q k^T sm_scale) v over
   * key columns < kv_limit_dense. */
  int64_t kv_limit_dense;
  /* optional device int32: when non-NULL, *seqlen_dev replaces kv_limit_sparse and
   * q_limit_sparse at run time (ref :58 reads cu_seqlens_q[1] on the device, :328-329). */
  const int32_t* seqlen_dev;
  int32_t out_dtype; /* == dtype, or JENGA_F32 (wan variant returns the query dtype, :530-532) */
  int32_t* err_flag; /* device int, may be NULL: set non-zero by in-kernel watchdogs */
  /* Fused Ulysses epilogue (sp_world > 0; ref hyvideo/modules/xdit_ring_atten.py:206-219 does
   * the same data movement with two all-to-alls after the kernel).  q/k/v hold this rank's
   * `heads` heads over the FULL sequence (image rows of all ranks in rank order, then the dense
   * text rows).  out_peers_host[r] (HOST array of sp_world device pointers, peer-mapped) is the
   * base of rank r's result buffer [batch, sp_rows + T, sp_heads_total, D], T = q_rows -
   * sp_world*sp_rows (the dense text rows; 0 when q_rows is shorter); each output row is stored
   * directly into its owner's buffer (sample b's image row t -> rank t / sp_rows; its dense rows ->
   * every rank, sp_world == 1 included), in sample b's slab, at heads [sp_rank*heads,
   * (sp_rank+1)*heads).  Every
   * entry must be non-NULL and 16-byte aligned.  `out` is ignored and may be NULL.  The caller
   * synchronises the ranks before reading (jenga_b200.ulysses.UlyssesFusedAttention). */
  int32_t sp_world, sp_rank, sp_heads_total;
  int64_t sp_rows;
  const uint64_t* out_peers_host;
  /* ABI 2: global head index of this launch's head 0 in the owners' buffers; -1 (or the struct
   * zero-filled with sp_head_base_valid == 0) means sp_rank*heads.  Lets one rank's head group be
   * processed as several launches (head sub-groups pipelined against the inbound exchange); then
   * sp_heads_total is the true total and need not equal heads*sp_world. */
  int32_t sp_head_base, sp_head_base_valid;
  /* ABI 2, dense shims: optional fp32 [B, H, q_rows] log-sum-exp (natural log) of every DENSE
   * row, what flash_attn's _flash_attn_forward returns as softmax_lse
   * (ref hyvideo/modules/attenion.py:221-246).  NULL = not written. */
  float* lse_out;
  /* ABI 2, opt-in FP8 P.V variant (SURVEY §8 f-3): when v_fp8 != NULL the P.V product reads V from
   * this contiguous [B, kv_rows, H, 128] e4m3 tensor (made by jenga_quantize_v_fp8, whose per-(b,h)
   * absmax goes in v_fp8_amax [B*H] f32) and rounds P to e4m3; `v` is ignored.  bf16 q/k only.
   * Own tolerance row (tests/test_fp8_gpu.py); never selected implicitly. */
  const void* v_fp8;
  const float* v_fp8_amax;
} JengaAttnArgs;

int jenga_carved_attn_fwd(const JengaAttnArgs* args, void* stream);

/* One-hot bool mask [BH, nq, nb] (ref: the tensor returned by
 * _build_block_index_with_importance_optimized, attention_block_triton_diffres.py:198-295)
 * -> packed bit rows [BH, nq, mask_words]. */
int jenga_mask_onehot_to_bits(const uint8_t* onehot, uint32_t* bits, int64_t rows, int32_t nb,
                              int32_t mask_words, void* stream);

/* ------------------------------------------------------------------------------------------
 * (a-8) block scoring and selection.
 * ref: hyvideo/modules/attention_block_triton_diffres.py:198-295
 *      (_build_block_index_with_importance_optimized); wan twin :306-411 adds
 *      first_frame_blocks (:400-406).
 *
 * Step 1 — jenga_block_pool: pooled[b,h,blk,:] = mean of the block's 128 rows (ref :216-217),
 *   rounded to `out_dtype`.  x is [B,S,H,D] (element strides), rows >= S count as zeros
 *   (the Wan/I2V variants zero-pad first).  in_dtype JENGA_F32 means "Wan q/k": every element
 *   is rounded to bf16 before pooling (wan/...:456-463) and, if cast_out != NULL, the bf16
 *   copy is written contiguously as [B,S,H,D].
 * Step 2 — jenga_select_blocks: scores = round(round(qp kp^T) D^-1/2) over the first n_img
 *   key blocks (:227,:235), fp32 softmax (:238), descending sort with ties in index order,
 *   n = max(#(cumsum <= p)+1, top_k) (:241-250), first n blocks, OR neighbour rows
 *   (:280-289), OR first-frame square (wan), OR text columns (:292-293).  Output: packed bit
 *   rows [BH, nq, mask_words] for jenga_carved_attn_fwd; out_counts (optional) gets n.
 *   nbr_bits are packed rows of the bool [nbr_rows, >= n_img] adjacency matrix
 *   (use jenga_mask_onehot_to_bits once per curve).
 * ---------------------------------------------------------------------------------------- */
int jenga_block_pool(const void* x, void* pooled, void* cast_out, int32_t in_dtype,
                     int32_t out_dtype, int32_t batch, int32_t heads, int32_t head_dim,
                     int64_t rows, int64_t stride_b, int64_t stride_s, int64_t stride_h,
                     int32_t n_blocks, void* stream);

typedef struct JengaSelectArgs {
  const void* q_pool; /* [BH, nq, D]       */
  const void* k_pool; /* [BH, nk_pool, D]  */
  int32_t dtype;      /* JENGA_BF16 | JENGA_F16 */
  int32_t batch_heads, head_dim;
  int32_t nq;      /* image query blocks                         */
  int32_t nk_pool; /* rows per head in k_pool (>= n_img)         */
  int32_t n_img;   /* ranked key blocks == text_start_block      */
  int32_t nb;      /* all key blocks                             */
  int32_t mask_words;
  int32_t top_k;
  float p_threshold; /* ref prob_threshold / p_remain_rates      */
  int32_t text_blocks;
  int32_t first_frame_blocks;
  const uint32_t* nbr_bits;
  int32_t nbr_rows, nbr_words;
  uint32_t* out_bits;
  int32_t* out_counts;
  /* Optional score workspace (device): batch_heads*nq*n_img floats
   * (jenga_select_blocks_workspace_bytes).  With it, and n_img <= 1024, the call runs as a tiled
   * pooled-score GEMM + a one-warp-per-row selection kernel (same results, ~3x faster); without
   * it a single fused kernel is used. */
  void* workspace;
  int64_t workspace_bytes;
} JengaSelectArgs;

int jenga_select_blocks(const JengaSelectArgs* args, void* stream);
int64_t jenga_select_blocks_workspace_bytes(int32_t batch_heads, int32_t nq, int32_t n_img);

/* ------------------------------------------------------------------------------------------
 * (a-12) Ulysses inbound exchange as ONE kernel of peer stores (ref xdit_ring_atten.py:120-131
 * does it with four SeqAllToAll4D collectives + .contiguous() copies): this rank's image rows
 * x[w][i, :, :] (w = q,k,v; i < n_loc; all `heads` heads) are written into every rank p's
 * buffer at [w, rank*n_loc + i, 0:heads/world, :] <- heads [p*heads/world, (p+1)*heads/world),
 * and the replicated text rows joint[w] into the LOCAL buffer at rows [world*n_loc, +n_text).
 * peer_qkv_host[p] (HOST array) = peer-mapped base of rank p's [3, world*n_loc + n_text,
 * heads/world, head_dim] buffer; every entry non-NULL and 16-byte aligned.  Element size 2 bytes.
 * ---------------------------------------------------------------------------------------- */
typedef struct JengaUlyssesScatterArgs {
  const void* x[3];
  const void* joint[3]; /* may be NULL when n_text == 0 */
  int64_t x_stride_s, joint_stride_s; /* element stride between tokens ([n, H, D] views) */
  int32_t world, rank, heads, head_dim;
  int64_t n_loc, n_text;
  const uint64_t* peer_qkv_host;
  /* head-group form (ABI 2): move only the local heads [head_begin, head_begin+head_count) of
   * every destination rank's group; head_count == 0 moves all heads/world of them. */
  int32_t head_begin, head_count;
} JengaUlyssesScatterArgs;

int jenga_ulysses_scatter(const JengaUlyssesScatterArgs* args, void* stream);

/* Ragged head split: the same exchange when `world` need not divide `heads`.
 * head_offsets_host (HOST array of world+1 int32) gives rank p the global heads
 * [off[p], off[p+1]); offsets run monotone from 0 to `heads` and no group exceeds
 * slots = ceil(heads/world) (jenga_b200.ulysses.head_offsets: sizes heads/world + (p < heads%world)).
 * Every rank's receive buffer is [3, world*n_loc + n_text, slots, head_dim]; slot s of rank p holds
 * global head off[p] + s, for s < off[p+1]-off[p] only (the other slots are not written).
 * head_begin/head_count select a slot range (head_count == 0: all slots); each destination takes
 * its intersection with its own group, which may be empty.  Text rows copy the local heads
 * [off[rank] + s).  With off[p] = p*heads/world the bytes written equal jenga_ulysses_scatter's. */
int jenga_ulysses_scatter_ragged(const JengaUlyssesScatterArgs* args, const int32_t* head_offsets_host,
                                 void* stream);

/* Batched form of both exchanges, one launch for `batch` samples: sample b reads x[w] + b*x_stride_b
 * and joint[w] + b*joint_stride_b (element strides, multiples of 8), and every rank's receive buffer
 * is [3, batch, world*n_loc + n_text, slots, head_dim]: sample b of q/k/v w starts at slab w*batch + b.
 * head_offsets_host == NULL is the divisible split (jenga_ulysses_scatter's rules, slots =
 * heads/world), otherwise the ragged one (jenga_ulysses_scatter_ragged's).  batch is 1..65535.  At
 * batch 1 the bytes written equal those of the unbatched entry point, which is this call at batch 1. */
typedef struct JengaUlyssesScatterBatchArgs {
  JengaUlyssesScatterArgs base;
  int32_t batch;
  int64_t x_stride_b, joint_stride_b;
} JengaUlyssesScatterBatchArgs;

int jenga_ulysses_scatter_batched(const JengaUlyssesScatterBatchArgs* args, const int32_t* head_offsets_host,
                                  void* stream);

/* ------------------------------------------------------------------------------------------
 * Host <-> device staging for callers whose q/k/v live in (pinned) host memory: a strided 2-D
 * copy on `stream` (cudaMemcpy2DAsync), used to move one head group of a [B,S,H,D] tensor
 * (width = heads_in_group*D*elem bytes, height = B*S rows) so that transfers of group g+1
 * overlap the attention of group g.  direction: 0 = host->device, 1 = device->host.
 * ---------------------------------------------------------------------------------------- */
int jenga_copy2d_async(void* dst, int64_t dst_pitch, const void* src, int64_t src_pitch,
                       int64_t width_bytes, int64_t rows, int32_t direction, void* stream);

/* ------------------------------------------------------------------------------------------
 * (a-5, a-6, part of a-8) HunyuanVideo attention prologue: per-head RMSNorm(q,k), RoPE(q,k)
 * on the image tokens, img||txt concatenation and block mean-pooling in one pass.
 * ref: hyvideo/modules/models_mul_block_gc_ha_multigpu.py:200-241 (double stream),
 *      :417-435 (single stream); norm_layers.py:32-59; posemb_layers.py:133-137,181-229;
 *      pooling attention_block_triton_diffres.py:216-217.
 * img_qkv / txt_qkv are the fused QKV projections viewed as [B, tokens, 3, H, D] with element
 * strides (batch, token, which-of-qkv, head); D == 128 contiguous.  Norm weights are [D] in
 * `dtype` (all NULL == elementwise_affine=False).  rope_cos/rope_sin are fp32 [rows, D]
 * tables (interleaved-pair layout of get_nd_rotary_pos_embed); rope_index (optional, int64
 * [img_tokens]) gathers table rows per token (freqs_cos[hilbert_order], jenga_hyvideo.py:117).
 * Outputs q,k,v are contiguous [B, S, H, D], S = img_tokens + txt_tokens; q_pool / k_pool
 * (optional, together) are [B, H, ceil(S/128), D].
 * ---------------------------------------------------------------------------------------- */
typedef struct JengaHyPrologueArgs {
  const void* img_qkv;
  const void* txt_qkv; /* may be NULL when txt_tokens == 0 */
  int32_t dtype;
  int32_t batch, heads, head_dim;
  int64_t img_tokens, txt_tokens;
  int64_t img_stride_b, img_stride_s, img_stride_w, img_stride_h;
  int64_t txt_stride_b, txt_stride_s, txt_stride_w, txt_stride_h;
  const void* w_img_q;
  const void* w_img_k;
  const void* w_txt_q;
  const void* w_txt_k;
  float eps;
  const float* rope_cos;
  const float* rope_sin;
  const int64_t* rope_index;
  void* q;
  void* k;
  void* v;
  void* q_pool;
  void* k_pool;
} JengaHyPrologueArgs;

int jenga_hy_prologue(const JengaHyPrologueArgs* args, void* stream);

/* ------------------------------------------------------------------------------------------
 * (a-5, a-6, Wan variant) WanRMSNorm over the full channel dim + 3-axis complex RoPE.
 * ref: wan/modules/model_mul.py:74-90 (WanRMSNorm), :40-71 (rope_apply incl. freq_remap),
 *      :145-151 (qkv_fn).  x: [B, L, H*128] projection output (bf16 or f32, element strides);
 * w: [H*128] norm weight (bf16 or f32; NULL = ones).  freqs: the reference's complex128 table
 * viewed as doubles [freq_rows, 64, 2]; grid = (F, H, W) latent grid; freq_remap (optional int64
 * [F*H*W]) = hilbert_order.  out: [B, L, H, 128] bf16 = bf16(float(fp64 rotation)), i.e. what
 * block_sparse_attention sees after its own cast (wan/...triton_diffres.py:456-463).
 * ---------------------------------------------------------------------------------------- */
typedef struct JengaWanPrologueArgs {
  const void* x;
  const void* w;
  int32_t x_dtype, w_dtype;
  int32_t batch, heads, head_dim;
  int64_t tokens;
  int64_t stride_b, stride_s;
  float eps;
  const double* freqs;
  int32_t freq_rows;
  int32_t grid_f, grid_h, grid_w;
  const int64_t* freq_remap;
  void* out;
} JengaWanPrologueArgs;

int jenga_wan_prologue(const JengaWanPrologueArgs* args, void* stream);

/* ------------------------------------------------------------------------------------------
 * (a-13) step-skip residual cache and TeaCache gate as device ops.
 * ref: jenga_hyvideo.py:128-179 (`img += self.previous_residual`; `self.previous_residual =
 *      img - ori_img`), jenga_hyvideo_multigpu.py:225-280, jenga_wan.py:595-648.
 * residual_apply:  x[i] += residual[i]          (in place; fp32 add, one rounding to `dtype`)
 * residual_store:  residual[i] = x_new[i] - x_old[i]
 * n = element count; dtype bf16/f16 (16-byte aligned pointers) or f32.
 * ---------------------------------------------------------------------------------------- */
int jenga_residual_apply(void* x, const void* residual, int64_t n, int32_t dtype, void* stream);
int jenga_residual_store(const void* x_new, const void* x_old, void* residual, int64_t n,
                         int32_t dtype, void* stream);

/* TeaCache gate of ONE parity (conditional / unconditional forward), jenga_wan.py:597-626:
 *   if force:  calc = 1, accum = 0                (cnt < ret_steps, cnt >= cutoff_steps, stage start)
 *   else:      rel = mean|cur-prev| / mean|prev|  (fp32 quotient, like the reference's .item())
 *              accum += polyval(coeff, rel)       (coeff[0] = highest power, numpy.poly1d; float64)
 *              calc = accum >= thresh ; if calc: accum = 0
 *   prev <- cur when update_prev (the reference's `.clone()`).
 * cur/prev: n elements, dtype must be JENGA_F32 (the reference asserts fp32 embeddings).
 * state: double[1] on the device (accum).
 * flag: int32, device or mapped pinned host memory (written before the kernel ends).
 * rel_out: optional double[1] (diagnostics). */
typedef struct JengaTeaCacheArgs {
  const void* cur;
  void* prev;
  int32_t dtype;
  int64_t n;
  double coeff[8];
  int32_t n_coeff;
  double thresh;
  int32_t force;
  int32_t update_prev;
  double* state;
  int32_t* flag;
  double* rel_out;
} JengaTeaCacheArgs;
int jenga_teacache_gate(const JengaTeaCacheArgs* args, void* stream);

/* ------------------------------------------------------------------------------------------
 * (f-1, first slice) elementwise chains of the DiT blocks around the attention, one pass each.
 * ref: hyvideo/modules/models_mul_block_gc_ha_multigpu.py:196-199,295-315,409,499-500;
 *      modulate_layers.py:31-68; activation_layers.py ("gelu_tanh").  bf16 only; rows are
 *      `channels` contiguous elements, `*_stride` elements apart (multiples of 8).
 * ln_modulate:   out = bf16( layer_norm_fp32(x) * bf16(1 + scale) + shift )   — the chain the
 *                reference runs under torch.autocast(bf16) (no affine, eps as given)
 * gate_residual: out = bf16( x + bf16(y * gate) )
 * gelu_tanh:     out = bf16( gelu_tanh_fp32(x) ), strided source and destination (fills the
 *                concatenation buffer of the single-stream block in place)
 * ---------------------------------------------------------------------------------------- */
int jenga_ln_modulate(const void* x, int64_t x_stride, const void* scale, const void* shift, void* out,
                      int64_t out_stride, int64_t rows, int32_t channels, float eps, void* stream);
int jenga_gate_residual(const void* x, int64_t x_stride, const void* y, int64_t y_stride, const void* gate,
                        void* out, int64_t out_stride, int64_t rows, int32_t channels, void* stream);
int jenga_gelu_tanh(const void* x, int64_t x_stride, void* out, int64_t out_stride, int64_t rows,
                    int32_t channels, void* stream);

/* Token-replace forms of ln_modulate / gate_residual (HunyuanVideo-I2V, i2v_condition_type ==
 * "token_replace").  ref: hyvideo_i2v/modules/modulate_layers.py:51-56,84-95.  Row r uses
 * tr_scale / tr_shift (tr_gate) when row_is_tr[r] != 0 and scale / shift (gate) otherwise; the
 * per-row arithmetic is that of the plain entry points.  row_is_tr: `rows` bytes on the device
 * (a torch.bool mask as it is).  Same validation as the plain forms, plus non-null and 16-byte
 * aligned tr vectors and a non-null row_is_tr. */
int jenga_ln_modulate_tr(const void* x, int64_t x_stride, const void* scale, const void* shift,
                         const void* tr_scale, const void* tr_shift, const uint8_t* row_is_tr, void* out,
                         int64_t out_stride, int64_t rows, int32_t channels, float eps, void* stream);
int jenga_gate_residual_tr(const void* x, int64_t x_stride, const void* y, int64_t y_stride, const void* gate,
                           const void* tr_gate, const uint8_t* row_is_tr, void* out, int64_t out_stride,
                           int64_t rows, int32_t channels, void* stream);

/* ----------------------------------------------------------------------------------------
 * (f-1, opt-in) W8A8 FP8 Linear: e4m3 activations with one scale per row, e4m3 weights with one
 * scale per output channel or per tensor, fp32 accumulation promoted every 128 channels of K.
 *
 * jenga_quantize_rows_fp8: scale[m] = amax(|x[m, :]|) / 448 (1 for an all-zero row),
 *   out[m, k] = e4m3_rn_satfinite(x[m, k] / scale[m]).  x bf16 rows of `cols` elements, `x_stride`
 *   elements apart (multiple of 8); out rows `out_stride` bytes apart (multiple of 16); cols % 16 == 0
 *   (JENGA_E_UNSUPPORTED otherwise).  Also quantises bf16 nn.Linear weights per output channel.
 * jenga_ln_modulate_fp8 / jenga_ln_modulate_tr_fp8: jenga_ln_modulate / _tr followed by
 *   jenga_quantize_rows_fp8 of its bf16 rows, in one pass (bit-identical to the two calls); out8 rows
 *   `out_stride` bytes apart (multiple of 16), a_scale [rows] f32.  Same validation as the bf16 forms,
 *   plus channels % 16 == 0.
 * jenga_linear_fp8: out[m, n] = bf16( sum_k a[m, k] w[n, k] * a_scale[m] * w_scale[n * w_scale_stride]
 *   + bias[n] ).  a: e4m3 [m, k], rows `a_stride` bytes apart (multiple of 16); w: contiguous e4m3
 *   [n, k] (the nn.Linear layout); w_scale_stride 1 (per channel) or 0 (per tensor); bias bf16 or f32
 *   (bias_dtype) or NULL; out bf16 rows `out_stride` elements apart (multiple of 8).  k % 16 == 0 and
 *   n % 8 == 0, JENGA_E_UNSUPPORTED otherwise; any m.
 * ---------------------------------------------------------------------------------------- */
typedef struct JengaLinearFp8Args {
  const void* a;
  int64_t a_stride;       /* bytes */
  const float* a_scale;   /* [m] */
  const void* w;
  const float* w_scale;
  int32_t w_scale_stride; /* 1: [n] per output channel; 0: one value */
  const void* bias;       /* [n] or NULL */
  int32_t bias_dtype;     /* JENGA_BF16 or JENGA_F32 */
  void* out;
  int64_t out_stride;     /* elements */
  int64_t m;
  int32_t n;
  int32_t k;
} JengaLinearFp8Args;

int jenga_quantize_rows_fp8(const void* x, int64_t x_stride, int64_t rows, int32_t cols, void* out,
                            int64_t out_stride, float* scale, void* stream);
int jenga_ln_modulate_fp8(const void* x, int64_t x_stride, const void* scale, const void* shift, void* out8,
                          int64_t out_stride, float* a_scale, int64_t rows, int32_t channels, float eps,
                          void* stream);
int jenga_ln_modulate_tr_fp8(const void* x, int64_t x_stride, const void* scale, const void* shift,
                             const void* tr_scale, const void* tr_shift, const uint8_t* row_is_tr, void* out8,
                             int64_t out_stride, float* a_scale, int64_t rows, int32_t channels, float eps,
                             void* stream);
int jenga_linear_fp8(const JengaLinearFp8Args* args, void* stream);

/* Wan2.1 forms (wan/modules/model_mul.py:303-346 WanAttentionBlock.forward under
 * torch.autocast(bf16)).  The residual stream is fp32 after block 0; parameter vectors (scale, shift,
 * gate, weight, bias) are fp32 [channels]; x is bf16 or fp32 (x_dtype JENGA_BF16 / JENGA_F32), y is
 * bf16.  LN(v) = layer_norm(v) in fp32 without affine, rstd * (v - mean); every other step is one fp32
 * rounding; bf16(.) is round-to-nearest-even.  Rows are `channels` contiguous elements, strides in
 * elements (multiples of 8, >= channels), pointers 16-byte aligned, channels % 8 == 0 and <= 6144.
 * Outputs never alias inputs.
 * wan_ln_modulate:   n = LN(float(x)), rounded to bf16 when x is bf16 (WanLayerNorm's .type_as(x),
 *                    :98-103); out = bf16( n * (1 + scale) + shift )                  (norm1, :331-333)
 * wan_residual_ln:   r = x + y * gate (gate NULL: r = x + y), written to `res` as fp32; then
 *                    affine != 0: out = bf16( fma(vec_a, LN(r), vec_b) )  weight / bias of norm3, the
 *                                 form ATen's layer_norm kernel computes        (gate 1 + norm3, :334-339)
 *                    affine == 0: out = bf16( LN(r) * (1 + vec_a) + vec_b )  scale / shift
 *                                                                   (cross residual + norm2, :339-340)
 * wan_gate_residual: out = x + y * gate, fp32                                    (gate 2, :341-342)
 * The _fp8 forms feed the opt-in FP8 Linears (jenga_linear_fp8): each is the bf16 form followed by
 * jenga_quantize_rows_fp8 of its bf16 rows, in one pass and bit-identical to the two calls; the bf16
 * rows are never written.  out8 e4m3 rows `out_stride` BYTES apart (multiple of 16), a_scale [rows]
 * f32, channels % 16 == 0 (JENGA_E_UNSUPPORTED otherwise); `res` of wan_residual_ln_fp8 is written as
 * by wan_residual_ln.
 * wan_ln_modulate_fp8:   norm1 + modulate, the one input of the self-attention q / k / v
 * wan_residual_ln_fp8:   gate 1 + norm3 (affine, the cross-attention q) or cross residual + norm2 +
 *                        modulate (ffn.0)
 * gelu_tanh_fp8:         jenga_gelu_tanh of bf16 rows (ffn.0's output), quantised (the ffn.2 input);
 *                        x_stride in elements (multiple of 8), channels <= 16384 */
int jenga_wan_ln_modulate(const void* x, int32_t x_dtype, int64_t x_stride, const float* scale, const float* shift,
                          void* out, int64_t out_stride, int64_t rows, int32_t channels, float eps, void* stream);
int jenga_wan_residual_ln(const void* x, int32_t x_dtype, int64_t x_stride, const void* y, int64_t y_stride,
                          const float* gate, float* res, int64_t res_stride, const float* vec_a, const float* vec_b,
                          int32_t affine, void* out, int64_t out_stride, int64_t rows, int32_t channels, float eps,
                          void* stream);
int jenga_wan_gate_residual(const void* x, int32_t x_dtype, int64_t x_stride, const void* y, int64_t y_stride,
                            const float* gate, float* out, int64_t out_stride, int64_t rows, int32_t channels,
                            void* stream);
int jenga_wan_ln_modulate_fp8(const void* x, int32_t x_dtype, int64_t x_stride, const float* scale,
                              const float* shift, void* out8, int64_t out_stride, float* a_scale, int64_t rows,
                              int32_t channels, float eps, void* stream);
int jenga_wan_residual_ln_fp8(const void* x, int32_t x_dtype, int64_t x_stride, const void* y, int64_t y_stride,
                              const float* gate, float* res, int64_t res_stride, const float* vec_a,
                              const float* vec_b, int32_t affine, void* out8, int64_t out_stride, float* a_scale,
                              int64_t rows, int32_t channels, float eps, void* stream);
int jenga_gelu_tanh_fp8(const void* x, int64_t x_stride, void* out8, int64_t out_stride, float* a_scale,
                        int64_t rows, int32_t channels, void* stream);

/* Wan2.1-I2V cross-attention in one launch (wan/modules/model_mul.py:223-249 WanI2VCrossAttention.forward,
 * the part between the norms and self.o, under bf16 autocast):
 *   out[b,r,h,:] = bf16( f32(A_img) + f32(A_txt) ),  A_seg = bf16( softmax(q k_seg^T sm_scale) v_seg )
 * Each segment is normalised by its own softmax sum with the arithmetic of the dense class of
 * jenga_carved_attn_fwd, so A_img and A_txt are bit for bit what a dense launch over that segment alone
 * returns.  q / out are [B, q_rows, H, 128], k_img / v_img [B, img_rows, H, 128], k_txt / v_txt
 * [B, txt_rows, H, 128]; all bf16 with head_dim contiguous and element strides (b, s, h) that are
 * positive multiples of 8; pointers 16-byte aligned; img_rows, txt_rows >= 1.  Rows >= q_rows are not
 * stored. */
typedef struct JengaWanCrossArgs {
  const void* q;
  const void* k_img;
  const void* v_img;
  const void* k_txt;
  const void* v_txt;
  void* out;
  int32_t dtype; /* JENGA_BF16 */
  int32_t batch, heads, head_dim;
  int64_t q_rows, img_rows, txt_rows;
  int64_t q_stride_b, q_stride_s, q_stride_h;
  int64_t ki_stride_b, ki_stride_s, ki_stride_h;
  int64_t vi_stride_b, vi_stride_s, vi_stride_h;
  int64_t kt_stride_b, kt_stride_s, kt_stride_h;
  int64_t vt_stride_b, vt_stride_s, vt_stride_h;
  int64_t o_stride_b, o_stride_s, o_stride_h;
  float sm_scale;
  int32_t* err_flag; /* device int, may be NULL: set non-zero by in-kernel watchdogs */
} JengaWanCrossArgs;
int jenga_wan_i2v_cross_attn(const JengaWanCrossArgs* args, void* stream);

/* (f-2) ProRes stage switch in one kernel: out = trilinear_up(latents + noise_pred*d_sigma) *
 * (1 - sigma_next) + noise * sigma_next, fp32, NCDHW contiguous.
 * ref: pipeline_hunyuan_video_prores.py:721-731; scheduling_flow_match_discrete.py:258-299.
 * latents/noise_pred: [batch_channels, in_t, in_h, in_w]; noise/out: [batch_channels, out_t, out_h, out_w].
 * d_sigma = sigmas[-1] - sigmas[i]; sigma_next = sigmas[index_for_timestep(timesteps[i+1])]. */
int jenga_prores_switch(const float* latents, const float* noise_pred, const float* noise, float* out,
                        int32_t batch_channels, int32_t in_t, int32_t in_h, int32_t in_w,
                        int32_t out_t, int32_t out_h, int32_t out_w, float d_sigma, float sigma_next,
                        void* stream);

/* (f-4) the curve tables and the block adjacency generated ON THE DEVICE (one thread per voxel runs
 * the reference's per-voxel index query, gilbert.py:12-38,68-272); bit-identical to the host tables.
 * linear_to_hilbert / hilbert_to_linear: device int64 [t*h*w] (either may be NULL).
 * bits: device uint32 [nb, words] packed adjacency rows (zeroed by the call), nb = ceil(t*h*w/block),
 * the format jenga_select_blocks takes as nbr_bits. */
int jenga_gilbert_mapping_device(int t, int h, int w, int sliced, int64_t* linear_to_hilbert,
                                 int64_t* hilbert_to_linear, void* stream);
int jenga_block_neighbor_bits_device(int t, int h, int w, int block, const int64_t* linear_to_hilbert,
                                     uint32_t* bits, int32_t words, void* stream);

/* (f-3) per-head FP8 quantisation of V for the opt-in FP8 P.V variant: amax[b*H+h] = max |v[b,:,h,:]|,
 * out[b,s,h,d] = e4m3_rn_satfinite(v * 448 / amax).  v: [B, S, H, 128] with element strides, bf16 or f16;
 * out: contiguous [B, S, H, 128] bytes; amax: [B*H] f32 (zeroed by the call). */
int jenga_quantize_v_fp8(const void* v, int32_t dtype, int32_t batch, int64_t rows, int32_t heads,
                         int64_t stride_b, int64_t stride_s, int64_t stride_h, void* out_fp8, float* amax,
                         void* stream);

/* (f-3) INT8 operands for the opt-in INT8 Q.K^T variant.  x: [B, rows, H, 128] bf16/f16, element strides.
 * smooth != 0: mean[b*H+h][0..128) = fp32 mean of x over its `rows` rows (written; caller-allocated
 *              f32 [B*H*128]), subtracted before quantising.  smooth == 0: nothing subtracted.
 * Per (b, h) and per group of `group_rows` rows (64 or 128):
 *   scale = max|x - mean| / 127 ;  out = clamp(rint((x - mean) / scale), -127, 127)   (0 where scale == 0)
 * out: contiguous int8 [B, out_rows, H, 128], out_rows a multiple of 128 and >= round_up(rows, 128).
 * Rows in [rows, out_rows) hold the quantised value of (0 - mean): they stand for the zero padding
 * that dense rows attend.  scale: f32 [B*H, out_rows / group_rows].  With smooth != 0, `out` also
 * serves as scratch for the per-block partial sums of the mean (deterministic, no atomics). */
int jenga_quantize_int8(const void* x, int32_t dtype, int32_t batch, int64_t rows, int32_t heads,
                        int64_t stride_b, int64_t stride_s, int64_t stride_h, int32_t group_rows,
                        int32_t smooth, float* mean, int8_t* out, int64_t out_rows, float* scale, void* stream);
/* jenga_quantize_int8(q, group_rows 64, smooth 0) that also writes, for every row i of every (b, h), the
 * fp32 shift[(b*H + h) * out_rows + i] = Q'_i . k_mean[b*H + h], Q'_i = the row's codes times its group
 * scale (0 on the padding rows).  k_mean is the mean jenga_quantize_int8(k, 128, smooth 1) wrote, so K
 * is quantised first.  Each row's dot product is summed in a fixed order (8 channels per thread, then a
 * shuffle tree over 16 threads), so the shift is deterministic.  The codes and scales are bit for bit
 * those of jenga_quantize_int8.  shift: f32 [B*H, out_rows], 4-byte aligned. */
int jenga_quantize_q_int8_lse_shift(const void* q, int32_t dtype, int32_t batch, int64_t rows, int32_t heads,
                                    int64_t stride_b, int64_t stride_s, int64_t stride_h, const float* k_mean,
                                    int8_t* out, int64_t out_rows, float* scale, float* shift, void* stream);

/* (f-3) opt-in INT8 Q.K^T variant of jenga_carved_attn_fwd (SageAttention's recipe): Q.K^T runs as
 * s8 x s8 -> s32 on the tensor cores from per-block-scaled int8 Q (64-row groups) and K (128-key
 * blocks, K smoothed by its per-head mean, which leaves every softmax unchanged).  `args` means what
 * it means for jenga_carved_attn_fwd (the FP8 P.V variant included) except that Q.K^T reads these
 * operands.  Refused here: lse_out (smoothing shifts the LSE by q.mean) and the Ulysses epilogue
 * (sp_world > 0), both built by jenga_carved_attn_fwd_qk_int8_ex below; FP8 P.V with f16 is not built.
 * Lower precision than the default path; never implicit. */
typedef struct JengaQkInt8Args {
  const int8_t* q_i8;   const float* q_scale;   /* from jenga_quantize_int8(q, group_rows 64, smooth 0)  */
  const int8_t* k_i8;   const float* k_scale;   /* from jenga_quantize_int8(k, group_rows 128, smooth 1) */
  int64_t q_rows_padded, kv_rows_padded;        /* the out_rows used for each                           */
} JengaQkInt8Args;
int jenga_carved_attn_fwd_qk_int8(const JengaAttnArgs* args, const JengaQkInt8Args* qk, void* stream);

/* jenga_carved_attn_fwd (qk == NULL) or jenga_carved_attn_fwd_qk_int8 (qk != NULL), with the work
 * ordered first by a small pass on the same stream: every dense query block, then each head's sparse
 * blocks by live-tile count, longest first.  Blocks that run side by side then walk rows of nearly
 * equal length, in step, and share K/V tiles through L2.  Every row computes exactly what it computes
 * without the schedule: the results are the same bit for bit.  The pass writes the order into
 * `workspace` (device, 4-byte aligned, jenga_carved_attn_sched_workspace_bytes(batch, heads,
 * nq_sparse, nq_dense) = 4 * batch * heads * (nq_sparse + nq_dense) bytes), which must stay untouched
 * until the launch completes; concurrent launches need separate workspaces. */
typedef struct JengaAttnSched {
  void* workspace;
  int64_t workspace_bytes;
} JengaAttnSched;
int jenga_carved_attn_fwd_sched(const JengaAttnArgs* args, const JengaQkInt8Args* qk /* nullable */,
                                const JengaAttnSched* sched, void* stream);
int64_t jenga_carved_attn_sched_workspace_bytes(int32_t batch, int32_t heads, int32_t nq_sparse, int32_t nq_dense);

/* The INT8 Q.K^T variant with everything jenga_carved_attn_fwd_qk_int8 refuses to do, and the work
 * order of jenga_carved_attn_fwd_sched when `sched` is non-NULL.  Checks what those two check, and:
 *   - the Ulysses epilogue (sp_world > 0) is built;
 *   - lse_out is built when q_lse_shift is given (from jenga_quantize_q_int8_lse_shift over the same Q
 *     and the mean of the same K): the natural-log LSE of each dense row is that of the smoothed scores
 *     plus sm_scale * shift, i.e. of Q'.(K' + mean) with Q', K' the dequantised operands.  lse_out
 *     without q_lse_shift returns JENGA_E_UNSUPPORTED; q_lse_shift must be 4-byte aligned.
 * Without lse_out and sp_world the results are bit for bit those of jenga_carved_attn_fwd_sched (or
 * jenga_carved_attn_fwd_qk_int8 when sched is NULL) with the same operands. */
typedef struct JengaQkInt8ExArgs {
  JengaQkInt8Args base;       /* the four operands and padded row counts                 */
  const float* q_lse_shift;   /* [B*H, q_rows_padded] f32, or NULL when lse_out is NULL  */
} JengaQkInt8ExArgs;
int jenga_carved_attn_fwd_qk_int8_ex(const JengaAttnArgs* args, const JengaQkInt8ExArgs* qk,
                                     const JengaAttnSched* sched /* nullable */, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* JENGA_B200_H_ */
