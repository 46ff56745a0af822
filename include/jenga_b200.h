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

#define JENGA_B200_ABI_VERSION 2

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
   * base of rank r's result buffer [sp_rows + dense rows, sp_heads_total, D]; each output row is
   * stored directly into its owner's buffer (image row t -> rank t / sp_rows; dense rows ->
   * every rank), at heads [sp_rank*heads, (sp_rank+1)*heads).  `out` is ignored.  The caller
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
 * heads/world, head_dim] buffer.  Element size 2 bytes.
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
  /* optional, used by the experimental vector kernel only (JENGA_WAN_PROLOGUE=vector; the default kernel
   * rotates in fp64 like the reference): the same table split into fp32 pairs,
   * [freq_rows, 64, 4] = (re_hi, im_hi, re_lo, im_lo) with hi = (float)x, lo = (float)(x - hi).  The
   * rotation then runs on the FP32 pipe with compensated products and sums (error ~2^-45 relative, i.e.
   * the correctly rounded fp32 of the complex128 product except ~1e-6 of the elements by one fp32 ulp,
   * invisible after the bf16 cast). */
  const float* freqs_hilo;
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

#ifdef __cplusplus
}
#endif
#endif /* JENGA_B200_H_ */
