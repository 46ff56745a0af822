// Parameters and mask walker of the carved-attention kernel (carved_attn.cu).
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
  // buffer over NVLink instead of `out`.  peer_out[r] = base of rank r's [sp_rows + dense rows,
  // sp_heads_total, D] buffer; this rank's heads are [sp_rank*heads, (sp_rank+1)*heads).
  int sp_world, sp_rank, sp_heads_total;
  int sp_head_base;           // global head index of local head 0 (default sp_rank*heads)
  long long sp_rows;          // image rows owned per rank
  unsigned long long peer_out[8];
  float* lse_out;             // optional [B, H, q_rows] natural-log LSE of the dense rows
  const float* v_fp8_amax;    // fp8 P.V variant: per (batch, head) absmax of V (scale = amax / 448)
  int* err_flag;
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


}  // namespace attn

}  // namespace jenga
