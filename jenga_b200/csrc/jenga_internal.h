// Internal glue shared by the translation units of libjenga_b200.so.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cstdint>

#include "jenga_b200.h"

namespace jenga {

// SMs of an H100 SXM: sizes the grids of the grid-stride (bandwidth-bound) kernels, whose results
// do not depend on it.
constexpr int kNumSMs = 132;

// Records a thread-local message and returns `code` (printf-style).
int set_error(int code, const char* fmt, ...);
int set_cuda_error(cudaError_t e, const char* what);

// cuTensorMapEncodeTiled resolved through cudaGetDriverEntryPoint (no link-time libcuda).
int encode_tensor_map(CUtensorMap* map, CUtensorMapDataType dt, uint32_t rank, void* base,
                      const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                      const cuuint32_t* box, const cuuint32_t* elem_strides,
                      CUtensorMapInterleave il, CUtensorMapSwizzle sw, CUtensorMapL2promotion l2,
                      CUtensorMapFloatOOBfill oob);

// qk != nullptr: the opt-in INT8 Q.K^T variant (jenga_carved_attn_fwd_qk_int8)
// sched != nullptr: order the work first (jenga_carved_attn_fwd_sched)
// qk_ex: called by jenga_carved_attn_fwd_qk_int8_ex, which also builds the Ulysses epilogue and, given
// q_lse_shift, lse_out with INT8 Q.K^T
int carved_attn_fwd_impl(const JengaAttnArgs* a, cudaStream_t stream, const JengaQkInt8Args* qk = nullptr,
                         const JengaAttnSched* sched = nullptr, bool qk_ex = false,
                         const float* q_lse_shift = nullptr);
int64_t carved_attn_sched_workspace_bytes(long long batch, long long heads, long long nq_sparse, long long nq_dense);
int block_pool_impl(const void* x, void* pooled, void* cast_out, int in_dtype, int out_dtype,
                    int batch, int heads, int head_dim, long long rows, long long sb, long long ss,
                    long long sh, int n_blocks, cudaStream_t stream);
int select_blocks_impl(const JengaSelectArgs* a, cudaStream_t stream);
int hy_prologue_impl(const JengaHyPrologueArgs* a, cudaStream_t stream);
int hy_prologue_bulk_try(const JengaHyPrologueArgs* a, cudaStream_t stream);  // > 0: not applicable
int wan_prologue_impl(const JengaWanPrologueArgs* a, cudaStream_t stream);

}  // namespace jenga
