// extern "C" surface of libjenga_b200.so (declared in include/jenga_b200.h) plus the small
// bandwidth-bound kernels that do not deserve their own translation unit.
#include <cstdarg>
#include <cstdio>
#include <cstring>

#include "jenga_internal.h"

namespace jenga {

static thread_local char g_err[512] = "";

int set_error(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}
int set_cuda_error(cudaError_t e, const char* what) {
  snprintf(g_err, sizeof(g_err), "%s: %s (%s)", what, cudaGetErrorName(e), cudaGetErrorString(e));
  return JENGA_E_CUDA;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn resolve_encode() {
  static EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) !=
            cudaSuccess ||
        qres != cudaDriverEntryPointSuccess)
      p = nullptr;
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  return fn;
}

int encode_tensor_map(CUtensorMap* map, CUtensorMapDataType dt, uint32_t rank, void* base,
                      const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                      const cuuint32_t* box, const cuuint32_t* elem_strides,
                      CUtensorMapInterleave il, CUtensorMapSwizzle sw, CUtensorMapL2promotion l2,
                      CUtensorMapFloatOOBfill oob) {
  EncodeTiledFn fn = resolve_encode();
  if (!fn) return set_error(JENGA_E_CUDA, "cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
  const CUresult r = fn(map, dt, rank, base, dims, strides_bytes, box, elem_strides, il, sw, l2, oob);
  if (r != CUDA_SUCCESS)
    return set_error(JENGA_E_CUDA, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
  return JENGA_OK;
}

// ------------------------------------------------------------------------------------------
// gather_rows: dst[b, i, :] = src[b, index[i], :]     (HBM-bound; 16-byte vectors)
// One warp per destination row chunk; index loaded once per row, broadcast by shuffle.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
gather_rows_kernel(const uint4* __restrict__ src, uint4* __restrict__ dst,
                   const long long* __restrict__ index, long long n_index, long long n_src_rows,
                   int vec_per_row, long long src_batch_vec, long long dst_batch_vec) {
  const int b = blockIdx.y;
  const uint4* s = src + b * src_batch_vec;
  uint4* d = dst + b * dst_batch_vec;
  const long long total = n_index * vec_per_row;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long row = i / vec_per_row;
    const int col = static_cast<int>(i - row * vec_per_row);
    long long srow = __ldg(index + row);
    if (srow < 0) srow += n_src_rows;  // torch-style negative index
    uint4 v = make_uint4(0, 0, 0, 0);
    if (srow >= 0 && srow < n_src_rows) v = __ldg(s + srow * vec_per_row + col);
    d[i] = v;
  }
}

// one-hot bytes [rows, nb] -> bit rows [rows, words]
__global__ void __launch_bounds__(256)
onehot_to_bits_kernel(const uint8_t* __restrict__ onehot, uint32_t* __restrict__ bits,
                      long long rows, int nb, int words) {
  const long long gw = (blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const long long total = rows * words;
  if (gw >= total) return;
  const long long row = gw / words;
  const int w = static_cast<int>(gw - row * words);
  const int col = w * 32 + lane;
  const bool on = col < nb && onehot[row * nb + col] != 0;
  const uint32_t word = __ballot_sync(0xffffffffu, on);
  if (lane == 0) bits[gw] = word;
}

// Ulysses inbound exchange: one pass over the local q,k,v, 16-byte stores into peer memory.
// A call moves the local heads [hg0, hg0+hg) of EVERY destination rank's head group (hg == h_loc
// moves everything); the head-group form lets the exchange of group g+1 run on a second stream
// under the attention of group g.  blockIdx.z is the sample: sample b reads x[w] + b*x_stride_bv and
// lands in slab (w*batch + b) of the [3, batch, N+T, slots, D] buffers (batch 1: slab w).
struct ScatterParams {
  const uint4* x[3];
  const uint4* joint[3];
  long long x_stride_v, joint_stride_v;  // uint4 units between tokens
  long long x_stride_bv, joint_stride_bv;  // uint4 units between samples
  int world, rank, heads, vec_per_head;  // vec_per_head = head_dim*2/16
  int hg0, hg;                           // local head range of this call
  long long n_loc, n_text;
  unsigned long long peer[8];
};
__global__ void __launch_bounds__(256)
ulysses_scatter_kernel(const ScatterParams p) {
  const int w = blockIdx.y;  // 0:q 1:k 2:v
  const uint4* x = p.x[w] + blockIdx.z * p.x_stride_bv;
  const uint4* joint = p.joint[w] + blockIdx.z * p.joint_stride_bv;
  const long long slab = static_cast<long long>(w) * gridDim.z + blockIdx.z;   // [3, batch] slab of the buffers
  const int h_loc = p.heads / p.world;
  const int vec_per_tok = p.world * p.hg * p.vec_per_head;     // vectors this call moves per image token
  const long long n_total = static_cast<long long>(p.world) * p.n_loc + p.n_text;
  const long long img_vecs = p.n_loc * vec_per_tok;
  const int txt_per_tok = p.hg * p.vec_per_head;
  const long long txt_vecs = p.n_text * static_cast<long long>(txt_per_tok);
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < img_vecs + txt_vecs;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    if (i < img_vecs) {
      const long long tok = i / vec_per_tok;
      const int c = static_cast<int>(i - tok * vec_per_tok);
      const int dst_rank = c / txt_per_tok;
      const int r = c - dst_rank * txt_per_tok;
      const int hl = p.hg0 + r / p.vec_per_head;               // local head at the destination
      const int v_in_head = r - (r / p.vec_per_head) * p.vec_per_head;
      const int head = dst_rank * h_loc + hl;                    // global head = column of x
      const uint4 v = __ldg(x + tok * p.x_stride_v + head * p.vec_per_head + v_in_head);
      uint4* dst = reinterpret_cast<uint4*>(p.peer[dst_rank]) +
                   ((slab * n_total + p.rank * p.n_loc + tok) * h_loc + hl) * p.vec_per_head +
                   v_in_head;
      *dst = v;
    } else {
      const long long k = i - img_vecs;
      const long long tok = k / txt_per_tok;
      const int r = static_cast<int>(k - tok * txt_per_tok);
      const int hl = p.hg0 + r / p.vec_per_head;
      const int v_in_head = r - (r / p.vec_per_head) * p.vec_per_head;
      const uint4 v = __ldg(joint + tok * p.joint_stride_v + (p.rank * h_loc + hl) * p.vec_per_head + v_in_head);
      uint4* dst = reinterpret_cast<uint4*>(p.peer[p.rank]) +
                   ((slab * n_total + p.world * p.n_loc + tok) * h_loc + hl) * p.vec_per_head +
                   v_in_head;
      *dst = v;
    }
  }
}

// Ragged form: destination p owns `cnt[p]` heads of this call, starting at slot hg0 of its
// group, whose global head 0 is off[p]; cstart[p] is the prefix of cnt (in heads) within one
// image token's vectors.  Every buffer has `slots` head slots.
struct ScatterRaggedParams {
  const uint4* x[3];
  const uint4* joint[3];
  long long x_stride_v, joint_stride_v;
  long long x_stride_bv, joint_stride_bv;
  int world, rank, slots, vec_per_head;
  int hg0;
  int off[9], cnt[8], cstart[9];   // cstart[world] = heads moved per image token
  long long n_loc, n_text;
  unsigned long long peer[8];
};
__global__ void __launch_bounds__(256)
ulysses_scatter_ragged_kernel(const ScatterRaggedParams p) {
  const int w = blockIdx.y;  // 0:q 1:k 2:v
  const uint4* x = p.x[w] + blockIdx.z * p.x_stride_bv;
  const uint4* joint = p.joint[w] + blockIdx.z * p.joint_stride_bv;
  const long long slab = static_cast<long long>(w) * gridDim.z + blockIdx.z;   // [3, batch] slab of the buffers
  const int vec_per_tok = p.cstart[p.world] * p.vec_per_head;
  const long long n_total = static_cast<long long>(p.world) * p.n_loc + p.n_text;
  const long long img_vecs = p.n_loc * vec_per_tok;
  const int txt_per_tok = p.cnt[p.rank] * p.vec_per_head;
  const long long txt_vecs = p.n_text * static_cast<long long>(txt_per_tok);
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < img_vecs + txt_vecs;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    if (i < img_vecs) {
      const long long tok = i / vec_per_tok;
      const int c = static_cast<int>(i - tok * vec_per_tok);
      const int j = c / p.vec_per_head;                          // head of this token's call
      const int v_in_head = c - j * p.vec_per_head;
      int dst_rank = 0;
      while (j >= p.cstart[dst_rank + 1]) ++dst_rank;
      const int slot = p.hg0 + (j - p.cstart[dst_rank]);
      const int head = p.off[dst_rank] + slot;                   // global head = column of x
      const uint4 v = __ldg(x + tok * p.x_stride_v + head * p.vec_per_head + v_in_head);
      uint4* dst = reinterpret_cast<uint4*>(p.peer[dst_rank]) +
                   ((slab * n_total + p.rank * p.n_loc + tok) * p.slots + slot) * p.vec_per_head +
                   v_in_head;
      *dst = v;
    } else {
      const long long k = i - img_vecs;
      const long long tok = k / txt_per_tok;
      const int r = static_cast<int>(k - tok * txt_per_tok);
      const int slot = p.hg0 + r / p.vec_per_head;
      const int v_in_head = r - (r / p.vec_per_head) * p.vec_per_head;
      const uint4 v = __ldg(joint + tok * p.joint_stride_v + (p.off[p.rank] + slot) * p.vec_per_head + v_in_head);
      uint4* dst = reinterpret_cast<uint4*>(p.peer[p.rank]) +
                   ((slab * n_total + p.world * p.n_loc + tok) * p.slots + slot) * p.vec_per_head +
                   v_in_head;
      *dst = v;
    }
  }
}

}  // namespace jenga

using namespace jenga;

extern "C" int jenga_abi_version(void) { return JENGA_B200_ABI_VERSION; }
extern "C" const char* jenga_last_error(void) { return g_err; }

extern "C" int jenga_carved_attn_fwd(const JengaAttnArgs* args, void* stream) {
  return carved_attn_fwd_impl(args, static_cast<cudaStream_t>(stream));
}

extern "C" int jenga_carved_attn_fwd_qk_int8(const JengaAttnArgs* args, const JengaQkInt8Args* qk, void* stream) {
  if (!qk) return set_error(JENGA_E_INVALID, "qk_int8: null pointer");
  return carved_attn_fwd_impl(args, static_cast<cudaStream_t>(stream), qk);
}

extern "C" int jenga_carved_attn_fwd_qk_int8_ex(const JengaAttnArgs* args, const JengaQkInt8ExArgs* qk,
                                                const JengaAttnSched* sched, void* stream) {
  if (!qk) return set_error(JENGA_E_INVALID, "qk_int8_ex: null pointer");
  return carved_attn_fwd_impl(args, static_cast<cudaStream_t>(stream), &qk->base, sched, true, qk->q_lse_shift);
}

extern "C" int jenga_carved_attn_fwd_sched(const JengaAttnArgs* args, const JengaQkInt8Args* qk,
                                           const JengaAttnSched* sched, void* stream) {
  if (!sched) return set_error(JENGA_E_INVALID, "sched: null pointer");
  return carved_attn_fwd_impl(args, static_cast<cudaStream_t>(stream), qk, sched);
}

extern "C" int64_t jenga_carved_attn_sched_workspace_bytes(int32_t batch, int32_t heads, int32_t nq_sparse,
                                                           int32_t nq_dense) {
  return carved_attn_sched_workspace_bytes(batch, heads, nq_sparse, nq_dense);
}

extern "C" int jenga_gather_rows(const void* src, void* dst, const int64_t* index, int64_t n_index,
                                 int64_t n_src_rows, int64_t row_bytes, int batch,
                                 int64_t src_batch_stride, int64_t dst_batch_stride, void* stream) {
  if (!src || !dst || !index) return set_error(JENGA_E_INVALID, "gather_rows: null pointer");
  if (n_index < 0 || n_src_rows <= 0 || batch <= 0)
    return set_error(JENGA_E_INVALID, "gather_rows: bad sizes");
  if (row_bytes <= 0 || row_bytes % 16 || src_batch_stride % 16 || dst_batch_stride % 16 ||
      reinterpret_cast<uintptr_t>(src) % 16 || reinterpret_cast<uintptr_t>(dst) % 16)
    return set_error(JENGA_E_INVALID, "gather_rows: rows must be 16-byte multiples and aligned");
  if (n_index == 0) return JENGA_OK;
  const int vec = static_cast<int>(row_bytes / 16);
  const long long total = n_index * vec;
  long long blocks = (total + 255) / 256;
  const long long cap = static_cast<long long>(kNumSMs) * 8 * 4;  // a few waves of 8 CTAs/SM; grid-stride beyond that
  if (blocks > cap) blocks = cap;
  dim3 grid(static_cast<unsigned>(blocks), static_cast<unsigned>(batch));
  gather_rows_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      static_cast<const uint4*>(src), static_cast<uint4*>(dst),
      reinterpret_cast<const long long*>(index), n_index, n_src_rows, vec, src_batch_stride / 16,
      dst_batch_stride / 16);
  cudaError_t ce = cudaGetLastError();
  return ce == cudaSuccess ? JENGA_OK : set_cuda_error(ce, "gather_rows launch");
}

extern "C" int jenga_mask_onehot_to_bits(const uint8_t* onehot, uint32_t* bits, int64_t rows,
                                         int32_t nb, int32_t mask_words, void* stream) {
  if (!onehot || !bits) return set_error(JENGA_E_INVALID, "onehot_to_bits: null pointer");
  if (rows <= 0 || nb <= 0 || mask_words * 32 < nb)
    return set_error(JENGA_E_INVALID, "onehot_to_bits: bad sizes");
  const long long warps = rows * mask_words;
  const long long blocks = (warps * 32 + 255) / 256;
  onehot_to_bits_kernel<<<static_cast<unsigned>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      onehot, bits, rows, nb, mask_words);
  cudaError_t ce = cudaGetLastError();
  return ce == cudaSuccess ? JENGA_OK : set_cuda_error(ce, "onehot_to_bits launch");
}

extern "C" int jenga_block_pool(const void* x, void* pooled, void* cast_out, int32_t in_dtype,
                                int32_t out_dtype, int32_t batch, int32_t heads, int32_t head_dim,
                                int64_t rows, int64_t stride_b, int64_t stride_s, int64_t stride_h,
                                int32_t n_blocks, void* stream) {
  return block_pool_impl(x, pooled, cast_out, in_dtype, out_dtype, batch, heads, head_dim, rows,
                         stride_b, stride_s, stride_h, n_blocks, static_cast<cudaStream_t>(stream));
}

extern "C" int jenga_select_blocks(const JengaSelectArgs* args, void* stream) {
  return select_blocks_impl(args, static_cast<cudaStream_t>(stream));
}

extern "C" int jenga_hy_prologue(const JengaHyPrologueArgs* args, void* stream) {
  return hy_prologue_impl(args, static_cast<cudaStream_t>(stream));
}

extern "C" int jenga_wan_prologue(const JengaWanPrologueArgs* args, void* stream) {
  return wan_prologue_impl(args, static_cast<cudaStream_t>(stream));
}

extern "C" int jenga_copy2d_async(void* dst, int64_t dst_pitch, const void* src, int64_t src_pitch,
                                  int64_t width_bytes, int64_t rows, int32_t direction, void* stream) {
  if (!dst || !src || width_bytes <= 0 || rows <= 0 || dst_pitch < width_bytes || src_pitch < width_bytes)
    return set_error(JENGA_E_INVALID, "copy2d: bad arguments");
  const cudaMemcpyKind kind = direction == 0 ? cudaMemcpyHostToDevice : cudaMemcpyDeviceToHost;
  cudaError_t ce = cudaMemcpy2DAsync(dst, static_cast<size_t>(dst_pitch), src, static_cast<size_t>(src_pitch),
                                     static_cast<size_t>(width_bytes), static_cast<size_t>(rows), kind,
                                     static_cast<cudaStream_t>(stream));
  return ce == cudaSuccess ? JENGA_OK : set_cuda_error(ce, "cudaMemcpy2DAsync");
}

// The exchange of `batch` samples, the batch strides in elements (checked by the caller).
static int ulysses_scatter_impl(const JengaUlyssesScatterArgs* a, int batch, int64_t x_stride_b,
                                int64_t joint_stride_b, cudaStream_t stream) {
  if (!a || !a->x[0] || !a->x[1] || !a->x[2] || !a->peer_qkv_host)
    return set_error(JENGA_E_INVALID, "ulysses_scatter: null pointer");
  if (a->world <= 0 || a->world > 8 || a->rank < 0 || a->rank >= a->world || a->heads % a->world ||
      a->head_dim % 8 || a->n_loc <= 0 || a->n_text < 0 || a->x_stride_s % 8 || a->joint_stride_s % 8)
    return set_error(JENGA_E_INVALID, "ulysses_scatter: bad shape");
  if (a->n_text > 0 && (!a->joint[0] || !a->joint[1] || !a->joint[2]))
    return set_error(JENGA_E_INVALID, "ulysses_scatter: joint tensors missing");
  for (int r = 0; r < a->world; ++r)
    if (!a->peer_qkv_host[r] || a->peer_qkv_host[r] % 16)
      return set_error(JENGA_E_INVALID, "ulysses_scatter: peer_qkv_host[%d] is null or not 16-byte aligned", r);
  ScatterParams p{};
  for (int w = 0; w < 3; ++w) {
    p.x[w] = static_cast<const uint4*>(a->x[w]);
    p.joint[w] = static_cast<const uint4*>(a->joint[w]);
  }
  p.x_stride_v = a->x_stride_s / 8;
  p.joint_stride_v = a->joint_stride_s / 8;
  p.x_stride_bv = x_stride_b / 8;
  p.joint_stride_bv = joint_stride_b / 8;
  p.world = a->world; p.rank = a->rank; p.heads = a->heads; p.vec_per_head = a->head_dim / 8;
  const int h_loc = a->heads / a->world;
  p.hg0 = a->head_count > 0 ? a->head_begin : 0;
  p.hg = a->head_count > 0 ? a->head_count : h_loc;
  if (p.hg0 < 0 || p.hg0 + p.hg > h_loc) return set_error(JENGA_E_INVALID, "ulysses_scatter: head group out of range");
  p.n_loc = a->n_loc; p.n_text = a->n_text;
  for (int r = 0; r < a->world; ++r) p.peer[r] = a->peer_qkv_host[r];
  const long long total = (a->n_loc * a->world + a->n_text) * p.hg * p.vec_per_head;
  long long blocks = (total + 255) / 256;
  if (blocks > static_cast<long long>(kNumSMs) * 16) blocks = static_cast<long long>(kNumSMs) * 16;
  dim3 grid(static_cast<unsigned>(blocks), 3, static_cast<unsigned>(batch));
  ulysses_scatter_kernel<<<grid, 256, 0, stream>>>(p);
  cudaError_t ce = cudaGetLastError();
  return ce == cudaSuccess ? JENGA_OK : set_cuda_error(ce, "ulysses_scatter launch");
}

static int ulysses_scatter_ragged_impl(const JengaUlyssesScatterArgs* a, const int32_t* off, int batch,
                                       int64_t x_stride_b, int64_t joint_stride_b, cudaStream_t stream) {
  if (!a || !off || !a->x[0] || !a->x[1] || !a->x[2] || !a->peer_qkv_host)
    return set_error(JENGA_E_INVALID, "ulysses_scatter_ragged: null pointer");
  if (a->world <= 0 || a->world > 8 || a->rank < 0 || a->rank >= a->world || a->heads <= 0 ||
      a->head_dim % 8 || a->n_loc <= 0 || a->n_text < 0 || a->x_stride_s % 8 || a->joint_stride_s % 8)
    return set_error(JENGA_E_INVALID, "ulysses_scatter_ragged: bad shape (world must be 1..8)");
  if (a->n_text > 0 && (!a->joint[0] || !a->joint[1] || !a->joint[2]))
    return set_error(JENGA_E_INVALID, "ulysses_scatter_ragged: joint tensors missing");
  if (off[0] != 0 || off[a->world] != a->heads)
    return set_error(JENGA_E_INVALID, "ulysses_scatter_ragged: head offsets must run from 0 to heads (%d), got %d..%d",
                     a->heads, off[0], off[a->world]);
  const int slots = (a->heads + a->world - 1) / a->world;
  for (int r = 0; r < a->world; ++r) {
    if (off[r + 1] < off[r])
      return set_error(JENGA_E_INVALID, "ulysses_scatter_ragged: head offsets decrease at rank %d", r);
    if (off[r + 1] - off[r] > slots)
      return set_error(JENGA_E_INVALID, "ulysses_scatter_ragged: rank %d's group of %d heads exceeds the %d slots",
                       r, off[r + 1] - off[r], slots);
  }
  for (int r = 0; r < a->world; ++r)
    if (!a->peer_qkv_host[r] || a->peer_qkv_host[r] % 16)
      return set_error(JENGA_E_INVALID, "ulysses_scatter_ragged: peer_qkv_host[%d] is null or not 16-byte aligned", r);
  ScatterRaggedParams p{};
  for (int w = 0; w < 3; ++w) {
    p.x[w] = static_cast<const uint4*>(a->x[w]);
    p.joint[w] = static_cast<const uint4*>(a->joint[w]);
  }
  p.x_stride_v = a->x_stride_s / 8;
  p.joint_stride_v = a->joint_stride_s / 8;
  p.x_stride_bv = x_stride_b / 8;
  p.joint_stride_bv = joint_stride_b / 8;
  p.world = a->world; p.rank = a->rank; p.slots = slots; p.vec_per_head = a->head_dim / 8;
  p.hg0 = a->head_count > 0 ? a->head_begin : 0;
  const int hg = a->head_count > 0 ? a->head_count : slots;
  if (p.hg0 < 0 || p.hg0 + hg > slots)
    return set_error(JENGA_E_INVALID, "ulysses_scatter_ragged: slot range out of range");
  p.cstart[0] = 0;
  for (int r = 0; r < a->world; ++r) {
    const int end = off[r + 1] - off[r] < p.hg0 + hg ? off[r + 1] - off[r] : p.hg0 + hg;
    p.off[r] = off[r];
    p.cnt[r] = end > p.hg0 ? end - p.hg0 : 0;
    p.cstart[r + 1] = p.cstart[r] + p.cnt[r];
  }
  p.off[a->world] = off[a->world];
  p.n_loc = a->n_loc; p.n_text = a->n_text;
  for (int r = 0; r < a->world; ++r) p.peer[r] = a->peer_qkv_host[r];
  const long long total = (a->n_loc * p.cstart[a->world] + a->n_text * p.cnt[a->rank]) * p.vec_per_head;
  if (total == 0) return JENGA_OK;
  long long blocks = (total + 255) / 256;
  if (blocks > static_cast<long long>(kNumSMs) * 16) blocks = static_cast<long long>(kNumSMs) * 16;
  dim3 grid(static_cast<unsigned>(blocks), 3, static_cast<unsigned>(batch));
  ulysses_scatter_ragged_kernel<<<grid, 256, 0, stream>>>(p);
  cudaError_t ce = cudaGetLastError();
  return ce == cudaSuccess ? JENGA_OK : set_cuda_error(ce, "ulysses_scatter_ragged launch");
}

extern "C" int jenga_ulysses_scatter(const JengaUlyssesScatterArgs* a, void* stream) {
  return ulysses_scatter_impl(a, 1, 0, 0, static_cast<cudaStream_t>(stream));
}

extern "C" int jenga_ulysses_scatter_ragged(const JengaUlyssesScatterArgs* a, const int32_t* off, void* stream) {
  return ulysses_scatter_ragged_impl(a, off, 1, 0, 0, static_cast<cudaStream_t>(stream));
}

extern "C" int jenga_ulysses_scatter_batched(const JengaUlyssesScatterBatchArgs* a, const int32_t* off,
                                             void* stream) {
  if (!a) return set_error(JENGA_E_INVALID, "ulysses_scatter_batched: null pointer");
  if (a->batch < 1 || a->batch > 65535)
    return set_error(JENGA_E_INVALID, "ulysses_scatter_batched: batch %d must be 1..65535", a->batch);
  if (a->x_stride_b % 8 || a->joint_stride_b % 8)
    return set_error(JENGA_E_INVALID, "ulysses_scatter_batched: batch strides (%lld, %lld) must be multiples of 8",
                     static_cast<long long>(a->x_stride_b), static_cast<long long>(a->joint_stride_b));
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  return off ? ulysses_scatter_ragged_impl(&a->base, off, a->batch, a->x_stride_b, a->joint_stride_b, st)
             : ulysses_scatter_impl(&a->base, a->batch, a->x_stride_b, a->joint_stride_b, st);
}

extern "C" int64_t jenga_select_blocks_workspace_bytes(int32_t batch_heads, int32_t nq, int32_t n_img) {
  if (batch_heads <= 0 || nq <= 0 || n_img <= 0) return 0;
  return static_cast<int64_t>(batch_heads) * nq * n_img * static_cast<int64_t>(sizeof(float));
}
