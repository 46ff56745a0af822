// Wan2.1-I2V cross-attention for sm_90a: the image and the text attention of one query block in one
// launch, summed as the reference sums them.
//
// Replaces WanI2VCrossAttention.forward's attention part (wan/modules/model_mul.py:240-247): two
// flash_attention calls over the 257 CLIP keys and the text keys, each returned as fp32
// (wan/modules/attention.py:130), added in fp32 and cast to bf16 by self.o under autocast:
//   out[r,h,:] = bf16( f32(A_img[r,h,:]) + f32(A_txt[r,h,:]) ),  A_seg = bf16(softmax(q K_seg^T D^-1/2) V_seg)
//
// One CTA per (batch*head, 128 query rows), head-major, running the pipeline of carved_attn_common.cuh
// with the dense-class arithmetic of the carved-attention kernel (carved_attn.cu) over the image tiles,
// then the text tiles as a second segment; each K/V pair has its own tensor maps.  So A_img and A_txt
// are bit for bit what one dense launch over that segment returns.  Rows past a tensor's extent are
// zero-filled by TMA and masked by the segment's column limit, so no padding copies are needed.  At
// the segment boundary A_img is normalised, rounded to bf16 as the dense epilogue rounds it and parked
// in the shared-memory Q tile: Q lives in registers by then, and each warp overwrites only its own 16
// Q rows.
#include "carved_attn_common.cuh"

namespace jenga {

namespace {

using namespace attn;

constexpr int kSmemBytes = 1024 /*align slack*/ + kOffEnd;

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

__global__ void __launch_bounds__(kThreads, 1)
wan_i2v_cross_attn_kernel(const __grid_constant__ CUtensorMap tm_q,
                          const __grid_constant__ CUtensorMap tm_ki, const __grid_constant__ CUtensorMap tm_vi,
                          const __grid_constant__ CUtensorMap tm_kt, const __grid_constant__ CUtensorMap tm_vt,
                          const CrossParams p) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_addr = smem_u32(smem_raw);
  uint8_t* smem = smem_raw + (((raw_addr + 1023u) & ~1023u) - raw_addr);
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
    for (int i = 0; i < VT_FULL; ++i) mbar_init(&bars[i], i >= K_EMPTY ? 8u : 1u);   // bf16 V: no V^T
    fence_mbar_init();
  }
  __syncthreads();

  if (warp >= kConsumerThreads / 32) {
    // =============================== producer warpgroup ===============================
    setmaxnreg_dec<24>();
    if (warp == kConsumerThreads / 32 && lane == 0) {
      produce<false, false>(smem, bars, p.err_flag, &tm_q, static_cast<int>(q_row0), h, b, [&](int j, KvMaps& m) {
        const bool img = j < p.n_img;
        m = {img ? &tm_ki : &tm_kt, img ? &tm_vi : &tm_vt};
        return j < n_tiles ? (img ? j : j - p.n_img) * kBlock : -1;
      });
    }
    return;
  }

  // =============================== consumers ===============================
  setmaxnreg_inc<240>();
  Consumer<true> cons(smem, bars, p.err_flag);
  // the parked bf16 A_img of this warp: its own 16 Q rows of the two Q boxes (2 x 2 KB), word k of a
  // lane at (k & 15) * 32 + lane of box k >> 4 — conflict-free, and no other warp reads it
  uint32_t* park = reinterpret_cast<uint32_t*>(smem + kOffQ + warp * 2048) + lane;
  auto park_at = [&](int k) -> uint32_t* { return park + (k >> 4) * (kBoxBytes / 4) + (k & 15) * 32; };
  // 1 / l of a finished segment
  auto inv_rows = [&](const float (&l)[2], float (&inv)[2]) {
#pragma unroll
    for (int r = 0; r < 2; ++r) inv[r] = 1.0f / row_sum(l[r]);
  };

  cons.load_q();
  cons.run(
      n_tiles,
      [&](int j, Tile& t) {   // the dense class of carved_attn.cu: no text_amp, c = qk_scale
        const bool img = j < p.n_img;
        t = {static_cast<long long>(img ? j : j - p.n_img) * kBlock, img ? p.img_rows : p.txt_rows, p.qk_scale, 0.f,
             j == p.n_img};
      },
      [&](const float (&l_img)[2]) {   // A_img = bf16(O / l), parked
        float inv[2];
        inv_rows(l_img, inv);
        __syncwarp();
#pragma unroll
        for (int k = 0; k < 32; ++k)
          *park_at(k) = pack2<true>(cons.o[2 * k] * inv[k & 1], cons.o[2 * k + 1] * inv[k & 1]);
      });

  // ---- out = bf16(f32(A_img) + f32(A_txt)); rows past q_rows are not stored ----
  float inv[2];
  inv_rows(cons.l_sum, inv);
#pragma unroll
  for (int k = 0; k < 32; ++k) {
    const int r = k & 1;
    const long long q_row = q_row0 + cons.row_lo + 8 * r;
    if (q_row >= p.q_rows) continue;
    const float2 ft = unpack2<true>(pack2<true>(cons.o[2 * k] * inv[r], cons.o[2 * k + 1] * inv[r]));
    const float2 fi = unpack2<true>(*park_at(k));
    const long long o_off = b * p.o_stride_b + q_row * p.o_stride_s + static_cast<long long>(h) * p.o_stride_h +
                            8 * (k >> 1) + 2 * cons.qd;
    *reinterpret_cast<uint32_t*>(p.out + o_off) = pack2<true>(ft.x + fi.x, ft.y + fi.y);
  }
}

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
  const int dt = JENGA_BF16;
  if ((rc = make_tile_map(&tm_q, a->q, dt, a->q_rows, a->heads, a->batch, a->q_stride_b, a->q_stride_s,
                          a->q_stride_h)) ||
      (rc = make_tile_map(&tm_ki, a->k_img, dt, a->img_rows, a->heads, a->batch, a->ki_stride_b, a->ki_stride_s,
                          a->ki_stride_h)) ||
      (rc = make_tile_map(&tm_vi, a->v_img, dt, a->img_rows, a->heads, a->batch, a->vi_stride_b, a->vi_stride_s,
                          a->vi_stride_h)) ||
      (rc = make_tile_map(&tm_kt, a->k_txt, dt, a->txt_rows, a->heads, a->batch, a->kt_stride_b, a->kt_stride_s,
                          a->kt_stride_h)) ||
      (rc = make_tile_map(&tm_vt, a->v_txt, dt, a->txt_rows, a->heads, a->batch, a->vt_stride_b, a->vt_stride_s,
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
