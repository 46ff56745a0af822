// Generalized-Hilbert tables on the device (SURVEY §8 f-4): the per-voxel index query of the
// reference (gilbert.py:12-38 gilbert_xyz2d, :68-272 gilbert_xyz2d_r) is embarrassingly parallel —
// one thread per voxel descends the same box subdivision the host walker (gilbert.cpp) enumerates,
// adding the volumes of the sub-boxes that precede the one containing its voxel.  Also the block
// adjacency (gilbert.py:597-677 / :679-766) produced directly as the packed bit rows the selection
// kernel consumes.  Serves short runs and many-resolution serving where even 22 ms of host work
// per (t,h,w) and the H2D copy of the tables are visible; results are bit-identical to the host
// tables (tests/test_gilbert_device_gpu.py).
#include "jenga_internal.h"

namespace jenga {
namespace {

struct V3 {
  int x, y, z;
};
__device__ __forceinline__ V3 add(V3 a, V3 b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
__device__ __forceinline__ V3 sub(V3 a, V3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
__device__ __forceinline__ V3 neg(V3 a) { return {-a.x, -a.y, -a.z}; }
__device__ __forceinline__ int sg(int v) { return (v > 0) - (v < 0); }
__device__ __forceinline__ V3 unit(V3 a) { return {sg(a.x), sg(a.y), sg(a.z)}; }
__device__ __forceinline__ int ext(V3 a) { return abs(a.x + a.y + a.z); }
__device__ __forceinline__ V3 halfv(V3 a) { return {a.x >> 1, a.y >> 1, a.z >> 1}; }  // Python // 2
__device__ __forceinline__ long long vol(V3 a, V3 b, V3 c) {
  return static_cast<long long>(ext(a)) * ext(b) * ext(c);
}
// is q inside the (signed, half-open) box that starts at p and spans a + b + c?  (gilbert.py:43-65)
__device__ __forceinline__ bool inside(V3 q, V3 p, V3 a, V3 b, V3 c) {
  const int d[3] = {a.x + b.x + c.x, a.y + b.y + c.y, a.z + b.z + c.z};
  const int qq[3] = {q.x, q.y, q.z}, pp[3] = {p.x, p.y, p.z};
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    if (d[i] < 0) {
      if (qq[i] > pp[i] || qq[i] <= pp[i] + d[i]) return false;
    } else {
      if (qq[i] < pp[i] || qq[i] >= pp[i] + d[i]) return false;
    }
  }
  return true;
}

// curve index of voxel q in the box (p; a, b, c) — iterative descent, same children in the same
// order as Walker::walk
__device__ long long curve_index(V3 q, V3 p, V3 a, V3 b, V3 c) {
  long long idx = 0;
  for (int guard = 0; guard < 96; ++guard) {
    const int w = ext(a), h = ext(b), d = ext(c);
    const V3 da = unit(a), db = unit(b), dc = unit(c);
    const V3 off = sub(q, p);
    if (h == 1 && d == 1) return idx + (da.x * off.x + da.y * off.y + da.z * off.z);
    if (w == 1 && d == 1) return idx + (db.x * off.x + db.y * off.y + db.z * off.z);
    if (w == 1 && h == 1) return idx + (dc.x * off.x + dc.y * off.y + dc.z * off.z);
    V3 a2 = halfv(a), b2 = halfv(b), c2 = halfv(c);
    const int w2 = ext(a2), h2 = ext(b2), d2 = ext(c2);
    if ((w2 & 1) && w > 2) a2 = add(a2, da);
    if ((h2 & 1) && h > 2) b2 = add(b2, db);
    if ((d2 & 1) && d > 2) c2 = add(c2, dc);
    // candidate children (start, a, b, c) in curve order; descend into the first that holds q
    V3 cp[5], ca[5], cb[5], cc[5];
    int n;
    if (2 * w > 3 * h && 2 * w > 3 * d) {
      n = 2;
      cp[0] = p; ca[0] = a2; cb[0] = b; cc[0] = c;
      cp[1] = add(p, a2); ca[1] = sub(a, a2); cb[1] = b; cc[1] = c;
    } else if (3 * h > 4 * d) {
      n = 3;
      cp[0] = p; ca[0] = b2; cb[0] = c; cc[0] = a2;
      cp[1] = add(p, b2); ca[1] = a; cb[1] = sub(b, b2); cc[1] = c;
      cp[2] = add(add(p, sub(a, da)), sub(b2, db)); ca[2] = neg(b2); cb[2] = c; cc[2] = neg(sub(a, a2));
    } else if (3 * d > 4 * h) {
      n = 3;
      cp[0] = p; ca[0] = c2; cb[0] = a2; cc[0] = b;
      cp[1] = add(p, c2); ca[1] = a; cb[1] = b; cc[1] = sub(c, c2);
      cp[2] = add(add(p, sub(a, da)), sub(c2, dc)); ca[2] = neg(c2); cb[2] = neg(sub(a, a2)); cc[2] = b;
    } else {
      n = 5;
      cp[0] = p; ca[0] = b2; cb[0] = c2; cc[0] = a2;
      cp[1] = add(p, b2); ca[1] = c; cb[1] = a2; cc[1] = sub(b, b2);
      cp[2] = add(add(p, sub(b2, db)), sub(c, dc)); ca[2] = a; cb[2] = neg(b2); cc[2] = neg(sub(c, c2));
      cp[3] = add(add(add(p, sub(a, da)), b2), sub(c, dc)); ca[3] = neg(c); cb[3] = neg(sub(a, a2)); cc[3] = sub(b, b2);
      cp[4] = add(add(p, sub(a, da)), sub(b2, db)); ca[4] = neg(b2); cb[4] = c2; cc[4] = neg(sub(a, a2));
    }
    int pick = n - 1;
    for (int i = 0; i < n - 1; ++i) {
      if (inside(q, cp[i], ca[i], cb[i], cc[i])) {
        pick = i;
        break;
      }
      idx += vol(ca[i], cb[i], cc[i]);
    }
    p = cp[pick]; a = ca[pick]; b = cb[pick]; c = cc[pick];
  }
  return -1;  // unreachable for valid boxes
}

__device__ __forceinline__ long long xyz2d(int x, int y, int z, int W, int H, int D) {
  const V3 q{x, y, z}, o{0, 0, 0}, X{W, 0, 0}, Y{0, H, 0}, Z{0, 0, D};
  if (W >= H && W >= D) return curve_index(q, o, X, Y, Z);
  if (H >= W && H >= D) return curve_index(q, o, Y, X, Z);
  return curve_index(q, o, Z, X, Y);
}

__global__ void __launch_bounds__(256)
gilbert3d_kernel(int t, int h, int w, long long* __restrict__ l2h, long long* __restrict__ h2l) {
  const long long n = static_cast<long long>(t) * h * w;
  for (long long lin = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; lin < n;
       lin += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(lin % w), y = static_cast<int>((lin / w) % h), z = static_cast<int>(lin / (static_cast<long long>(w) * h));
    const long long idx = xyz2d(x, y, z, w, h, t);
    if (l2h) l2h[lin] = idx;
    if (h2l) h2l[idx] = lin;
  }
}

// sliced curve (gilbert.py:332-434): one 2-D curve per frame; frame z is mirrored in x and/or y so
// that it starts at the corner nearest to where frame z-1 ended.
__global__ void __launch_bounds__(256)
gilbert_sliced_kernel(int t, int h, int w, long long* __restrict__ l2h, long long* __restrict__ h2l) {
  const long long hw = static_cast<long long>(h) * w, n = hw * t;
  // where the unflipped 2-D curve ends: the voxel with index hw-1 — the curve's last line lies on a
  // box edge, so testing the four corners is enough; fall back to a scan-free search over the border
  __shared__ int s_ex, s_ey;
  if (threadIdx.x == 0) {
    s_ex = -1;
    const int cx[4] = {0, w - 1, 0, w - 1}, cy[4] = {0, 0, h - 1, h - 1};
    for (int i = 0; i < 4 && s_ex < 0; ++i)
      if (xyz2d(cx[i], cy[i], 0, w, h, 1) == hw - 1) { s_ex = cx[i]; s_ey = cy[i]; }
    for (int x = 0; x < w && s_ex < 0; ++x)
      for (int y = 0; y < h; y += (h > 1 ? h - 1 : 1))
        if (xyz2d(x, y, 0, w, h, 1) == hw - 1) { s_ex = x; s_ey = y; break; }
    for (int y = 0; y < h && s_ex < 0; ++y)
      for (int x = 0; x < w; x += (w > 1 ? w - 1 : 1))
        if (xyz2d(x, y, 0, w, h, 1) == hw - 1) { s_ex = x; s_ey = y; break; }
    for (int y = 0; y < h && s_ex < 0; ++y)      // last resort: everywhere
      for (int x = 0; x < w; ++x)
        if (xyz2d(x, y, 0, w, h, 1) == hw - 1) { s_ex = x; s_ey = y; break; }
  }
  __syncthreads();
  const int ex0 = s_ex, ey0 = s_ey;
  for (long long lin = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; lin < n;
       lin += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(lin % w), y = static_cast<int>((lin / w) % h), z = static_cast<int>(lin / hw);
    bool fx = false, fy = false;
    for (int zz = 0; zz < z; ++zz) {          // flips of frame zz+1 from the end of frame zz (:372-405)
      const int ex = fx ? w - 1 - ex0 : ex0, ey = fy ? h - 1 - ey0 : ey0;
      fx = 2 * ex >= w;
      fy = 2 * ey >= h;
    }
    const int ax = fx ? w - 1 - x : x, ay = fy ? h - 1 - y : y;
    const long long idx = z * hw + xyz2d(ax, ay, 0, w, h, 1);
    if (l2h) l2h[lin] = idx;
    if (h2l) h2l[idx] = lin;
  }
}

__global__ void __launch_bounds__(256)
neighbour_bits_kernel(int t, int h, int w, int block, const long long* __restrict__ l2h,
                      unsigned int* __restrict__ bits, int words) {
  const long long n = static_cast<long long>(t) * h * w;
  for (long long lin = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; lin < n;
       lin += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int x = static_cast<int>(lin % w), y = static_cast<int>((lin / w) % h), z = static_cast<int>(lin / (static_cast<long long>(w) * h));
    const int me = static_cast<int>(l2h[lin] / block);
    unsigned int* row = bits + static_cast<long long>(me) * words;
    int last = -1;
    for (int dz = -1; dz <= 1; ++dz) {
      const int nz = z + dz;
      if (nz < 0 || nz >= t) continue;
      for (int dy = -1; dy <= 1; ++dy) {
        const int ny = y + dy;
        if (ny < 0 || ny >= h) continue;
        for (int dx = -1; dx <= 1; ++dx) {
          const int nx = x + dx;
          if (nx < 0 || nx >= w) continue;
          const int other = static_cast<int>(l2h[(static_cast<long long>(nz) * h + ny) * w + nx] / block);
          if (other != last) {   // most neighbours share a block: skip repeated atomics
            atomicOr(row + (other >> 5), 1u << (other & 31));
            last = other;
          }
        }
      }
    }
  }
}

}  // namespace
}  // namespace jenga

using namespace jenga;

extern "C" int jenga_gilbert_mapping_device(int t, int h, int w, int sliced, int64_t* linear_to_hilbert,
                                            int64_t* hilbert_to_linear, void* stream) {
  if (t <= 0 || h <= 0 || w <= 0) return set_error(JENGA_E_INVALID, "gilbert_device: empty grid");
  if (!linear_to_hilbert && !hilbert_to_linear) return set_error(JENGA_E_INVALID, "gilbert_device: no output");
  const long long n = static_cast<long long>(t) * h * w;
  long long blocks = (n + 255) / 256;
  if (blocks > static_cast<long long>(kNumSMs) * 8) blocks = static_cast<long long>(kNumSMs) * 8;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  if (sliced)
    gilbert_sliced_kernel<<<static_cast<unsigned>(blocks), 256, 0, s>>>(t, h, w, reinterpret_cast<long long*>(linear_to_hilbert),
                                                                       reinterpret_cast<long long*>(hilbert_to_linear));
  else
    gilbert3d_kernel<<<static_cast<unsigned>(blocks), 256, 0, s>>>(t, h, w, reinterpret_cast<long long*>(linear_to_hilbert),
                                                                  reinterpret_cast<long long*>(hilbert_to_linear));
  const cudaError_t ce = cudaGetLastError();
  return ce == cudaSuccess ? JENGA_OK : set_cuda_error(ce, "gilbert_device launch");
}

extern "C" int jenga_block_neighbor_bits_device(int t, int h, int w, int block, const int64_t* linear_to_hilbert,
                                                uint32_t* bits, int32_t words, void* stream) {
  if (!linear_to_hilbert || !bits || block <= 0 || t <= 0 || h <= 0 || w <= 0)
    return set_error(JENGA_E_INVALID, "neighbor_bits_device: bad argument");
  const long long n = static_cast<long long>(t) * h * w;
  const long long nb = (n + block - 1) / block;
  if (static_cast<long long>(words) * 32 < nb) return set_error(JENGA_E_INVALID, "neighbor_bits_device: words too small");
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  cudaError_t ce = cudaMemsetAsync(bits, 0, static_cast<size_t>(nb) * words * 4, s);
  if (ce != cudaSuccess) return set_cuda_error(ce, "neighbor_bits_device memset");
  long long blocks = (n + 255) / 256;
  if (blocks > static_cast<long long>(kNumSMs) * 8) blocks = static_cast<long long>(kNumSMs) * 8;
  neighbour_bits_kernel<<<static_cast<unsigned>(blocks), 256, 0, s>>>(t, h, w, block,
                                                                     reinterpret_cast<const long long*>(linear_to_hilbert), bits, words);
  ce = cudaGetLastError();
  return ce == cudaSuccess ? JENGA_OK : set_cuda_error(ce, "neighbor_bits_device launch");
}
