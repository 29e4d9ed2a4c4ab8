// SIMT kernels of the SuperPoint + SuperGlue matcher (everything that is not a GEMM / 3x3 conv).
// Reference: etc/feature_matching_baselines/SuperGlue/models/{superpoint,superglue}.py.
#include "spsg_ops.cuh"

#include <cuda_bf16.h>

#include <algorithm>
#include <type_traits>

namespace mfr {

namespace {

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ------------------------------------------------------------------------------------------ conv1a
// 3x3, pad 1, 1 -> 64 channels, bias, ReLU (superpoint.py:119,148). thread = output channel. OutT: float or bf16
template <typename OutT>
__global__ void __launch_bounds__(64) conv1a_kernel(const float* __restrict__ img, const float* __restrict__ w,
                                                    const float* __restrict__ bias, OutT* __restrict__ out,
                                                    int H, int W) {
  __shared__ float patch[3][66];
  const int n = blockIdx.z, y = blockIdx.y, x0 = blockIdx.x * 64;
  for (int idx = threadIdx.x; idx < 3 * 66; idx += 64) {
    const int ky = idx / 66, kx = idx - ky * 66;
    const int iy = y - 1 + ky, ix = x0 - 1 + kx;
    patch[ky][kx] = (iy >= 0 && iy < H && ix >= 0 && ix < W) ? img[(static_cast<size_t>(n) * H + iy) * W + ix] : 0.f;
  }
  const int c = threadIdx.x;
  float wr[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) wr[k] = w[c * 9 + k];
  const float b = bias[c];
  __syncthreads();
  const int xe = min(64, W - x0);
  for (int px = 0; px < xe; ++px) {
    float a = b;
#pragma unroll
    for (int ky = 0; ky < 3; ++ky)
#pragma unroll
      for (int kx = 0; kx < 3; ++kx) a = fmaf(wr[ky * 3 + kx], patch[ky][px + kx], a);
    const float r = fmaxf(a, 0.f);
    if constexpr (std::is_same<OutT, float>::value) out[((static_cast<size_t>(n) * H + y) * W + x0 + px) * 64 + c] = r;
    else out[((static_cast<size_t>(n) * H + y) * W + x0 + px) * 64 + c] = __float2bfloat16_rn(r);
  }
}

// ------------------------------------------------------------------------------------------ maxpool 2x2
__global__ void maxpool2_kernel(const float* __restrict__ in, float* __restrict__ out, int N, int H, int W, int C4) {
  const int Ho = H / 2, Wo = W / 2;
  const size_t total = static_cast<size_t>(N) * Ho * Wo * C4;
  const size_t idx = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c4 = static_cast<int>(idx % C4);
  size_t p = idx / C4;
  const int x = static_cast<int>(p % Wo); p /= Wo;
  const int y = static_cast<int>(p % Ho);
  const int n = static_cast<int>(p / Ho);
  const float4* s = reinterpret_cast<const float4*>(in) + (static_cast<size_t>(n) * H + 2 * y) * W * C4;
  const float4 a = s[(2 * x) * C4 + c4], b = s[(2 * x + 1) * C4 + c4];
  const float4 c = s[(static_cast<size_t>(W) + 2 * x) * C4 + c4], d = s[(static_cast<size_t>(W) + 2 * x + 1) * C4 + c4];
  float4 o;
  o.x = fmaxf(fmaxf(a.x, b.x), fmaxf(c.x, d.x));
  o.y = fmaxf(fmaxf(a.y, b.y), fmaxf(c.y, d.y));
  o.z = fmaxf(fmaxf(a.z, b.z), fmaxf(c.z, d.z));
  o.w = fmaxf(fmaxf(a.w, b.w), fmaxf(c.w, d.w));
  reinterpret_cast<float4*>(out)[idx] = o;
}

// bf16 [N][H][W][8 C8] -> [N][H/2][W/2][8 C8], 8 channels per thread (the max of bf16 values is exact)
__global__ void maxpool2_bf16_kernel(const uint4* __restrict__ in, uint4* __restrict__ out, int N, int H, int W, int C8) {
  const int Ho = H / 2, Wo = W / 2;
  const size_t total = static_cast<size_t>(N) * Ho * Wo * C8;
  const size_t idx = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c8 = static_cast<int>(idx % C8);
  size_t p = idx / C8;
  const int x = static_cast<int>(p % Wo); p /= Wo;
  const int y = static_cast<int>(p % Ho);
  const int n = static_cast<int>(p / Ho);
  const uint4* s = in + (static_cast<size_t>(n) * H + 2 * y) * W * C8;
  uint4 v[4] = {s[(2 * x) * C8 + c8], s[(2 * x + 1) * C8 + c8], s[(static_cast<size_t>(W) + 2 * x) * C8 + c8],
                s[(static_cast<size_t>(W) + 2 * x + 1) * C8 + c8]};
  const __nv_bfloat162* a = reinterpret_cast<const __nv_bfloat162*>(&v[0]);
  const __nv_bfloat162* b = reinterpret_cast<const __nv_bfloat162*>(&v[1]);
  const __nv_bfloat162* c = reinterpret_cast<const __nv_bfloat162*>(&v[2]);
  const __nv_bfloat162* d = reinterpret_cast<const __nv_bfloat162*>(&v[3]);
  uint4 o;
  __nv_bfloat162* r = reinterpret_cast<__nv_bfloat162*>(&o);
#pragma unroll
  for (int i = 0; i < 4; ++i) r[i] = __hmax2(__hmax2(a[i], b[i]), __hmax2(c[i], d[i]));
  out[idx] = o;
}

// ------------------------------------------------------------------------------------------ detector head
// softmax over 65 channels, drop the dustbin, depth-to-space 8x8 (superpoint.py:163-166).
// logits [N][h][w][ldc >= 65] -> scores [N][h*8][w*8]; one warp per cell.
__global__ void __launch_bounds__(256) score_map_kernel(const float* __restrict__ logits, int ldc,
                                                        float* __restrict__ scores, int N, int h, int w) {
  const int cell = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (cell >= N * h * w) return;
  const int lane = threadIdx.x & 31;
  const float* p = logits + static_cast<size_t>(cell) * ldc;
  const float a = p[lane], b = p[32 + lane], c = lane == 0 ? p[64] : -INFINITY;
  const float m = warp_max(fmaxf(fmaxf(a, b), c));
  const float ea = __expf(a - m), eb = __expf(b - m), ec = lane == 0 ? __expf(c - m) : 0.f;
  const float inv = 1.f / warp_sum(ea + eb + ec);
  const int x = cell % w, y = (cell / w) % h, n = cell / (w * h);
  float* o = scores + (static_cast<size_t>(n) * h * 8 + y * 8) * (w * 8) + x * 8;
  // channel k -> (dy, dx) = (k / 8, k % 8)
  o[(lane >> 3) * (w * 8) + (lane & 7)] = ea * inv;
  o[(4 + (lane >> 3)) * (w * 8) + (lane & 7)] = eb * inv;
}

// ------------------------------------------------------------------------------------------ NMS (superpoint.py:47-62)
// max over a (2r+1)^2 window, -inf padding, as two separable passes (max is exact, so this equals
// torch's max_pool2d bit for bit).
__global__ void rowmax_kernel(const float* __restrict__ in, float* __restrict__ out, int N, int H, int W, int r) {
  const size_t idx = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= static_cast<size_t>(N) * H * W) return;
  const int x = static_cast<int>(idx % W);
  const float* row = in + (idx - x);
  float m = -INFINITY;
  for (int k = max(0, x - r); k <= min(W - 1, x + r); ++k) m = fmaxf(m, row[k]);
  out[idx] = m;
}
__global__ void colmax_kernel(const float* __restrict__ in, float* __restrict__ out, int N, int H, int W, int r) {
  const size_t idx = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= static_cast<size_t>(N) * H * W) return;
  const int x = static_cast<int>(idx % W);
  const int y = static_cast<int>((idx / W) % H);
  const float* base = in + (idx - static_cast<size_t>(y) * W - x) + x;
  float m = -INFINITY;
  for (int k = max(0, y - r); k <= min(H - 1, y + r); ++k) m = fmaxf(m, base[static_cast<size_t>(k) * W]);
  out[idx] = m;
}
// step 0: mask = (s == pool(s))                      [mask as float 0/1]
__global__ void nms_init_kernel(const float* __restrict__ s, const float* __restrict__ pooled,
                                float* __restrict__ mask, size_t n) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) mask[i] = s[i] == pooled[i] ? 1.f : 0.f;
}
// supp = pool(mask) > 0 ; supp_scores = supp ? 0 : s
__global__ void nms_supp_kernel(const float* __restrict__ s, const float* __restrict__ pooled_mask,
                                float* __restrict__ supp_scores, size_t n) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n) supp_scores[i] = pooled_mask[i] > 0.f ? 0.f : s[i];
}
// mask |= (supp_scores == pool(supp_scores)) & !supp
__global__ void nms_update_kernel(const float* __restrict__ supp_scores, const float* __restrict__ pooled_supp,
                                  const float* __restrict__ pooled_mask, float* __restrict__ mask, size_t n) {
  const size_t i = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i < n && supp_scores[i] == pooled_supp[i] && !(pooled_mask[i] > 0.f)) mask[i] = 1.f;
}

// ------------------------------------------------------------------------------------------ keypoint selection
// candidates: mask && score > thr && inside the border, in row-major order (torch.nonzero order);
// then the max_kp highest scores in descending order (torch.topk), or all of them in row-major order
// when there are not more than max_kp (superpoint.py:170-187). One block per image.
constexpr int kMaxCand = 16384;
constexpr int kRadixBits = 11;

__device__ __forceinline__ bool is_candidate(float s, float m, int i, int H, int W, float thr, int border) {
  const int y = i / W, x = i - y * W;
  return m > 0.f && s > thr && y >= border && y < H - border && x >= border && x < W - border;
}
// sort key: descending key order = descending score, then lower pixel index first (scores are >= 0, so their bits
// order like the values)
__device__ __forceinline__ unsigned long long cand_key(float s, int i) {
  return (static_cast<unsigned long long>(__float_as_uint(s)) << 32) |
         static_cast<unsigned long long>(0xffffffffu - static_cast<unsigned>(i));
}
// inclusive prefix sum over a block of 1024 threads; wsum must not be in use by another scan
__device__ __forceinline__ int block_scan1024(int v, int* wsum) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v += t;
  }
  if (lane == 31) wsum[wid] = v;
  __syncthreads();
  if (wid == 0) {
    int ws = wsum[lane];
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, ws, o);
      if (lane >= o) ws += t;
    }
    wsum[lane] = ws;
  }
  __syncthreads();
  return v + (wid > 0 ? wsum[wid - 1] : 0);
}

// Shared memory: 128 KB of keys (dynamic) and the 8 KB radix histogram: one block per SM, so the register budget is
// that of one 1024-thread block.
__global__ void __launch_bounds__(1024, 1) select_keypoints_kernel(
    const float* __restrict__ scores, const float* __restrict__ mask, int H, int W, float thr, int border,
    int max_kp, float* __restrict__ kpts /*[N][max_kp][2]*/, float* __restrict__ kscores /*[N][max_kp]*/,
    int* __restrict__ counts) {
  extern __shared__ unsigned long long s_key[];   // cand_key of the first kMaxCand candidates
  __shared__ int wsum[32];
  __shared__ int base;
  __shared__ unsigned hist[1 << kRadixBits];
  __shared__ unsigned long long sel_prefix;
  __shared__ int sel_rank, gathered;
  const int n = blockIdx.x;
  const float* sc = scores + static_cast<size_t>(n) * H * W;
  const float* mk = mask + static_cast<size_t>(n) * H * W;
  if (threadIdx.x == 0) base = 0;
  __syncthreads();
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int total = H * W;
  for (int i0 = 0; i0 < total; i0 += 1024) {
    const int i = i0 + threadIdx.x;
    int flag = 0;
    float s = 0.f;
    if (i < total) {
      s = sc[i];
      flag = is_candidate(s, mk[i], i, H, W, thr, border) ? 1 : 0;
    }
    int inc = flag;
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += t;
    }
    if (lane == 31) wsum[wid] = inc;
    __syncthreads();
    if (wid == 0) {
      int ws = wsum[lane];
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, ws, o);
        if (lane >= o) ws += t;
      }
      wsum[lane] = ws;
    }
    __syncthreads();
    if (flag) {
      const int slot = base + (wid > 0 ? wsum[wid - 1] : 0) + inc - 1;
      if (slot < kMaxCand) s_key[slot] = cand_key(s, i);
    }
    __syncthreads();
    if (threadIdx.x == 0) base += wsum[31];
    __syncthreads();
  }
  int ncand = min(base, kMaxCand);
  const bool row_major = base <= max_kp;
  if (base > kMaxCand) {
    // s_key holds only the first kMaxCand candidates in row-major order. Radix-select the max_kp-th largest key
    // over the whole image, most significant 11-bit digit first (digits [53, 64), [42, 53), ..., [0, 9)), then
    // gather the max_kp keys at or above it (keys are distinct) for the sort below.
    unsigned long long prefix = 0ull, pmask = 0ull;   // the selected key's digits found so far
    int rank = max_kp;                                // its rank among the keys that match them
    for (int hi = 64; hi > 0; hi -= kRadixBits) {
      const int lo = max(hi - kRadixBits, 0);
      const unsigned dmask = (1u << (hi - lo)) - 1u;
      for (int b = threadIdx.x; b < (1 << kRadixBits); b += 1024) hist[b] = 0u;
      __syncthreads();
      for (int i = threadIdx.x; i < total; i += 1024) {
        const float s = sc[i];
        if (!is_candidate(s, mk[i], i, H, W, thr, border)) continue;
        const unsigned long long key = cand_key(s, i);
        if ((key & pmask) == prefix) atomicAdd(&hist[static_cast<unsigned>(key >> lo) & dmask], 1u);
      }
      __syncthreads();
      // thread t holds digits 2047 - 2t and 2046 - 2t: the scan counts the keys above each digit
      const int d1 = 2047 - 2 * static_cast<int>(threadIdx.x), d0 = d1 - 1;
      const int c1 = static_cast<int>(hist[d1]), c = c1 + static_cast<int>(hist[d0]);
      const int incl = block_scan1024(c, wsum);
      const int excl = incl - c;
      if (excl < rank && rank <= incl) {
        const bool top = excl + c1 >= rank;
        sel_prefix = prefix | (static_cast<unsigned long long>(top ? d1 : d0) << lo);
        sel_rank = rank - (top ? excl : excl + c1);
      }
      __syncthreads();
      prefix = sel_prefix;
      rank = sel_rank;
      pmask |= static_cast<unsigned long long>(dmask) << lo;
      __syncthreads();
    }
    if (threadIdx.x == 0) gathered = 0;
    __syncthreads();
    for (int i = threadIdx.x; i < total; i += 1024) {
      const float s = sc[i];
      if (!is_candidate(s, mk[i], i, H, W, thr, border)) continue;
      const unsigned long long key = cand_key(s, i);
      if (key >= prefix) {
        const int slot = atomicAdd(&gathered, 1);
        if (slot < max_kp) s_key[slot] = key;
      }
    }
    __syncthreads();
    ncand = max_kp;
  }
  float* ko = kpts + static_cast<size_t>(n) * max_kp * 2;
  float* so = kscores + static_cast<size_t>(n) * max_kp;
  if (row_major) {   // keep torch.nonzero (row-major) order
    for (int k = threadIdx.x; k < max_kp; k += blockDim.x) {
      float x = 0.f, y = 0.f, s = 0.f;
      if (k < ncand) {
        const unsigned pix = 0xffffffffu - static_cast<unsigned>(s_key[k] & 0xffffffffull);
        s = __uint_as_float(static_cast<unsigned>(s_key[k] >> 32));
        y = static_cast<float>(pix / W);
        x = static_cast<float>(pix % W);
      }
      ko[2 * k] = x; ko[2 * k + 1] = y; so[k] = s;
    }
    if (threadIdx.x == 0) counts[n] = ncand;
    return;
  }
  // bitonic sort, descending by (score, then lower pixel index first)
  int npow = 1;
  while (npow < ncand) npow <<= 1;
  for (int k = ncand + threadIdx.x; k < npow; k += blockDim.x) s_key[k] = 0ull;
  __syncthreads();
  for (int size = 2; size <= npow; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      for (int t = threadIdx.x; t < npow / 2; t += blockDim.x) {
        const int lo = (t / stride) * 2 * stride + (t % stride);
        const int hi = lo + stride;
        const bool desc = ((lo & size) == 0);
        const unsigned long long a = s_key[lo], b = s_key[hi];
        if ((a < b) == desc) { s_key[lo] = b; s_key[hi] = a; }
      }
      __syncthreads();
    }
  }
  for (int k = threadIdx.x; k < max_kp; k += blockDim.x) {
    const unsigned pix = 0xffffffffu - static_cast<unsigned>(s_key[k] & 0xffffffffull);
    ko[2 * k] = static_cast<float>(pix % W);
    ko[2 * k + 1] = static_cast<float>(pix / W);
    so[k] = __uint_as_float(static_cast<unsigned>(s_key[k] >> 32));
  }
  if (threadIdx.x == 0) counts[n] = max_kp;
}

// ------------------------------------------------------------------------------------------ descriptors
// in-place L2 normalisation over 256 channels (F.normalize, eps 1e-12); warp per pixel
__global__ void __launch_bounds__(256) l2norm256_kernel(float* __restrict__ x, size_t rows) {
  const size_t r = static_cast<size_t>(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (r >= rows) return;
  const int lane = threadIdx.x & 31;
  float4* p = reinterpret_cast<float4*>(x + r * 256);
  float4 a = p[lane], b = p[32 + lane];
  const float ss = warp_sum(a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w + b.x * b.x + b.y * b.y + b.z * b.z + b.w * b.w);
  const float inv = 1.f / fmaxf(sqrtf(ss), 1e-12f);
  a.x *= inv; a.y *= inv; a.z *= inv; a.w *= inv; b.x *= inv; b.y *= inv; b.z *= inv; b.w *= inv;
  p[lane] = a; p[32 + lane] = b;
}

// bilinear grid_sample (align_corners=False, zero padding) of the dense descriptor map at the
// keypoints + L2 normalisation (superpoint.py:80-92). dense [N][h][w][256]; out tokens [N][max_kp][ldo].
__global__ void __launch_bounds__(256) sample_desc_kernel(const float* __restrict__ dense,
                                                          const float* __restrict__ kpts,
                                                          const int* __restrict__ counts, int h, int w,
                                                          int max_kp, float* __restrict__ out, long long ldo) {
  const int n = blockIdx.y;
  const int k = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (k >= max_kp) return;
  const int lane = threadIdx.x & 31;
  float* o = out + (static_cast<size_t>(n) * max_kp + k) * ldo;
  if (k >= counts[n]) {   // unused slots are zero tokens
    for (int c = lane; c < 256; c += 32) o[c] = 0.f;
    return;
  }
  const float s = 8.f;
  float kx = kpts[(static_cast<size_t>(n) * max_kp + k) * 2], ky = kpts[(static_cast<size_t>(n) * max_kp + k) * 2 + 1];
  kx = (kx - s / 2 + 0.5f) / (w * s - s / 2 - 0.5f) * 2.f - 1.f;
  ky = (ky - s / 2 + 0.5f) / (h * s - s / 2 - 0.5f) * 2.f - 1.f;
  // grid_sample, align_corners=False: pixel = ((g + 1) * size - 1) / 2
  const float px = ((kx + 1.f) * w - 1.f) * 0.5f, py = ((ky + 1.f) * h - 1.f) * 0.5f;
  const float fx = floorf(px), fy = floorf(py);
  const int x0 = static_cast<int>(fx), y0 = static_cast<int>(fy);
  const float ax = px - fx, ay = py - fy;
  const float w00 = (1.f - ax) * (1.f - ay), w01 = ax * (1.f - ay), w10 = (1.f - ax) * ay, w11 = ax * ay;
  const float* d = dense + static_cast<size_t>(n) * h * w * 256;
  float v[8];
  float ss = 0.f;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = lane + 32 * j;
    float a = 0.f;
    if (y0 >= 0 && y0 < h) {
      if (x0 >= 0 && x0 < w) a = fmaf(w00, d[(static_cast<size_t>(y0) * w + x0) * 256 + c], a);
      if (x0 + 1 >= 0 && x0 + 1 < w) a = fmaf(w01, d[(static_cast<size_t>(y0) * w + x0 + 1) * 256 + c], a);
    }
    if (y0 + 1 >= 0 && y0 + 1 < h) {
      if (x0 >= 0 && x0 < w) a = fmaf(w10, d[(static_cast<size_t>(y0 + 1) * w + x0) * 256 + c], a);
      if (x0 + 1 >= 0 && x0 + 1 < w) a = fmaf(w11, d[(static_cast<size_t>(y0 + 1) * w + x0 + 1) * 256 + c], a);
    }
    v[j] = a;
    ss = fmaf(a, a, ss);
  }
  const float inv = 1.f / fmaxf(sqrtf(warp_sum(ss)), 1e-12f);
#pragma unroll
  for (int j = 0; j < 8; ++j) o[lane + 32 * j] = v[j] * inv;
}

// keypoint encoder input: [(x - W/2) / (0.7 max(W,H)), (y - H/2) / (0.7 max), score, 0] (superglue.py:63-82)
__global__ void kenc_input_kernel(const float* __restrict__ kpts, const float* __restrict__ kscores,
                                  float* __restrict__ out, int total, float cx, float cy, float inv_scale) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  float4 o;
  o.x = (kpts[2 * i] - cx) * inv_scale;
  o.y = (kpts[2 * i + 1] - cy) * inv_scale;
  o.z = kscores[i];
  o.w = 0.f;
  reinterpret_cast<float4*>(out)[i] = o;
}

// ------------------------------------------------------------------------------------------ softmax attention on the tensor cores
// The scores Q_h K_h^T / 8 and the product P V_h are tensor-core GEMMs (conv_gemm, per-(image, head) B operand); in between:
//   sg_softmax_rows : P[img][h][q][:] = softmax over the source image's nk keys (0 beyond them), in place
//   sg_transpose_v  : Vt[img][h][d][k] = qkv[img][k][512 + 64 h + d]  (the P V GEMM needs V K-major along the keys)
__global__ void __launch_bounds__(256) sg_softmax_rows_kernel(float* __restrict__ S, const int* __restrict__ counts,
                                                              int src_xor, int max_kp) {
  __shared__ float sh[8];
  const int q = blockIdx.x, h = blockIdx.y, img = blockIdx.z;
  const int nq = counts[img], nk = counts[img ^ src_xor];
  float* row = S + ((static_cast<size_t>(img) * 4 + h) * max_kp + q) * max_kp;
  const int t = threadIdx.x;
  if (q >= nq) {                             // absent keypoints: zero message, so that padded rows stay bounded through the layers
    for (int k = t; k < max_kp; k += 256) row[k] = 0.f;
    return;
  }
  float v[4];
  float m = -INFINITY;
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int k = t + 256 * e;
    v[e] = (k < nk) ? row[k] : -INFINITY;
    m = fmaxf(m, v[e]);
  }
  for (int k = t + 1024; k < nk; k += 256) m = fmaxf(m, row[k]);    // max_kp > 1024 (not used by the reference config)
  m = warp_max(m);
  if ((t & 31) == 0) sh[t >> 5] = m;
  __syncthreads();
  m = sh[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) m = fmaxf(m, sh[w]);
  __syncthreads();
  float s = 0.f;
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    v[e] = (t + 256 * e < nk) ? __expf(v[e] - m) : 0.f;
    s += v[e];
  }
  for (int k = t + 1024; k < nk; k += 256) s += __expf(row[k] - m);
  s = warp_sum(s);
  if ((t & 31) == 0) sh[t >> 5] = s;
  __syncthreads();
  s = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) s += sh[w];
  const float inv = s > 0.f ? 1.f / s : 0.f;
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int k = t + 256 * e;
    if (k < max_kp) row[k] = v[e] * inv;
  }
  for (int k = t + 1024; k < max_kp; k += 256) row[k] = (k < nk) ? __expf(row[k] - m) * inv : 0.f;
}

__global__ void __launch_bounds__(256) sg_transpose_v_kernel(const float* __restrict__ qkv, long long ld,
                                                             float* __restrict__ vt, int max_kp) {
  __shared__ float tile[32][33];
  const int img = blockIdx.z, c0 = blockIdx.y * 32, k0 = blockIdx.x * 32;   // c = 64 h + d in [0, 256)
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;                   // 32 x 8
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int k = k0 + ty + 8 * j;
    tile[ty + 8 * j][tx] = k < max_kp ? qkv[(static_cast<size_t>(img) * max_kp + k) * ld + 512 + c0 + tx] : 0.f;
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int c = c0 + ty + 8 * j, k = k0 + tx;
    if (k < max_kp) vt[(static_cast<size_t>(img) * 256 + c) * max_kp + k] = tile[tx][ty + 8 * j];
  }
}

// ------------------------------------------------------------------------------------------ Sinkhorn (superglue.py:141-170)
// couplings Z[(n0+1) x (n1+1)]: Z[i][j] = S[i][j] (i < n0, j < n1), bin score alpha otherwise.
__device__ __forceinline__ void lse_push(float& m, float& s, float x) {
  if (x > m) { s = s * __expf(m - x) + 1.f; m = x; } else { s += __expf(x - m); }
}
// u[i] = log_mu[i] - logsumexp_j(Z[i][j] + v[j]); one block per row i in [0, n0]
__global__ void __launch_bounds__(256) sinkhorn_rows_kernel(const float* __restrict__ S, int ldS,
                                                            const int* __restrict__ counts, float alpha,
                                                            const float* __restrict__ v, float* __restrict__ u) {
  __shared__ float shm[8], shs[8];
  const int pair = blockIdx.y;
  counts += 2 * pair; S += static_cast<size_t>(pair) * ldS * ldS; v += pair * (ldS + 1); u += pair * (ldS + 1);
  const int n0 = counts[0], n1 = counts[1];
  const int i = blockIdx.x;
  if (i > n0) return;
  float m = -INFINITY, s = 0.f;
  for (int j = threadIdx.x; j <= n1; j += 256) {
    const float z = (i < n0 && j < n1) ? S[static_cast<size_t>(i) * ldS + j] : alpha;
    lse_push(m, s, z + v[j]);
  }
  // merge (m, s) pairs
  for (int o = 16; o > 0; o >>= 1) {
    const float om = __shfl_xor_sync(0xffffffffu, m, o), os = __shfl_xor_sync(0xffffffffu, s, o);
    const float nm = fmaxf(m, om);
    s = (m == -INFINITY ? 0.f : s * __expf(m - nm)) + (om == -INFINITY ? 0.f : os * __expf(om - nm));
    m = nm;
  }
  if ((threadIdx.x & 31) == 0) { shm[threadIdx.x >> 5] = m; shs[threadIdx.x >> 5] = s; }
  __syncthreads();
  if (threadIdx.x == 0) {
    float M = shm[0], Ssum = shs[0];
    for (int k = 1; k < 8; ++k) {
      const float nm = fmaxf(M, shm[k]);
      Ssum = (M == -INFINITY ? 0.f : Ssum * __expf(M - nm)) + (shm[k] == -INFINITY ? 0.f : shs[k] * __expf(shm[k] - nm));
      M = nm;
    }
    const float norm = -__logf(static_cast<float>(n0 + n1));
    const float log_mu = i < n0 ? norm : __logf(static_cast<float>(n1)) + norm;
    u[i] = log_mu - (M + __logf(Ssum));
  }
}
// v[j] = log_nu[j] - logsumexp_i(Z[i][j] + u[i]); block = 32 columns x 8 row groups
__global__ void __launch_bounds__(256) sinkhorn_cols_kernel(const float* __restrict__ S, int ldS,
                                                            const int* __restrict__ counts, float alpha,
                                                            const float* __restrict__ u, float* __restrict__ v) {
  __shared__ float shm[8][33], shs[8][33];
  const int pair = blockIdx.y;
  counts += 2 * pair; S += static_cast<size_t>(pair) * ldS * ldS; v += pair * (ldS + 1); u += pair * (ldS + 1);
  const int n0 = counts[0], n1 = counts[1];
  const int j = blockIdx.x * 32 + (threadIdx.x & 31);
  const int g = threadIdx.x >> 5;
  float m = -INFINITY, s = 0.f;
  if (j <= n1) {
    for (int i = g; i <= n0; i += 8) {
      const float z = (i < n0 && j < n1) ? S[static_cast<size_t>(i) * ldS + j] : alpha;
      lse_push(m, s, z + u[i]);
    }
  }
  shm[g][threadIdx.x & 31] = m;
  shs[g][threadIdx.x & 31] = s;
  __syncthreads();
  if (g == 0 && j <= n1) {
    float M = shm[0][threadIdx.x], Ssum = shs[0][threadIdx.x];
    for (int k = 1; k < 8; ++k) {
      const float om = shm[k][threadIdx.x], os = shs[k][threadIdx.x];
      const float nm = fmaxf(M, om);
      Ssum = (M == -INFINITY ? 0.f : Ssum * __expf(M - nm)) + (om == -INFINITY ? 0.f : os * __expf(om - nm));
      M = nm;
    }
    const float norm = -__logf(static_cast<float>(n0 + n1));
    const float log_nu = j < n1 ? norm : __logf(static_cast<float>(n0)) + norm;
    v[j] = log_nu - (M + __logf(Ssum));
  }
}
__global__ void fill_kernel(float* p, int n, float val) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = val;
}

// ------------------------------------------------------------------------------------------ matches (superglue.py:266-276)
// row / column arg-max of Z[:-1, :-1] = S + u_i + v_j - norm (lowest index on ties)
__global__ void __launch_bounds__(256) sg_rowmax_kernel(const float* __restrict__ S, int ldS,
                                                        const int* __restrict__ counts, const float* __restrict__ u,
                                                        const float* __restrict__ v, float* __restrict__ rmax,
                                                        int* __restrict__ rarg) {
  __shared__ float shv[8];
  __shared__ int shi[8];
  const int pair = blockIdx.y;
  counts += 2 * pair; S += static_cast<size_t>(pair) * ldS * ldS; v += pair * (ldS + 1); u += pair * (ldS + 1);
  rmax += pair * ldS; rarg += pair * ldS;
  const int n0 = counts[0], n1 = counts[1];
  const int i = blockIdx.x;
  if (i >= n0) return;
  float best = -INFINITY;
  int arg = 0x7fffffff;
  for (int j = threadIdx.x; j < n1; j += 256) {
    const float z = S[static_cast<size_t>(i) * ldS + j] + v[j];
    if (z > best) { best = z; arg = j; }
  }
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
    if (ob > best || (ob == best && oa < arg)) { best = ob; arg = oa; }
  }
  if ((threadIdx.x & 31) == 0) { shv[threadIdx.x >> 5] = best; shi[threadIdx.x >> 5] = arg; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < 8; ++k)
      if (shv[k] > best || (shv[k] == best && shi[k] < arg)) { best = shv[k]; arg = shi[k]; }
    rmax[i] = best + u[i];
    rarg[i] = arg;
  }
}
__global__ void __launch_bounds__(256) sg_colarg_kernel(const float* __restrict__ S, int ldS,
                                                        const int* __restrict__ counts, const float* __restrict__ u,
                                                        int* __restrict__ carg) {
  __shared__ float shv[8][33];
  __shared__ int shi[8][33];
  const int pair = blockIdx.y;
  counts += 2 * pair; S += static_cast<size_t>(pair) * ldS * ldS; u += pair * (ldS + 1); carg += pair * ldS;
  const int n0 = counts[0], n1 = counts[1];
  const int j = blockIdx.x * 32 + (threadIdx.x & 31);
  const int g = threadIdx.x >> 5;
  float best = -INFINITY;
  int arg = 0x7fffffff;
  if (j < n1)
    for (int i = g; i < n0; i += 8) {
      const float z = S[static_cast<size_t>(i) * ldS + j] + u[i];
      if (z > best) { best = z; arg = i; }
    }
  shv[g][threadIdx.x & 31] = best;
  shi[g][threadIdx.x & 31] = arg;
  __syncthreads();
  if (g == 0 && j < n1) {
    for (int k = 1; k < 8; ++k) {
      const float ob = shv[k][threadIdx.x];
      const int oa = shi[k][threadIdx.x];
      if (ob > best || (ob == best && oa < arg)) { best = ob; arg = oa; }
    }
    carg[j] = arg;
  }
}
// mutual check + threshold + ordered compaction of the matched keypoint coordinates (one block)
__global__ void __launch_bounds__(1024) sg_matches_kernel(const int* __restrict__ counts, const float* __restrict__ rmax,
                                                          const int* __restrict__ rarg, const int* __restrict__ carg,
                                                          float thr, const float* __restrict__ kpts, int max_kp,
                                                          int* __restrict__ matches0, float* __restrict__ mscores0,
                                                          float* __restrict__ mk0, float* __restrict__ mk1,
                                                          int* __restrict__ m_offsets, int n_pairs) {
  __shared__ int wsum[32];
  __shared__ int base;
  __shared__ int s_out0;
  if (threadIdx.x == 0) { s_out0 = 0; m_offsets[0] = 0; }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int pair = 0; pair < n_pairs; ++pair) {
  const int n0 = counts[2 * pair], n1 = counts[2 * pair + 1];
  const float norm = -__logf(static_cast<float>(n0 + n1));
  if (threadIdx.x == 0) base = 0;
  __syncthreads();
  const int out0 = s_out0;
  const float* rmax_p = rmax + pair * max_kp;
  const int* rarg_p = rarg + pair * max_kp;
  const int* carg_p = carg + pair * max_kp;
  const float* kpts_p = kpts + static_cast<size_t>(pair) * 2 * max_kp * 2;
  int* matches_p = matches0 + pair * max_kp;
  float* mscores_p = mscores0 + pair * max_kp;
  for (int i0 = 0; i0 < max_kp; i0 += 1024) {
    const int i = i0 + threadIdx.x;
    int flag = 0, j = -1;
    float ms = 0.f;
    if (i < n0 && n1 > 0) {
      j = rarg_p[i];
      const bool mutual = carg_p[j] == i;
      ms = mutual ? __expf(rmax_p[i] - norm) : 0.f;
      flag = (mutual && ms > thr) ? 1 : 0;
    }
    if (i < max_kp) {
      matches_p[i] = flag ? j : -1;
      mscores_p[i] = ms;
    }
    int inc = flag;
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += t;
    }
    if (lane == 31) wsum[wid] = inc;
    __syncthreads();
    if (wid == 0) {
      int ws = wsum[lane];
      for (int o = 1; o < 32; o <<= 1) {
        const int t = __shfl_up_sync(0xffffffffu, ws, o);
        if (lane >= o) ws += t;
      }
      wsum[lane] = ws;
    }
    __syncthreads();
    if (flag) {
      const int slot = out0 + base + (wid > 0 ? wsum[wid - 1] : 0) + inc - 1;
      mk0[2 * slot] = kpts_p[2 * i];
      mk0[2 * slot + 1] = kpts_p[2 * i + 1];
      mk1[2 * slot] = kpts_p[(static_cast<size_t>(max_kp) + j) * 2];
      mk1[2 * slot + 1] = kpts_p[(static_cast<size_t>(max_kp) + j) * 2 + 1];
    }
    __syncthreads();
    if (threadIdx.x == 0) base += wsum[31];
    __syncthreads();
  }
  if (threadIdx.x == 0) { m_offsets[pair + 1] = out0 + base; s_out0 = out0 + base; }
  __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------ shared map frame
// Pair-interleaved SuperPoint outputs from one map image and B queries: image 2b <- the map, 2b + 1 <- query b.
// blockIdx.y = output image; x grid-strides over the image's descriptors, keypoints and scores as 16-byte elements.
__global__ void __launch_bounds__(256) pair_interleave_kernel(
    const int* __restrict__ m_cnt, const float4* __restrict__ m_kp, const float4* __restrict__ m_ks,
    const float4* __restrict__ m_d, const int* __restrict__ q_cnt, const float4* __restrict__ q_kp,
    const float4* __restrict__ q_ks, const float4* __restrict__ q_d, int max_kp, int* __restrict__ cnt,
    float4* __restrict__ kp, float4* __restrict__ ks, float4* __restrict__ d) {
  const int img = blockIdx.y, b = img >> 1;
  const bool q = img & 1;
  const int nd = max_kp * 64, nkp = max_kp / 2, nks = max_kp / 4;   // float4 per image
  if (blockIdx.x == 0 && threadIdx.x == 0) cnt[img] = q ? q_cnt[b] : m_cnt[0];
  const float4* sd = q ? q_d + static_cast<size_t>(b) * nd : m_d;
  const float4* skp = q ? q_kp + static_cast<size_t>(b) * nkp : m_kp;
  const float4* sks = q ? q_ks + static_cast<size_t>(b) * nks : m_ks;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nd + nkp + nks; i += gridDim.x * blockDim.x) {
    if (i < nd) d[static_cast<size_t>(img) * nd + i] = sd[i];
    else if (i < nd + nkp) kp[static_cast<size_t>(img) * nkp + i - nd] = skp[i - nd];
    else ks[static_cast<size_t>(img) * nks + i - nd - nkp] = sks[i - nd - nkp];
  }
}

}  // namespace

// ================================================================================================
// launch wrappers
// ================================================================================================
#define GRID1(n, b) static_cast<unsigned>(((n) + (b) - 1) / (b))

int sp_conv1a(const float* img, const float* w, const float* bias, float* out, int N, int H, int W, cudaStream_t st) {
  conv1a_kernel<float><<<dim3((W + 63) / 64, H, N), 64, 0, st>>>(img, w, bias, out, H, W);
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}
int sp_conv1a_bf16(const float* img, const float* w, const float* bias, void* out, int N, int H, int W, cudaStream_t st) {
  conv1a_kernel<__nv_bfloat16><<<dim3((W + 63) / 64, H, N), 64, 0, st>>>(img, w, bias, static_cast<__nv_bfloat16*>(out), H, W);
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}
int maxpool2x2(const float* in, float* out, int N, int H, int W, int C, cudaStream_t st) {
  if (C % 4) return MFR_ERR_ARG;
  const size_t total = static_cast<size_t>(N) * (H / 2) * (W / 2) * (C / 4);
  maxpool2_kernel<<<GRID1(total, 256), 256, 0, st>>>(in, out, N, H, W, C / 4);
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}
int maxpool2x2_bf16(const void* in, void* out, int N, int H, int W, int C, cudaStream_t st) {
  if (C % 8) return MFR_ERR_ARG;
  const size_t total = static_cast<size_t>(N) * (H / 2) * (W / 2) * (C / 8);
  maxpool2_bf16_kernel<<<GRID1(total, 256), 256, 0, st>>>(static_cast<const uint4*>(in), static_cast<uint4*>(out), N, H, W, C / 8);
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}
int sp_score_map(const float* logits, int ldc, float* scores, int N, int h, int w, cudaStream_t st) {
  score_map_kernel<<<GRID1(static_cast<size_t>(N) * h * w, 8), 256, 0, st>>>(logits, ldc, scores, N, h, w);
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}
int sp_nms(const float* scores, float* mask, float* t0, float* t1, float* t2, float* t3, int N, int H, int W, int r,
           cudaStream_t st) {
  const size_t n = static_cast<size_t>(N) * H * W;
  const unsigned g = GRID1(n, 256);
  auto pool = [&](const float* in, float* tmp, float* out) {
    rowmax_kernel<<<g, 256, 0, st>>>(in, tmp, N, H, W, r);
    colmax_kernel<<<g, 256, 0, st>>>(tmp, out, N, H, W, r);
  };
  pool(scores, t0, t1);
  nms_init_kernel<<<g, 256, 0, st>>>(scores, t1, mask, n);
  for (int it = 0; it < 2; ++it) {
    pool(mask, t0, t1);                                   // t1 = pool(mask)
    nms_supp_kernel<<<g, 256, 0, st>>>(scores, t1, t2, n);  // t2 = supp_scores
    pool(t2, t0, t3);                                     // t3 = pool(supp_scores)
    nms_update_kernel<<<g, 256, 0, st>>>(t2, t3, t1, mask, n);
  }
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}
int sp_select_keypoints(const float* scores, const float* mask, int N, int H, int W, float thr, int border,
                        int max_kp, float* kpts, float* kscores, int* counts, cudaStream_t st) {
  static bool attr_seen[64] = {};
  if (first_call_on_device(attr_seen))
    cudaFuncSetAttribute(select_keypoints_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMaxCand * 8);
  select_keypoints_kernel<<<N, 1024, kMaxCand * 8, st>>>(scores, mask, H, W, thr, border, max_kp, kpts, kscores, counts);
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}
int l2norm256(float* x, size_t rows, cudaStream_t st) {
  l2norm256_kernel<<<GRID1(rows, 8), 256, 0, st>>>(x, rows);
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}
int sp_sample_descriptors(const float* dense, const float* kpts, const int* counts, int N, int h, int w, int max_kp,
                          float* out, long long ldo, cudaStream_t st) {
  sample_desc_kernel<<<dim3((max_kp + 7) / 8, N), 256, 0, st>>>(dense, kpts, counts, h, w, max_kp, out, ldo);
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}
int sg_kenc_input(const float* kpts, const float* kscores, float* out, int total, int H, int W, cudaStream_t st) {
  const float sc = 1.f / (0.7f * static_cast<float>(std::max(H, W)));
  kenc_input_kernel<<<GRID1(total, 256), 256, 0, st>>>(kpts, kscores, out, total, W * 0.5f, H * 0.5f, sc);
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}
int sg_softmax_rows(float* S, const int* counts, int cross, int max_kp, int n_img, cudaStream_t st) {
  sg_softmax_rows_kernel<<<dim3(max_kp, 4, n_img), 256, 0, st>>>(S, counts, cross ? 1 : 0, max_kp);
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}
int sg_transpose_v(const float* qkv, long long ld, float* vt, int max_kp, int n_img, cudaStream_t st) {
  sg_transpose_v_kernel<<<dim3((max_kp + 31) / 32, 8, n_img), 256, 0, st>>>(qkv, ld, vt, max_kp);
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}
int sg_sinkhorn(const float* S, int ldS, const int* counts, float alpha, int iters, int max_kp, int n_pairs,
                float* u, float* v, cudaStream_t st) {
  if (ldS != max_kp) return MFR_ERR_ARG;
  fill_kernel<<<GRID1(n_pairs * (max_kp + 1), 256), 256, 0, st>>>(u, n_pairs * (max_kp + 1), 0.f);
  fill_kernel<<<GRID1(n_pairs * (max_kp + 1), 256), 256, 0, st>>>(v, n_pairs * (max_kp + 1), 0.f);
  for (int it = 0; it < iters; ++it) {
    sinkhorn_rows_kernel<<<dim3(max_kp + 1, n_pairs), 256, 0, st>>>(S, ldS, counts, alpha, v, u);
    sinkhorn_cols_kernel<<<dim3((max_kp + 1 + 31) / 32, n_pairs), 256, 0, st>>>(S, ldS, counts, alpha, u, v);
  }
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}
int sg_extract_matches(const float* S, int ldS, const int* counts, const float* u, const float* v, float thr,
                       const float* kpts, int max_kp, float* rmax, int* rarg, int* carg, int* matches0,
                       float* mscores0, float* mk0, float* mk1, int* m_offsets, int n_pairs, cudaStream_t st) {
  if (ldS != max_kp) return MFR_ERR_ARG;
  sg_rowmax_kernel<<<dim3(max_kp, n_pairs), 256, 0, st>>>(S, ldS, counts, u, v, rmax, rarg);
  sg_colarg_kernel<<<dim3((max_kp + 31) / 32, n_pairs), 256, 0, st>>>(S, ldS, counts, u, carg);
  sg_matches_kernel<<<1, 1024, 0, st>>>(counts, rmax, rarg, carg, thr, kpts, max_kp, matches0, mscores0, mk0, mk1,
                                        m_offsets, n_pairs);
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}

int sp_pair_interleave(const int* map_counts, const float* map_kpts, const float* map_scores, const float* map_desc,
                       const int* q_counts, const float* q_kpts, const float* q_scores, const float* q_desc, int B, int max_kp,
                       int* counts, float* kpts, float* scores, float* desc, cudaStream_t st) {
  if (B < 1 || (max_kp % 4)) return MFR_ERR_ARG;
  const int per_img = max_kp * 64 + max_kp / 2 + max_kp / 4;
  pair_interleave_kernel<<<dim3(GRID1(per_img, 256 * 4), 2 * B), 256, 0, st>>>(
      map_counts, reinterpret_cast<const float4*>(map_kpts), reinterpret_cast<const float4*>(map_scores),
      reinterpret_cast<const float4*>(map_desc), q_counts, reinterpret_cast<const float4*>(q_kpts),
      reinterpret_cast<const float4*>(q_scores), reinterpret_cast<const float4*>(q_desc), max_kp, counts,
      reinterpret_cast<float4*>(kpts), reinterpret_cast<float4*>(scores), reinterpret_cast<float4*>(desc));
  MFR_CUDA_CHECK(cudaGetLastError());
  return MFR_OK;
}

}  // namespace mfr
